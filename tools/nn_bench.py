"""Throughput of the network kernel alone (positions/s, tensor-roofline fraction) -- ch5 net by default, batch in HBM.

python tools/nn_bench.py [res_blocks] [iters] [filters] [impl] [n ...]
  filters: cnn_filter_num (default 256); impl: RZ_NET_IMPL_* (default 2, the tensor-core tower; 1 = the generic fp32
  kernel); n: batch sizes (default 296 32768).  With filters or impl given, each line also carries them."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "reversi-alpha-zero_b200"))
FLOP_PER_POS = 2 * 755_343_616


def flop_per_position(filters=256, res_blocks=10, value_fc=256):
    """algorithmic flop of one position: conv0, 2R tower convolutions, 1x1 head convolutions, the dense layers"""
    F = filters
    return 2 * (64 * F * 18 + res_blocks * 2 * 64 * F * 9 * F + 64 * 3 * F + 128 * 64 + 64 * value_fc + value_fc)


def run(n=32768, iters=5, warmup=2, res_blocks=10, filters=256, impl=2, tag=False):
    import torch
    from reversi_zero_b200.agent import model as M
    from reversi_zero_b200 import net as N, device as D
    mc = M.ModelConfig(res_layer_num=res_blocks, cnn_filter_num=filters)
    flop = flop_per_position(filters, res_blocks, mc.value_fc_size)
    net = N.Net(mc)
    net.load_weights(M.build_random_weights(mc, 0))
    rng = np.random.default_rng(0)
    a = rng.integers(0, 2 ** 64, size=n, dtype=np.uint64); r = rng.integers(0, 2 ** 64, size=n, dtype=np.uint64)
    d_own, d_en = D.to_device(a & r), D.to_device(a & ~r)
    d_pol, d_val = D.empty(n * 64, np.float32), D.empty(n, np.float32)
    s = torch.cuda.current_stream()
    for _ in range(warmup):
        net.predict_dev(d_own, d_en, d_pol, d_val, n, impl, D.stream_ptr(s))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(s)
    for _ in range(iters):
        net.predict_dev(d_own, d_en, d_pol, d_val, n, impl, D.stream_ptr(s))
    e1.record(s)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    tflops = n * flop / ms / 1e9
    # share of the H100 SXM data-sheet dense FP16 tensor rate (989 TFLOP/s at 700 W), not a measured peak
    r = dict(n=n, res_blocks=res_blocks, flop_per_position=flop, ms=ms, pos_per_s=n / ms * 1e3, tflops=tflops,
             frac_of_datasheet_fp16=tflops / 989.0, gpu=torch.cuda.get_device_name())
    if tag:
        r.update(filters=filters, impl=impl)
    return r


if __name__ == "__main__":
    rb = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    iters = int(sys.argv[2]) if len(sys.argv) > 2 else 5
    filters = int(sys.argv[3]) if len(sys.argv) > 3 else 256
    impl = int(sys.argv[4]) if len(sys.argv) > 4 else 2
    ns = [int(a) for a in sys.argv[5:]] or [296, 32768]
    for n in ns:
        r = run(n, iters=iters, res_blocks=rb, filters=filters, impl=impl, tag=len(sys.argv) > 3)
        print(json.dumps(r))
