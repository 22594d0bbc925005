"""Time of one device training step (rz_trainer_step_dev) for the ch5 network: ms per step from CUDA events after
warm-up, records/s, and algorithmic TFLOP/s of the 3x3 convolutions (forward, input gradient and weight gradient GEMMs;
the heads and BatchNorm are not counted).  The GPU name and power limit are read in the same run.

    python tools/train_bench.py [--batches 256 1024] [--steps 30] [--warmup 5] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "reversi-alpha-zero_b200"))


def conv_flop_per_step(mc, batch):
    F, R = mc.cnn_filter_num, mc.res_layer_num
    fwd = 2 * batch * 64 * 9 * (2 * F + 2 * R * F * F)
    return 3 * fwd


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in out.split(","))
        return dict(gpu=name, power_limit=power, max_sm_clock=clock)
    except Exception as e:  # the measurement itself does not depend on it
        return dict(gpu_info_error=str(e))


def run(batch, steps, warmup, n_records=65536):
    import torch
    from reversi_zero_b200.agent import model as M
    from reversi_zero_b200 import train as T
    mc = M.ModelConfig()  # ch5: 256 filters, 10 residual blocks, value_fc 256
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0)
    states = (torch.rand((n_records, 2, 8, 8), generator=g, device=dev) < 0.3).to(torch.uint8)
    policy = torch.rand((n_records, 64), generator=g, device=dev)
    policy /= policy.sum(dim=1, keepdim=True)
    z = torch.randint(-1, 2, (n_records,), generator=g, device=dev).float()
    perm = torch.randperm(n_records, generator=g, device=dev).to(torch.int32)
    tr = T.Trainer(mc, max_batch=batch)
    tr.load_blob(M.weights_to_blob(mc, M.build_random_weights(mc, 0)))
    idx = lambda k: perm[(k * batch) % (n_records - batch):][:batch].contiguous()
    for k in range(warmup):
        tr.step(states, policy, z, idx(k), 0.01)
    torch.cuda.synchronize()
    ids = [idx(k) for k in range(steps)]
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for k in range(steps):
        loss = tr.step(states, policy, z, ids[k], 0.01)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    flop = conv_flop_per_step(mc, batch)
    res = dict(config="ch5", batch=batch, steps=steps, ms_per_step=ms, records_per_s=batch / ms * 1e3,
               conv_tflop_per_step=flop / 1e12, conv_tflops=flop / ms / 1e9, final_loss=[float(x) for x in loss.cpu()],
               torch_device=torch.cuda.get_device_name(dev))
    tr.close()
    return res


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[256, 1024])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    info = gpu_info()
    lines = [json.dumps({**info, **run(b, a.steps, a.warmup)}) for b in a.batches]
    for line in lines:
        print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")
