"""Latency of the policy/value tower at the batch sizes of a single-game search, split (RZ_NET_IMPL_SPLIT) vs throughput
(RZ_NET_IMPL_TCGEN05) tower, and one 400-simulation search (K = 8) under AUTO and with the throughput tower forced.
Prints one JSON line; the card's name, power limit and max SM clock are read in the same run.

    python tools/search_latency_bench.py [--blocks 10 19] [--min-seconds 1.0]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "reversi-alpha-zero_b200")):
    sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import mcts  # noqa: E402
from reversi_zero_b200 import engine as E  # noqa: E402
from reversi_zero_b200.agent import model as M  # noqa: E402
from reversi_zero_b200.net import Net, IMPL_AUTO, IMPL_TCGEN05, IMPL_SPLIT  # noqa: E402

NS = (1, 2, 4, 8, 16, 32, 64)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def tower_ms(net, n, impl, min_seconds):
    rng = np.random.default_rng(n)
    occ = torch.from_numpy(rng.integers(0, 2 ** 63, size=n, dtype=np.int64)).cuda()
    r = torch.from_numpy(rng.integers(0, 2 ** 63, size=n, dtype=np.int64)).cuda()
    own, enemy = occ & r, occ & ~r
    pol, val = torch.empty((n, 64), device="cuda"), torch.empty((n,), device="cuda")
    for _ in range(20):
        net.predict_dev(own, enemy, pol, val, n, impl)
    torch.cuda.synchronize()
    reps, ms = 50, 0.0
    while True:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            net.predict_dev(own, enemy, pol, val, n, impl)
        b.record()
        b.synchronize()
        ms = a.elapsed_time(b)
        if ms >= 1000.0 * min_seconds:
            return ms / reps
        reps = int(reps * max(2.0, 1.2 * 1000.0 * min_seconds / max(ms, 1e-3)))


def search_ms(net, impl, reps=5):
    pp = mcts.PlayParams(simulation_num_per_move=400, parallel_search_num=8, c_puct=5, noise_eps=0.0)
    own, enemy = 0x00000000081d0603, 0x0002043814020100   # a midgame position
    eng = E.Engine(E.engine_cfg_from_play_config(pp, games=1, seed=3, net_impl=impl), net)
    eng.search_root(own, enemy, 1, 0)
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        eng.search_root(own, enemy, 1, 0)   # fresh tree each time
        t.append(1000.0 * (time.perf_counter() - t0))
    eng.close()
    return float(np.median(t))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, nargs="+", default=[10, 19])
    ap.add_argument("--min-seconds", type=float, default=1.0)
    args = ap.parse_args()
    out = dict(card=card(), tower_ms={})
    for blocks in args.blocks:
        mc = M.ModelConfig(cnn_filter_num=256, res_layer_num=blocks, value_fc_size=256)
        net = Net(mc)
        net.load_weights(M.build_random_weights(mc, 0))
        out["tower_ms"][f"{blocks}_blocks"] = {
            name: {str(n): round(tower_ms(net, n, impl, args.min_seconds), 4) for n in NS}
            for name, impl in (("split", IMPL_SPLIT), ("throughput", IMPL_TCGEN05))}
        if blocks == 10:
            out["search_400_sims_ms"] = dict(auto=round(search_ms(net, IMPL_AUTO), 2), throughput=round(search_ms(net, IMPL_TCGEN05), 2))
            out["auto_impl_at_8"] = net.select_impl(8)
        net.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
