"""Deep exact endgame solver (rz_solve_deep) over seeded positions at 14..24 empties: median and max seconds, probes,
leaves, re-splits and node steps per second per empty count, the lane solver (rz_solve) at 12 empties for scale, and the
card's name and power limit read in the same run.  Prints one JSON line; --out also writes it to a file.

    python tools/deep_solver_bench.py [--empties 14 16 18 20 22 24] [--positions 4] [--timeout 60] [--out f.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "reversi-alpha-zero_b200")):
    sys.path.insert(0, p)

from oracle import bitboard as ob  # noqa: E402
from reversi_zero_b200.lib import reversi_solver as zs  # noqa: E402


def positions(seed, n, empties):
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        e = ob.Env().reset()
        while not e.done and 60 - e.turn > empties:
            o, en = e.own_enemy()
            legal = ob.find_correct_moves(o, en)
            ms = [i for i in range(64) if legal >> i & 1]
            e.step(ms[rng.integers(len(ms))])
        if not e.done and 60 - e.turn == empties:
            out.append(e.own_enemy())
    return out


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().split("\n")[0]
    except (OSError, subprocess.TimeoutExpired):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--empties", type=int, nargs="+", default=[14, 16, 18, 20, 22, 24])
    ap.add_argument("--positions", type=int, default=4)
    ap.add_argument("--timeout", type=float, default=60.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "timeout_s": a.timeout, "rows": []}
    # lane solver at 12 empties, for scale: one launch over the batch, and one position at a time
    p12 = positions(12, 256, 12)
    o, e = np.array([p[0] for p in p12], np.uint64), np.array([p[1] for p in p12], np.uint64)
    zs.solve_batch(o[:4], e[:4], True)
    t0 = time.perf_counter()
    zs.solve_batch(o, e, True)
    batch_s = time.perf_counter() - t0
    one = []
    for i in range(16):
        t0 = time.perf_counter()
        zs.solve_batch(o[i:i + 1], e[i:i + 1], True)
        one.append(time.perf_counter() - t0)
    deep12 = []
    zs.solve_deep_batch(o[:2], e[:2])  # allocates the workspace
    for i in range(16):
        _, _, st = zs.solve_deep_batch(o[i:i + 1], e[i:i + 1], stats=True)
        deep12.append(st[0]["seconds"])
    res["lane_12"] = {"batch_256_s": batch_s, "one_median_s": float(np.median(one)), "one_max_s": float(np.max(one)),
                      "deep_one_median_s": float(np.median(deep12))}
    print(json.dumps({"lane_12": res["lane_12"]}), flush=True)
    for k in a.empties:
        pos = positions(1000 + k, a.positions, k)
        sts, timeouts = [], 0
        for own, enemy in pos:
            mv, _, st = zs.solve_deep_batch([own], [enemy], timeout=a.timeout, stats=True)
            timeouts += int(mv[0] < 0)
            sts.append(st[0])
            print(json.dumps({"empties": k, "move": int(mv[0]), **st[0]}), flush=True)
        secs = [s["seconds"] for s in sts]
        row = {"empties": k, "positions": len(pos), "timeouts": timeouts, "median_s": float(np.median(secs)),
               "max_s": float(np.max(secs)), "probes": float(np.mean([s["probes"] for s in sts])),
               "leaves": float(np.mean([s["leaves"] for s in sts])), "resplits": float(np.mean([s["resplits"] for s in sts])),
               "slices": float(np.mean([s["slices"] for s in sts])),
               "node_steps_per_s": float(sum(s["node_steps"] for s in sts) / max(1e-9, sum(secs)))}
        res["rows"].append(row)
        print(json.dumps(row), flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
