"""Deep exact endgame solver (rz_solve_deep) over seeded positions at 14..24 empties: median and max seconds, timeouts,
probes, leaves, re-splits, node steps and the transposition table's counts per empty count; the lane solver (rz_solve)
and the deep solver at 12 empties for scale; and the card's name and power limit read in the same run.  Prints one JSON
line per row and a summary line; --out also writes the summary to a file.

Each position is solved cold (the table emptied before it) unless --sequence N is given: then the positions of one
seeded game from N empties down to 13 are solved in order with the table kept, as NBoard asks for them.  --lib runs
other builds of librz_engine.so in the same process (a build without a table, such as the parent commit's, runs without
clearing); the builds take turns position by position, each repeated --repeat times, so they share the card's state.

    python tools/deep_solver_bench.py [--empties 14 16 18 20 22 24] [--positions 4] [--timeout 60] [--sequence 24]
                                      [--lib OTHER/librz_engine.so ...] [--repeat 1] [--out f.json]
"""
import argparse
import ctypes as C
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
from reversi_zero_b200 import _cabi  # noqa: E402
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


def game_sequence(seed, start):
    """the positions of one seeded random game from `start` empties down to 13 (the side to move of an unfinished game
    always has a move: the environment passes for it)"""
    rng = np.random.default_rng(seed)
    while True:
        e, out = ob.Env().reset(), []
        while not e.done:
            o, en = e.own_enemy()
            if 13 <= 64 - bin(o | en).count("1") <= start:
                out.append((o, en))
            legal = ob.find_correct_moves(o, en)
            ms = [i for i in range(64) if legal >> i & 1]
            e.step(ms[rng.integers(len(ms))])
        if out and 64 - bin(out[0][0] | out[0][1]).count("1") == start:
            return out


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().split("\n")[0]
    except (OSError, subprocess.TimeoutExpired):
        return "unknown"


class Build:
    """one librz_engine.so: the tree's (through _cabi) or another loaded beside it"""

    def __init__(self, path=None):
        self.path = os.path.abspath(path) if path else _cabi.LIB_PATH
        self.lib = C.CDLL(self.path) if path else _cabi.lib()
        self.lib.rz_solve_deep.restype = C.c_int
        self.lib.rz_solve_deep.argtypes = _cabi.SIGNATURES["rz_solve_deep"][1]
        self.table = getattr(self.lib, "rz_solve_deep_table_stats", None) is not None
        if self.table:
            for name in ("rz_solve_deep_clear", "rz_solve_deep_table_stats"):
                fn = getattr(self.lib, name)
                fn.restype, fn.argtypes = _cabi.SIGNATURES[name]

    def clear(self):
        if self.table and self.lib.rz_solve_deep_clear() != 0:
            raise RuntimeError("rz_solve_deep_clear failed")

    def table_stats(self):
        if not self.table:
            return None
        st = _cabi.DeepTableStats()
        if self.lib.rz_solve_deep_table_stats(C.byref(st)) != 0:
            raise RuntimeError("rz_solve_deep_table_stats failed")
        return {k: getattr(st, k) for k, _ in _cabi.DeepTableStats._fields_}

    def solve(self, own, enemy, timeout):
        o, e = np.array([own], np.uint64), np.array([enemy], np.uint64)
        mv, sc, st = np.empty(1, np.int8), np.empty(1, np.int8), _cabi.DeepSolveStats()
        rc = self.lib.rz_solve_deep(o.ctypes.data_as(_cabi.u64p), e.ctypes.data_as(_cabi.u64p), mv.ctypes.data_as(_cabi.i8p),
                                    sc.ctypes.data_as(_cabi.i8p), 1, float(timeout), C.byref(st))
        if rc != 0:
            raise RuntimeError(f"rz_solve_deep failed ({rc}) in {self.path}")
        return int(mv[0]), int(sc[0]), {k: getattr(st, k) for k, _ in _cabi.DeepSolveStats._fields_ if k != "pad"}


def add_table_delta(acc, before, after):
    """the table's counts over one solve added to acc; occupied and bytes are the last ones seen"""
    if before is None:
        return None
    acc = dict(acc or {})
    for k in after:
        acc[k] = after[k] if k in ("occupied", "bytes") else acc.get(k, 0) + after[k] - before[k]
    return acc


def run_row(builds, label, pos, timeout, cold, repeat):
    """solve `pos` with every build, taking turns position by position -> one row per build"""
    sts = [[] for _ in builds]
    answers = [[] for _ in builds]
    tables = [None for _ in builds]
    if not cold:
        for b in builds:
            b.clear()
    for i, (own, enemy) in enumerate(pos):
        order = list(range(len(builds)))
        if i % 2:
            order.reverse()
        for r in range(repeat):
            for j in order:
                if cold:
                    builds[j].clear()
                before = builds[j].table_stats()
                mv, sc, st = builds[j].solve(own, enemy, timeout)
                tables[j] = add_table_delta(tables[j], before, builds[j].table_stats())
                sts[j].append(st)
                if r == 0:
                    answers[j].append((mv, sc))
                print(json.dumps({"row": label, "build": j, "position": i, "move": mv, "score": sc, **st}), flush=True)
    rows = []
    for j, b in enumerate(builds):
        secs = [s["seconds"] for s in sts[j]]
        rows.append({"row": label, "build": j, "positions": len(pos), "repeat": repeat,
                     "timeouts": sum(int(m < 0) for m, _ in answers[j]),
                     "median_s": float(np.median(secs)), "max_s": float(np.max(secs)), "sum_s": float(np.sum(secs)),
                     "node_steps": int(sum(s["node_steps"] for s in sts[j])),
                     "probes": float(np.mean([s["probes"] for s in sts[j]])),
                     "leaves": float(np.mean([s["leaves"] for s in sts[j]])),
                     "resplits": float(np.mean([s["resplits"] for s in sts[j]])),
                     "slices": float(np.mean([s["slices"] for s in sts[j]])),
                     "node_steps_per_s": float(sum(s["node_steps"] for s in sts[j]) / max(1e-9, sum(secs))),
                     "table": tables[j],
                     "seconds_each": secs})
    # answers of builds agree wherever neither timed out
    for j in range(1, len(builds)):
        for a, b in zip(answers[0], answers[j]):
            if a[0] >= 0 and b[0] >= 0 and a != b:
                raise RuntimeError(f"builds 0 and {j} disagree on {label}: {a} vs {b}")
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--empties", type=int, nargs="*", default=[14, 16, 18, 20, 22, 24])
    ap.add_argument("--positions", type=int, default=4)
    ap.add_argument("--timeout", type=float, default=60.0)
    ap.add_argument("--sequence", type=int, default=None, help="also solve one seeded game from N empties down to 13")
    ap.add_argument("--lib", action="append", default=[], help="another build of librz_engine.so (repeatable)")
    ap.add_argument("--repeat", type=int, default=1)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    builds = [Build()] + [Build(p) for p in a.lib]
    res = {"card": card(), "timeout_s": a.timeout, "builds": [b.path for b in builds], "rows": []}
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
    for b in builds:
        b.solve(p12[0][0], p12[0][1], a.timeout)  # allocates the workspace
    res["lane_12"] = {"batch_256_s": batch_s, "one_median_s": float(np.median(one)), "one_max_s": float(np.max(one))}
    print(json.dumps({"lane_12": res["lane_12"]}), flush=True)
    rows = run_row(builds, 12, p12[:16], a.timeout, True, a.repeat)
    for k in a.empties:
        rows += run_row(builds, k, positions(1000 + k, a.positions, k), a.timeout, True, a.repeat)
    if a.sequence:
        rows += run_row(builds, f"sequence_{a.sequence}", game_sequence(2000 + a.sequence, a.sequence), a.timeout, False, 1)
    for row in rows:
        print(json.dumps({k: v for k, v in row.items() if k != "seconds_each"}), flush=True)
    res["rows"] = rows
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
