"""The value of every root move (rz_solve_deep_moves, NBoard's exact hints) over seeded positions at 10..20 empties, with
the card's name and power limit read in the same run.  Per position, each arm starts from an empty transposition table,
and the arms take turns in an order that alternates from position to position:
  moves_all    solve_moves with n_best = 0 (every move exact), one forest per round;
  moves_best3  solve_moves with n_best = 3 (the best three exact);
  children     the host-only alternative: rz_solve_deep of each move's child in turn, with the table kept between them
               (negated where the opponent moves, not after its pass; a move that ends the game counts its discs);
  root         one rz_solve_deep of the root (best move and value only), for scale;
  lane         up to 12 empties: every child in one lane-solver launch (ReversiSolver.solve_moves' path there).
Arms moves_all and children must give the same values; the tool stops with an error otherwise.  Prints one JSON line per
position and arm, one per row with the medians, and a summary line; --out also writes the summary to a file.

    python tools/deep_moves_bench.py [--empties 10 12 14 16 18 20] [--positions 4] [--timeout 120] [--out f.json]
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


def arm_moves(own, enemy, n_best, timeout):
    got, st = zs.solve_moves(own, enemy, n_best, timeout, stats=True)
    return got, st["node_steps"], st["probes"]


def arm_children(own, enemy, timeout):
    """rz_solve_deep of each child in turn, the table kept -> ({square: (v, v)}, node steps, solves)"""
    legal = ob.find_correct_moves(own, enemy)
    out, steps, solves = {}, 0, 0
    for a in range(64):
        if not legal >> a & 1:
            continue
        fl = ob.calc_flip(a, own, enemy)
        o2, e2 = own | fl | (1 << a), enemy ^ fl
        if ob.find_correct_moves(e2, o2):
            kid, sign = (e2, o2), -1
        elif ob.find_correct_moves(o2, e2):
            kid, sign = (o2, e2), 1
        else:
            v = bin(o2).count("1") - bin(e2).count("1")
            out[a] = (v, v)
            continue
        mv, sc, st = zs.solve_deep_batch([kid[0]], [kid[1]], timeout, stats=True)
        steps += st[0]["node_steps"]
        solves += 1
        v = sign * int(sc[0]) if mv[0] >= 0 else None
        out[a] = (v, v) if v is not None else (-64, 64)
    return out, steps, solves


def arm_root(own, enemy, timeout):
    mv, sc, st = zs.solve_deep_batch([own], [enemy], timeout, stats=True)
    return {int(mv[0]): (int(sc[0]), int(sc[0]))} if mv[0] >= 0 else {}, st[0]["node_steps"], st[0]["probes"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--empties", type=int, nargs="*", default=[10, 12, 14, 16, 18, 20])
    ap.add_argument("--positions", type=int, default=4)
    ap.add_argument("--timeout", type=float, default=120.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "timeout_s": a.timeout, "rows": []}
    print(json.dumps({"card": res["card"]}), flush=True)
    arms = {"moves_all": lambda o, e: arm_moves(o, e, 0, a.timeout),
            "moves_best3": lambda o, e: arm_moves(o, e, 3, a.timeout),
            "children": lambda o, e: arm_children(o, e, a.timeout),
            "root": lambda o, e: arm_root(o, e, a.timeout)}
    lane_solver = zs.ReversiSolver()
    warm = positions(5, 1, 14)[0]
    for f in arms.values():   # workspace, modules and the lane solver loaded before anything is timed
        f(*warm)
    lane_solver.solve_moves(*positions(6, 1, 10)[0], 1)
    for k in a.empties:
        names = list(arms) + (["lane"] if k <= zs.LANE_MAX_EMPTIES else [])
        secs = {n: [] for n in names}
        steps = {n: 0 for n in names}
        for i, (own, enemy) in enumerate(positions(3000 + k, a.positions, k)):
            order = names if i % 2 == 0 else names[::-1]
            vals = {}
            for n in order:
                zs.clear_deep_table()
                t0 = time.perf_counter()
                if n == "lane":
                    got, st, extra = lane_solver.solve_moves(own, enemy, 1), 0, 1
                else:
                    got, st, extra = arms[n](own, enemy)
                dt = time.perf_counter() - t0
                secs[n].append(dt)
                steps[n] += st
                vals[n] = got
                print(json.dumps({"empties": k, "position": i, "arm": n, "seconds": dt, "node_steps": st,
                                  "forests_or_solves": extra, "moves": len(got),
                                  "exact": sum(lo == hi for lo, hi in got.values())}), flush=True)
            if vals["moves_all"] != vals["children"]:
                raise RuntimeError(f"solve_moves and the children's solves disagree at {k} empties, position {i}: "
                                   f"{vals['moves_all']} vs {vals['children']}")
            if "lane" in vals and vals["lane"] != vals["moves_all"]:
                raise RuntimeError(f"lane and deep paths disagree at {k} empties, position {i}")
        row = {"empties": k, "positions": a.positions}
        for n in names:
            row[n] = {"median_s": float(np.median(secs[n])), "max_s": float(np.max(secs[n])), "node_steps": int(steps[n])}
        print(json.dumps(row), flush=True)
        res["rows"].append(row)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
