"""Whole-game analysis on the device (play_game/analysis.py), measured on a seeded full game with a ch5 network of
random weights at 400 simulations:

(a) the searched positions all at once through ``Engine.search_roots`` (64 slots) against the same positions one at a
    time through a one-slot engine, alternated three times; the root statistics must be identical;
(b) with ``use_solver_turn: 40`` and ``solver_max_empties: 20``, the exact part in retrograde order (fewest empties first)
    with the deep solver's table kept, against each position solved after ``clear_deep_table()``.

    python tools/analysis_bench.py [--seed 7] [--sims 400] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, "reversi-alpha-zero_b200"), ROOT]

import numpy as np  # noqa: E402

from reversi_zero_b200 import engine as E, net as N  # noqa: E402
from reversi_zero_b200.agent import model as M  # noqa: E402
from reversi_zero_b200.agent.player import search_play_config  # noqa: E402
from reversi_zero_b200.config import load_yaml  # noqa: E402
from reversi_zero_b200.lib import reversi_solver as zs  # noqa: E402
from reversi_zero_b200.lib.bitboard import bit_count, find_correct_moves, calc_flip  # noqa: E402
from reversi_zero_b200.play_game import analysis as A  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        return out
    except Exception as ex:  # noqa: BLE001
        return f"unknown ({ex})"


def seeded_game(seed):
    rng = np.random.default_rng(seed)
    own, enemy, actions = 1 << 28 | 1 << 35, 1 << 27 | 1 << 36, []
    while True:
        m = find_correct_moves(own, enemy)
        if not m:
            if not find_correct_moves(enemy, own):
                return actions
            actions.append(None)
            own, enemy = enemy, own
            continue
        ms = [i for i in range(64) if m >> i & 1]
        a = ms[rng.integers(len(ms))]
        f = calc_flip(a, own, enemy)
        own, enemy = enemy ^ f, own | f | 1 << a
        actions.append(a)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seed", type=int, default=7)
    ap.add_argument("--sims", type=int, default=400)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    cfg = load_yaml(os.path.join(ROOT, "tests", "golden", "ref_config", "ch5.yml"), project_dir=tempfile.mkdtemp())
    cfg.play_with_human.update_play_config(cfg.play)
    cfg.play.simulation_num_per_move = args.sims
    net = N.Net(cfg.model)
    net.load_weights(M.build_random_weights(cfg.model, 5))
    actions = seeded_game(args.seed)
    pos = A.enumerate_positions(1 << 28 | 1 << 35, 1 << 27 | 1 << 36, 1, actions)
    roots = [(k[2], k[3]) for k in A.classify(pos) if k[0] != "over"]
    roots = list(dict.fromkeys(roots))
    per_sim = int(cfg.nboard.hint_callback_per_sim)
    chunks = A.chunk_steps(args.sims, per_sim)
    pc = search_play_config(cfg, cfg.play)

    # (a) searched positions: 64 slots at once against one slot at a time
    own, enemy = [r[0] for r in roots], [r[1] for r in roots]
    t_many, t_one, ref = [], [], None
    for rep in range(args.reps):
        for which in ("many", "one"):
            # a fresh evaluation cache each time, so neither side is served by the other's or its own earlier leaves
            eng = E.Engine(E.engine_cfg_from_play_config(pc, games=A.ANALYSIS_SLOTS if which == "many" else 1,
                                                         max_searches_per_game=1 if which == "many" else 0,
                                                         eval_cache_mb=A.ANALYSIS_CACHE_MB if which == "many" else 0), net)
            t0 = time.perf_counter()
            if which == "many":
                for k, step in enumerate(chunks):
                    eng.set_simulation_num(step)
                    n, w = eng.search_roots(own, enemy, 1, keep_tree=k > 0)
            else:
                n, w = np.zeros((len(roots), 64), np.int32), np.zeros((len(roots), 64), np.float32)
                for i, (o, e) in enumerate(roots):
                    for k, step in enumerate(chunks):
                        eng.set_simulation_num(step)
                        n[i], w[i] = eng.search_root(o, e, 1, 0, keep_tree=k > 0)
            dt = time.perf_counter() - t0
            eng.close()
            (t_many if which == "many" else t_one).append(dt)
            if ref is None:
                ref = (n.copy(), w.copy())
            assert np.array_equal(ref[0], n) and np.array_equal(ref[1].view(np.uint32), w.view(np.uint32)), (rep, which)
    print(json.dumps({"part": "a", "positions": len(roots), "sims": args.sims, "chunks": len(chunks),
                      "search_roots_s": [round(t, 3) for t in t_many], "one_slot_s": [round(t, 3) for t in t_one],
                      "identical": True}), flush=True)

    # (b) the exact part: retrograde with the table kept against each position cold
    exact = [r for r in roots if bit_count(r[0] | r[1]) - 4 >= 40 and 12 < 64 - bit_count(r[0] | r[1]) <= 20]
    exact.sort(key=lambda r: 64 - bit_count(r[0] | r[1]))
    zs.clear_deep_table()
    retro = [zs.solve_deep_batch([o], [e], 30.0, stats=True) for o, e in exact]
    cold = []
    for o, e in exact:
        zs.clear_deep_table()
        cold.append(zs.solve_deep_batch([o], [e], 30.0, stats=True))
    rows = []
    for (o, e), r, c in zip(exact, retro, cold):
        assert r[0][0] < 0 or c[0][0] < 0 or (r[0][0], r[1][0]) == (c[0][0], c[1][0])
        rows.append({"empties": 64 - bit_count(o | e), "retro_s": round(r[2][0]["seconds"], 3), "cold_s": round(c[2][0]["seconds"], 3),
                     "retro_steps": r[2][0]["node_steps"], "cold_steps": c[2][0]["node_steps"],
                     "retro_timeout": bool(r[0][0] < 0), "cold_timeout": bool(c[0][0] < 0)})
    print(json.dumps({"part": "b", "rows": rows,
                      "retro_total_s": round(sum(x["retro_s"] for x in rows), 3), "cold_total_s": round(sum(x["cold_s"] for x in rows), 3),
                      "retro_total_steps": sum(x["retro_steps"] for x in rows), "cold_total_steps": sum(x["cold_steps"] for x in rows)}),
          flush=True)


if __name__ == "__main__":
    main()
