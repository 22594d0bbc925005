"""Opening-book measurements on the GPU (csrc/rz_openings.cu rz_openings_book_graph, lib/book.py, NBoard's go).

(a) The graph: nodes, edges and wall time (a host clock around the synchronous call, median of --reps) at 6, 8 and 10 plies.
(b) Leaf search: positions per second of ``search_positions`` over the first --leaves 8-ply openings, at 400 simulations
    with a ch5 network (256 x 10, random-init weights), b200.games_per_gpu roots per call.
(c) The whole book at --plies (default 8) with that network: graph, searches and backup, and the backup alone.
(d) ``go`` latency: a book move against a level-N search (``set depth N``) of the same one-slot player, from the same
    position after one ply.
(e) Agreement: how often the book move equals the move of a single 400-simulation search at ply P - 1 (on --agree
    positions of level P - 1).

    python tools/book_bench.py [--out book_bench.json] [--plies 8] [--leaves 16384] [--depth 10] [--agree 200]

Needs a CUDA device; the card's name and power limit are read in the same run and stored with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "reversi-alpha-zero_b200")]

from reversi_zero_b200 import net as N  # noqa: E402
from reversi_zero_b200.agent import model as M  # noqa: E402
from reversi_zero_b200.agent.player import ReversiPlayer  # noqa: E402
from reversi_zero_b200.config import Config  # noqa: E402
from reversi_zero_b200.lib import book as BK  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in out.split(","))
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def ch5_net(seed):
    mc = M.ModelConfig(256, 3, 10, 1e-4, 256)
    net = N.Net(mc)
    net.load_weights(M.build_random_weights(mc, seed))
    return net


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="book_bench.json")
    ap.add_argument("--plies", type=int, default=8)
    ap.add_argument("--leaves", type=int, default=16384)
    ap.add_argument("--depth", type=int, default=10)
    ap.add_argument("--agree", type=int, default=200)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    res = dict(card=card(), graph=[])
    BK.book_graph(4)  # module load and first allocations
    for plies in (6, 8, 10):
        ts = []
        for _ in range(args.reps):
            t0 = time.perf_counter()
            g = BK.book_graph(plies)
            ts.append(time.perf_counter() - t0)
        row = dict(plies=plies, nodes=int(g.own.size), edges=int(g.edge_square.size), seconds_median=float(np.median(ts)),
                   seconds=ts)
        res["graph"].append(row)
        print(f"graph {row}", flush=True)
    cfg = Config()
    net = ch5_net(1)
    chunk = int(cfg.b200.games_per_gpu)
    g = BK.book_graph(8)
    first = BK.level_starts(g.level_counts)
    own, enemy = g.own[first[8]:][:args.leaves], g.enemy[first[8]:][:args.leaves]
    eng = BK.search_engine(cfg, net, 400, chunk, seed=1)
    BK.search_positions(eng, own[:chunk], enemy[:chunk], chunk)  # warm-up
    t0 = time.perf_counter()
    BK.search_positions(eng, own, enemy, chunk)
    dt = time.perf_counter() - t0
    eng.close()
    res["leaf_search"] = dict(positions=int(own.size), simulations=400, slots=chunk, seconds=dt, positions_per_s=own.size / dt)
    print(f"leaf search {res['leaf_search']}", flush=True)
    t0 = time.perf_counter()
    book = BK.build_book(cfg, net, args.plies, 400, seed=1)
    total = time.perf_counter() - t0
    g = BK.book_graph(args.plies)
    flags = BK.node_flags(g)
    searched = np.where(flags == BK.INTERIOR, 0.0, book.values)
    t0 = time.perf_counter()
    BK.backup(g, flags, searched)
    res["book"] = dict(plies=args.plies, nodes=int(book.values.size), searched=int((flags != BK.INTERIOR).sum()),
                       incomplete=int((flags == BK.INCOMPLETE).sum()), seconds=total, backup_seconds=time.perf_counter() - t0)
    print(f"book {res['book']}", flush=True)
    # go: a book move against a level-N search of the one-slot player, from the position after the first ply
    pc = SimpleNamespace(**vars(cfg.play))
    cfg.play_with_human.update_play_config(pc)
    pc.required_visit_to_decide_action = args.depth * cfg.nboard.simulation_num_per_depth_about
    pc.thinking_loop = min(30, int(pc.required_visit_to_decide_action * 5 / pc.simulation_num_per_move))
    player = ReversiPlayer(cfg, net, pc, enable_resign=False)
    pos = (int(g.own[1]), int(g.enemy[1]))
    book_t, search_t = [], []
    for _ in range(5):
        t0 = time.perf_counter()
        BK.best_move(book.moves(*pos))
        book_t.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        player.action(*pos)
        search_t.append(time.perf_counter() - t0)
    player.engine.close()
    res["go"] = dict(depth=args.depth, book_seconds_median=float(np.median(book_t)), search_seconds_median=float(np.median(search_t)))
    print(f"go {res['go']}", flush=True)
    # agreement at ply P - 1: the book move against the most visited move of one 400-simulation search
    lv = args.plies - 1
    nodes = [i for i in range(int(first[lv]), int(first[lv + 1])) if flags[i] == BK.INTERIOR][:args.agree]
    eng = BK.search_engine(cfg, net, 400, len(nodes), seed=1)
    n, _ = eng.search_roots(g.own[nodes], g.enemy[nodes], 1)
    eng.close()
    agree = sum(int(np.argmax(n[k])) == BK.best_move(book.moves(int(g.own[i]), int(g.enemy[i])))[0] for k, i in enumerate(nodes))
    res["agreement"] = dict(ply=lv, positions=len(nodes), same_move=int(agree))
    print(f"agreement {res['agreement']}", flush=True)
    net.close()
    with open(args.out, "wt") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
