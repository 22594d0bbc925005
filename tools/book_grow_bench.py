"""Measurements of a growing opening book on the GPU (csrc/rz_openings.cu rz_openings_book_children, lib/book.py grow and
learn_game).

(a) The children call: wall time (a host clock around the synchronous call, median of --reps) over every node of the
    8-ply graph's level 7 against level 8's keys.
(b) Growth: an 8-ply book searched at --sims simulations with a ch5 network (256 x 10, random-init weights) grown by
    --grow nodes in rounds of --batch, with the depth cost --cost and max_level 40.  Reports positions searched per
    second and how the time splits between the searches, the children calls and the host's selection, merge and backup.
(c) NBoard's ``learn``: the wall time of learn_game on a seeded random game of 60 plies plus the book's save, with a
    fresh engine as NBoardEngine.learn makes it, median of 3 games.

    python tools/book_grow_bench.py [--out book_grow_bench.json] [--sims 400] [--grow 3000] [--batch 256] [--cost 0.05]

Needs a CUDA device; the card's name and power limit are read in the same run and stored with the numbers.
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "reversi-alpha-zero_b200"), os.path.join(ROOT, "tools")]

from book_bench import card, ch5_net  # noqa: E402
from reversi_zero_b200.config import Config  # noqa: E402
from reversi_zero_b200.lib import bitboard as bb, book as BK  # noqa: E402


class Timed:
    """a callable that adds its wall time and call count up"""

    def __init__(self, fn):
        self.fn, self.seconds, self.calls, self.items = fn, 0.0, 0, 0

    def __call__(self, *args):
        t0 = time.perf_counter()
        out = self.fn(*args)
        self.seconds += time.perf_counter() - t0
        self.calls += 1
        self.items += len(args[0])
        return out


def random_game(rng, plies=60):
    own, enemy = BK.START
    moves = []
    while len(moves) < plies:
        legal = [s for s in range(64) if (bb.find_correct_moves(own, enemy) >> s) & 1]
        if not legal:
            if not bb.find_correct_moves(enemy, own):
                break
            moves.append(None)
            own, enemy = enemy, own
            continue
        a = int(rng.choice(legal))
        moves.append(a)
        fl = bb.calc_flip(a, own, enemy)
        own, enemy = enemy ^ fl, own | fl | (1 << a)
    return moves


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="book_grow_bench.json")
    ap.add_argument("--sims", type=int, default=400)
    ap.add_argument("--grow", type=int, default=3000)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--cost", type=float, default=0.05)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    res = dict(card=card())
    g = BK.book_graph(8)
    first = BK.level_starts(g.level_counts)
    a, b, c = (int(first[k]) for k in (7, 8, 9))
    BK.book_children(g.own[:1], g.enemy[:1], [], [])   # module load and first allocations
    ts = []
    for _ in range(args.reps):
        t0 = time.perf_counter()
        ch = BK.book_children(g.own[a:b], g.enemy[a:b], g.key_hi[b:c], g.key_lo[b:c])
        ts.append(time.perf_counter() - t0)
    res["children"] = dict(nodes=b - a, edges=int(ch.edge_square.size), seconds_median=float(np.median(ts)), seconds=ts)
    print(f"children {res['children']}", flush=True)
    cfg = Config()
    net = ch5_net(1)
    t0 = time.perf_counter()
    book = BK.build_book(cfg, net, 8, args.sims, seed=1)
    res["build"] = dict(plies=8, nodes=int(book.values.size), seconds=time.perf_counter() - t0)
    print(f"build {res['build']}", flush=True)
    search = BK.Searcher(cfg, net, book)
    children = Timed(BK.book_children)
    timed_search = Timed(search)
    try:
        t0 = time.perf_counter()
        grown = BK.grow(book, args.grow, args.batch, BK.MAX_LEVEL, args.cost, children, timed_search)
        total = time.perf_counter() - t0
    finally:
        search.close()
    host = total - children.seconds - timed_search.seconds
    res["grow"] = dict(expansions=args.grow, batch=args.batch, depth_cost=args.cost, simulations=args.sims,
                       nodes_before=int(book.values.size), nodes_after=int(grown.values.size), levels=grown.levels,
                       searched=timed_search.items, seconds=total, search_seconds=timed_search.seconds,
                       positions_per_s=timed_search.items / max(timed_search.seconds, 1e-9),
                       children_seconds=children.seconds, children_calls=children.calls,
                       host_seconds=host, level_counts=grown.level_counts.tolist())
    print(f"grow {res['grow']}", flush=True)
    rng = np.random.default_rng(7)
    learn = []
    with tempfile.TemporaryDirectory() as tmp:
        for _ in range(3):
            moves = random_game(rng)
            t0 = time.perf_counter()
            s = BK.Searcher(cfg, net, grown)
            try:
                learned, k = BK.learn_game(grown, moves, BK.MAX_LEVEL, search=s)
            finally:
                s.close()
            BK.save_book(os.path.join(tmp, "book.npz"), learned)
            learn.append(dict(seconds=time.perf_counter() - t0, expanded=k,
                              searched=int(learned.values.size - grown.values.size)))
    res["learn"] = dict(games=learn, seconds_median=float(np.median([x["seconds"] for x in learn])))
    print(f"learn {res['learn']}", flush=True)
    net.close()
    with open(args.out, "wt") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
