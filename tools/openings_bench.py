"""Opening-suite measurements on the GPU (csrc/rz_openings.cu, lib/openings.py, rz_engine_set_openings).

(a) The enumerator: distinct openings and wall time (a host clock around the synchronous call) for 1 .. --max-plies
    plies; a level that does not fit in device memory ends the list.
(b) Scoring: the time of ``balanced_suite`` for an 8-ply suite with a ch5 network (256 x 10, random-init weights).
(c) Matches: --games games between two ch5 networks (random-init, seeds 1 and 2) under eval's rules
    (``eval_play_config`` of the default configuration: 400 simulations, argmax moves, no root noise), from the initial
    position and from the 8-ply suite of (b): distinct move sequences (opening included) and games/s.

    python tools/openings_bench.py [--out openings_bench.json] [--games 400] [--max-plies 12]

Needs a CUDA device; the card's name and power limit are read in the same run and stored with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "reversi-alpha-zero_b200")]

from reversi_zero_b200 import _cabi, net as N  # noqa: E402
from reversi_zero_b200.agent import model as M  # noqa: E402
from reversi_zero_b200.config import Config  # noqa: E402
from reversi_zero_b200.lib import openings as OP  # noqa: E402
from reversi_zero_b200.worker import evaluate as EV  # noqa: E402


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
    ap.add_argument("--out", default="openings_bench.json")
    ap.add_argument("--games", type=int, default=400)
    ap.add_argument("--max-plies", type=int, default=12)
    args = ap.parse_args()
    res = dict(card=card(), enumerate=[])
    OP.enumerate_openings(4)  # module load and first allocations
    for plies in range(1, args.max_plies + 1):
        t0 = time.perf_counter()
        try:
            ops = OP.enumerate_openings(plies)
        except _cabi.RzError as e:
            res["enumerate"].append(dict(plies=plies, error=str(e)))
            break
        dt = time.perf_counter() - t0
        res["enumerate"].append(dict(plies=plies, openings=int(ops.own.size), seconds=dt))
        print(f"plies {plies}: {ops.own.size} openings, {dt * 1e3:.1f} ms", flush=True)
        del ops
    nets = [ch5_net(1), ch5_net(2)]
    OP.balanced_suite(nets[0], 4, 10, 0.2, seed=1)  # warm-up of the evaluator
    t0 = time.perf_counter()
    suite = OP.balanced_suite(nets[0], 8, 500, 0.2, seed=20260922)
    res["score"] = dict(plies=8, openings=67239, kept=len(suite), seconds=time.perf_counter() - t0)
    print(f"score: {res['score']}", flush=True)
    cfg = Config()
    res["match"] = []
    for name, s in (("initial", None), ("suite8", [e.moves for e in suite])):
        t0 = time.perf_counter()
        results, games = EV.play_match(cfg, nets[0], nets[1], args.games, seed=7, suite=s)
        dt = time.perf_counter() - t0
        seqs = set()
        for i, g in enumerate(games):
            opening = tuple(EV.match_openings(args.games, s)[i]) if s else ()
            seqs.add(opening + tuple(p["action"] for p in g["plies"]))
        row = dict(start=name, games=len(games), distinct_sequences=len(seqs), seconds=dt, games_per_s=len(games) / dt,
                   challenger_wins=sum(r == 1 for r in results), draws=sum(r is None for r in results))
        res["match"].append(row)
        print(f"match: {row}", flush=True)
    for net in nets:
        net.close()
    with open(args.out, "wt") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
