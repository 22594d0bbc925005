"""League measurements on the GPU (worker/league.py, rz_engine_set_nets).

(a) Cost of the generalised path: a two-model league (``set_nets`` with an alternating table) against the same games
    played through ``set_second_net``; ch5 networks (256 x 10, random-init), eval settings at 100 simulations, 512 games.
    The two are alternated ``--repeats`` times; their games must be identical.
(b) Throughput of a large league: eight ch5 networks with different random-init seeds, 28 pairs x 32 games, in one
    engine: games/s, node expansions/s, evaluator launches per wave and the tower's share of wave time.

    python tools/league_bench.py [--out league_bench.json]

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

import numpy as np  # noqa: E402

from reversi_zero_b200 import engine as E, net as N  # noqa: E402
from reversi_zero_b200.agent import model as M  # noqa: E402
from reversi_zero_b200.config import Config  # noqa: E402
from reversi_zero_b200.worker import league as L  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (x.strip() for x in out.split(","))
    return dict(name=name, power_limit=power, max_sm_clock=clock)


def make_nets(n, mc):
    nets = []
    for seed in range(n):
        net = N.Net(mc)
        net.load_weights(M.build_random_weights(mc, 1000 + seed))
        nets.append(net)
    return nets


def run_engine(pc, nets, games, black=None, white=None, seed=11):
    cfg = E.engine_cfg_from_play_config(pc, games=min(games, 4096), seed=seed, eval_mode=E.EVAL_NET, max_games=games,
                                        eval_cache_mb=-1)
    eng = E.Engine(cfg, nets[0])
    if black is None:
        eng.set_second_net(nets[1])
    else:
        eng.set_nets(nets, black, white)
    t0 = time.perf_counter()
    eng.run(finished_target=games)   # returns after the device has finished the last wave
    wall = time.perf_counter() - t0
    out = sorted(eng.poll(), key=lambda g: g["game_id"])
    st = eng.stats()
    eng.close()
    return wall, out, st


def key(g):
    return (g["game_id"], g["winner"], g["black"], g["white"], g["black_net"], g["white_net"],
            tuple((p["action"], tuple(p["N"])) for p in g["plies"]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--sims", type=int, default=100)
    ap.add_argument("--games", type=int, default=512)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--nets", type=int, default=8)
    ap.add_argument("--games-per-pair", type=int, default=32)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("league_bench.py measures on a CUDA device; none is visible")
    res = dict(card=card())
    cfg = Config()
    cfg.eval = dict(play_config=dict(simulation_num_per_move=args.sims))
    pc = L.league_play_config(cfg)
    ch5 = M.ModelConfig(256, 3, 10, 1e-4, 256)
    nets = make_nets(max(2, args.nets), ch5)

    # (a) two models: set_nets with the alternating table against set_second_net, alternated
    local = np.arange(args.games)
    black, white = (local & 1).astype(np.uint8), (1 - (local & 1)).astype(np.uint8)
    run_engine(pc, nets[:2], 64, black[:64], white[:64])   # warm-up: module loading, tower set-up
    walls = dict(set_second_net=[], set_nets=[])
    ref = None
    for _ in range(args.repeats):
        for name in ("set_second_net", "set_nets"):
            wall, games, st = run_engine(pc, nets[:2], args.games, *((None, None) if name == "set_second_net" else (black, white)))
            walls[name].append(wall)
            keys = [key(g) for g in games]
            assert len(keys) == args.games
            if ref is None:
                ref = keys
            assert keys == ref, f"{name}: games differ from the first run"
    res["a"] = dict(games=args.games, sims=args.sims, wall_s=walls, identical=True,
                    median_s={k: float(np.median(v)) for k, v in walls.items()})
    print(json.dumps(res["a"]), flush=True)

    # (b) a large league in one engine
    black, white = L.schedule(args.nets, args.games_per_pair)
    total = int(black.size)
    wall, games, st = run_engine(pc, nets[:args.nets], total, black, white)
    assert len(games) == total
    res["b"] = dict(nets=args.nets, pairs=args.nets * (args.nets - 1) // 2, games=total, sims=args.sims, wall_s=wall,
                    games_per_s=total / wall, expansions_per_s=st["expansions"] / wall, waves=st["waves"],
                    evaluator_launches_per_wave=st["nn_launches"] / st["waves"], nn_ms=st["nn_ms"], mcts_ms=st["mcts_ms"],
                    tower_share=st["nn_ms"] / (st["nn_ms"] + st["mcts_ms"]), nn_over_mcts=st["nn_ms"] / st["mcts_ms"])
    print(json.dumps(res["b"]), flush=True)
    for net in nets:
        net.close()
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
