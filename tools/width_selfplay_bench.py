"""Self-play throughput as a function of the network width: bench.py's ch5 workload (4096 games, 400 simulations, K = 8,
warm start, solver and resignation off) with cnn_filter_num set per run (10 blocks, value head 256, random-init weights).

python tools/width_selfplay_bench.py [--filters 256 128 64] [--steps 3] [--warmup 3] [--games 4096]

Prints one JSON line per width: games/s (games finished in the timed window), node expansions/s, the tower's share of
wave time (one slot group, so that the events around each tower launch bracket that kernel alone), the implementation
AUTO ran, and the card name, power limit and median SM clock read in the same run."""
import argparse
import json
import os
import subprocess
import sys
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "reversi-alpha-zero_b200"))
import bench  # noqa: E402  (the workload definition and helpers; not modified here)


def power_limit_w(index=0):
    try:
        out = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout
        return float(out.strip().splitlines()[0])
    except Exception:
        return None


def run(filters, steps, warmup, games):
    import torch
    from reversi_zero_b200.agent import model as M
    from reversi_zero_b200 import net as N, engine as E
    mc = M.ModelConfig(**dict(bench.MODEL_KW, cnn_filter_num=filters))
    net = N.Net(mc)
    net.load_blob(M.weights_to_blob(mc, M.build_random_weights(mc, 0)))
    pp = SimpleNamespace(required_visit_to_decide_action=400, start_rethinking_turn=8, allowed_resign_turn=20,
                         disable_resignation_rate=0.1, **bench.PLAY_KW)
    profile, profile_src = bench.warm_start_profile()
    wps = bench.waves_per_step()

    def make_engine(groups):
        cfg = E.engine_cfg_from_play_config(pp, games=games, seed=20260922, eval_mode=E.EVAL_NET, warm_start=True,
                                            overlap_groups=groups)
        eng = E.Engine(cfg, net)
        if profile is not None:
            eng.set_warm_start_profile(profile)
        return eng

    eng = make_engine(0)
    eng.run(max_waves=warmup * wps)
    eng.poll()
    s0 = eng.stats()
    sampler = bench.ClockSampler(0)
    torch.cuda.synchronize()
    sampler.start()
    eng.run(max_waves=steps * wps)
    torch.cuda.synchronize()
    clocks = sampler.stop()
    s1 = eng.stats()
    eng.close()
    d = {k: s1[k] - s0[k] for k in s1}
    secs = d["run_ms"] / 1e3
    eng1 = make_engine(1)   # tower share: one slot group
    eng1.run(max_waves=warmup * 4)
    r0 = eng1.stats()
    eng1.run(max_waves=48)
    r1 = eng1.stats()
    eng1.close()
    roof = {k: r1[k] - r0[k] for k in r1}
    out = dict(filters=filters, res_blocks=mc.res_layer_num, impl_auto=net.select_impl(games * bench.PLAY_KW["parallel_search_num"]),
               games_per_s=d["games_finished"] / secs, expansions_per_s=d["expansions"] / secs,
               tower_share_of_wave=roof["nn_ms"] / roof["run_ms"] if roof["run_ms"] else None,
               games_finished=d["games_finished"], seconds=secs, steps=steps, games=games,
               gpu=torch.cuda.get_device_name(), power_limit_w=power_limit_w(), sm_mhz=clocks["sm_mhz"],
               clock_reasons=clocks["reasons"], warm_start=profile_src)
    net.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--filters", type=int, nargs="+", default=[256, 128, 64])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--games", type=int, default=4096)
    args = ap.parse_args()
    for f in args.filters:
        print(json.dumps(run(f, args.steps, args.warmup, args.games)), flush=True)


if __name__ == "__main__":
    main()
