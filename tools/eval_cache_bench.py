"""Evaluation cache on bench.py's workload (ch5 random-init, 4096 games, 400 simulations, K = 8, warm start with
profiles/full_games.json, solver and resignation off): engines with the cache off and on, alternately, in one process.

python tools/eval_cache_bench.py [--pairs 5] [--steps 3] [--warmup 3] [--games 4096]

Per run it prints one JSON line: games finished in the timed window per second (bench.py's `value`), the renewal estimate
(expansions/s over expansions per complete game), expansions, the rows the tower really ran (`tower_rows`), the cache's
lookups and hits -- in total, for the games the engine started from the opening during the run, and per turn of the
searched root -- the within-wave repeats, the tower's own rate from tower_rows, and the card, power limit and median SM
clock read in the same run.  The last line summarises the pairs: mean gain and the spread of each arm.

Warm-started slots play their first game from a randomly played opening (engine warm_start), whose positions rarely
repeat across games, so the hit rate that says what the cache does in a long run is the one over games started inside
the run (turn buckets 0..59)."""
import argparse
import json
import os
import statistics
import sys
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "reversi-alpha-zero_b200"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench  # noqa: E402  (the workload definition and helpers; not modified here)
from width_selfplay_bench import power_limit_w  # noqa: E402


def run_one(net, pp, games, steps, warmup, cache_mb):
    import torch
    from reversi_zero_b200 import engine as E
    profile, profile_src = bench.warm_start_profile()
    wps = bench.waves_per_step()
    cfg = E.engine_cfg_from_play_config(pp, games=games, seed=20260922, eval_mode=E.EVAL_NET, warm_start=True, eval_cache_mb=cache_mb)
    eng = E.Engine(cfg, net)
    if profile is not None:
        eng.set_warm_start_profile(profile)
    eng.run(max_waves=warmup * wps)
    eng.poll()
    s0 = eng.stats()
    l0, h0 = eng.cache_turn_stats()
    sampler = bench.ClockSampler(0)
    torch.cuda.synchronize()
    sampler.start()
    eng.run(max_waves=steps * wps)
    torch.cuda.synchronize()
    clocks = sampler.stop()
    s1 = eng.stats()
    l1, h1 = eng.cache_turn_stats()
    eng.close()
    d = {k: s1[k] - s0[k] for k in s1}
    lk, ht = (l1 - l0).astype(int), (h1 - h0).astype(int)
    secs = d["run_ms"] / 1e3
    epg, _ = bench.expansions_per_game()
    fresh_l, fresh_h = int(lk[:60].sum()), int(ht[:60].sum())
    return dict(cache="on" if cache_mb >= 0 else "off", value=d["games_finished"] / secs, renewal_estimate=d["expansions"] / secs / epg,
                games_finished=d["games_finished"], seconds=secs, expansions=d["expansions"], tower_rows=d["tower_rows"],
                expansions_over_tower_rows=d["expansions"] / max(1, d["tower_rows"]),
                cache_lookups=d["cache_lookups"], cache_hits=d["cache_hits"], hit_rate=d["cache_hits"] / max(1, d["cache_lookups"]),
                fresh_lookups=fresh_l, fresh_hits=fresh_h, fresh_hit_rate=fresh_h / max(1, fresh_l),
                warm_lookups=int(lk[60]), warm_hits=int(ht[60]), cache_repeats=d["cache_repeats"],
                by_turn={t: [int(lk[t]), int(ht[t])] for t in range(60) if lk[t]},
                tower_tflops_from_tower_rows=d["tower_rows"] * bench.FLOP_PER_EXPANSION / (d["nn_ms"] / 1e3) / 1e12 if d["nn_ms"] else None,
                gpu=torch.cuda.get_device_name(), power_limit_w=power_limit_w(), sm_mhz=clocks["sm_mhz"], clock_reasons=clocks["reasons"],
                steps=steps, warmup=warmup, games=games, warm_start=profile_src)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--games", type=int, default=4096)
    args = ap.parse_args()
    from reversi_zero_b200.agent import model as M
    from reversi_zero_b200 import net as N
    mc = M.ModelConfig(**bench.MODEL_KW)
    net = N.Net(mc)
    net.load_blob(M.weights_to_blob(mc, M.build_random_weights(mc, 0)))
    pp = SimpleNamespace(required_visit_to_decide_action=400, start_rethinking_turn=8, allowed_resign_turn=20,
                         disable_resignation_rate=0.1, **bench.PLAY_KW)
    runs = {"off": [], "on": []}
    for _ in range(args.pairs):
        for mb in (-1, 0):
            r = run_one(net, pp, args.games, args.steps, max(3, args.warmup), mb)
            runs[r["cache"]].append(r)
            print(json.dumps(r), flush=True)
    net.close()

    def arm(rs, key):
        v = [r[key] for r in rs]
        return dict(mean=statistics.mean(v), min=min(v), max=max(v), spread=(max(v) - min(v)) / statistics.mean(v))
    print(json.dumps(dict(summary=True, pairs=args.pairs, value_off=arm(runs["off"], "value"), value_on=arm(runs["on"], "value"),
                          renewal_off=arm(runs["off"], "renewal_estimate"), renewal_on=arm(runs["on"], "renewal_estimate"),
                          gain_value=statistics.mean(r["value"] for r in runs["on"]) / statistics.mean(r["value"] for r in runs["off"]) - 1,
                          gain_renewal=statistics.mean(r["renewal_estimate"] for r in runs["on"]) /
                          statistics.mean(r["renewal_estimate"] for r in runs["off"]) - 1,
                          expansions_over_tower_rows=statistics.mean(r["expansions_over_tower_rows"] for r in runs["on"]),
                          hit_rate=statistics.mean(r["hit_rate"] for r in runs["on"]),
                          fresh_hit_rate=statistics.mean(r["fresh_hit_rate"] for r in runs["on"]))), flush=True)


if __name__ == "__main__":
    main()
