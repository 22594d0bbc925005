"""bench.py's reference arm (CPU side of the contract): `--impl reference --steps K --warmup W` honours K and W, prints
one JSON line on the real stdout and describes the SAME workload (`config`) as the CUDA arm.  No GPU involved."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_windowed_cpu_runner_counts_per_window():
    from oracle import selfplay_cpu
    model_kw = dict(cnn_filter_num=16, cnn_filter_size=3, res_layer_num=1, value_fc_size=16)
    play_kw = dict(simulation_num_per_move=16, parallel_search_num=4, c_puct=5, virtual_loss=3, noise_eps=0.25,
                   dirichlet_alpha=0.5, change_tau_turn=4, thinking_loop=1, resign_threshold=None,
                   share_mtcs_info_in_self_play=True)
    wins, tot = selfplay_cpu.measure_windows(model_kw, play_kw, windows=3, window_s=1.0, processes=2)
    assert len(wins) == 3
    for w in wins:
        assert w["processes"] == 2 and w["expansions"] > 0 and w["expansions_per_s"] > 0 and 1 <= w["mean_batch"] <= 4
    # a 16-simulation game on a 1-block net lasts well under a second: the streams play games back to back
    assert tot["games_finished"] >= 2 and tot["plies"] >= 60


def test_reference_arm_line_and_shared_config():
    sys.path.insert(0, ROOT)
    import bench
    # the workload description both arms print is a function of the arguments only
    args = argparse.Namespace(games=4096, sims=400, gpus=1)
    assert bench.workload_config(args) == bench.workload_config(args)
    assert "cores" not in bench.workload_config(args)
    env = dict(os.environ, RZ_BENCH_REFERENCE_TOTAL_S="6", CUDA_VISIBLE_DEVICES="")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "3", "--warmup", "3"],
                         stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, env=env, timeout=300, check=True).stdout
    lines = [x for x in out.splitlines() if x.strip()]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["steps"] == 3 and d["warmup"] == 3 and d["gpu_launches"] == 0
    assert d["metric"] == "self_play_games_per_sec" and d["unit"] == "games/s" and d["higher_is_better"] is True
    assert d["config"] == bench.workload_config(args)
    assert d["value"] > 0 and d["e2e"] == dict(value=d["value"], unit="games/s", h2d_bytes_per_step=0, d2h_bytes_per_step=0)
    cb = d["cpu_baseline"]
    assert cb["kind"] == "port" and cb["cores"] >= 1 and cb["value"] == d["value"] and "windows" in cb["sample"]


def test_reference_arm_under_torchrun_prints_one_line_from_rank_0():
    """the driver launches the reference arm like the CUDA arm (torchrun, one rank per GPU): rank 0 alone measures and prints,
    the other ranks exit 0 without work"""
    env = dict(os.environ, RZ_BENCH_REFERENCE_TOTAL_S="6", CUDA_VISIBLE_DEVICES="")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
                        "--master-port", "29541", os.path.join(ROOT, "bench.py"), "--impl", "reference", "--gpus", "2", "--steps", "3",
                        "--warmup", "3"], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, env=env, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    lines = [x for x in r.stdout.splitlines() if x.strip().startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    assert d["impl"] == "reference" and d["n_gpus"] == 2 and d["value"] > 0 and d["config"]["parallelism"].startswith("dp2")
