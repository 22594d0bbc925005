"""GPU tests of opening suites: the device enumerator against its host twin, games from openings against the oracle
(two networks and four), a table of empty openings against no table, the refusals of rz_engine_set_openings, a balanced
suite from a random-weight network, eval and league from a suite, and the `openings` command."""
import ctypes as C
import json
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from oracle import mcts, nn as onn
from reversi_zero_b200 import _cabi
from reversi_zero_b200.lib import openings as OP
from test_engine_gpu import make_engine, params
from test_openings_host import run_check

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "reversi-alpha-zero_b200", "csrc")


@pytest.fixture(scope="module")
def check_exe(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    exe = str(tmp_path_factory.mktemp("openings_check") / "openings_check")
    subprocess.run([nvcc, "-O2", "-std=c++17", "--expt-relaxed-constexpr", "-Wno-deprecated-gpu-targets", "-I", CSRC,
                    os.path.join(ROOT, "tests", "support", "openings_check.cu"), "-o", exe], check=True)
    return exe


@pytest.mark.parametrize("plies", range(1, 10))
def test_enumerator_matches_host_twin(check_exe, plies):
    counts, out = run_check(check_exe, plies)
    ops = OP.enumerate_openings(plies)
    assert list(ops.level_counts) == counts
    assert list(zip(ops.own.tolist(), ops.enemy.tolist(), ops.moves.tolist())) == out


def test_enumerator_repeats_and_size_query():
    a, b = OP.enumerate_openings(8), OP.enumerate_openings(8)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    n = C.c_size_t()
    assert _cabi.lib().rz_openings_enumerate(8, None, None, None, 0, C.byref(n), None) == 0 and n.value == a.own.size == 67239
    small = np.zeros(10, np.uint64), np.zeros(10, np.uint64), np.zeros((10, 8), np.uint8)
    rc = _cabi.lib().rz_openings_enumerate(8, small[0].ctypes.data_as(_cabi.u64p), small[1].ctypes.data_as(_cabi.u64p),
                                           small[2].ctypes.data_as(_cabi.u8p), 10, C.byref(n), None)
    assert rc == -5 and n.value == 67239


def pick_openings(k, plies=6, stride=97):
    ops = OP.enumerate_openings(plies)
    return [ops.moves[(i * stride) % ops.own.size].tolist() for i in range(k)]


def oracle_check(g, pp, seed, opening, s_black, s_white):
    """the game equals the oracle's two-evaluator game started after `opening`, with black's evaluator first"""
    o = mcts.SelfPlayGame(pp, onn.FakeNetAPI(s_black), seed=seed, game_id=g["game_id"], api_b=onn.FakeNetAPI(s_white), black_net=0)
    for a in opening:
        o.env.step(a)
    o.play()
    theirs = sorted(o.plies + o.solved_plies, key=lambda r: r["turn"])
    played = [p for p in g["plies"] if p["action"] >= 0]
    assert [(p["own"], p["enemy"], p["action"], list(p["N"]) if p["recorded"] else None) for p in played] == \
           [(p["own"], p["enemy"], p["action"], list(p["N"]) if "N" in p else None) for p in theirs]
    assert g["winner"] == o.env.winner and (g["black"], g["white"]) == (o.env.black, o.env.white)
    assert g["opening_plies"] == len(opening) and g["turn"] == o.env.turn


MATCH_KW = [dict(), dict(use_solver_turn=54, use_solver_turn_in_simulation=51, resign_threshold=-0.35, allowed_resign_turn=10,
                         disable_resignation_rate=0)]


@pytest.mark.parametrize("kw", MATCH_KW)
def test_second_net_games_from_openings_equal_oracle(kw):
    pp = params(simulation_num_per_move=24, share_mtcs_info_in_self_play=False, change_tau_turn=0, **kw)
    openings = pick_openings(12)
    eng = make_engine(pp, games=5, seed=51, max_games=12)
    eng.set_second_net(None, enable=True)
    eng.set_openings(openings)
    eng.run(finished_target=12)
    games = sorted(eng.poll(), key=lambda g: g["game_id"])
    eng.close()
    assert len(games) == 12
    for i, g in enumerate(games):
        assert g["plies"][0]["own"] | g["plies"][0]["enemy"] == sum(OP.replay(openings[i]))
        oracle_check(g, pp, 51, openings[i], 1.0 if i % 2 == 0 else -1.0, -1.0 if i % 2 == 0 else 1.0)


def test_four_networks_from_openings_equal_oracle():
    scales = [1.0, -1.0, 0.5, -0.25]
    ordered = [(i, j) for i in range(4) for j in range(4) if i != j]
    black, white = np.array(ordered, dtype=np.uint8).T
    pp = params(simulation_num_per_move=20, share_mtcs_info_in_self_play=False, change_tau_turn=0)
    openings = pick_openings(12, plies=8, stride=1013)
    eng = make_engine(pp, games=5, seed=53, max_games=12, overlap_groups=2)
    eng.set_nets([None] * 4, black, white, fake_scales=scales)
    eng.set_openings(openings)
    eng.run(finished_target=12)
    games = sorted(eng.poll(), key=lambda g: g["game_id"])
    eng.close()
    for k, g in enumerate(games):
        oracle_check(g, pp, 53, openings[k], scales[ordered[k][0]], scales[ordered[k][1]])


def game_key(g):
    return (g["game_id"], g["black"], g["white"], g["winner"], g["turn"], g["expansions"], g["simulations"], g["opening_plies"],
            [(p["own"], p["enemy"], p["action"], list(p["N"]), p["recorded"], p["n"], p["q"]) for p in g["plies"]])


def test_empty_openings_equal_no_table():
    pp = params(simulation_num_per_move=24, share_mtcs_info_in_self_play=False, change_tau_turn=2, noise_eps=0.25)
    runs = []
    for table in (False, True):
        eng = make_engine(pp, games=3, seed=57, max_games=6)
        eng.set_second_net(None, enable=True)
        if table:
            eng.set_openings([[]] * 6)
        eng.run(finished_target=6)
        runs.append([game_key(g) for g in sorted(eng.poll(), key=lambda g: g["game_id"])])
        eng.close()
    assert runs[0] == runs[1] and all(k[7] == 0 for k in runs[0])


def test_refusals_leave_engine_usable():
    pp = params(simulation_num_per_move=8, share_mtcs_info_in_self_play=False, change_tau_turn=0)
    eng = make_engine(pp, games=2, seed=59, max_games=2)
    good = pick_openings(2)
    with pytest.raises(_cabi.RzError, match="illegal"):
        eng.set_openings([[0], []])
    with pytest.raises(ValueError, match="at most 20"):
        eng.set_openings([list(range(21)), []])
    from test_openings_host import forcing_pass_sequence
    seq, _ = forcing_pass_sequence()
    with pytest.raises(_cabi.RzError, match="must pass|ends the game"):
        eng.set_openings([seq, []])
    with pytest.raises(_cabi.RzError, match="max_games"):
        eng.set_openings(good[:1])   # max_games 2 > 1 opening
    n_moves = np.array([21, 0], np.uint8)
    moves = np.zeros((2, 20), np.uint8)
    assert _cabi.lib().rz_engine_set_openings(eng._h, moves.ctypes.data_as(_cabi.u8p), n_moves.ctypes.data_as(_cabi.u8p), 2) == -1
    eng.set_openings(good)
    eng.run(finished_target=2)
    games = sorted(eng.poll(), key=lambda g: g["game_id"])
    assert [g["opening_plies"] for g in games] == [6, 6]
    assert [g["turn"] for g in games] == [6 + sum(p["action"] >= 0 for p in g["plies"]) for g in games]
    with pytest.raises(_cabi.RzError, match="first wave"):
        eng.set_openings(good)
    eng.close()
    warm = make_engine(pp, games=2, seed=59, max_games=2, warm_start=True)
    with pytest.raises(_cabi.RzError, match="warm_start"):
        warm.set_openings(good)
    warm.close()


def random_net(seed=1):
    from reversi_zero_b200.agent import model as M
    from reversi_zero_b200 import net as N
    mc = M.ModelConfig(256, 3, 10, 1e-4, 256)
    net = N.Net(mc)
    net.load_weights(M.build_random_weights(mc, seed))
    return net


def test_balanced_suite_values_and_seed():
    net = random_net()
    suite = OP.balanced_suite(net, 6, 200, 0.05, seed=3)
    again = OP.balanced_suite(net, 6, 200, 0.05, seed=3)
    other = OP.balanced_suite(net, 6, 200, 0.05, seed=4)
    assert suite == again and [e.moves for e in suite] != [e.moves for e in other]
    planes = np.zeros((len(suite), 2, 8, 8), np.uint8)
    for i, e in enumerate(suite):
        own, enemy = OP.replay(e.moves)
        planes[i, 0] = np.array([(own >> s) & 1 for s in range(64)], np.uint8).reshape(8, 8)
        planes[i, 1] = np.array([(enemy >> s) & 1 for s in range(64)], np.uint8).reshape(8, 8)
    _, v = net.predict_planes(planes)
    for e, vv in zip(suite, v):
        assert abs(e.value - vv) < 1e-3
        if abs(abs(vv) - 0.05) > 1e-3:
            assert abs(vv) <= 0.05
    net.close()


def small_config(tmp_path, **league):
    from reversi_zero_b200.config import Config
    cfg = Config(project_dir=str(tmp_path), data_dir=str(tmp_path / "data"))
    cfg.model.update(dict(cnn_filter_num=16, res_layer_num=1, value_fc_size=16))
    cfg.play.update(dict(c_puct=5, parallel_search_num=4))
    cfg.eval = dict(play_config=dict(simulation_num_per_move=16, c_puct=1), openings="suite.txt")
    cfg.league.update(dict(openings="suite.txt", **league))
    cfg.resource.create_directories()
    return cfg


def write_blobs(tmp_path, names):
    from reversi_zero_b200.agent import model as M
    mc = M.ModelConfig(16, 3, 1, 1e-4, 16)
    os.makedirs(tmp_path / "gen", exist_ok=True)
    for k, name in enumerate(names):
        np.save(tmp_path / "gen" / name, M.weights_to_blob(mc, M.build_random_weights(mc, 10 + k)))


def test_eval_and_league_from_suite(tmp_path):
    from reversi_zero_b200 import net as N
    from reversi_zero_b200.worker import evaluate as EV, league as L
    suite = pick_openings(3, plies=4)
    OP.save_suite(str(tmp_path / "suite.txt"), suite)
    cfg = small_config(tmp_path, models=["gen/a.rzblob.npy", "gen/b.rzblob.npy", "gen/c.rzblob.npy"], game_num_per_pair=5)
    write_blobs(tmp_path, ["a.rzblob.npy", "b.rzblob.npy", "c.rzblob.npy"])
    nets = []
    for name in ("a", "b"):
        net = N.Net(cfg.model)
        net.load_blob(np.load(tmp_path / "gen" / f"{name}.rzblob.npy"))
        nets.append(net)
    loaded = EV.EvaluateWorker(cfg).load_openings()
    assert loaded == suite
    results, games = EV.play_match(cfg, nets[0], nets[1], 8, seed=5, suite=loaded)
    assert len(games) == 8
    seen = {}
    for i, g in enumerate(games):
        op = suite[(i // 2) % 3]
        assert g["opening_plies"] == 4 and g["black_net"] == i % 2
        own, enemy = OP.replay(op)
        assert (g["plies"][0]["own"], g["plies"][0]["enemy"]) == (own, enemy)
        seen.setdefault(tuple(op), set()).add(g["black_net"])
    assert all(v == {0, 1} for v in seen.values()) and len(seen) == 3
    for net in nets:
        net.close()
    out = [json.load(open(L.LeagueWorker(cfg).start())) for _ in range(2)]
    assert out[0]["openings"] == dict(path="suite.txt", sha256=OP.suite_digest(str(tmp_path / "suite.txt")), count=3)
    assert dict(out[0], timestamp=None) == dict(out[1], timestamp=None) and out[0]["games"] == 15
    for p in out[0]["pairs"]:
        assert sum(p["as_black"]) + sum(p["as_white"]) == 5
    cfg.league.openings = None
    plain = json.load(open(L.LeagueWorker(cfg).start()))
    assert plain["openings"] is None


def test_openings_command_writes_a_suite(tmp_path):
    write_blobs(tmp_path, ["m.rzblob.npy"])
    yml = tmp_path / "o.yml"
    yml.write_text("model: {cnn_filter_num: 16, res_layer_num: 1, value_fc_size: 16}\n"
                   "openings: {plies: 5, count: 20, max_abs_value: 0.5, seed: 9, model: gen/m.rzblob.npy, path: out/suite.txt}\n")
    env = dict(os.environ, PROJECT_DIR=str(tmp_path), PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "reversi-alpha-zero_b200"), ROOT]))
    subprocess.run([sys.executable, "-m", "reversi_zero_b200.run", "openings", "-c", str(yml)], env=env, cwd=str(tmp_path),
                   check=True, timeout=600)
    suite = OP.load_suite(str(tmp_path / "out" / "suite.txt"))
    assert 1 <= len(suite) <= 20 and all(len(m) == 5 for m in suite)
