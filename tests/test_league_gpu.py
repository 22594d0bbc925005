"""GPU tests of leagues: N networks in one engine (rz_engine_set_nets) against the two-network path and the oracle, real
networks of mixed widths, the refusals of rz_engine_set_nets, the league worker and command, and eval's archive of
promoted models."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import mcts, nn as onn
from reversi_zero_b200 import _cabi, engine as E
from test_engine_gpu import make_engine, params, replay_check

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MATCH_KW = [dict(), dict(use_solver_turn=54, use_solver_turn_in_simulation=51, resign_threshold=-0.35, allowed_resign_turn=10,
                         disable_resignation_rate=0, noise_eps=0.0)]


def game_key(g):
    return (g["game_id"], g["black"], g["white"], g["winner"], g["black_net"], g["white_net"], g["expansions"], g["simulations"],
            [(p["own"], p["enemy"], p["pid"], p["action"], list(p["N"]), p["loops"], p["recorded"], p["n"], p["q"]) for p in g["plies"]])


def oracle_check(g, pp, seed, s_black, s_white):
    """the game equals the oracle's two-evaluator game with black's evaluator first"""
    replay_check(g)
    o = mcts.SelfPlayGame(pp, onn.FakeNetAPI(s_black), seed=seed, game_id=g["game_id"], api_b=onn.FakeNetAPI(s_white), black_net=0).play()
    theirs = sorted(o.plies + o.solved_plies, key=lambda r: r["turn"])
    played = [p for p in g["plies"] if p["action"] >= 0]
    assert [(p["own"], p["enemy"], p["action"], list(p["N"]) if p["recorded"] else None) for p in played] == \
           [(p["own"], p["enemy"], p["action"], list(p["N"]) if "N" in p else None) for p in theirs]
    assert g["winner"] == o.env.winner and (len(g["plies"]) > len(played)) == (o.actions[-1] is None)


@pytest.mark.parametrize("kw", MATCH_KW)
def test_two_fake_networks_equal_set_second_net(kw):
    pp = params(simulation_num_per_move=30, share_mtcs_info_in_self_play=False, change_tau_turn=0, **kw)
    runs = []
    for use_table in (False, True):
        eng = make_engine(pp, games=3, seed=41, max_games=6)
        if use_table:
            local = np.arange(6)
            eng.set_nets([None, None], local & 1, 1 - (local & 1), fake_scales=[1.0, -1.0])
        else:
            eng.set_second_net(None, enable=True)
        eng.run(finished_target=6)
        runs.append(sorted(eng.poll(), key=lambda g: g["game_id"]))
        eng.close()
    assert [g["black_net"] for g in runs[0]] == [0, 1, 0, 1, 0, 1]
    assert [g["white_net"] for g in runs[0]] == [1, 0, 1, 0, 1, 0]
    assert [game_key(g) for g in runs[0]] == [game_key(g) for g in runs[1]]


def test_four_fake_networks_equal_oracle():
    scales = [1.0, -1.0, 0.5, -0.25]  # powers of two: the engine's fp32 products equal the oracle's bit for bit
    ordered = [(i, j) for i in range(4) for j in range(4) if i != j]
    black, white = np.array(ordered, dtype=np.uint8).T
    pp = params(simulation_num_per_move=24, share_mtcs_info_in_self_play=False, change_tau_turn=0)
    eng = make_engine(pp, games=5, seed=43, max_games=12, overlap_groups=2)
    eng.set_nets([None] * 4, black, white, fake_scales=scales)
    eng.run(finished_target=12)
    games = sorted(eng.poll(), key=lambda g: g["game_id"])
    st = eng.stats()
    eng.close()
    assert len(games) == 12 and st["nn_launches"] == 0
    for k, g in enumerate(games):
        assert g["game_id"] == k and (g["black_net"], g["white_net"]) == ordered[k]
        oracle_check(g, pp, 43, scales[ordered[k][0]], scales[ordered[k][1]])
    assert len({(g["winner"], g["black"]) for g in games}) > 2


def small_config(tmp_path, **league):
    from reversi_zero_b200.config import Config
    cfg = Config(project_dir=str(tmp_path), data_dir=str(tmp_path / "data"))
    cfg.model.update(dict(cnn_filter_num=16, res_layer_num=1, value_fc_size=16))
    cfg.play.update(dict(c_puct=5, parallel_search_num=4))
    cfg.eval = dict(play_config=dict(simulation_num_per_move=16, c_puct=1))
    cfg.league.update(league)
    cfg.resource.create_directories()
    return cfg


def test_real_networks_of_mixed_widths_equal_two_network_engines(tmp_path):
    from reversi_zero_b200.agent import model as M
    from reversi_zero_b200 import net as N
    from reversi_zero_b200.worker import league as L
    cfg = small_config(tmp_path, play_config=dict(simulation_num_per_move=12))
    ch5 = M.ModelConfig(256, 3, 10, 1e-4, 256)
    narrow = M.ModelConfig(64, 3, 2, 1e-4, 64)
    nets = []
    for mc, seed in ((ch5, 1), (ch5, 2), (narrow, 3)):
        net = N.Net(mc)
        net.load_weights(M.build_random_weights(mc, seed))
        nets.append(net)
    games_per_pair = 4
    recs = L.play_league(cfg, nets, games_per_pair, seed=7, first_game_id=100)
    black, white = L.schedule(3, games_per_pair)
    assert [(r["black"], r["white"]) for r in recs] == list(zip(black, white))
    assert [r["game_id"] for r in recs] == list(range(100, 112))
    pc = L.league_play_config(cfg)
    league_games = {}
    eng_cfg = E.engine_cfg_from_play_config(pc, games=12, seed=7, eval_mode=E.EVAL_NET, max_games=12, first_game_id=100,
                                     eval_cache_mb=-1)
    eng = E.Engine(eng_cfg, nets[0])
    eng.set_nets(nets, black, white)
    eng.run(finished_target=12)
    for g in eng.poll():
        league_games[g["game_id"]] = g
    eng.close()
    assert {g["game_id"]: g["winner"] for g in league_games.values()} == {r["game_id"]: r["winner"] for r in recs}
    for r in recs:  # the same game alone in a two-network engine, black's network first: tower rows do not depend on the batch
        one = E.Engine(E.engine_cfg_from_play_config(pc, games=1, seed=7, eval_mode=E.EVAL_NET, max_games=1, first_game_id=r["game_id"],
                                                   eval_cache_mb=-1),
                       nets[r["black"]])
        one.set_second_net(nets[r["white"]])
        one.run(finished_target=1)
        (g,) = one.poll()
        one.close()
        replay_check(g)
        mine = dict(league_games[r["game_id"]], black_net=0, white_net=1)
        assert game_key(mine) == game_key(g), r
    for net in nets:
        net.close()


def test_set_nets_refusals_leave_the_engine_usable():
    pp = params(simulation_num_per_move=16, share_mtcs_info_in_self_play=False, change_tau_turn=0)
    b4, w4 = np.array([0, 1, 2, 3, 3, 2], np.uint8), np.array([1, 2, 3, 0, 1, 0], np.uint8)
    eng = make_engine(pp, games=3, seed=5, max_games=6)
    for nets, b, w in (([None], b4[:6] * 0, w4 * 0), ([None] * 17, b4, w4), ([None] * 3, b4, w4)):
        with pytest.raises(_cabi.RzError):
            eng.set_nets(nets, b, w)
    with pytest.raises(_cabi.RzError):
        eng.set_nets([None] * 4, b4[:5], w4[:5])   # max_games 6 > 5 games in the table
    eng.set_max_games(0)
    with pytest.raises(_cabi.RzError):
        eng.set_nets([None] * 4, b4, w4)           # max_games 0: no bound on the table
    eng.set_max_games(6)
    eng.set_nets([None] * 4, b4, w4, fake_scales=[1.0, -1.0, 0.5, -0.25])
    with pytest.raises(_cabi.RzError):
        eng.set_max_games(7)                       # past the table
    eng.run(max_waves=1)
    with pytest.raises(_cabi.RzError):
        eng.set_nets([None] * 4, b4, w4)           # after the first wave
    eng.run(finished_target=6)
    games = sorted(eng.poll(), key=lambda g: g["game_id"])
    eng.close()
    assert [(g["black_net"], g["white_net"]) for g in games] == list(zip(b4, w4))
    scales = [1.0, -1.0, 0.5, -0.25]
    for g in games:
        oracle_check(g, pp, 5, scales[g["black_net"]], scales[g["white_net"]])
    # under the network evaluator: a NULL network is refused; four networks keep the evaluation cache off
    from reversi_zero_b200.agent import model as M
    from reversi_zero_b200 import net as N
    mc = M.ModelConfig(16, 3, 1, 1e-4, 16)
    nets = []
    for seed in range(4):
        net = N.Net(mc)
        net.load_weights(M.build_random_weights(mc, seed))
        nets.append(net)
    eng = E.Engine(E.engine_cfg_from_play_config(pp, games=3, seed=5, eval_mode=E.EVAL_NET, max_games=6), nets[0])
    with pytest.raises(_cabi.RzError):
        eng.set_nets([nets[0], None, nets[2], nets[3]], b4, w4)
    eng.set_nets(nets, b4, w4)
    eng.run(finished_target=6)
    st = eng.stats()
    games = eng.poll()
    eng.close()
    assert len(games) == 6 and st["cache_lookups"] == 0 and st["cache_hits"] == 0 and st["tower_rows"] > 0
    for g in games:
        replay_check(g)
    for net in nets:
        net.close()


def write_blobs(cfg, tmp_path):
    from reversi_zero_b200.agent import model as M
    d = tmp_path / "gen"
    d.mkdir()
    paths = []
    for name, seed in (("a", 1), ("b", 2), ("c", 1)):   # a and c are byte-identical
        p = d / f"{name}.rzblob.npy"
        np.save(p, M.weights_to_blob(cfg.model, M.build_random_weights(cfg.model, seed, perturb_bn=True)))
        paths.append(p)
    assert paths[0].read_bytes() == paths[2].read_bytes()


def test_league_worker_end_to_end(tmp_path):
    from reversi_zero_b200.worker import league as L
    cfg = small_config(tmp_path, models=["gen/*.rzblob.npy"], game_num_per_pair=4)
    write_blobs(cfg, tmp_path)
    out = [json.load(open(L.LeagueWorker(cfg).start())) for _ in range(2)]
    res = out[0]
    assert res["games"] == 12 and res["games_per_pair"] == 4 and res["anchor"] == 0
    assert [m["path"] for m in res["models"]] == ["gen/a.rzblob.npy", "gen/b.rzblob.npy", "gen/c.rzblob.npy"]
    assert res["models"][0]["sha256"] == res["models"][2]["sha256"] != res["models"][1]["sha256"]
    pairs = {(p["model"], p["opponent"]): p for p in res["pairs"]}
    assert len(pairs) == 6
    for (i, j), p in pairs.items():
        q = pairs[(j, i)]
        assert (p["W"], p["D"], p["L"]) == (q["L"], q["D"], q["W"]) and p["W"] + p["D"] + p["L"] == 4
        assert p["as_black"] == q["as_white"][::-1] and sum(p["as_black"]) == sum(p["as_white"]) == 2   # colours balanced
    for m in res["models"]:
        assert np.isfinite(m["elo"]) and np.isfinite(m["ci95"]) and m["games"] == 8
        assert m["score"] == sum(p["W"] + 0.5 * p["D"] for (i, _), p in pairs.items() if i == m["index"])
    assert res["models"][0]["elo"] == 0.0 and res["models"][0]["ci95"] == 0.0
    assert out[0]["timestamp"] != out[1]["timestamp"]
    assert dict(out[0], timestamp=None) == dict(out[1], timestamp=None)
    # the command: python -m reversi_zero_b200.run league -c <yml>
    yml = tmp_path / "league.yml"
    yml.write_text("model: {cnn_filter_num: 16, res_layer_num: 1, value_fc_size: 16}\n"
                   "eval: {play_config: {simulation_num_per_move: 16, c_puct: 1}}\n"
                   "league: {models: [gen/a.rzblob.npy, gen/b.rzblob.npy], game_num_per_pair: 2, anchor: 1}\n")
    env = dict(os.environ, PROJECT_DIR=str(tmp_path), PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "reversi-alpha-zero_b200"), ROOT]))
    before = set(os.listdir(tmp_path / "logs"))
    subprocess.run([sys.executable, "-m", "reversi_zero_b200.run", "league", "-c", str(yml)], env=env, cwd=str(tmp_path),
                   check=True, timeout=600)
    (new,) = set(os.listdir(tmp_path / "logs")) - before - {"main.log"}
    res = json.load(open(tmp_path / "logs" / new))
    assert res["games"] == 2 and res["anchor"] == 1 and res["models"][1]["elo"] == 0.0
    log = (tmp_path / "logs" / "main.log").read_text()
    assert "league: 2 models, 2 games per pair" in log and "gen/b.rzblob.npy" in log


@pytest.mark.parametrize("keep", [True, False])
def test_eval_keeps_promoted_models(tmp_path, keep):
    from reversi_zero_b200.agent import model as M
    from reversi_zero_b200.worker import evaluate as EV
    cfg = small_config(tmp_path)
    cfg.eval = dict(game_num=4, replace_rate=0.0, play_config=dict(simulation_num_per_move=8, c_puct=1))  # always promotes
    cfg.b200.keep_promoted_models = keep
    np.save(cfg.resource.model_best_blob_path, M.weights_to_blob(cfg.model, M.build_random_weights(cfg.model, 1)))
    name = cfg.resource.next_generation_model_dirname_tmpl % "20260922-000000.000000"
    ng_dir = os.path.join(cfg.resource.next_generation_model_dir, name)
    os.makedirs(ng_dir)
    ng_blob = M.weights_to_blob(cfg.model, M.build_random_weights(cfg.model, 2))
    np.save(os.path.join(ng_dir, EV.NEXT_GENERATION_BLOB), ng_blob)
    best = open(cfg.resource.model_best_blob_path, "rb").read()
    assert EV.EvaluateWorker(cfg).start(max_models=1) == 1
    promoted = os.path.join(cfg.resource.model_dir, "promoted")
    assert np.array_equal(np.load(cfg.resource.model_best_blob_path), ng_blob)   # promoted
    if not keep:
        assert not os.path.exists(promoted)
        return
    files = sorted(os.listdir(promoted))
    assert len(files) == 2 and name + ".rzblob.npy" in files and all(f.startswith("model_") for f in files)
    (first,) = [f for f in files if f != name + ".rzblob.npy"]
    assert open(os.path.join(promoted, first), "rb").read() == best
    assert np.array_equal(np.load(os.path.join(promoted, name + ".rzblob.npy")), ng_blob)
    # a restart does not archive the best blob again: a promoted blob with its content exists
    assert EV.EvaluateWorker(cfg).archive_best_model() is None and len(os.listdir(promoted)) == 2
