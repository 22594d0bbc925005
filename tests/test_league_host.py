"""CPU suite of the league (worker/league.py): the Elo fit, the schedule, the model list and its refusals, the ABI of
rz_engine_set_nets and the `league` command."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest

from reversi_zero_b200 import _cabi, run
from reversi_zero_b200.agent import model as M
from reversi_zero_b200.config import create_config
from reversi_zero_b200.worker import league as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def games(pairs):
    """[(black, white, winner, count)] -> records"""
    out = []
    for b, w, win, k in pairs:
        out += [dict(game_id=len(out) + i, black=b, white=w, winner=win, disc_diff=0) for i in range(k)]
    return out


@pytest.mark.parametrize("w,l,p", [(7, 3, 1), (10, 0, 1), (3, 9, 2), (5, 5, 1), (12, 4, 0)])
def test_fit_elo_two_models_closed_form(w, l, p):
    recs = games([(0, 1, 1, w // 2), (1, 0, 2, w - w // 2), (0, 1, 2, l // 2), (1, 0, 1, l - l // 2)])
    r, ci = L.fit_elo(recs, 2, prior_draws=p)
    assert r[0] == 0.0 and ci[0] == 0.0
    want = 400 * math.log10((w + p / 2) / (l + p / 2))
    assert abs((r[0] - r[1]) - want) < 1e-7
    # the 95 % interval of a two-model fit: 1.96 / sqrt(n p (1 - p)) natural units
    n, q = w + l + p, (w + p / 2) / (w + l + p)
    assert abs(ci[1] - 1.96 / math.sqrt(n * q * (1 - q)) * 400 / math.log(10)) < 1e-6


def league_records(seed=0, n=4):
    rng = np.random.default_rng(seed)
    strength = np.linspace(0, 1.5, n)
    recs = []
    black, white = L.schedule(n, 12)
    for b, w in zip(black, white):
        p = 1 / (1 + math.exp(strength[w] - strength[b]))
        u = rng.random()
        recs.append(dict(game_id=len(recs), black=int(b), white=int(w), winner=3 if abs(u - p) < 0.05 else (1 if u < p else 2),
                         disc_diff=0))
    return recs


def test_fit_elo_relabel_and_anchor_invariance():
    recs = league_records()
    r, ci = L.fit_elo(recs, 4)
    perm = [2, 0, 3, 1]  # model i is called perm[i]
    relabelled = [dict(r_, black=perm[r_["black"]], white=perm[r_["white"]]) for r_ in recs]
    r2, ci2 = L.fit_elo(relabelled, 4, anchor=perm[0])
    for i in range(4):
        assert abs(r2[perm[i]] - r[i]) < 1e-7 and abs(ci2[perm[i]] - ci[i]) < 1e-7
    r3, ci3 = L.fit_elo(recs, 4, anchor=2)  # moving the anchor shifts every rating by one constant
    assert np.allclose(r3 - r, -r[2], atol=1e-7) and r3[2] == 0.0 and ci3[2] == 0.0


def test_fit_elo_sweep_is_finite_and_transitive_order():
    sweep = games([(0, 1, 1, 5), (1, 0, 2, 5)])
    r, ci = L.fit_elo(sweep, 2)
    assert np.all(np.isfinite(r)) and np.all(np.isfinite(ci)) and r[1] < -300
    with pytest.raises(ValueError):
        L.fit_elo(sweep, 2, prior_draws=0)
    # 0 beats 1 beats 2, 0 beats 2 more often
    recs = games([(0, 1, 1, 6), (1, 0, 1, 3), (1, 2, 1, 6), (2, 1, 1, 3), (0, 2, 1, 8), (2, 0, 1, 1), (1, 0, 3, 1)])
    r, _ = L.fit_elo(recs, 3)
    assert r[0] > r[1] > r[2]


def test_fit_elo_repeated_records_narrow_by_sqrt_k():
    recs = league_records(3)
    r, ci = L.fit_elo(recs, 4, prior_draws=0)
    for k in (2, 5):
        rk, cik = L.fit_elo(recs * k, 4, prior_draws=0)
        assert np.allclose(rk, r, atol=1e-7)
        assert np.allclose(cik * math.sqrt(k), ci, rtol=1e-9, atol=1e-12)


@pytest.mark.parametrize("n,gpp", [(2, 1), (2, 5), (3, 4), (5, 3), (16, 2)])
def test_schedule(n, gpp):
    black, white = L.schedule(n, gpp)
    pairs = [(i, j) for i in range(n) for j in range(i + 1, n)]
    P = len(pairs)
    assert black.dtype == np.uint8 and white.dtype == np.uint8 and black.size == white.size == P * gpp
    assert np.all(black != white) and black.max() < n and white.max() < n
    for k in range(black.size):  # interleaving: game k belongs to pair k mod P, the lower index is black in even rounds
        i, j = pairs[k % P]
        assert (black[k], white[k]) == ((i, j) if (k // P) % 2 == 0 else (j, i))
    for i, j in pairs:
        as_black = int(np.sum((black == i) & (white == j)))
        as_white = int(np.sum((black == j) & (white == i)))
        assert as_black + as_white == gpp and abs(as_black - as_white) <= 1
    for bad in ((1, 4), (17, 1), (3, 0)):
        with pytest.raises(ValueError):
            L.schedule(*bad)


def make_blob(path, mc, seed=0):
    np.save(path, M.weights_to_blob(mc, M.build_random_weights(mc, seed)))


def small_config(tmp_path, league):
    cfg = create_config(dict(model=dict(cnn_filter_num=16, res_layer_num=1, value_fc_size=16), league=league),
                        project_dir=str(tmp_path), data_dir=str(tmp_path / "data"))
    return cfg


def test_yaml_league_section_and_model_list(tmp_path):
    import yaml
    text = """
model: {cnn_filter_num: 16, res_layer_num: 1, value_fc_size: 16}
league:
  models:
    - gen/a.rzblob.npy
    - gen/b*.rzblob.npy
    - {path: wide.rzblob.npy, model: {cnn_filter_num: 32}}
  game_num_per_pair: 6
  play_config: {simulation_num_per_move: 20}
  anchor: 1
"""
    (tmp_path / "gen").mkdir()
    base = M.ModelConfig(16, 3, 1, 1e-4, 16)
    make_blob(tmp_path / "gen" / "a.rzblob.npy", base)
    make_blob(tmp_path / "gen" / "b2.rzblob.npy", base, 2)
    make_blob(tmp_path / "gen" / "b1.rzblob.npy", base, 1)
    make_blob(tmp_path / "wide.rzblob.npy", M.ModelConfig(32, 3, 1, 1e-4, 16))
    cfg = create_config(yaml.safe_load(text), project_dir=str(tmp_path), data_dir=str(tmp_path / "data"))
    assert cfg.league.game_num_per_pair == 6 and cfg.league.anchor == 1
    entries = L.LeagueWorker(cfg).model_entries()
    assert [os.path.relpath(p, tmp_path) for p, _ in entries] == ["gen/a.rzblob.npy", "gen/b1.rzblob.npy", "gen/b2.rzblob.npy",
                                                                 "wide.rzblob.npy"]
    assert [mc.cnn_filter_num for _, mc in entries] == [16, 16, 16, 32]
    assert cfg.model.cnn_filter_num == 16  # the override does not leak into the shared model section
    pc = L.league_play_config(cfg)
    assert pc.simulation_num_per_move == 20 and pc.thinking_loop == 1 and pc.noise_eps == 0  # eval's rules underneath
    assert pc.share_mtcs_info_in_self_play is False


def test_default_model_list_is_the_promoted_directory(tmp_path):
    cfg = small_config(tmp_path, None)
    d = os.path.join(cfg.resource.model_dir, "promoted")
    os.makedirs(d)
    for name in ("model_2.rzblob.npy", "model_1.rzblob.npy", "other.npy"):
        make_blob(os.path.join(d, name), cfg.model)
    assert [os.path.basename(p) for p, _ in L.LeagueWorker(cfg).model_entries()] == ["model_1.rzblob.npy", "model_2.rzblob.npy"]


def test_refusals_name_the_files(tmp_path):
    mc = M.ModelConfig(16, 3, 1, 1e-4, 16)
    for i in range(18):
        make_blob(tmp_path / f"m{i:02d}.rzblob.npy", mc)
    with pytest.raises(ValueError, match=r"at least 2 models, found 1: .*m00\.rzblob\.npy"):
        L.LeagueWorker(small_config(tmp_path, dict(models=["m00.rzblob.npy"]))).model_entries()
    with pytest.raises(ValueError, match=r"at least 2 models, found 0"):
        L.LeagueWorker(small_config(tmp_path, None)).model_entries()
    with pytest.raises(ValueError, match=r"at most 16 models, found 18: .*m17\.rzblob\.npy"):
        L.LeagueWorker(small_config(tmp_path, dict(models=["m*.rzblob.npy"]))).model_entries()
    with pytest.raises(ValueError, match=r"missing file\(s\): .*nothere\.rzblob\.npy"):
        L.LeagueWorker(small_config(tmp_path, dict(models=["m00.rzblob.npy", "nothere.rzblob.npy"]))).model_entries()
    with pytest.raises(ValueError, match=r"zz\*\.npy matches no file"):
        L.LeagueWorker(small_config(tmp_path, dict(models=["m00.rzblob.npy", "zz*.npy"]))).model_entries()
    with pytest.raises(ValueError, match=r"m01\.rzblob\.npy holds \d+ floats, but its model configuration \(64 filters"):
        L.LeagueWorker(small_config(tmp_path, dict(models=["m00.rzblob.npy", dict(path="m01.rzblob.npy",
                                                                                  model=dict(cnn_filter_num=64))]))).model_entries()


def test_set_nets_abi():
    with open(os.path.join(ROOT, "include", "rz_engine.h")) as f:
        header = re.sub(r"\s+", " ", f.read())
    assert "#define RZ_MAX_NETS 16" in header
    assert ("int rz_engine_set_nets(rz_engine* e, rz_net* const* nets, const float* fake_scale, int n_nets, const uint8_t* black_net, "
            "const uint8_t* white_net, uint64_t n_games);") in header
    assert "uint8_t white_net;" in header
    res, args = _cabi.SIGNATURES["rz_engine_set_nets"]
    assert res is C.c_int and args == [C.c_void_p, C.POINTER(C.c_void_p), _cabi.f32p, C.c_int, _cabi.u8p, _cabi.u8p, C.c_uint64]
    assert getattr(_cabi.lib(), "rz_engine_set_nets", None) is not None
    # white_net takes the place of the first pad byte: the game record keeps its layout and size
    assert C.sizeof(_cabi.Game) == 56 and _cabi.Game.white_net.offset == _cabi.Game.black_net.offset + 1
    assert _cabi.Game.table_nodes.offset == 48


def test_parser_accepts_league():
    args = run.create_parser().parse_args(["league", "-c", "x.yml"])
    assert args.cmd == "league" and args.config_file == "x.yml"
    assert "league" in run.CMD_LIST
