"""GPU tests of the engine's evaluation cache: a leaf served from the cache gets the bits the tower would have produced, so
seeded games are identical with the cache on and off -- with a table small enough to evict all the time, with two slot
groups that insert and look up concurrently, and after new weights are loaded into the engine's network."""
import numpy as np
import pytest

from oracle import mcts
from reversi_zero_b200 import engine as E, net as N
from reversi_zero_b200.agent import model as M

pytestmark = pytest.mark.gpu

MC = M.ModelConfig(cnn_filter_num=256, res_layer_num=2, value_fc_size=256)
PP = mcts.PlayParams(simulation_num_per_move=48, parallel_search_num=8, c_puct=5, noise_eps=0.25, dirichlet_alpha=0.5,
                     change_tau_turn=4, thinking_loop=1, resign_threshold=None, share_mtcs_info_in_self_play=True)
GAMES = 64


def make_net(seed):
    net = N.Net(MC)
    net.load_weights(M.build_random_weights(MC, seed))
    return net


@pytest.fixture(scope="module")
def net():
    return make_net(0)


def play(net, cache_mb, groups):
    eng = E.Engine(E.engine_cfg_from_play_config(PP, games=GAMES, seed=7, eval_mode=E.EVAL_NET, max_games=GAMES,
                                                 overlap_groups=groups, eval_cache_mb=cache_mb), net)
    eng.run(finished_target=GAMES)
    games = sorted(eng.poll(), key=lambda g: g["game_id"])
    st = eng.stats()
    lookups, hits = eng.cache_turn_stats()
    eng.close()
    assert len(games) == GAMES
    return games, st, lookups, hits


def assert_same_games(a, b):
    for ga, gb in zip(a, b):
        for k in ("game_id", "winner", "black", "white", "expansions", "simulations", "turn"):
            assert ga[k] == gb[k], (ga["game_id"], k)
        assert len(ga["plies"]) == len(gb["plies"])
        for pa, pb in zip(ga["plies"], gb["plies"]):
            assert (pa["own"], pa["enemy"], pa["action"], pa["n"], pa["q"]) == (pb["own"], pb["enemy"], pb["action"], pb["n"], pb["q"])
            assert np.array_equal(pa["N"], pb["N"])


@pytest.mark.parametrize("cache_mb,groups", [(64, 1), (1, 1), (64, 2)])
def test_games_identical_with_cache(net, cache_mb, groups):
    """(64, 1): the plain case; (1, 1): 455 sets of 8 entries, so inserts keep evicting; (64, 2): two slot groups share the
    table on two streams."""
    off, st_off, lk_off, _ = play(net, -1, groups)
    on, st_on, lookups, hits = play(net, cache_mb, groups)
    assert_same_games(off, on)
    assert st_off["cache_lookups"] == 0 and st_off["cache_hits"] == 0 and int(lk_off.sum()) == 0
    assert st_off["tower_rows"] == st_off["expansions"]
    assert st_on["expansions"] == st_off["expansions"]
    assert st_on["cache_hits"] > 0
    assert st_on["cache_lookups"] == st_on["expansions"] == int(lookups.sum())
    assert st_on["cache_hits"] == int(hits.sum())
    assert st_on["tower_rows"] + st_on["cache_hits"] == st_off["tower_rows"]
    assert lookups[60] == 0  # no warm start: every game is played from the opening


def test_weight_reload_invalidates_cache():
    """Every slot searches the same root, so the second slot onwards is served from the cache.  After new weights are
    loaded, a search must equal that of a fresh engine on the new weights: no entry of the old network is used."""
    own, enemy = 0x00000000081d0603, 0x0002043814020100
    net = make_net(1)
    eng = E.Engine(E.engine_cfg_from_play_config(PP, games=16, seed=5, eval_mode=E.EVAL_NET, eval_cache_mb=64), net)
    n_old, _ = eng.search_root(own, enemy, 1, 3)
    assert eng.stats()["cache_hits"] > 0
    net.load_weights(M.build_random_weights(MC, 2))
    got = [eng.search_root(own, enemy, 1, s) for s in (0, 3, 15)]
    eng.close()
    fresh = E.Engine(E.engine_cfg_from_play_config(PP, games=16, seed=5, eval_mode=E.EVAL_NET, eval_cache_mb=-1), net)
    want = [fresh.search_root(own, enemy, 1, s) for s in (0, 3, 15)]
    fresh.close()
    for (n, w), (n_ref, w_ref) in zip(got, want):
        assert np.array_equal(n, n_ref) and np.array_equal(w, w_ref)
    assert not np.array_equal(got[1][0], n_old)  # the two networks really search differently
