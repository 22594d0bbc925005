"""GPU suite for the 64- and 128-filter wgmma tower (csrc/rz_net_tc_narrow.cu): the fp32 oracle (oracle/nn.py) on
ragged batches, the number-format bound on trained-like weights, bit-for-bit determinism and independence of where a
board lands in a tile, AUTO's selection, the engine's counted path against the oracle search, and the trainer's blob."""
import numpy as np
import pytest
import torch

from oracle import bitboard as ob, mcts, nn as onn
from reversi_zero_b200 import _cabi, device as D, engine as E, net as N, train as T
from reversi_zero_b200.agent import model as M
from reversi_zero_b200.agent.api import ReversiModelAPI

pytestmark = pytest.mark.gpu

WIDTHS = [64, 128]
NAMES = ("policy", "value", "logits", "vlogit", "tower")
ROOT = (0x00000000081d0603, 0x0002043814020100)


def selfplay_positions(n, seed):
    """positions from random playouts (side-to-move frame), some of them dihedral-transformed"""
    rng = np.random.default_rng(seed)
    own, enemy = [], []
    while len(own) < n:
        e = ob.Env().reset()
        while not e.done and len(own) < n:
            o, en = e.own_enemy()
            t = int(rng.integers(8))
            own.append(ob.dihedral(o, t)); enemy.append(ob.dihedral(en, t))
            legal = ob.find_correct_moves(o, en)
            ms = [i for i in range(64) if legal >> i & 1]
            e.step(ms[rng.integers(len(ms))])
    return np.array(own, np.uint64), np.array(enemy, np.uint64)


def make_net(F, R, seed, perturb=False, V=256):
    mc = M.ModelConfig(cnn_filter_num=F, res_layer_num=R, value_fc_size=V)
    w = M.build_random_weights(mc, seed, perturb_bn=perturb)
    net = N.Net(mc)
    net.load_weights(w)
    return net, w


def heads(net, own, enemy, impl=N.IMPL_TCGEN05, tower=True, stream=None):
    """the debug entry point: probabilities, value, both logits and (optionally) the fp32 tower output [n][F][8][8]"""
    n, F = own.size, net.mc.cnn_filter_num
    d_own, d_en = D.to_device(own), D.to_device(enemy)
    out = dict(policy=D.empty(n * 64, np.float32), value=D.empty(n, np.float32), logits=D.empty(n * 64, np.float32),
               vlogit=D.empty(n, np.float32))
    tow = D.empty(n * 64 * F, np.float32) if tower else None
    net.debug_heads_impl_dev(d_own, d_en, out["policy"], out["value"], out["logits"], out["vlogit"], n, impl, tower_t=tow,
                             stream_ptr=stream)
    torch.cuda.synchronize()
    got = {k: v.cpu().numpy() for k, v in out.items()}
    got["policy"], got["logits"] = got["policy"].reshape(n, 64), got["logits"].reshape(n, 64)
    if tower:
        got["tower"] = tow.cpu().numpy().reshape(n, 64, F).transpose(0, 2, 1).reshape(n, F, 8, 8)
    return got


def predict_dev(net, own, enemy, impl=N.IMPL_AUTO, stream=None):
    n = own.size
    d_own, d_en = D.to_device(own), D.to_device(enemy)
    p, v = D.empty(n * 64, np.float32), D.empty(n, np.float32)
    net.predict_dev(d_own, d_en, p, v, n, impl, D.stream_ptr(stream) if stream is not None else None)
    torch.cuda.synchronize()
    return p.cpu().numpy().reshape(n, 64), v.cpu().numpy()


def same_bits(a, b):
    return all(np.array_equal(np.asarray(a[k]).view(np.int32), np.asarray(b[k]).view(np.int32)) for k in a)


# ---- 1. against the fp32 oracle ------------------------------------------------------------------------------------
@pytest.mark.parametrize("F", WIDTHS)
@pytest.mark.parametrize("R,kind", [(0, "new"), (1, "new"), (2, "new"), (10, "new"), (0, "perturbed"), (1, "perturbed"),
                                    (2, "perturbed")])
def test_narrow_tower_vs_oracle(F, R, kind):
    """ragged batches against 4 / 8 boards per tile, and more tiles than CTAs (1100 positions); `--new` weights and
    perturbed BatchNorm.  1e-3 on probabilities, value and both logits.  At 10 blocks the fp16 operand format alone costs
    up to 9.1e-4 on these policy logits (scale 2.5), so there the logits are held to the format bound of
    test_narrow_trained_like_weights_format_bound instead.  Trained-like weights of a 10-block tower are tested below."""
    net, w = make_net(F, R, 100 * R + F, perturb=kind == "perturbed")
    own, enemy = selfplay_positions(1100, R + F)
    planes = onn.planes_from_bitboards(own, enemy)
    ref = dict(zip(NAMES, onn.forward_logits(w, planes, R)))
    tol = dict(policy=1e-3, value=1e-3, logits=1e-3, vlogit=1e-3)
    if R >= 10:
        fmt = dict(zip(NAMES, onn.forward_fp16_operands(w, planes, R)))
        for k in ("logits", "vlogit"):
            tol[k] = max(1e-3, 1.6 * np.abs(fmt[k] - ref[k]).max() + 3e-4)
    for n in (1, 2, 3, 5, 7, 9, 263, 1100):
        got = heads(net, own[:n], enemy[:n])
        for k in ("logits", "vlogit", "policy", "value"):
            err = np.abs(got[k] - ref[k][:n]).max()
            assert err <= tol[k], (n, k, err, tol[k])
        terr, scale = np.abs(got["tower"] - ref["tower"][:n]).max(), np.abs(ref["tower"][:n]).max()
        assert terr <= 4e-3 * max(scale, 1.0), (n, terr, scale)
        p, v = predict_dev(net, own[:n], enemy[:n])   # the production entry point (AUTO) gives the same bits
        assert same_bits(dict(p=p, v=v), dict(p=got["policy"], v=got["value"])), n
    api = ReversiModelAPI(None, net)   # host-buffer path
    p2, v2 = api.predict(planes[:5])
    assert np.abs(p2 - ref["policy"][:5]).max() <= 1e-3 and np.abs(v2[:, 0] - ref["value"][:5]).max() <= 1e-3
    net.close()


# ---- 2. trained-like weights ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("F", WIDTHS)
@pytest.mark.parametrize("kind", ["perturbed", "calibrated"])
def test_narrow_trained_like_weights_format_bound(F, kind):
    """the kernel adds nothing to the error of its number format (oracle/nn.py forward_fp16_operands), with the floors of
    test_net_gpu.py::test_tcgen05_trained_like_weights_format_bound; probabilities stay within 1e-3"""
    mc = M.ModelConfig(cnn_filter_num=F, res_layer_num=10, value_fc_size=256)
    w = M.build_random_weights(mc, 5, perturb_bn=True)
    if kind == "calibrated":
        oc, ec = selfplay_positions(256, 11)
        onn.calibrate_bn(w, onn.planes_from_bitboards(oc, ec), 10)
    own, enemy = selfplay_positions(64, 5)
    planes = onn.planes_from_bitboards(own, enemy)
    net = N.Net(mc)
    net.load_weights(w)
    got = heads(net, own, enemy)
    ref = dict(zip(NAMES, onn.forward_logits(w, planes, 10)))
    fmt = dict(zip(NAMES, onn.forward_fp16_operands(w, planes, 10)))
    for k, floor in (("tower", 1e-3), ("logits", 3e-4), ("vlogit", 3e-4)):
        kernel_err, format_err = np.abs(got[k] - ref[k]).max(), np.abs(fmt[k] - ref[k]).max()
        assert kernel_err <= 1.6 * format_err + floor, (kind, k, kernel_err, format_err)
    assert np.abs(got["policy"] - ref["policy"]).max() <= 1e-3
    net.close()


# ---- 3. determinism and placement independence ---------------------------------------------------------------------
@pytest.mark.parametrize("F", WIDTHS)
def test_narrow_repeat_clusters_and_streams_give_the_same_bits(F):
    net, _ = make_net(F, 10, 7 + F)
    own, enemy = selfplay_positions(301, 4)
    ref = heads(net, own, enemy)
    assert same_bits(ref, heads(net, own, enemy))
    try:
        outs = {}
        for cluster in (1, 2):
            N.set_tower_cluster(cluster)
            outs[cluster] = heads(net, own, enemy)
        assert same_bits(outs[1], outs[2]) and same_bits(outs[2], ref)
    finally:
        N.set_tower_cluster(2)
    p0, v0 = predict_dev(net, own[:64], enemy[:64])
    streams = [torch.cuda.Stream() for _ in range(12)]
    for s in streams:
        p, v = predict_dev(net, own[:64], enemy[:64], stream=s)
        assert p.tobytes() == p0.tobytes() and v.tobytes() == v0.tobytes()
    net.close()


@pytest.mark.parametrize("F", WIDTHS)
def test_narrow_outputs_do_not_depend_on_the_tile_slot(F):
    """a position gives the same bits alone, in a batch and in a permuted batch: wherever its board lands in a tile"""
    net, _ = make_net(F, 2, 3 + F, perturb=True)
    own, enemy = selfplay_positions(37, 9)
    batch = heads(net, own, enemy)
    perm = np.random.default_rng(1).permutation(own.size)
    shuffled = heads(net, own[perm], enemy[perm])
    assert same_bits({k: v[perm] for k, v in batch.items()}, shuffled)
    for i in (0, 1, 5, 11, 36):
        alone = heads(net, own[i:i + 1], enemy[i:i + 1])
        assert same_bits({k: v[i:i + 1] for k, v in batch.items()}, alone), i
    net.close()


# ---- 4. selection --------------------------------------------------------------------------------------------------
def test_auto_selects_the_tensor_core_tower_by_width():
    for F in (64, 128, 256):
        net = N.Net(M.ModelConfig(cnn_filter_num=F, res_layer_num=1, value_fc_size=256))
        assert [net.select_impl(n) for n in (1, 8, 296, 32768)] == [N.IMPL_TCGEN05] * 4, F
        net.close()
    for F, V in ((16, 16), (32, 64), (96, 256), (128, 513)):
        net = N.Net(M.ModelConfig(cnn_filter_num=F, res_layer_num=1, value_fc_size=V))
        assert net.select_impl(1) == N.IMPL_GENERIC and net.select_impl(4096) == N.IMPL_GENERIC, (F, V)
        net.close()


@pytest.mark.parametrize("F,V,match", [(32, 64, "64, 128 or 256"), (96, 256, "64, 128 or 256"), (128, 513, "value_fc_size <= 512")])
def test_tensor_core_paths_reject_unsupported_shapes(F, V, match):
    net, _ = make_net(F, 1, 2, V=V)
    own, enemy = selfplay_positions(3, 2)
    d_own, d_en = D.to_device(own), D.to_device(enemy)
    p, v, lg, vl = D.empty(3 * 64, np.float32), D.empty(3, np.float32), D.empty(3 * 64, np.float32), D.empty(3, np.float32)
    with pytest.raises(_cabi.RzError, match=match):
        net.predict_dev(d_own, d_en, p, v, 3, N.IMPL_TCGEN05)
    with pytest.raises(_cabi.RzError, match=match):
        net.debug_tower_dev(d_own, d_en, p, v, D.empty(3 * 64 * F, np.float32), 3)
    with pytest.raises(_cabi.RzError, match=match):
        net.debug_heads_dev(d_own, d_en, p, v, lg, vl, 3)
    if V <= 512:
        with pytest.raises(_cabi.RzError, match=match):
            net.debug_heads_impl_dev(d_own, d_en, p, v, lg, vl, 3, N.IMPL_TCGEN05)
    with pytest.raises(_cabi.RzError):
        net.debug_heads_impl_dev(d_own, d_en, p, v, lg, vl, 3, N.IMPL_SPLIT)
    net.predict_dev(d_own, d_en, p, v, 3, N.IMPL_AUTO)   # AUTO runs the generic kernel
    torch.cuda.synchronize()
    assert torch.isfinite(v).all()
    net.close()


# ---- 5. engine integration -----------------------------------------------------------------------------------------
def test_search_with_a_128_filter_net_matches_the_oracle_in_every_slot():
    """the engine's counted launches under AUTO against the oracle search whose evaluator is the same network on the host
    path: both see the same bits for every leaf, so root visits and values are identical in every slot"""
    net, _ = make_net(128, 2, 4, perturb=True)
    pp = mcts.PlayParams(simulation_num_per_move=48, parallel_search_num=4, noise_eps=0.0, c_puct=5, change_tau_turn=4,
                         thinking_loop=1, resign_threshold=None, share_mtcs_info_in_self_play=True)
    eng = E.Engine(E.engine_cfg_from_play_config(pp, games=24, seed=31, eval_mode=E.EVAL_NET), net)
    api = ReversiModelAPI(None, net, N.IMPL_TCGEN05)
    for slot in range(24):
        n, w = eng.search_root(*ROOT, 1, slot)
        game = mcts.SelfPlayGame(pp, api, seed=31, game_id=slot)
        game.search(*ROOT, 1)
        node = game.table[ROOT]
        assert list(n) == list(node.N), slot
        assert np.array_equal(w, node.W), slot
    eng.close()
    net.close()


def replay_check(g):
    env = ob.Env().reset()
    for ply in g["plies"]:
        own, enemy = env.own_enemy()
        assert (ply["own"], ply["enemy"], ply["pid"]) == (own, enemy, env.next_player)
        legal = ob.find_correct_moves(own, enemy)
        assert all((legal >> int(a)) & 1 for a in np.nonzero(ply["N"])[0])
        assert ply["action"] == -1 or (legal >> ply["action"]) & 1
        env.step(None if ply["action"] < 0 else ply["action"])
    assert env.done and env.winner == g["winner"] and (env.black, env.white) == (g["black"], g["white"])


def test_games_with_a_64_filter_net_replay_and_repeat():
    net, _ = make_net(64, 2, 8)
    pp = mcts.PlayParams(simulation_num_per_move=16, parallel_search_num=4, c_puct=5, noise_eps=0.25)

    def play():
        eng = E.Engine(E.engine_cfg_from_play_config(pp, games=32, seed=5, max_games=32), net)
        eng.run(finished_target=32)
        games = sorted(eng.poll(), key=lambda g: g["game_id"])
        assert eng.stats()["nn_launches"] > 0
        eng.close()
        return games

    first, second = play(), play()
    assert len(first) == 32
    for g in first:
        replay_check(g)
    key = lambda gs: [(g["game_id"], g["winner"], [(p["action"], list(p["N"])) for p in g["plies"]]) for g in gs]
    assert key(first) == key(second)
    net.close()


# ---- 6. trainer to inference ---------------------------------------------------------------------------------------
def test_trained_128_filter_blob_runs_on_the_narrow_tower():
    mc = M.ModelConfig(cnn_filter_num=128, res_layer_num=2, value_fc_size=256)
    own, enemy = selfplay_positions(512, 12)
    planes = onn.planes_from_bitboards(own, enemy)
    rng = np.random.default_rng(12)
    pol = rng.random((512, 64)).astype(np.float32)
    pol /= pol.sum(1, keepdims=True)
    z = rng.choice([-1.0, 1.0], 512).astype(np.float32)
    states = torch.from_numpy(np.ascontiguousarray(planes, np.uint8)).cuda()
    policy, zt = torch.from_numpy(pol).cuda(), torch.from_numpy(z).cuda()
    tr = T.Trainer(mc, max_batch=128)
    tr.load_blob(M.weights_to_blob(mc, M.build_random_weights(mc, 2)))
    for i in range(3):
        tr.step(states, policy, zt, torch.arange(128 * i, 128 * i + 128, dtype=torch.int32, device="cuda"), 0.05)
    blob_t = tr.blob_dev()
    net = N.Net(mc)
    net.load_blob_dev(blob_t)
    torch.cuda.synchronize()
    assert net.select_impl(100) == N.IMPL_TCGEN05
    p, v = net.predict_planes(planes[:100])
    p_ref, v_ref = onn.forward(M.blob_to_weights(mc, blob_t.cpu().numpy()), planes[:100], 2)
    assert np.abs(p - p_ref).max() < 1e-3 and np.abs(v - v_ref).max() < 1e-3
    net.close()
    tr.close()
