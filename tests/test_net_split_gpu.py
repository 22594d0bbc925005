"""GPU suite for the split tower (csrc/rz_net_split.cu, RZ_NET_IMPL_SPLIT): bit-identical to the throughput tower
(RZ_NET_IMPL_TCGEN05) in policy, value, policy logits, value logit and the fp32 tower output; AUTO's switch between them;
and a one-slot search that sees the same statistics under either."""
import numpy as np
import pytest
import torch

from oracle import mcts
from reversi_zero_b200 import engine as E
from reversi_zero_b200.agent import model as M
from reversi_zero_b200.net import Net, IMPL_AUTO, IMPL_TCGEN05, IMPL_SPLIT

pytestmark = pytest.mark.gpu

T = 0   # rz_net.cu kSplitMaxBatch: AUTO never picks the split tower (it was not faster on an H100)


def positions(n, seed):
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 2 ** 63, size=n, dtype=np.int64)
    r = rng.integers(0, 2 ** 63, size=n, dtype=np.int64)
    m = rng.integers(0, 2 ** 63, size=n, dtype=np.int64)
    occ = a & m if seed % 2 else a | m
    return torch.from_numpy(occ & r).cuda(), torch.from_numpy(occ & ~r).cuda()


def make_net(res_blocks, seed, perturb=0.0, value_fc=256):
    mc = M.ModelConfig(cnn_filter_num=256, res_layer_num=res_blocks, value_fc_size=value_fc)
    w = M.build_random_weights(mc, seed)
    blob = M.weights_to_blob(mc, w)
    if perturb:   # relative noise on every weight; BatchNorm variances stay positive
        rng = np.random.default_rng(seed + 1)
        blob = (blob * (1 + perturb * rng.standard_normal(blob.shape))).astype(np.float32)
    net = Net(mc)
    net.load_blob(blob)
    return net


def run(net, own, enemy, impl, stream=None):
    n = own.shape[0]
    out = dict(policy=torch.empty((n, 64), device="cuda"), value=torch.empty((n,), device="cuda"),
               logits=torch.empty((n, 64), device="cuda"), vlogit=torch.empty((n,), device="cuda"),
               tower=torch.empty((n, 64, 256), device="cuda"))
    net.debug_heads_impl_dev(own, enemy, out["policy"], out["value"], out["logits"], out["vlogit"], n, impl, tower_t=out["tower"],
                             stream_ptr=stream)
    return out


def same(a, b):
    for k in a:
        assert torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)), k


@pytest.mark.parametrize("res_blocks", [0, 1, 2, 10, 19])
def test_split_is_bit_identical_to_the_throughput_tower(res_blocks):
    for variant, perturb in (("new", 0.0), ("perturbed", 0.05)):
        net = make_net(res_blocks, 11 + res_blocks, perturb)
        for n in (1, 2, 3, 7, 8, 16, 17, 40):
            own, enemy = positions(n, 100 * res_blocks + n)
            a, b = run(net, own, enemy, IMPL_TCGEN05), run(net, own, enemy, IMPL_SPLIT)
            torch.cuda.synchronize()
            assert torch.isfinite(a["value"]).all()
            same(a, b)
        net.close()


def test_small_value_head_and_auto():
    net = make_net(2, 5, value_fc=7)
    own, enemy = positions(5, 3)
    same(run(net, own, enemy, IMPL_TCGEN05), run(net, own, enemy, IMPL_SPLIT))
    same(run(net, own, enemy, IMPL_AUTO), run(net, own, enemy, IMPL_SPLIT))   # AUTO picks either; the bytes are the same


def test_select_impl_switches_at_threshold():
    net = make_net(1, 1)
    assert [net.select_impl(n) for n in (1, 8, 16, 4096)] == [IMPL_SPLIT if n <= T else IMPL_TCGEN05 for n in (1, 8, 16, 4096)]
    small = Net(M.ModelConfig(cnn_filter_num=16, res_layer_num=1, value_fc_size=16))
    assert small.select_impl(1) == 1   # generic kernel below 256 filters


def test_repeat_launches_and_concurrent_streams_give_the_same_bytes():
    net = make_net(10, 7)
    own, enemy = positions(8, 9)
    ref = run(net, own, enemy, IMPL_SPLIT)
    for _ in range(5):
        same(ref, run(net, own, enemy, IMPL_SPLIT))
    streams = [torch.cuda.Stream() for _ in range(12)]
    outs = []
    for s in streams:
        with torch.cuda.stream(s):
            outs.append(run(net, own, enemy, IMPL_SPLIT, stream=C_stream(s)))
    torch.cuda.synchronize()
    for o in outs:
        same(ref, o)


def C_stream(s):
    import ctypes
    return ctypes.c_void_p(s.cuda_stream)


def test_one_slot_search_sees_the_same_statistics():
    """a ch5 network, K = 8: the engine's counted path (capacity 8, device-side count below it) with either tower"""
    mc = M.ModelConfig(cnn_filter_num=256, res_layer_num=10, value_fc_size=256)
    net = Net(mc)
    net.load_weights(M.build_random_weights(mc, 3))
    pp = mcts.PlayParams(simulation_num_per_move=400, parallel_search_num=8, c_puct=5, noise_eps=0.0)
    own, enemy = 0x00000000081d0603, 0x0002043814020100
    res = []
    for impl in (IMPL_SPLIT, IMPL_TCGEN05):
        eng = E.Engine(E.engine_cfg_from_play_config(pp, games=1, seed=3, net_impl=impl), net)
        res.append(eng.search_root(own, enemy, 1, 0))
        eng.close()
    (n0, w0), (n1, w1) = res
    assert n0.sum() >= 399 and np.array_equal(n0, n1) and np.array_equal(w0.view(np.int32), w1.view(np.int32))
