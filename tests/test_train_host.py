"""CPU suite for the device trainer: the fp64 oracle step (oracle/train.py) against central finite differences and a
hand computation of the Keras update rules, the TF32 format model, and the trainer's configuration checks (which run
before any CUDA call)."""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import nn as onn, train as ot
from reversi_zero_b200 import _cabi
from reversi_zero_b200.agent import model as M

MINI = dict(cnn_filter_num=16, res_layer_num=1, value_fc_size=8)


def _batch(n, seed):
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 2 ** 64, n, dtype=np.uint64)
    r = rng.integers(0, 2 ** 64, n, dtype=np.uint64)
    planes = onn.planes_from_bitboards(a & r, a & ~r)
    policy = rng.dirichlet(np.full(64, 0.3), n).astype(np.float32)
    z = rng.choice([-1.0, 0.0, 1.0], n).astype(np.float32)
    return planes, policy, z


def _weights(mc, seed):
    w = M.build_random_weights(mc, seed, perturb_bn=True)
    return {k: v.astype(np.float64) for k, v in w.items()}


def test_oracle_gradient_matches_central_differences():
    mc = M.ModelConfig(**MINI)
    w = _weights(mc, 1)
    planes, policy, z = _batch(4, 2)
    l2 = 1e-4
    (total, _, _), grads, _ = ot.loss_and_grad(w, planes, policy, z, 1, l2)

    def loss_at(ww):
        return ot.loss_and_grad(ww, planes, policy, z, 1, l2)[0][0]

    rng = np.random.default_rng(3)
    h = 1e-6  # small enough that no ReLU input of the 4 x 64 pixels changes sign inside the stencil
    for name, g in grads.items():
        for _ in range(2):  # random unit directions: every element of the tensor takes part
            d = rng.standard_normal(g.shape)
            d /= np.linalg.norm(d)
            wp, wm = dict(w), dict(w)
            wp[name] = w[name] + h * d
            wm[name] = w[name] - h * d
            fd = (loss_at(wp) - loss_at(wm)) / (2 * h)
            an = float((g * d).sum())
            if name.endswith(".bias") and not name.startswith(("policy_fc", "value_fc")):
                assert abs(fd) < 1e-8 and abs(an) < 1e-12, (name, fd, an)  # conv bias under training-mode BN: exactly 0
            else:
                assert abs(fd - an) <= 1e-6 * abs(an) + 1e-12, (name, fd, an)


def test_oracle_moving_statistics_and_keras_sgd_by_hand():
    mc = M.ModelConfig(**MINI)
    w = _weights(mc, 4)
    planes, policy, z = _batch(6, 5)
    w1, v1, _, g1 = ot.step(w, None, planes, policy, z, 0.1, 1, 1e-4)
    # conv0's batch statistics by hand
    k = torch.from_numpy(w["conv0.kernel"]).permute(3, 2, 0, 1)
    y = F.conv2d(torch.from_numpy(planes).double(), k, torch.from_numpy(w["conv0.bias"]), padding=1).numpy()
    mean, var = y.mean(axis=(0, 2, 3)), y.var(axis=(0, 2, 3))
    np.testing.assert_allclose(w1["conv0.bn_mean"], 0.99 * w["conv0.bn_mean"] + 0.01 * mean, rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(w1["conv0.bn_var"], 0.99 * w["conv0.bn_var"] + 0.01 * var, rtol=1e-12, atol=1e-14)
    # Keras SGD with an lr change: v = 0.9 v - lr g; w = w + v (not torch.optim.SGD's v = 0.9 v + g; w -= lr v)
    w2, v2, _, g2 = ot.step(w1, v1, planes, policy, z, 0.01, 1, 1e-4)
    for name in g1:
        np.testing.assert_allclose(v1[name], -0.1 * g1[name], rtol=1e-12, atol=1e-15)
        np.testing.assert_allclose(w2[name], w[name] - 0.1 * g1[name] + 0.9 * (-0.1 * g1[name]) - 0.01 * g2[name], rtol=1e-10,
                                   atol=1e-13)
    torch_sgd = w1["policy_fc.kernel"] - 0.01 * (0.9 * g1["policy_fc.kernel"] + g2["policy_fc.kernel"])
    assert np.abs(torch_sgd - w2["policy_fc.kernel"]).max() > 1e-4  # the two forms really differ after an lr change
    # the L2 term counts kernels only and is not divided by the batch size
    wk = dict(w)
    wk["policy_fc.bias"] = w["policy_fc.bias"] + 1.0
    l_a = ot.loss_and_grad(w, planes, policy, z, 1, 0.5)[0]
    l_b = ot.loss_and_grad(w, planes, policy, z, 1, 0.0)[0]
    expected = 0.5 * sum((v ** 2).sum() for n, v in w.items() if n.endswith(".kernel"))
    assert abs((l_a[0] - l_b[0]) - expected) < 1e-9 * expected


def test_tf32_rounding_and_format_model():
    x = torch.tensor([1.0, 1.0 + 2 ** -11, 1.0 + 2 ** -10, -(1.0 + 2 ** -11), 3.0e-3, 0.0], dtype=torch.float64)
    r = ot.tf32(x)
    assert r[0] == 1.0 and r[1] == 1.0 + 2 ** -10 and r[2] == 1.0 + 2 ** -10 and r[3] == -(1.0 + 2 ** -10) and r[5] == 0.0
    assert (ot.tf32(r) == r).all()
    mc = M.ModelConfig(**MINI)
    w = _weights(mc, 6)
    planes, policy, z = _batch(8, 7)
    l64, g64, _ = ot.loss_and_grad(w, planes, policy, z, 1, 1e-4)
    lfm, gfm, _ = ot.loss_and_grad(w, planes, policy, z, 1, 1e-4, tf32_convs=True)
    assert abs(lfm[0] - l64[0]) < 1e-3 * abs(l64[0])
    for k in ("res0.conv1.kernel", "conv0.kernel", "policy_fc.kernel"):
        err = np.linalg.norm(gfm[k] - g64[k]) / np.linalg.norm(g64[k])
        assert 0 < err < 5e-2, (k, err)  # TF32's 2^-11 unit roundoff, amplified by the BN backward's cancellation


@pytest.mark.parametrize("batch,cin,cout", [(1, 2, 16), (3, 48, 16), (2, 16, 80)])
def test_conv_gemm_restatement_matches_torch(batch, cin, cout):
    """oracle/train.py's gather-and-matmul convolutions (the reference of tests/test_train_shapes_gpu.py) are the
    convolution, input gradient and weight gradient of F.conv2d(padding=1) on Keras-layout kernels"""
    g = torch.Generator().manual_seed(batch * cin + cout)
    x = torch.randn(batch, cin, 8, 8, generator=g, dtype=torch.float64)
    k = torch.randn(3, 3, cin, cout, generator=g, dtype=torch.float64)
    dy = torch.randn(batch, cout, 8, 8, generator=g, dtype=torch.float64)
    kt = k.permute(3, 2, 0, 1)
    pix = lambda t: t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])   # NCHW -> [B*64][C]
    ok = lambda a, b: torch.allclose(a, b, rtol=1e-12, atol=1e-12)
    assert ok(ot.conv3x3(pix(x), k.reshape(9, cin, cout)), pix(F.conv2d(x, kt, padding=1)))
    assert ok(ot.conv3x3_dgrad(pix(dy), k.reshape(9, cin, cout)), pix(torch.nn.grad.conv2d_input(x.shape, kt, dy, padding=1)))
    assert ok(ot.conv3x3_wgrad(pix(x), pix(dy)),
              torch.nn.grad.conv2d_weight(x, kt.shape, dy, padding=1).permute(2, 3, 1, 0).reshape(9, cin, cout))


@pytest.mark.parametrize("cfg,batch", [(MINI, 6), (dict(cnn_filter_num=48, res_layer_num=2, value_fc_size=24), 5)],
                         ids=["mini", "48x2"])
def test_stage_chain_matches_autograd(cfg, batch):
    """oracle/train.py's per-stage references (the fp64 side of tests/test_train_stages_gpu.py), chained in the device
    step's order and layout, give loss_and_grad's losses, batch statistics and every gradient to 1e-10 relative"""
    mc = M.ModelConfig(**cfg)
    w = _weights(mc, 8)
    planes, policy, z = _batch(batch, 9)
    policy[0] = np.eye(64)[17]   # a one-hot target
    l2 = 1e-4
    losses, grads, stats = ot.loss_and_grad(w, planes, policy, z, mc.res_layer_num, l2)
    sl, sg, ss = ot.stage_loss_and_grad({k: torch.from_numpy(v) for k, v in w.items()}, planes, policy, z, mc.res_layer_num, l2)
    for a, b in zip(sl, losses):
        assert abs(a - b) <= 1e-10 * abs(b), (sl, losses)
    rel = lambda a, b: np.linalg.norm(np.asarray(a, np.float64).ravel() - np.asarray(b).ravel()) / max(np.linalg.norm(b), 1e-300)
    assert set(sg) == set(grads)
    for name, g in grads.items():
        if name.endswith(".bias") and not name.startswith(("policy_fc", "value_fc")):   # exactly 0 up to rounding in both
            assert np.abs(sg[name].numpy()).max() < 1e-12 and np.abs(g).max() < 1e-12, name
        else:
            assert sg[name].shape == g.shape and rel(sg[name].numpy(), g) <= 1e-10, (name, rel(sg[name].numpy(), g))
    assert set(ss) == set(stats)
    for name, (m, v) in stats.items():
        assert rel(ss[name][0].numpy(), m) <= 1e-10 and rel(ss[name][1].numpy(), v) <= 1e-10, name


def test_stage_update_is_keras_sgd():
    """the update stage: L2 on kernels only, Keras momentum form, moving averages"""
    w, vel, g = (torch.tensor([0.5, -2.0], dtype=torch.float64), torch.tensor([0.1, 0.3], dtype=torch.float64),
                 torch.tensor([1.0, -1.0], dtype=torch.float64))
    nw, nv, ng = ot.sgd_update(w, vel, g, 0.1, 0.9, 1e-2, kernel=True)
    assert torch.allclose(ng, torch.tensor([1.01, -1.04], dtype=torch.float64), rtol=0, atol=1e-15)
    assert torch.allclose(nv, 0.9 * vel - 0.1 * ng, rtol=0, atol=1e-15) and torch.allclose(nw, w + nv, rtol=0, atol=1e-15)
    assert torch.equal(ot.sgd_update(w, vel, g, 0.1, 0.9, 1e-2, kernel=False)[2], g)
    assert ot.moving_average(2.0, 4.0, 0.99) == pytest.approx(2.02, rel=1e-15)


DEBUG_SYMBOLS = ("rz_trainer_debug_tensor_dev", "rz_trainer_debug_keep_backward")


def test_debug_tensor_symbols_resolve():
    lib = C.CDLL(_cabi.LIB_PATH)
    for name in DEBUG_SYMBOLS:
        assert getattr(lib, name, None) is not None, name
        assert name in _cabi.SIGNATURES


@pytest.mark.parametrize("filters,res,kernel,batch", [(24, 1, 3, 8), (8, 1, 3, 8), (272, 1, 3, 8), (16, 1, 5, 8), (16, 1, 3, 0)])
def test_trainer_rejects_unsupported_configurations(filters, res, kernel, batch):
    ncfg = _cabi.NetCfg(filters, res, 8, kernel)
    tcfg = _cabi.TrainCfg(batch, 0.9, 1e-4, 0.99)
    h = C.c_void_p()
    assert _cabi.lib().rz_trainer_create(C.byref(ncfg), C.byref(tcfg), 0, C.byref(h)) == -1  # RZ_EINVAL
    assert not h.value
