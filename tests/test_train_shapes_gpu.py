"""GPU suite for the device trainer (csrc/rz_train.cu) across the shapes it accepts.

- Its convolution GEMMs, through the rz_trainer_debug_conv_dev hook: bit-exact on one-hot impulses (every output one
  product or zero) and on TF32 rounding ties, and within a per-element bound of an fp64 reference on dense operands, at
  widths 16 to 256, batches that end in half an M tile and in a short last split-K slice.
- The whole step against the fp64 oracle and its TF32 format model at widths 32 to 256, value heads 1 to 4096, 0 to 2
  residual blocks, batches below max_batch, and an epoch tail of the `opt` worker.
- Steps that do not depend on max_batch, bit for bit.
- The trained blob of a width without a tensor-core tower on the generic inference kernel, and that kernel against the
  fp32 oracle wherever AUTO sends it."""
import numpy as np
import pytest
import torch

from oracle import nn as onn, train as ot
from reversi_zero_b200 import net as N, train as T
from reversi_zero_b200.agent import model as M
from test_train_gpu import _check_against_oracle, _host, _oracle_steps, _weights, records  # noqa: F401 (records: fixture)

pytestmark = pytest.mark.gpu

WIDTHS = [16, 48, 64, 128, 144, 208, 256]
FWD_OPS = (T.CONV0_FWD, T.CONV_FWD, T.CONV_DGRAD)
WGRAD_OPS = (T.CONV_WGRAD, T.CONV0_WGRAD)
ALL_OPS = FWD_OPS + WGRAD_OPS
OP_NAMES = {T.CONV0_FWD: "conv0_fwd", T.CONV_FWD: "fwd", T.CONV_DGRAD: "dgrad", T.CONV_WGRAD: "wgrad", T.CONV0_WGRAD: "conv0_wgrad"}
# (filters, batch) whose weight-gradient split-K ends in a short slice; all but the last have an odd batch
EDGE_SHAPES = [(48, 67), (128, 97), (144, 37), (256, 100)]


def _cin(op, F):
    return 16 if op in (T.CONV0_FWD, T.CONV0_WGRAD) else F


def wgrad_split(cin, F, batch):
    """the step's weight-gradient split-K for this batch (wgrad_splits / launch_wgrad in rz_train.cu): records per
    slice, slices used"""
    tiles = -(-9 * cin // 128) * -(-F // 128)
    per = -(-batch // min(-(-264 // tiles), batch))
    return per, -(-batch // per)


def test_split_table_of_the_edge_shapes():
    """the edge shapes do reach the split-K edges they are chosen for: (splits, records per slice, slices, last slice)"""
    want = {48: (66, 2, 34, 1), 128: (30, 4, 25, 1), 144: (12, 4, 10, 1), 256: (8, 13, 8, 9)}
    for F, batch in EDGE_SHAPES:
        per, used = wgrad_split(F, F, batch)
        assert (min(-(-264 // (-(-9 * F // 128) * -(-F // 128))), batch), per, used, batch - (used - 1) * per) == want[F]


def _trainer(F, max_batch):
    return T.Trainer(M.ModelConfig(cnn_filter_num=F, res_layer_num=0, value_fc_size=1), max_batch=max_batch)


def _exact(rng, shape):
    """small integers x 2^-8: exact in TF32, and every product and sum below stays exact in fp32"""
    return torch.as_tensor(rng.integers(-127, 128, shape).astype(np.float32) / 256, device="cuda")


def _reference(op, x, k, bias, add):
    """fp64 reference of one hook op, operands rounded to TF32 exactly where the kernel rounds them (forward: activations
    and weights; input gradient: dy and the mirrored weights; weight gradient: input and dy), bias and add unrounded after
    the sum.  Returns (value, sum of |products|)."""
    r = lambda t: ot.tf32(t).double()
    if op in WGRAD_OPS:
        a = r(x[:, :2] if op == T.CONV0_WGRAD else x)
        return ot.conv3x3_wgrad(a, r(add)), ot.conv3x3_wgrad(a.abs(), r(add).abs())
    a, b = r(x[:, :2] if op == T.CONV0_FWD else x), r(k)
    f = ot.conv3x3_dgrad if op == T.CONV_DGRAD else ot.conv3x3
    ref, mag = f(a, b), f(a.abs(), b.abs())
    for t in (bias, add):
        if t is not None:
            ref = ref + t.double()
    return ref, mag


def _run(tr, op, batch, x, k, bias, add):
    got = tr.debug_conv(op, x, batch, kernel=None if op in WGRAD_OPS else k, bias=None if op in WGRAD_OPS else bias, add=add)
    return got.double(), _reference(op, x, k, bias, add)


def _operands(rng, op, F, batch, gen):
    """x [M][Cin], kernel [9][Cin_real][F], bias [F], add (= dy of the weight gradient) [M][F]"""
    conv0 = op in (T.CONV0_FWD, T.CONV0_WGRAD)
    return gen(rng, (64 * batch, _cin(op, F))), gen(rng, (9, 2 if conv0 else F, F)), gen(rng, (F,)), gen(rng, (64 * batch, F))


# ---- (a) impulses: every output is one product (plus bias and add) or zero, so it must be exact -----------------------
PIXELS = [0, 7, 56, 63, 3, 40, 36]   # the four corners, a top and a left edge pixel, the centre


@pytest.mark.parametrize("op", ALL_OPS, ids=lambda o: OP_NAMES[o])
@pytest.mark.parametrize("F,batch", EDGE_SHAPES + [(16, 3), (208, 5)])
def test_conv_impulses_are_exact(F, batch, op):
    """a one-hot activation (and, for the weight gradient, a one-hot dy) against dense operands, at the corners, edges and
    centre; on the first record, the last one and the first of the short last split-K slice; on the first and last
    channel (and conv0's padding channel 15, which must contribute nothing).  Catches a wrong tap, a wrong mirror, padding
    that leaks across records or boards, a missing mask and a dropped tail, exactly."""
    rng = np.random.default_rng(F * 1000 + batch + op)
    tr = _trainer(F, batch)
    x0, k, bias, add = _operands(rng, op, F, batch, _exact)
    cin = _cin(op, F)
    per, used = wgrad_split(cin, F, batch)
    recs = sorted({0, batch - 1, (used - 1) * per})
    chans = [0, 1, 15] if op in (T.CONV0_FWD, T.CONV0_WGRAD) else [0, F - 1]
    sides = ["x", "dy"] if op in WGRAD_OPS else ["x"]
    n = 0
    for side in sides:
        for b in recs:
            for p in PIXELS:
                for c in (chans if side == "x" else [0, F - 1]):
                    s = float(rng.integers(1, 128)) / 256 * (-1) ** n
                    x, a = (torch.zeros_like(x0), add) if side == "x" else (x0, torch.zeros_like(add))
                    (x if side == "x" else a)[b * 64 + p, c] = s
                    got, (ref, _) = _run(tr, op, batch, x, k, bias, a)
                    bad = (got != ref).nonzero()
                    assert bad.numel() == 0, (side, b, p, c, bad[:4].tolist(), got[tuple(bad[0])].item(), ref[tuple(bad[0])].item())
                    n += 1
    tr.close()


# ---- (b) TF32 rounding: ties go away from zero --------------------------------------------------------------------
TIES = [1 + 2 ** -11, -(1 + 2 ** -11), 1 + 2 ** -11 - 2 ** -23, 1 + 2 ** -11 + 2 ** -23, 1 + 2 ** -12 + 2 ** -20,
        1 + 2 ** -10 + 2 ** -11]


def test_tie_values_round_away_from_zero_in_the_oracle():
    r = ot.tf32(torch.tensor(TIES, dtype=torch.float32)).tolist()
    assert r == [1 + 2 ** -10, -(1 + 2 ** -10), 1.0, 1 + 2 ** -10, 1.0, 1 + 2 ** -9]


@pytest.mark.parametrize("op", ALL_OPS, ids=lambda o: OP_NAMES[o])
@pytest.mark.parametrize("side", ["A", "B"])
def test_conv_operands_round_ties_away(op, side):
    """one operand a one-hot on a TF32 tie (or just below or above one), the other exact: each output is
    tf32(x) * w exactly, with tf32 = round to nearest, ties away (cvt.rna).  Ties to even or raw fp32 bits differ.
    A is the activation (dy for the input gradient, the input for the weight gradient), B the weights (dy for the weight
    gradient)."""
    F, batch = 64, 3
    rng = np.random.default_rng(op * 2 + (side == "B"))
    tr = _trainer(F, batch)
    x0, k0, bias, add0 = _operands(rng, op, F, batch, _exact)
    for i, v in enumerate(TIES):
        x, k, add = x0, k0, add0
        if side == "A":
            x = torch.zeros_like(x0)
            x[64 + 9 * i, i % 2] = v
        elif op in WGRAD_OPS:
            add = torch.zeros_like(add0)
            add[64 + 9 * i, 5 * i] = v
        else:
            k = torch.zeros_like(k0)
            k[i, i % 2, 7 * i] = v
        got, (ref, _) = _run(tr, op, batch, x, k, bias, add)
        assert torch.equal(got, ref), (v, (got != ref).nonzero()[:4].tolist())
    tr.close()


# ---- (c) dense operands against fp64 ------------------------------------------------------------------------------
DENSE_SHAPES = [(F, b) for F in WIDTHS for b in (1, 3)] + EDGE_SHAPES + [(48, 1001)]
BOUND = 2.0 ** -16   # per element, times the sum of |products|: well under one product's size at every K here


def _normal(rng, shape):
    return torch.as_tensor(rng.standard_normal(shape, dtype=np.float32), device="cuda")


@pytest.mark.parametrize("op", ALL_OPS, ids=lambda o: OP_NAMES[o])
@pytest.mark.parametrize("F,batch", DENSE_SHAPES)
def test_conv_dense_vs_fp64(F, batch, op):
    """|got - ref| <= 2^-16 * sum |a * b| + 2^-23 * |ref| per element, against the fp64 product of the TF32-rounded
    operands; conv0's padding channels 2..15 hold random values that the zero padding of the weight image must cancel.
    Prints the worst |got - ref| / sum |a * b|."""
    rng = np.random.default_rng(F * 7 + batch * 3 + op)
    tr = _trainer(F, batch)
    x, k, bias, add = _operands(rng, op, F, batch, _normal)
    got, (ref, mag) = _run(tr, op, batch, x, k, bias, add)
    err = (got - ref).abs()
    ratio = (err / mag).max().item()
    print(f"\n{OP_NAMES[op]} F={F} B={batch}: worst |err| / sum|ab| = {ratio:.2e} = 2^{np.log2(max(ratio, 1e-300)):.1f}")
    assert bool((err <= BOUND * mag + 2.0 ** -23 * ref.abs()).all()), ratio
    tr.close()


def test_debug_conv_rejects_bad_arguments():
    tr = _trainer(64, 4)
    x, k = torch.zeros(64 * 4, 64, device="cuda"), torch.zeros(9, 64, 64, device="cuda")
    tr.debug_conv(T.CONV_FWD, x, 4, kernel=k)
    tr.debug_conv(T.CONV_WGRAD, x, 4, add=x)
    for op, xx, args in [(T.CONV_FWD, x, dict(batch=5, kernel=k)), (T.CONV_FWD, x, dict(batch=0, kernel=k)),
                         (T.CONV_FWD, None, dict(batch=4, kernel=k)), (T.CONV_FWD, x, dict(batch=4)),
                         (T.CONV_DGRAD, x, dict(batch=4)), (T.CONV_WGRAD, x, dict(batch=4)),
                         (T.CONV_WGRAD, x, dict(batch=4, kernel=k, add=x)), (T.CONV0_WGRAD, None, dict(batch=4, add=x)),
                         (7, x, dict(batch=4, kernel=k)), (-1, x, dict(batch=4, kernel=k))]:
        with pytest.raises(RuntimeError, match="failed \\(-1\\)"):
            tr.debug_conv(op, xx, **args)
    torch.cuda.synchronize()
    tr.close()


# ---- (d) the whole step against the fp64 oracle -------------------------------------------------------------------
def _trainer_run(mc, w0, records, idxs, lrs, max_batch):
    tr = T.Trainer(mc, max_batch=max_batch)
    tr.load_blob(M.weights_to_blob(mc, w0))
    losses = []
    for idx, lr in zip(idxs, lrs):
        loss = tr.step(*records, torch.as_tensor(np.asarray(idx, np.int32), device="cuda"), lr)
        losses.append(tuple(float(x) for x in loss.cpu().numpy()))
    out = M.blob_to_weights(mc, tr.blob()), losses, M.blob_to_weights(mc, tr.last_grad())
    tr.close()
    return out


@pytest.mark.parametrize("F,R,V,batch,max_batch,kind", [
    (32, 1, 16, 64, 64, "calibrated"),      # mini's value head
    (48, 1, 1, 67, 67, "new"),              # 5-lane column reductions, V = 1
    (64, 2, 256, 100, 100, "calibrated"),   # narrow-tower width
    (128, 2, 256, 97, 256, "calibrated"),   # narrow-tower width, uneven split-K, partial batch
    (144, 1, 513, 37, 37, "calibrated"),    # two N tiles, the second 16 wide
    (208, 0, 4096, 5, 5, "new"),            # no residual block, head_fc_kernel above 48 KB of shared memory
    (256, 1, 256, 100, 256, "calibrated"),  # uneven split-K at 8 splits, under a larger max_batch
])
def test_step_shapes_match_oracle(records, F, R, V, batch, max_batch, kind):
    mc = M.ModelConfig(cnn_filter_num=F, res_layer_num=R, value_fc_size=V)
    idx = np.random.default_rng(F + V).choice(records[0].shape[0], batch, replace=False)
    host = _host(records, idx)
    w0 = _weights(mc, kind, host[0])
    w, losses, g = _trainer_run(mc, w0, records, [idx], [0.02], max_batch)
    o64 = _oracle_steps(mc, w0, [host], [0.02])
    ofm = _oracle_steps(mc, w0, [host], [0.02], tf32_convs=True)
    report = []
    _check_against_oracle(mc, w0, w, g, losses[0], (o64[0], o64[1][0], o64[2]), (ofm[0], ofm[1][0], ofm[2]), report)
    worst = max(report, key=lambda r: r[1])
    ratios = [r[1] / r[2] for r in report if r[2] > 0]
    print(f"\nF={F} R={R} V={V} B={batch}/{max_batch} {kind}: worst gradient {worst[0]}: kernel {worst[1]:.2e} format model "
          f"{worst[2]:.2e}; kernel/format median {np.median(ratios):.2f}, max {max(ratios):.2f}")


def test_epoch_tail_with_learning_rate_change(records):
    """the `opt` worker's end of an epoch: two full batches and a short one under max_batch = 64, momentum carried"""
    mc = M.ModelConfig(cnn_filter_num=64, res_layer_num=1, value_fc_size=64)
    perm = np.random.default_rng(12).permutation(records[0].shape[0])
    idxs = [perm[:64], perm[64:128], perm[128:145]]
    lrs = [0.05, 0.05, 0.01]
    w0 = _weights(mc, "calibrated", _host(records, idxs[0])[0])
    w, losses, _ = _trainer_run(mc, w0, records, idxs, lrs, 64)
    batches = [_host(records, i) for i in idxs]
    o64 = _oracle_steps(mc, w0, batches, lrs)
    ofm = _oracle_steps(mc, w0, batches, lrs, tf32_convs=True)
    for s in range(3):
        for a, b, c in zip(losses[s], o64[1][s], ofm[1][s]):
            assert abs(a - b) <= 1.5 * abs(c - b) + 1e-4 * abs(b), (s, losses[s], o64[1][s], ofm[1][s])
    _check_against_oracle(mc, w0, w, None, None, (o64[0], o64[1][2], o64[2]), (ofm[0], ofm[1][2], ofm[2]))


# ---- (e) max_batch changes nothing --------------------------------------------------------------------------------
def _bits(mc, blob, records, idxs, max_batch):
    tr = T.Trainer(mc, max_batch=max_batch)
    tr.load_blob(blob)
    losses = [tr.step(*records, torch.as_tensor(np.asarray(i, np.int32), device="cuda"), 0.02).cpu().numpy() for i in idxs]
    out = np.concatenate(losses), tr.blob(), tr.last_grad()
    tr.close()
    return [a.view(np.uint32) for a in out]


@pytest.mark.parametrize("batches", [[1, 1], [17, 17], [100, 100], [100, 17, 1, 64, 100]], ids=["B1", "B17", "B100", "mixed"])
def test_steps_do_not_depend_on_max_batch(records, batches):
    """the split-K and every reduction depend on the batch alone: Trainer(max_batch = largest batch) and
    Trainer(max_batch = 1024) give the same losses, weights and gradient, bit for bit"""
    mc = M.ModelConfig(cnn_filter_num=128, res_layer_num=2, value_fc_size=256)
    rng = np.random.default_rng(sum(batches))
    idxs = [rng.choice(records[0].shape[0], b, replace=False) for b in batches]
    blob = M.weights_to_blob(mc, M.build_random_weights(mc, 4))
    a, b = _bits(mc, blob, records, idxs, max(batches)), _bits(mc, blob, records, idxs, 1024)
    for name, u, v in zip(("losses", "weights", "gradient"), a, b):
        assert np.array_equal(u, v), (name, int((u != v).sum()))


# ---- (f) the generic inference kernel, where AUTO sends it ---------------------------------------------------------
def _positions(records, n):
    return _host(records, np.arange(0, 13 * n, 13))[0]


def _check_generic(mc, w, planes, tp=2e-5, tv=5e-5):
    net = N.Net(mc)
    net.load_weights(w)
    p_ref, v_ref = onn.forward(w, planes, mc.res_layer_num)
    for n in (1, planes.shape[0]):
        assert net.select_impl(n) == N.IMPL_GENERIC, n
        p, v = net.predict_planes(planes[:n])
        pg, vg = net.predict_planes(planes[:n], N.IMPL_GENERIC)
        assert np.array_equal(p.view(np.uint32), pg.view(np.uint32)) and np.array_equal(v.view(np.uint32), vg.view(np.uint32)), n
        perr, verr = np.abs(p - p_ref[:n]).max(), np.abs(v - v_ref[:n]).max()
        assert perr <= tp and verr <= tv, (n, perr, verr)
    net.close()


def test_trained_48_filter_blob_runs_on_the_generic_kernel(records):
    """a width without a tensor-core tower, trained for three steps, loaded into Net: AUTO picks the generic kernel, which
    matches the fp32 oracle on the trained blob"""
    mc = M.ModelConfig(cnn_filter_num=48, res_layer_num=1, value_fc_size=1)
    rng = np.random.default_rng(48)
    tr = T.Trainer(mc, max_batch=67)
    tr.load_blob(M.weights_to_blob(mc, M.build_random_weights(mc, 6)))
    for _ in range(3):
        tr.step(*records, torch.as_tensor(rng.choice(records[0].shape[0], 67, replace=False).astype(np.int32), device="cuda"), 0.05)
    w = M.blob_to_weights(mc, tr.blob())
    tr.close()
    _check_generic(mc, w, _positions(records, 300))


@pytest.mark.parametrize("F,R,V", [(3, 1, 16), (48, 1, 1), (96, 2, 513), (200, 1, 64), (256, 1, 1024), (256, 1, 4096)])
def test_generic_kernel_where_auto_sends_it(records, F, R, V):
    """one position and 300 (> 2 x 132 SMs, so CTAs loop over positions); (256, 1, 4096) takes 221,952 B of shared memory
    and one CTA per SM"""
    mc = M.ModelConfig(cnn_filter_num=F, res_layer_num=R, value_fc_size=V)
    _check_generic(mc, M.build_random_weights(mc, F + V, perturb_bn=True), _positions(records, 300))
