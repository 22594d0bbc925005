"""GPU suite for the device trainer (csrc/rz_train.cu) stage by stage: one step with the backward taps on
(Trainer.debug_keep_backward / debug_tensor), then every kernel other than the convolution GEMMs (which
tests/test_train_shapes_gpu.py pins) against its fp64 reference in oracle/train.py, evaluated on the tensors that kernel
was actually given.  TF32 noise from upstream then drops out, and each stage is held to the rounding of its own
arithmetic: a few ulp, or the accumulation bound of its own sum.  The GEMM stages are checked for wiring only (operand,
layer, bias, skip connection), within the GEMM suite's bound.  A second step checks the update with momentum.

Each bound is written as `err <= LIMIT[stage] * unit`, where `unit` is the per-element bound that follows from the
kernel's arithmetic; LIMIT is at most 1 and at most 16 times the worst ratio measured over this file's cases (DESIGN §5,
"Training step").  Prints the worst err / unit per stage."""
import numpy as np
import pytest
import torch

from oracle import train as ot
from reversi_zero_b200 import train as T
from reversi_zero_b200.agent import model as M
from test_train_gpu import _host, _weights, records  # noqa: F401 (records: fixture)

pytestmark = pytest.mark.gpu

E = lambda k: 2.0 ** k
# err <= LIMIT * unit per stage; 1.0 is the bound read from the kernel's arithmetic
LIMIT = {
    "forward GEMM": 1.0, "BN mean": 1.0, "BN variance": 1.0, "BN invstd": 1.0, "BN apply": 1.0, "head conv": 1.0,
    "head forward": 1.0, "batch losses": 1.0, "total loss": 1.0, "Dense gradients": 1.0, "head BN gradients": 1.0,
    "head conv gradients": 1.0, "head conv input gradient": 1.0, "BN backward": 1.0, "BN backward sums": 1.0,
    "input gradient GEMM": 1.0, "weight gradient GEMM": 1.0, "update velocity": 1.0, "update weights": 1.0,
    "moving averages": 1.0,
}

# (filters, residual blocks, value_fc, batch, max_batch, weights, edge edits)
CASES = [
    (16, 1, 64, 64, 64, "new", True),
    (48, 1, 1, 67, 67, "calibrated", True),       # column reductions whose lanes do not divide 256
    (64, 2, 256, 100, 128, "calibrated", False),
    (128, 0, 513, 37, 64, "new", True),           # no residual block
    (208, 0, 4096, 5, 5, "calibrated", True),     # head_fc_kernel above 48 KB of shared memory
    (256, 2, 256, 1, 256, "new", False),
    (256, 2, 256, 32, 256, "calibrated", True),
    (256, 10, 256, 8, 8, "calibrated", False),    # ch5
]
LR1, LR2 = 0.02, 0.01
CONST, BIG, DEAD = 1, 2, 3    # conv0 channels of the edge edits (res0.conv1 too: CONST + 3, DEAD + 3)
LOG_EPS32 = float(np.float32(ot.LOG_EPS))   # the kernel's 1e-7f inside the log (Keras adds K.epsilon() in float32)


def _offsets(mc):
    off, out = 0, {}
    for name, shape in M.tensor_specs(mc):
        out[name] = (off, int(np.prod(shape)))
        off += int(np.prod(shape))
    return out


def _edges(mc, w, planes):
    """weight edits that put each kernel at an edge: a constant conv output channel (variance 0, xhat 0), a channel whose
    mean is 300 x its spread, a dead channel (A = 0, sum dz = 0, dy = 0), logits scaled so that many p fall near and below
    the 1e-7 inside the log, and a value head near tanh's saturation, where 1 - v^2 and v - z cancel"""
    w = {k: np.array(v, np.float32) for k, v in w.items()}
    F = mc.cnn_filter_num
    w["conv0.kernel"][..., CONST] = 0
    x0 = ot.planes_to_x0(torch.from_numpy(planes).double())
    y = ot.conv3x3(x0, torch.from_numpy(w["conv0.kernel"].reshape(9, 2, F)).double())[:, BIG]
    w["conv0.bias"][BIG] = 300 * float(y.std()) - float(y.mean())
    w["conv0.bn_beta"][DEAD] = -1e3
    if mc.res_layer_num:
        w["res0.conv1.kernel"][..., CONST + 3] = 0
        w["res0.conv1.bn_beta"][DEAD + 3] = -1e3
    w["policy_fc.kernel"] *= 30
    w["policy_fc.bias"] *= 30
    w["value_fc2.bias"][:] = 7
    return w


def _targets(records, idx, edges):
    """the dataset's policy and z, with one-hot and all-zero policy targets and z in {-1, 0, 1} on the batch's records"""
    _, pol, z = records
    if not edges:
        return pol, z
    pol, z = pol.clone(), z.clone()
    for k, r in enumerate(idx.tolist()):
        if k % 4 < 3:
            pol[r] = 0
        if k % 4 < 2:
            pol[r, 0 if k % 4 == 0 else (11 * k) % 64] = 1
        z[r] = (-1.0, 0.0, 1.0)[k % 3]
    return pol, z


class Checker:
    """collects the worst err / unit per stage and every failed check, so that one run reports all of them"""
    def __init__(self):
        self.worst, self.fails = {}, []

    def __call__(self, stage, got, ref, unit, what=""):
        # + 2^-149: a value below fp32's normal range is stored with the subnormal spacing
        got, ref, unit = got.double(), torch.as_tensor(ref).double(), torch.as_tensor(unit).double() + E(-149)
        err = (got - ref).abs()
        ratio = torch.where(err == 0, torch.zeros_like(err), err / unit)
        r = float(ratio.max()) if ratio.numel() else 0.0
        self.worst[stage] = max(self.worst.get(stage, 0.0), r)
        if r > LIMIT[stage]:
            i = int(ratio.reshape(-1).argmax())
            self.fails.append(f"{stage} {what}: err / unit = {r:.3g} > {LIMIT[stage]} at flat index {i} of {tuple(got.shape)}: got "
                              f"{got.reshape(-1)[i].item()!r}, ref {ref.reshape(-1)[i].item()!r}, unit {unit.reshape(-1)[i].item():.3g}")

    def exact(self, ok, what):
        if not bool(ok):
            self.fails.append(f"not exact: {what}")


def _ulp(x):
    """spacing of float32 at |x| (fp64 tensor)"""
    _, e = torch.frexp(x.float().abs().clamp_min(2.0 ** -126))
    return torch.ldexp(torch.ones_like(x), (e - 24).to(torch.int64)).double()


def _tf(t):
    return ot.tf32(t.float()).double()


@pytest.mark.parametrize("F,R,V,batch,max_batch,kind,edges", CASES,
                         ids=[f"{c[0]}x{c[1]}-V{c[2]}-B{c[3]}of{c[4]}-{c[5]}{'-edges' if c[6] else ''}" for c in CASES])
def test_stages_against_fp64(records, F, R, V, batch, max_batch, kind, edges):
    mc = M.ModelConfig(cnn_filter_num=F, res_layer_num=R, value_fc_size=V)
    L, N = 1 + 2 * R, records[0].shape[0]
    rng = np.random.default_rng(F * 31 + R * 7 + batch)
    idx_np = rng.choice(N, batch, replace=False)
    idx2_np = rng.choice(N, batch, replace=False)
    host = _host(records, idx_np)
    w0 = _weights(mc, kind, host[0])
    if edges:
        w0 = _edges(mc, w0, host[0])
    blob0 = M.weights_to_blob(mc, w0)
    idx = torch.as_tensor(idx_np.astype(np.int32), device="cuda")
    pol_all, z_all = _targets(records, idx_np, edges)
    states = records[0]
    l2 = float(np.float32(mc.l2_reg))
    dev = lambda a: torch.as_tensor(np.asarray(a), dtype=torch.float64, device="cuda")
    W = {k: dev(v) for k, v in w0.items()}
    off = _offsets(mc)
    check = Checker()

    tr = T.Trainer(mc, max_batch=max_batch)
    tr.load_blob(blob0)
    tr.debug_keep_backward(True)
    loss1 = tr.step(states, pol_all, z_all, idx, LR1)
    D = lambda name, layer=0: tr.debug_tensor(name, layer).double()
    grad1 = dev(tr.last_grad())
    G = lambda name: grad1[off[name][0]:off[name][0] + off[name][1]]
    stat1 = D("stat")
    names = ["conv0"] + [f"res{i}.conv{j}" for i in range(R) for j in (1, 2)]
    Y, A = [D("y", l) for l in range(L)], [D("a", l) for l in range(L)]
    ST = [D("stats", s) for s in range(L + 2)]

    def sums(s, C):
        """sum dz and sum dz * xhat of slot s: packed at stride C after mean and invstd ([F] each)"""
        flat = ST[s].reshape(-1)[2 * F:]
        return flat[:C], flat[C:2 * C]
    Mrows = 64 * batch

    # ---- gather: x0 is the records' planes exactly, channels 2..15 zero
    x0 = tr.debug_tensor("x0")
    want = ot.planes_to_x0(states[idx.long()].float())
    assert torch.equal(x0[:, :2], want) and bool((x0[:, 2:] == 0).all())
    x0 = x0[:, :2].double()

    def k3(n):
        return W[f"{n}.kernel"].reshape(9, -1, F)

    # ---- forward GEMM wiring: Y(l) = conv3x3(tf32(A(l - 1)), tf32(W_l)) + b_l
    for l, n in enumerate(names):
        a, b = _tf(A[l - 1] if l else x0), _tf(k3(n))
        ref = ot.conv3x3(a, b) + W[f"{n}.bias"]
        check("forward GEMM", Y[l], ref, E(-16) * ot.conv3x3(a.abs(), b.abs()) + E(-23) * ref.abs(), n)

    # ---- BN statistics (tower layers and the two head slots)
    hc, ah, dh, dyh = D("hc"), D("ah"), D("dh"), D("dyh")
    bn_slots = [(n, Y[l], slice(0, F)) for l, n in enumerate(names)] + [("policy_conv", hc[:, :2], slice(0, 2)),
                                                                        ("value_conv", hc[:, 2:], slice(0, 1))]
    for s, (n, y, cols) in enumerate(bn_slots):
        C = y.shape[1]
        mean, inv = ST[s][0, :C], ST[s][1, :C]
        ref = y.mean(0)
        check("BN mean", mean, ref, E(-23) * ref.abs() + E(-40) * y.abs().mean(0), n)
        o = off[f"{n}.bn_mean"][0]
        check.exact(torch.equal(stat1[o:o + C], mean), f"{n}: moving-average mean")   # the mean the layer normalised with
        var = stat1[off[f"{n}.bn_var"][0]:][:C]
        ref = ((y - mean) ** 2).mean(0)
        check("BN variance", var, ref, 2 * _ulp(ref), n)
        ref = 1 / torch.sqrt(var + float(np.float32(1e-3)))
        check("BN invstd", inv, ref, 2 * _ulp(ref), n)

    # ---- BN apply (+ residual on conv2 of each block) + ReLU, with the kernel's mean and invstd
    def apply_ref(y, s, gamma, beta, res=None):
        C = y.shape[1]
        xg = (y - ST[s][0, :C]) * ST[s][1, :C] * gamma
        v = xg + beta + (0 if res is None else res)
        return torch.relu(v), E(-20) * (xg.abs() + beta.abs() + (0 if res is None else res.abs()))

    for l, n in enumerate(names):
        ref, unit = apply_ref(Y[l], l, W[f"{n}.bn_gamma"], W[f"{n}.bn_beta"], A[l - 2] if l >= 2 and l % 2 == 0 else None)
        check("BN apply", A[l], ref, unit, n)
    for s, n, c in ((L, "policy_conv", slice(0, 2)), (L + 1, "value_conv", slice(2, 3))):
        ref, unit = apply_ref(hc[:, c], s, W[f"{n}.bn_gamma"], W[f"{n}.bn_beta"])
        check("BN apply", ah[:, c], ref, unit, n)

    # ---- heads: 1x1 convs, then the Dense heads, losses and their backward in fp64
    kpc, kvc = W["policy_conv.kernel"].reshape(F, 2), W["value_conv.kernel"].reshape(F, 1)
    tower = A[L - 1]
    ref = ot.head_conv(tower, kpc, W["policy_conv.bias"], kvc, W["value_conv.bias"])
    mag = ot.head_conv(tower.abs(), kpc.abs(), W["policy_conv.bias"].abs(), kvc.abs(), W["value_conv.bias"].abs())
    check("head conv", hc, ref, E(-22) * ref.abs() + E(-45) * mag)

    i_l = idx.long()
    y_pol, zb = pol_all[i_l].double(), z_all[i_l].double()
    pfk, pfb, v1k, v1b, v2k, v2b = (W[k] for k in ("policy_fc.kernel", "policy_fc.bias", "value_fc1.kernel", "value_fc1.bias",
                                                   "value_fc2.kernel", "value_fc2.bias"))
    h = ot.head_fc(ah, pfk, pfb, v1k, v1b, v2k, v2b, y_pol, zb, log_eps=LOG_EPS32)
    got = {k: D(k) for k in ("hp", "hv", "dl", "h1", "dh1", "dv", "lp", "lv")}
    check.exact(torch.equal(got["hp"], h["hp"]) and torch.equal(got["hv"], h["hv"]), "hp, hv: copies of ah")
    # error scales, in units of one fp64 rounding: of the logits (and so of p, relatively), and of v
    p, v, d = h["p"], h["v"], h["v"] - zb
    ep = 1 + 2 * (h["hp"].abs() @ pfk.abs() + pfb.abs()).max(1).values
    ev = 1 + (1 - v * v) * (h["h1"].abs() @ v2k[:, 0].abs() + v2b.abs())
    gg = -y_pol / (p + LOG_EPS32)
    pgabs = (p * gg).abs().sum(1, keepdim=True)
    t_dl = ((p * gg).abs() + p * pgabs) / batch * ep[:, None]
    t_dv = 2 / batch * ev * ((1 - v * v) + 2 * d.abs())
    t_dh1 = t_dv[:, None] * v2k[:, 0].abs()
    terms = dict(
        h1=h["hv"].abs() @ v1k.abs() + v1b.abs(),
        lp=(y_pol * torch.log(p + LOG_EPS32)).abs().sum(1) + (y_pol * ep[:, None]).sum(1),
        lv=2 * d.abs() * ev, dl=t_dl, dv=t_dv, dh1=t_dh1)
    for k, t in terms.items():
        check("head forward", got[k], h[k], E(-22) * h[k].abs() + E(-45) * t, k)
    t_dh = torch.cat([((h["dl"].abs() + t_dl) @ pfk.abs().T).reshape(batch, 2, 64).permute(0, 2, 1).reshape(-1, 2),
                      ((h["dh1"].abs() + t_dh1) @ v1k.abs().T).reshape(-1, 1)], 1)
    check("head forward", dh, h["dh"], E(-22) * h["dh"].abs() + E(-45) * t_dh, "dh")
    if edges:   # the edits do reach the edges
        assert float((p < 1e-6).double().mean()) > 0.3 and float((1 - v * v).min()) < 1e-3, (float((p < 1e-6).double().mean()),
                                                                                             float((1 - v * v).min()))

    # ---- batch losses and the loss of the step
    pv = D("loss_pv")
    ref = torch.stack([got["lp"].mean(), got["lv"].mean()])
    check("batch losses", pv, ref, batch * E(-23) * ref.abs())
    l1 = loss1.double()
    check.exact(l1[1] == pv[0] and l1[2] == pv[1], "returned policy / value loss")
    k_mask = torch.zeros(tr.blob_floats, dtype=torch.bool, device="cuda")
    for name, (o, cnt) in off.items():
        if name.endswith(".kernel"):
            k_mask[o:o + cnt] = True
    blob0_d = dev(blob0)
    sw2 = (blob0_d[k_mask] ** 2).sum()
    check("total loss", l1[0], pv[0] + pv[1] + l2 * sw2, E(-22) * (pv[0].abs() + pv[1].abs()) + E(-14) * l2 * sw2)

    # ---- head gradients: Dense kernels / biases, head BN gamma / beta, policy_conv / value_conv kernels
    def with_l2(name, raw, mag):
        """expected last_grad of a kernel: raw + 2 * l2 * w0 (update_kernel writes the L2 term back into grad)"""
        if name.endswith(".kernel"):
            t = 2 * l2 * W[name].reshape(raw.shape)
            return raw + t, E(-22) * (raw.abs() + t.abs()) + E(-45) * mag
        return raw, E(-22) * raw.abs() + E(-45) * mag

    fg = ot.head_fc_grads(got["hp"], got["hv"], got["dl"], got["h1"], got["dh1"], got["dv"])
    fm = ot.head_fc_grads(got["hp"].abs(), got["hv"].abs(), got["dl"].abs(), got["h1"].abs(), got["dh1"].abs(), got["dv"].abs())
    for n, k in (("policy_fc", "pf"), ("value_fc1", "v1"), ("value_fc2", "v2")):
        for part in ("kernel", "bias"):
            ref, unit = with_l2(f"{n}.{part}", fg[k + part[0]], fm[k + part[0]])
            check("Dense gradients", G(f"{n}.{part}"), ref.reshape(-1), unit.reshape(-1), f"{n}.{part}")

    def bn_sums(g, a, y, s, what):
        """sum dz and sum dz * xhat against the stats slot and the blob's beta / gamma gradients; xhat as the kernel forms
        it, (y - mean) * invstd in fp32, and each product and sum in fp64"""
        C = y.shape[1]
        dz = torch.where(a > 0, g, torch.zeros_like(g))
        xh = ((y.float() - ST[s][0, :C].float()) * ST[s][1, :C].float()).double()
        stage = "head BN gradients" if s >= L else "BN backward sums"
        for got_sum, ref, mag in zip(sums(s, C), (dz.sum(0), (dz * xh).sum(0)), (dz.abs().sum(0), (dz * xh).abs().sum(0))):
            check(stage, got_sum, ref, E(-22) * ref.abs() + E(-45) * mag, what)
        n = bn_slots[s][0]
        check.exact(torch.equal(G(f"{n}.bn_beta"), sums(s, C)[0]) and torch.equal(G(f"{n}.bn_gamma"), sums(s, C)[1]), f"{n}: beta / gamma gradient")
        check.exact((G(f"{n}.bias") == 0).all(), f"{n}: conv bias gradient 0")
        return dz

    bn_sums(dh[:, :2], ah[:, :2], hc[:, :2], L, "policy_conv")
    bn_sums(dh[:, 2:], ah[:, 2:], hc[:, 2:], L + 1, "value_conv")
    for n, cols, shape in (("policy_conv", slice(0, 2), (F, 2)), ("value_conv", slice(2, 3), (F, 1))):
        ref, unit = with_l2(f"{n}.kernel", tower.T @ dyh[:, cols], tower.abs().T @ dyh[:, cols].abs())
        check("head conv gradients", G(f"{n}.kernel"), ref.reshape(-1), unit.reshape(-1), n)
    # dyh itself: the head BN backward
    for s, n, c in ((L, "policy_conv", slice(0, 2)), (L + 1, "value_conv", slice(2, 3))):
        C = c.stop - c.start
        dz = torch.where(ah[:, c] > 0, dh[:, c], torch.zeros_like(dh[:, c]))
        xh = (hc[:, c] - ST[s][0, :C]) * ST[s][1, :C]
        gi, (sdz, sdzx) = W[f"{n}.bn_gamma"] * ST[s][1, :C], sums(s, C)
        ref = gi * (dz - (sdz + xh * sdzx) / Mrows)
        check("BN backward", dyh[:, c], ref, E(-20) * gi.abs() * (dz.abs() + (sdz.abs() + xh.abs() * sdzx.abs()) / Mrows), n)

    # ---- gradient into the tower and the tower's backward
    Gt = [D("g", l) for l in range(L)]
    DY = [D("dy", l) for l in range(L)]
    ref = ot.head_conv_dgrad(dyh, kpc, kvc)
    check("head conv input gradient", Gt[L - 1], ref, E(-22) * ot.head_conv_dgrad(dyh.abs(), kpc.abs(), kvc.abs()))
    for l, n in enumerate(names):
        dz = bn_sums(Gt[l], A[l], Y[l], l, n)
        if l >= 2 and l % 2 == 0:
            check.exact(torch.equal(D("dz", l), dz), f"{n}: dz is the ReLU mask of G")
        xh = (Y[l] - ST[l][0]) * ST[l][1]
        gi = W[f"{n}.bn_gamma"] * ST[l][1]
        ref = gi * (dz - (ST[l][2] + xh * ST[l][3]) / Mrows)
        check("BN backward", DY[l], ref, E(-20) * gi.abs() * (dz.abs() + (ST[l][2].abs() + xh.abs() * ST[l][3].abs()) / Mrows), n)
        if l:   # input gradient: G(l - 1) = dgrad(dY(l)) (+ dz(l + 1), the skip connection, below conv1)
            a, b = _tf(DY[l]), _tf(k3(n))
            ref = ot.conv3x3_dgrad(a, b) + (D("dz", l + 1) if l % 2 else 0)
            check("input gradient GEMM", Gt[l - 1], ref, E(-16) * ot.conv3x3_dgrad(a.abs(), b.abs()) + E(-23) * ref.abs(), n)
        a, b = _tf(A[l - 1] if l else x0), _tf(DY[l])
        raw = ot.conv3x3_wgrad(a, b)
        t = 2 * l2 * k3(n).reshape(raw.shape)
        check("weight gradient GEMM", G(f"{n}.kernel"), (raw + t).reshape(-1),
              (E(-16) * ot.conv3x3_wgrad(a.abs(), b.abs()) + E(-23) * (raw.abs() + t.abs())).reshape(-1), n)
    if edges:
        m0 = ST[0][0, BIG]
        assert float(m0.abs() / torch.sqrt(stat1[off["conv0.bn_var"][0] + BIG])) > 100
        assert stat1[off["conv0.bn_var"][0] + CONST] == 0 and bool((Y[0][:, CONST] == ST[0][0, CONST]).all())
        assert bool((A[0][:, DEAD] == 0).all()) and ST[0][2, DEAD] == 0 and bool((DY[0][:, DEAD] == 0).all())

    # ---- update, on a second step (momentum not zero)
    w1, v1 = (t.double() for t in tr.replica_state(0))
    idx2 = torch.as_tensor(idx2_np.astype(np.int32), device="cuda")
    loss2 = tr.step(states, pol_all, z_all, idx2, LR2).double()
    w2, v2 = (t.double() for t in tr.replica_state(0))
    g2, stat2, pv2 = dev(tr.last_grad()), D("stat"), D("loss_pv")
    trainable = torch.ones_like(k_mask)
    for name, (o, cnt) in off.items():
        if not ot.is_trainable(name):
            trainable[o:o + cnt] = False
    mu, lr = float(np.float32(T.MOMENTUM)), float(np.float32(LR2))
    tv = trainable
    check("update velocity", v2[tv], mu * v1[tv] - lr * g2[tv], E(-23) * (mu * v1[tv].abs() + lr * g2[tv].abs()))
    check("update weights", w2[tv], w1[tv] + v2[tv], E(-23) * (w1[tv].abs() + v2[tv].abs()))
    bm = float(np.float32(T.BN_MOMENTUM))
    c = float(np.float32(1) - np.float32(T.BN_MOMENTUM))
    mv = ~tv
    check("moving averages", w2[mv], bm * w1[mv] + c * stat2[mv], E(-23) * (bm * w1[mv].abs() + c * stat2[mv].abs()))
    sw2 = (w1[k_mask] ** 2).sum()
    check("total loss", loss2[0], pv2[0] + pv2[1] + l2 * sw2, E(-22) * (pv2[0].abs() + pv2[1].abs()) + E(-14) * l2 * sw2)
    tr.close()
    print(f"\nF={F} R={R} V={V} B={batch}/{max_batch} {kind}{' edges' if edges else ''}: worst err / unit per stage: "
          + ", ".join(f"{k} {v:.3g}" for k, v in check.worst.items()))
    assert not check.fails, "\n".join(check.fails)


def test_debug_tensor_rejects_bad_requests(records):
    mc = M.ModelConfig(cnn_filter_num=16, res_layer_num=1, value_fc_size=8)
    tr = T.Trainer(mc, max_batch=4)
    tr.load_blob(M.weights_to_blob(mc, M.build_random_weights(mc, 1)))
    with pytest.raises(RuntimeError, match="no step has run"):
        tr.debug_tensor("y")
    idx = torch.arange(3, dtype=torch.int32, device="cuda")
    tr.step(*records, idx, 0.01)
    assert tr.debug_tensor("y", 2).shape == (192, 16)
    for name, layer in (("g", 0), ("y", 3), ("stats", 5), ("dz", 1), ("hc", 1)):
        with pytest.raises(RuntimeError, match="failed \\(-[14]\\)"):
            tr.debug_tensor(name, layer)
    tr.debug_keep_backward(True)
    tr.step(*records, idx, 0.01)
    assert tr.debug_tensor("g", 0).shape == (192, 16) and tr.debug_tensor("dz", 2).shape == (192, 16)
    tr.debug_keep_backward(False)
    with pytest.raises(RuntimeError, match="failed \\(-4\\)"):
        tr.debug_tensor("g", 0)
    tr.close()
