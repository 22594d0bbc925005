"""One training step of the reference's network (worker/optimize.py:73-86 -> Keras fit on agent/model.py:28-72,104-110)
restated in torch autograd, CPU.  Test infrastructure only.

PARITY UNPINNED against Keras itself (Keras 2.1.2 / TensorFlow 1.4.1 are not installable, see oracle/nn.py).  This
follows the published semantics:
  - BatchNormalization in training mode: batch mean and biased variance over (batch, 8, 8), epsilon 1e-3; moving
    statistics moving = bn_momentum * moving + (1 - bn_momentum) * batch statistic (biased variance, no zero-debias),
    computed before the weight update;
  - loss = mean(sum -y log(p + 1e-7)) + mean((v - z)^2) + l2_reg * sum of squared Conv2D / Dense kernels;
  - Keras SGD with momentum: v = momentum * v - lr * g; w = w + v (kernels, biases, BN gamma / beta).

`step(..., tf32=True)` is the FORMAT MODEL of the device trainer: the operands of every 3x3 convolution GEMM (forward,
input gradient, weight gradient) rounded to TF32 (round to nearest, ties away, like cvt.rna.tf32.f32), everything else
exact (fp64).  Its distance from the fp64 step is what the number format alone costs.
"""
import numpy as np
import torch
import torch.nn.functional as F

from .nn import BN_EPS

LOG_EPS = 1e-7


def tf32(t):
    """round to TF32 (10 explicit mantissa bits), nearest with ties away from zero; returns t's dtype"""
    b = t.float().contiguous().view(torch.int32)
    b = (b + 0x1000) & ~0x1FFF
    return b.view(torch.float32).to(t.dtype)


class _Tf32Conv3x3(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, k):
        xr, kr = tf32(x), tf32(k)
        ctx.save_for_backward(xr, kr)
        return F.conv2d(xr, kr, padding=1)

    @staticmethod
    def backward(ctx, gy):
        xr, kr = ctx.saved_tensors
        gr = tf32(gy)
        gx = torch.nn.grad.conv2d_input(xr.shape, kr, gr, padding=1)
        gk = torch.nn.grad.conv2d_weight(xr, kr.shape, gr, padding=1)
        return gx, gk


def _shift_rows(batch, device):
    """src[tap][m]: the row that pixel m of a pixel-major [batch*64][C] tensor reads at tap = kh*3 + kw (offset
    (kh-1, kw-1)), or batch*64 (a zero row) when that falls off the board"""
    m = torch.arange(64 * batch, device=device)
    y, x = (m % 64) // 8, m % 8
    src = []
    for tap in range(9):
        yy, xx = y + tap // 3 - 1, x + tap % 3 - 1
        ok = (yy >= 0) & (yy < 8) & (xx >= 0) & (xx < 8)
        src.append(torch.where(ok, m - m % 64 + yy * 8 + xx, 64 * batch))
    return src


def _gather(x, src):
    return torch.cat([x, x.new_zeros(1, x.shape[1])])[src]


def conv3x3(x, k):
    """the device trainer's convolution GEMMs restated as plain gathers and matrix products, in x's dtype and device.
    x [B*64][Cin] pixel-major, k [9][Cin][Cout] (blob layout, tap = kh*3 + kw): out[m] = sum_tap x[shift(m, tap)] @ k[tap]"""
    src = _shift_rows(x.shape[0] // 64, x.device)
    return sum(_gather(x, src[t]) @ k[t] for t in range(9))


def conv3x3_dgrad(dy, k):
    """gradient of conv3x3 with respect to x for output gradient dy [B*64][Cout]: each tap's dy @ k[tap]^T added back to
    the pixel it was read from"""
    M = dy.shape[0]
    src = _shift_rows(M // 64, dy.device)
    out = dy.new_zeros(M + 1, k.shape[1])
    for t in range(9):
        out.index_add_(0, src[t], dy @ k[t].T)
    return out[:M]


def conv3x3_wgrad(x, dy):
    """gradient of conv3x3 with respect to k: [9][Cin][Cout]"""
    src = _shift_rows(x.shape[0] // 64, x.device)
    return torch.stack([_gather(x, src[t]).T @ dy for t in range(9)])


# ---- the device step stage by stage ----------------------------------------------------------------------------------
# One plain function per stage of csrc/rz_train.cu, in its layout: activations pixel-major [B*64][C], kernels in blob
# layout ([9][Cin][Cout] for 3x3, [Cin][Cout] for 1x1 and Dense), in the dtype and on the device of the arguments.
# `stage_loss_and_grad` chains them into the whole step; tests/test_train_host.py ties that chain to loss_and_grad.
def planes_to_x0(planes):
    """[B][2][8][8] planes -> [B*64][2]: x0[b*64 + p][c] = planes[b][c][p]"""
    return planes.reshape(planes.shape[0], 2, 64).permute(0, 2, 1).reshape(-1, 2)


def bn_stats(y):
    """training-mode BatchNorm statistics of y [M][C]: batch mean and biased variance"""
    mean = y.mean(0)
    return mean, ((y - mean) ** 2).mean(0)


def bn_invstd(var):
    return 1 / torch.sqrt(var + BN_EPS)


def bn_apply(y, mean, invstd, gamma, beta, res=None):
    """relu(gamma * (y - mean) * invstd + beta [+ res])"""
    v = gamma * (y - mean) * invstd + beta
    return torch.relu(v if res is None else v + res)


def bn_backward(g, a, y, mean, invstd, gamma):
    """BatchNorm + ReLU backward for g = d loss / d a: dz = g where a > 0, xhat = (y - mean) * invstd;
    -> (dy, dz, sum dz (beta's gradient), sum dz * xhat (gamma's gradient)),
    dy = gamma * invstd * (dz - (sum dz + xhat * sum dz * xhat) / M)"""
    dz = torch.where(a > 0, g, torch.zeros_like(g))
    xh = (y - mean) * invstd
    sdz, sdzx = dz.sum(0), (dz * xh).sum(0)
    return gamma * invstd * (dz - (sdz + xh * sdzx) / y.shape[0]), dz, sdz, sdzx


def head_conv(x, kpc, bpc, kvc, bvc):
    """the two 1x1 head convolutions of x [M][F]: hc [M][3] = (x @ kpc + bpc [2 columns], x @ kvc + bvc [1 column])"""
    return torch.cat([x @ kpc + bpc, x @ kvc + bvc], 1)


def head_conv_wgrad(x, dyh):
    """kernel gradients of the head convolutions for dyh = d loss / d hc [M][3]: (policy_conv [F][2], value_conv [F][1])"""
    g = x.T @ dyh
    return g[:, :2], g[:, 2:]


def head_conv_dgrad(dyh, kpc, kvc):
    """gradient of the tower output through the head convolutions: [M][F]"""
    return dyh[:, :2] @ kpc.T + dyh[:, 2:] @ kvc.T


def head_fc(ah, pfk, pfb, v1k, v1b, v2k, v2b, policy, z, log_eps=LOG_EPS):
    """per record: the Dense heads, the losses and their backward down to dh = d loss / d ah [B*64][3].  ah [B*64][3];
    policy [B][64]; z [B].  Returns a dict of hp [B][128] (channels-first flatten), hv [B][64], logits, p, lp, h1, v,
    lv, dl (d loss / d logits), dh1 (d loss / d value_fc1 pre-activation), dv (d loss / d value_fc2 pre-activation),
    dh; the losses are per record, the gradients those of the batch-mean loss.  log_eps: the epsilon inside the log
    (the device adds float32's 1e-7, as Keras' float32 graph does)."""
    B = ah.shape[0] // 64
    hp = ah[:, :2].reshape(B, 64, 2).permute(0, 2, 1).reshape(B, 128)
    hv = ah[:, 2].reshape(B, 64)
    logits = hp @ pfk + pfb
    p = torch.softmax(logits, 1)
    lp = -(policy * torch.log(p + log_eps)).sum(1)
    h1 = torch.relu(hv @ v1k + v1b)
    v = torch.tanh(h1 @ v2k[:, 0] + v2b[0])
    lv = (v - z) ** 2
    gg = -policy / (p + log_eps)                        # d lp / d p
    dl = p * (gg - (p * gg).sum(1, keepdim=True)) / B
    dv = 2 * (v - z) * (1 - v * v) / B
    dh1 = torch.where(h1 > 0, dv[:, None] * v2k[:, 0], torch.zeros_like(h1))
    dhp, dhv = dl @ pfk.T, dh1 @ v1k.T
    dh = torch.cat([dhp.reshape(B, 2, 64).permute(0, 2, 1).reshape(-1, 2), dhv.reshape(-1, 1)], 1)
    return dict(hp=hp, hv=hv, logits=logits, p=p, lp=lp, h1=h1, v=v, lv=lv, dl=dl, dh1=dh1, dv=dv, dh=dh)


def head_fc_grads(hp, hv, dl, h1, dh1, dv):
    """the Dense layers' gradients, summed over the batch: policy_fc kernel / bias, value_fc1 kernel / bias, value_fc2
    kernel [V][1] / bias [1]"""
    return dict(pfk=hp.T @ dl, pfb=dl.sum(0), v1k=hv.T @ dh1, v1b=dh1.sum(0), v2k=(h1.T @ dv)[:, None], v2b=dv.sum(0, keepdim=True))


def sgd_update(w, vel, g, lr, momentum, l2_reg, kernel):
    """Keras SGD with momentum on one tensor: g += 2 * l2_reg * w on Conv2D / Dense kernels; v = momentum * v - lr * g;
    w = w + v.  -> (w, v, g)"""
    if kernel:
        g = g + 2 * l2_reg * w
    v = momentum * vel - lr * g
    return w + v, v, g


def moving_average(moving, batch_stat, bn_momentum):
    return bn_momentum * moving + (1 - bn_momentum) * batch_stat


def stage_loss_and_grad(w, planes, policy, z, n_res, l2_reg):
    """loss_and_grad restated as the device step's chain of stages: -> (total, policy, value) losses as floats,
    {trainable name: gradient}, {conv name: (batch mean, batch var)}; tensors in w's dtype and device (w: name ->
    tensor, blob shapes)"""
    T = lambda a: torch.as_tensor(np.ascontiguousarray(a)).to(w["conv0.kernel"])
    x, y_pol, zz = planes_to_x0(T(planes)), T(policy), T(z)
    names = ["conv0"] + [f"res{i}.conv{j}" for i in range(n_res) for j in (1, 2)]
    L = len(names)
    k3 = lambda n: w[f"{n}.kernel"].reshape(9, -1, w[f"{n}.kernel"].shape[-1])
    bn = lambda n: (w[f"{n}.bn_gamma"], w[f"{n}.bn_beta"])
    stats, grads, Y, A, S = {}, {}, [], [], []
    for l, n in enumerate(names):                         # tower forward
        Y.append(conv3x3(A[l - 1] if l else x, k3(n)) + w[f"{n}.bias"])
        mean, var = bn_stats(Y[l])
        stats[n] = (mean, var)
        S.append((mean, bn_invstd(var)))
        A.append(bn_apply(Y[l], *S[l], *bn(n), res=A[l - 2] if l >= 2 and l % 2 == 0 else None))
    kpc, kvc = w["policy_conv.kernel"].reshape(-1, 2), w["value_conv.kernel"].reshape(-1, 1)
    hc = head_conv(A[-1], kpc, w["policy_conv.bias"], kvc, w["value_conv.bias"])
    hs = {}
    for n, cols in (("policy_conv", slice(0, 2)), ("value_conv", slice(2, 3))):
        mean, var = bn_stats(hc[:, cols])
        stats[n] = (mean, var)
        hs[n] = (cols, mean, bn_invstd(var))
    ah = torch.cat([bn_apply(hc[:, c], m, s, *bn(n)) for n, (c, m, s) in hs.items()], 1)
    h = head_fc(ah, w["policy_fc.kernel"], w["policy_fc.bias"], w["value_fc1.kernel"], w["value_fc1.bias"], w["value_fc2.kernel"],
                w["value_fc2.bias"], y_pol, zz)
    fg = head_fc_grads(h["hp"], h["hv"], h["dl"], h["h1"], h["dh1"], h["dv"])
    for n, k in (("policy_fc", "pf"), ("value_fc1", "v1"), ("value_fc2", "v2")):
        grads[f"{n}.kernel"], grads[f"{n}.bias"] = fg[k + "k"], fg[k + "b"]
    dyh = []
    for n, (c, m, s) in hs.items():
        dy, _, sdz, sdzx = bn_backward(h["dh"][:, c], ah[:, c], hc[:, c], m, s, w[f"{n}.bn_gamma"])
        dyh.append(dy)
        grads[f"{n}.bn_beta"], grads[f"{n}.bn_gamma"], grads[f"{n}.bias"] = sdz, sdzx, dy.sum(0)
    dyh = torch.cat(dyh, 1)
    gpc, gvc = head_conv_wgrad(A[-1], dyh)
    grads["policy_conv.kernel"], grads["value_conv.kernel"] = gpc.reshape(1, 1, -1, 2), gvc.reshape(1, 1, -1, 1)
    g, skip = head_conv_dgrad(dyh, kpc, kvc), None      # g: gradient of A(l); skip: dz of the block's conv2
    for l in range(L - 1, -1, -1):                        # tower backward
        n = names[l]
        dy, dz, sdz, sdzx = bn_backward(g, A[l], Y[l], *S[l], w[f"{n}.bn_gamma"])
        grads[f"{n}.bn_beta"], grads[f"{n}.bn_gamma"], grads[f"{n}.bias"] = sdz, sdzx, dy.sum(0)
        grads[f"{n}.kernel"] = conv3x3_wgrad(A[l - 1] if l else x, dy).reshape(w[f"{n}.kernel"].shape)
        if l:
            g = conv3x3_dgrad(dy, k3(n))
            if l % 2 == 1 and skip is not None:
                g = g + skip
            skip = dz if l % 2 == 0 else None
    lp, lv = h["lp"].mean(), h["lv"].mean()
    l2 = sum((t ** 2).sum() for k, t in w.items() if k.endswith(".kernel"))
    for k in grads:
        if k.endswith(".kernel"):
            grads[k] = grads[k] + 2 * l2_reg * w[k]
    return (float(lp + lv + l2_reg * l2), float(lp), float(lv)), grads, stats


def is_trainable(name):
    return not (name.endswith(".bn_mean") or name.endswith(".bn_var"))


def _forward_train(P, x, n_res, tf32_convs):
    """training-mode forward; P: name -> tensor.  Returns logits, value (N,), {conv name: (batch mean, batch var)}"""
    stats = {}

    def conv_bn(x, name, residual=None):
        k = P[f"{name}.kernel"].permute(3, 2, 0, 1)
        if k.shape[-1] == 3:
            y = (_Tf32Conv3x3.apply(x, k) if tf32_convs else F.conv2d(x, k, padding=1))
        else:
            y = F.conv2d(x, k)
        y = y + P[f"{name}.bias"].view(1, -1, 1, 1)
        mean = y.mean(dim=(0, 2, 3))
        var = y.var(dim=(0, 2, 3), unbiased=False)
        stats[name] = (mean.detach(), var.detach())
        y = (y - mean.view(1, -1, 1, 1)) / torch.sqrt(var.view(1, -1, 1, 1) + BN_EPS)
        y = y * P[f"{name}.bn_gamma"].view(1, -1, 1, 1) + P[f"{name}.bn_beta"].view(1, -1, 1, 1)
        if residual is not None:
            y = y + residual
        return F.relu(y)

    x = conv_bn(x, "conv0")
    for i in range(n_res):
        x = conv_bn(conv_bn(x, f"res{i}.conv1"), f"res{i}.conv2", residual=x)
    p = conv_bn(x, "policy_conv").reshape(x.shape[0], -1)
    logits = p @ P["policy_fc.kernel"] + P["policy_fc.bias"]
    v = conv_bn(x, "value_conv").reshape(x.shape[0], -1)
    v = F.relu(v @ P["value_fc1.kernel"] + P["value_fc1.bias"])
    value = torch.tanh(v @ P["value_fc2.kernel"] + P["value_fc2.bias"]).reshape(-1)
    return logits, value, stats


def loss_and_grad(w, planes, policy, z, n_res, l2_reg, dtype=torch.float64, tf32_convs=False):
    """-> (total, policy, value) losses as floats, {trainable name: gradient ndarray}, {conv name: (mean, var)}"""
    P = {k: torch.tensor(np.asarray(v), dtype=dtype, requires_grad=is_trainable(k)) for k, v in w.items()}
    x = torch.from_numpy(np.ascontiguousarray(planes)).to(dtype)
    y = torch.from_numpy(np.ascontiguousarray(policy)).to(dtype)
    zz = torch.from_numpy(np.ascontiguousarray(z)).to(dtype)
    logits, value, stats = _forward_train(P, x, n_res, tf32_convs)
    prob = torch.softmax(logits, dim=1)
    lp = (-(y * torch.log(prob + LOG_EPS)).sum(dim=1)).mean()
    lv = ((value - zz) ** 2).mean()
    l2 = sum((t ** 2).sum() for k, t in P.items() if k.endswith(".kernel"))
    total = lp + lv + l2_reg * l2
    names = [k for k in P if is_trainable(k)]
    grads = torch.autograd.grad(total, [P[k] for k in names])
    return ((float(total.detach()), float(lp.detach()), float(lv.detach())), {k: g.detach().numpy() for k, g in zip(names, grads)},
            {k: (m.numpy(), v.numpy()) for k, (m, v) in stats.items()})


def step(w, vel, planes, policy, z, lr, n_res, l2_reg, momentum=0.9, bn_momentum=0.99, dtype=torch.float64, tf32_convs=False):
    """One Keras SGD step.  w: {name: ndarray} (blob tensors), vel: {trainable name: ndarray} or None (zero momentum).
    Returns new weights, new velocities, losses (total, policy, value), gradients (trainable names)."""
    npdt = np.float64 if dtype == torch.float64 else np.float32
    w = {k: np.asarray(v, npdt) for k, v in w.items()}
    losses, grads, stats = loss_and_grad(w, planes, policy, z, n_res, l2_reg, dtype, tf32_convs)
    vel = {k: np.zeros_like(g) for k, g in grads.items()} if vel is None else vel
    new_w, new_v = dict(w), {}
    for k, g in grads.items():
        new_v[k] = (momentum * vel[k] - lr * g).astype(npdt)
        new_w[k] = (w[k] + new_v[k]).astype(npdt)
    for name, (m, v) in stats.items():
        new_w[f"{name}.bn_mean"] = (bn_momentum * w[f"{name}.bn_mean"] + (1 - bn_momentum) * m).astype(npdt)
        new_w[f"{name}.bn_var"] = (bn_momentum * w[f"{name}.bn_var"] + (1 - bn_momentum) * v).astype(npdt)
    return new_w, new_v, losses, grads
