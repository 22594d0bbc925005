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
