"""fp32 restatement of the reference's Keras forward pass (agent/model.py:28-72) in torch, CPU.

Test infrastructure only.  PARITY UNPINNED against Keras itself: Keras 2.1.2 / TensorFlow 1.4.1
(reference requirements.txt:25,59) are not installable here and the reference has no test touching
the model; this follows the published layer semantics -- Conv2D(padding=same, use_bias=True,
channels_first) -> BatchNormalization(axis=1, epsilon=1e-3, inference statistics) -> ReLU; residual
add before the last ReLU (model.py:60-72); Flatten on channels_first = (C,H,W) row-major reshape;
Dense(softmax) / Dense(relu) -> Dense(tanh).  Weights come in Keras layouts (kernel (kh,kw,Cin,Cout),
Dense kernel (in,out)) as produced by reversi_zero_b200.agent.model.
"""
import numpy as np
import torch
import torch.nn.functional as F

BN_EPS = 1e-3


def _conv_bn(x, w, name, relu=True, residual=None, pad=1):
    k = torch.from_numpy(w[f"{name}.kernel"]).permute(3, 2, 0, 1).contiguous()  # (kh,kw,ci,co)->(co,ci,kh,kw)
    y = F.conv2d(x, k, torch.from_numpy(w[f"{name}.bias"]), padding=pad)
    g, b, m, v = (torch.from_numpy(w[f"{name}.bn_{p}"]).view(1, -1, 1, 1) for p in ("gamma", "beta", "mean", "var"))
    y = (y - m) / torch.sqrt(v + BN_EPS) * g + b
    if residual is not None:
        y = y + residual
    return F.relu(y) if relu else y


@torch.no_grad()
def forward(w, planes, n_res, return_tower=False, dtype=torch.float32):
    """planes: (N,2,8,8) {0,1}. Returns policy (N,64) softmax probs, value (N,) tanh."""
    x = torch.from_numpy(np.ascontiguousarray(planes)).to(dtype)
    if dtype != torch.float32:
        w = {k: v.astype(np.float64) for k, v in w.items()}
    x = _conv_bn(x, w, "conv0")
    for i in range(n_res):
        y = _conv_bn(x, w, f"res{i}.conv1")
        x = _conv_bn(y, w, f"res{i}.conv2", residual=x)
    tower = x
    p = _conv_bn(x, w, "policy_conv", pad=0).reshape(x.shape[0], -1)
    logits = p @ torch.from_numpy(w["policy_fc.kernel"]) + torch.from_numpy(w["policy_fc.bias"])
    policy = torch.softmax(logits, dim=1)
    v = _conv_bn(x, w, "value_conv", pad=0).reshape(x.shape[0], -1)
    v = F.relu(v @ torch.from_numpy(w["value_fc1.kernel"]) + torch.from_numpy(w["value_fc1.bias"]))
    value = torch.tanh(v @ torch.from_numpy(w["value_fc2.kernel"]) + torch.from_numpy(w["value_fc2.bias"])).reshape(-1)
    if return_tower:
        return policy.numpy(), value.numpy(), logits.numpy(), tower.numpy()
    return policy.numpy(), value.numpy()


def _fold(w, name):
    g, b, m, v = (torch.from_numpy(w[f"{name}.bn_{p}"]) for p in ("gamma", "beta", "mean", "var"))
    s = g / torch.sqrt(v + BN_EPS)
    return s.view(1, -1, 1, 1), ((torch.from_numpy(w[f"{name}.bias"]) - m) * s + b).view(1, -1, 1, 1)


@torch.no_grad()
def forward_fp16_operands(w, planes, n_res, round_weights=True, round_acts=True):
    """The SAME network evaluated the way the tensor-core tower is specified to evaluate it: convolution operands rounded
    to fp16 (round-to-nearest-even; weights of all 1 + 2R convolutions, activations of the 2R tower convolutions -- the
    first layer's {0,1} planes are exact), products and sums exact (fp64 here; the tensor core accumulates in fp32),
    folded BatchNorm / residual stream / heads in fp32.  The difference between this and `forward` is the error the
    *number format* costs; whatever the kernel adds on top is the kernel's own (tools/nn_diag.py prints both).
    Returns policy, value, logits, value_logit, tower."""
    def h(t):
        return t.half().float()

    def conv(x, name, ra):
        k = torch.from_numpy(w[f"{name}.kernel"]).permute(3, 2, 0, 1).contiguous()
        k = h(k) if round_weights else k
        x = h(x) if (ra and round_acts) else x
        s, sh = _fold(w, name)
        return F.conv2d(x.double(), k.double(), padding=1).float() * s + sh

    x = F.relu(conv(torch.from_numpy(np.ascontiguousarray(planes)).float(), "conv0", False))
    for i in range(n_res):
        y = F.relu(conv(x, f"res{i}.conv1", True))
        x = F.relu(conv(y, f"res{i}.conv2", True) + x)
    return heads(w, x)


@torch.no_grad()
def heads(w, x):
    """policy / value heads (agent/model.py:43-56) in fp32 from a tower output x (N, C, 8, 8)"""
    def c1(name):
        k = torch.from_numpy(w[f"{name}.kernel"]).permute(3, 2, 0, 1).contiguous()
        s, sh = _fold(w, name)
        return F.relu(F.conv2d(x, k) * s + sh).reshape(x.shape[0], -1)
    logits = c1("policy_conv") @ torch.from_numpy(w["policy_fc.kernel"]) + torch.from_numpy(w["policy_fc.bias"])
    v = F.relu(c1("value_conv") @ torch.from_numpy(w["value_fc1.kernel"]) + torch.from_numpy(w["value_fc1.bias"]))
    pre = (v @ torch.from_numpy(w["value_fc2.kernel"]) + torch.from_numpy(w["value_fc2.bias"])).reshape(-1)
    return torch.softmax(logits, 1).numpy(), torch.tanh(pre).numpy(), logits.numpy(), pre.numpy(), x.numpy()


@torch.no_grad()
def forward_logits(w, planes, n_res):
    """fp32 reference with the head outputs before softmax / tanh: policy, value, logits, value_logit, tower"""
    return forward_fp16_operands(w, planes, n_res, round_weights=False, round_acts=False)


@torch.no_grad()
def calibrate_bn(w, planes, n_res):
    """Trained-like weights for the tolerance tests: the BatchNormalization moving statistics of every layer are set to
    the statistics of that layer's own pre-activation over `planes` (what training leaves behind: every layer's output is
    normalised, then scaled / shifted by gamma / beta), keeping whatever gamma, beta and biases `w` has.  In place."""
    x = torch.from_numpy(np.ascontiguousarray(planes)).float()

    def layer(x, name, res=None):
        k = torch.from_numpy(w[f"{name}.kernel"]).permute(3, 2, 0, 1).contiguous()
        y = F.conv2d(x, k, torch.from_numpy(w[f"{name}.bias"]), padding=k.shape[-1] // 2)
        w[f"{name}.bn_mean"] = y.mean(dim=(0, 2, 3)).numpy().copy()
        w[f"{name}.bn_var"] = y.var(dim=(0, 2, 3), unbiased=False).numpy().copy()
        s, sh = _fold(w, name)
        y = F.conv2d(x, k, padding=k.shape[-1] // 2) * s + sh
        return F.relu(y if res is None else y + res)

    x = layer(x, "conv0")
    for i in range(n_res):
        x = layer(layer(x, f"res{i}.conv1"), f"res{i}.conv2", x)
    layer(x, "policy_conv")
    layer(x, "value_conv")
    return w


def planes_from_bitboards(own, enemy):
    """(N,) u64 pairs -> (N,2,8,8) uint8 planes [own, enemy], plane[y][x] = bit y*8+x (bit_to_array)."""
    own = np.asarray(own, np.uint64).reshape(-1, 1)
    enemy = np.asarray(enemy, np.uint64).reshape(-1, 1)
    sh = np.arange(64, dtype=np.uint64).reshape(1, 64)
    o = ((own >> sh) & np.uint64(1)).astype(np.uint8).reshape(-1, 8, 8)
    e = ((enemy >> sh) & np.uint64(1)).astype(np.uint8).reshape(-1, 8, 8)
    return np.stack([o, e], axis=1)


class OracleNetAPI:
    """Object with the ReversiModelAPI.predict contract (agent/api.py:30-45) backed by `forward`."""

    def __init__(self, weights, n_res, threads=None):
        self.w, self.n_res = weights, n_res
        self.rows = 0
        self.calls = 0
        if threads:
            torch.set_num_threads(threads)

    def predict(self, x):
        x = np.asarray(x)
        single = x.ndim == 3
        if single:
            x = x.reshape(1, 2, 8, 8)
        p, v = forward(self.w, x, self.n_res)
        self.rows += x.shape[0]
        self.calls += 1
        v = v.reshape(-1, 1)
        return (p[0], v[0]) if single else (p, v)


class FakeNetAPI:
    """Deterministic, dihedral-invariant stand-in used for exact MCTS parity tests (reference, oracle
    and CUDA engine all implement it): policy = 1/64 everywhere, value = (#own - #enemy)/64."""

    def __init__(self, sign=1.0):
        """sign = -1: the engine's deterministic "second network" of evaluation matches (value negated)."""
        self.rows = 0
        self.calls = 0
        self.sign = np.float32(sign)

    def predict(self, x):
        x = np.asarray(x)
        single = x.ndim == 3
        if single:
            x = x.reshape(1, 2, 8, 8)
        n = x.shape[0]
        p = np.full((n, 64), 1.0 / 64, dtype=np.float32)
        cnt = x.reshape(n, 2, 64).astype(np.int32).sum(axis=2)
        v = (self.sign * ((cnt[:, 0] - cnt[:, 1]).astype(np.float32) / np.float32(64))).reshape(n, 1)
        self.rows += n
        self.calls += 1
        return (p[0], v[0]) if single else (p, v)
