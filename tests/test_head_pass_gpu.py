"""The dense heads after the wgmma towers (rz_net_heads.cu) held to SHA-256 digests of policy, value, policy logits and value
logit, for what tests/test_tower_ring_gpu.py does not cover: value heads of 1, 100 and 512 units on the 256-filter tower,
the 64- and 128-filter towers at n = 1, 5, 263 and 4 096, and the engine's counted path, whose device-side count is below
the batch capacity and whose rows past the count must keep what they held.  The digests in golden/head_pass_digest.json
were recorded with the heads still inside the tower kernels, one tile at a time; the batched head pass must reproduce them
bit for bit.

    python tests/test_head_pass_gpu.py --record    # rewrite golden/head_pass_digest.json from the current kernels
"""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "head_pass_digest.json")
SEED = 11
RES_BLOCKS = 1
# (filters, value_fc) -> batch sizes
CASES = {(256, 1): (1, 263), (256, 100): (1, 263), (256, 512): (1, 263),
         (128, 256): (1, 5, 263, 4096), (64, 256): (1, 5, 263, 4096)}
# (filters, value_fc, device-side count, capacity): the count is one of the recorded batch sizes of that network
COUNTED = ((256, 100, 263, 300), (128, 256, 5, 263), (64, 256, 263, 4096))
SENTINEL = -7.5


def _key(filters, value_fc, n):
    return f"f{filters}_v{value_fc}_n{n}"


def _positions(n):
    rng = np.random.default_rng(SEED)
    a = rng.integers(0, 2 ** 64, size=n, dtype=np.uint64)
    r = rng.integers(0, 2 ** 64, size=n, dtype=np.uint64)
    return a & r, a & ~r


def _net(filters, value_fc):
    from reversi_zero_b200.agent import model as M
    from reversi_zero_b200 import net as N
    mc = M.ModelConfig(cnn_filter_num=filters, res_layer_num=RES_BLOCKS, value_fc_size=value_fc)
    net = N.Net(mc)
    net.load_weights(M.build_random_weights(mc, SEED, perturb_bn=True))
    return net


def _digest(t):
    return hashlib.sha256(t.cpu().numpy()).hexdigest()


def head_digests(filters, value_fc):
    import torch
    from reversi_zero_b200 import device as D
    sizes = CASES[(filters, value_fc)]
    own, enemy = _positions(max(sizes))
    net = _net(filters, value_fc)
    out = {}
    try:
        for n in sizes:
            bufs = dict(policy=D.empty(n * 64, np.float32), value=D.empty(n, np.float32), logits=D.empty(n * 64, np.float32),
                        vlogit=D.empty(n, np.float32))
            net.debug_heads_dev(D.to_device(own[:n]), D.to_device(enemy[:n]), bufs["policy"], bufs["value"], bufs["logits"],
                                bufs["vlogit"], n)
            torch.cuda.synchronize()
            out[_key(filters, value_fc, n)] = {k: _digest(v) for k, v in bufs.items()}
    finally:
        net.close()
    return out


def _golden():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.mark.gpu
@pytest.mark.parametrize("filters,value_fc", sorted(CASES))
def test_heads_match_recorded_digests(filters, value_fc):
    want = _golden()
    for key, d in head_digests(filters, value_fc).items():
        assert d == want[key], (key, {k: d[k] == want[key][k] for k in d})


@pytest.mark.gpu
@pytest.mark.parametrize("filters,value_fc,count,capacity", COUNTED)
def test_counted_batch_matches_digests_and_keeps_rows_past_the_count(filters, value_fc, count, capacity):
    import torch
    from reversi_zero_b200 import device as D
    want = _golden()[_key(filters, value_fc, count)]
    own, enemy = _positions(max(CASES[(filters, value_fc)]))   # the recorded batch's positions ...
    pad_own, pad_enemy = _positions(capacity)                  # ... then others up to the capacity
    own, enemy = np.concatenate([own[:count], pad_own[count:]]), np.concatenate([enemy[:count], pad_enemy[count:]])
    net = _net(filters, value_fc)
    try:
        policy = torch.full((capacity * 64,), SENTINEL, dtype=torch.float32, device="cuda")
        value = torch.full((capacity,), SENTINEL, dtype=torch.float32, device="cuda")
        count_t = torch.tensor([count], dtype=torch.int32, device="cuda")
        # the positions past the count are real positions, so that a kernel that ignored the count would overwrite them
        net.predict_counted_dev(D.to_device(own), D.to_device(enemy), policy, value, count_t, capacity)
        torch.cuda.synchronize()
    finally:
        net.close()
    assert _digest(policy[:count * 64]) == want["policy"]
    assert _digest(value[:count]) == want["value"]
    assert bool((policy[count * 64:] == SENTINEL).all()) and bool((value[count:] == SENTINEL).all())


if __name__ == "__main__":
    assert sys.argv[1:] == ["--record"], __doc__
    root = os.path.dirname(HERE)
    sys.path[:0] = [root, os.path.join(root, "reversi-alpha-zero_b200")]
    rec = {}
    for filters, value_fc in sorted(CASES):
        rec.update(head_digests(filters, value_fc))
    with open(GOLDEN, "w") as f:
        json.dump(rec, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"wrote {len(rec)} digests to {GOLDEN}")
