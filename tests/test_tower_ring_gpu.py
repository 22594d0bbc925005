"""The wgmma tower (rz_net_tc.cu) held to SHA-256 digests of its outputs: policy, value, policy logits, value logit and the
fp32 tower output of a seeded batch, for batches that leave CTAs without tiles (n = 1, 2, 3), end on an odd tile and give
pairs a dummy tile (263), and run every CTA through many tiles (32 768), for 0, 1, 10 and 19 residual blocks and both
cluster variants.  The digests in golden/tower_digest.json were recorded with a weight ring of three 32 KB stages and
a separate layer-0 weight buffer.  A schedule change that keeps the K order, the fp16 operands and the epilogue
arithmetic must reproduce them bit for bit.

    python tests/test_tower_ring_gpu.py --record    # rewrite golden/tower_digest.json from the current kernel
"""
import hashlib
import json
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "tower_digest.json")
SIZES = (1, 2, 3, 263, 32768)
BLOCKS = (0, 1, 10, 19)
SEED = 7


def tower_digests(res_blocks, cluster):
    import torch
    from reversi_zero_b200.agent import model as M
    from reversi_zero_b200 import net as N, device as D
    mc = M.ModelConfig(cnn_filter_num=256, res_layer_num=res_blocks, value_fc_size=256)
    net = N.Net(mc)
    net.load_weights(M.build_random_weights(mc, SEED, perturb_bn=True))
    rng = np.random.default_rng(SEED)
    a = rng.integers(0, 2 ** 64, size=max(SIZES), dtype=np.uint64)
    r = rng.integers(0, 2 ** 64, size=max(SIZES), dtype=np.uint64)
    out = {}
    try:
        N.set_tower_cluster(cluster)
        for n in SIZES:
            d_own, d_en = D.to_device(a[:n] & r[:n]), D.to_device(a[:n] & ~r[:n])
            bufs = dict(policy=D.empty(n * 64, np.float32), value=D.empty(n, np.float32), logits=D.empty(n * 64, np.float32),
                        vlogit=D.empty(n, np.float32), tower=D.empty(n * 64 * 256, np.float32))
            net.debug_heads_dev(d_own, d_en, bufs["policy"], bufs["value"], bufs["logits"], bufs["vlogit"], n, tower_t=bufs["tower"])
            torch.cuda.synchronize()
            out[f"b{res_blocks}_n{n}"] = {k: hashlib.sha256(v.cpu().numpy()).hexdigest() for k, v in bufs.items()}
            del bufs
    finally:
        N.set_tower_cluster(2)
        net.close()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("cluster", (1, 2))
@pytest.mark.parametrize("res_blocks", BLOCKS)
def test_tower_outputs_match_recorded_digests(res_blocks, cluster):
    with open(GOLDEN) as f:
        want = json.load(f)
    got = tower_digests(res_blocks, cluster)
    for key, d in got.items():
        assert d == want[key], (key, cluster, {k: d[k] == want[key][k] for k in d})


if __name__ == "__main__":
    assert sys.argv[1:] == ["--record"], __doc__
    root = os.path.dirname(HERE)
    sys.path[:0] = [root, os.path.join(root, "reversi-alpha-zero_b200")]
    rec = {}
    for b in BLOCKS:
        d1, d2 = tower_digests(b, 1), tower_digests(b, 2)
        assert d1 == d2, b   # the two cluster variants compute the same bits
        rec.update(d2)
    with open(GOLDEN, "w") as f:
        json.dump(rec, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"wrote {len(rec)} digests to {GOLDEN}")
