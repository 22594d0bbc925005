"""GPU suite for the data-parallel training step (rz_trainer_create_group, csrc/rz_train.cu).

A group of replicas runs one step split into contiguous shards of the batch, and must give exactly the bits of the one-
device step: losses, gradient, weights, momentum and moving statistics.  Every test here runs on one H100 by repeating
device 0 in the device list; the tests on distinct devices run only where two or more GPUs are visible.
- A group of one (and the plain trainer) reproduces digests recorded from the build before groups existed.
- Groups of 2, 3, 4 and 8 replicas equal the single trainer after every step, and every replica's weights and momentum
  equal the primary's: empty shards, a conv0 weight-gradient split that straddles two shards, a batch off the split
  grid, a network without residual blocks, an epoch tail and a batch that changes from step to step.
- An out-of-range index in the last shard, non-default streams, reruns, two live groups, and the `opt` worker.
- One run of small group cases under compute-sanitizer's memcheck, which also sees writes past a buffer that no later
  read would reveal."""
import hashlib
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

from reversi_zero_b200 import net as N, train as T
from reversi_zero_b200.agent import model as M

pytestmark = pytest.mark.gpu

N_RECORDS = 700
LRS = [0.02, 0.02, 0.02, 0.005, 0.005]
# name -> (filters, res_blocks, value_fc, batch, max_batch)
SHAPES = {"16x1": (16, 1, 16, 64, 64), "48x1": (48, 1, 1, 67, 67), "128x2": (128, 2, 256, 97, 256),
          "256x1": (256, 1, 256, 100, 100), "ch5": (256, 10, 256, 256, 256)}


def _dataset(n=N_RECORDS, seed=5):
    """seeded training arrays on cuda:0: disjoint own / enemy planes, a sharp policy, z in {-1, 0, 1}"""
    rng = np.random.default_rng(seed)
    occ = rng.random((n, 64)) < 0.6
    own = occ & (rng.random((n, 64)) < 0.5)
    states = np.stack([own, occ & ~own], 1).reshape(n, 2, 8, 8).astype(np.uint8)
    p = rng.random((n, 64)) ** 4
    p = (p / p.sum(1, keepdims=True)).astype(np.float32)
    z = rng.choice([-1.0, 0.0, 1.0], n).astype(np.float32)
    return tuple(torch.as_tensor(a, device="cuda") for a in (states, p, z))


def _mc(name):
    F, R, V, _, _ = SHAPES[name]
    return M.ModelConfig(cnn_filter_num=F, res_layer_num=R, value_fc_size=V)


def _blob(mc, seed=3):
    return M.weights_to_blob(mc, M.build_random_weights(mc, seed, perturb_bn=True))


def _indices(batches, seed, n=N_RECORDS):
    rng = np.random.default_rng(seed)
    return [torch.as_tensor(rng.choice(n, b, replace=False).astype(np.int32), device="cuda") for b in batches]


def _digest(losses, blob, grad):
    return {k: hashlib.sha256(np.ascontiguousarray(v).view(np.uint32).tobytes()).hexdigest()[:32]
            for k, v in (("loss", np.concatenate(losses)), ("weights", blob), ("grad", grad))}


def _digest_run(name, make_trainer):
    mc = _mc(name)
    _, _, _, B, max_batch = SHAPES[name]
    data = _dataset()
    tr = make_trainer(mc, max_batch)
    tr.load_blob(_blob(mc))
    losses = [tr.step(*data, i, lr).cpu().numpy() for i, lr in zip(_indices([B] * len(LRS), 17), LRS)]
    out = _digest(losses, tr.blob(), tr.last_grad())
    tr.close()
    return out


# sha256 (first 128 bits) of the losses of 5 steps, the weights and the last gradient at each shape of SHAPES, recorded
# from the one-device trainer of the build before groups existed
PARENT_DIGESTS = {
    "16x1": {
        "loss": "e6ebbc7818d56d7105541e9522f6ca2d",
        "weights": "7a718e58ca208b9e8d5335f122f30908",
        "grad": "570483c11702f04573943e47d8da18ed"
    },
    "48x1": {
        "loss": "df610378bd5c5e1814a65d647445f40d",
        "weights": "3a498d6e9ba390006af4be50fcbe73f2",
        "grad": "5c6345749f894214923b0e095eaea01c"
    },
    "128x2": {
        "loss": "355050dd266fd90c2c47fd8fe928245f",
        "weights": "2865fd9df51cc342b0c81f7d4630127e",
        "grad": "ee1a329cc00756f4a8651c0b089ca329"
    },
    "256x1": {
        "loss": "4ecabf407cc249add0e314adf9768ae9",
        "weights": "861c249abda50f1cb7df7869fec0890b",
        "grad": "ce3217038975106ef3b10a867722f499"
    },
    "ch5": {
        "loss": "7bada0d2063ff98fd11a396f7b67220b",
        "weights": "53307c06031b69990c7f829bae8c68fe",
        "grad": "8886068ac086452a2f5297eb78aadb57"
    },
}


@pytest.mark.parametrize("name", list(SHAPES))
@pytest.mark.parametrize("kind", ["plain", "group_of_one"])
def test_one_device_reproduces_the_recorded_digests(name, kind):
    make = (lambda mc, mb: T.Trainer(mc, max_batch=mb)) if kind == "plain" else (lambda mc, mb: T.Trainer(mc, max_batch=mb, devices=[0]))
    assert _digest_run(name, make) == PARENT_DIGESTS[name]


def _bits(t):
    return t.contiguous().view(torch.int32)


def _state(tr, r):
    w, v = tr.replica_state(r)
    return _bits(w), _bits(v)


def _check_equal(ref, grp, n, step, loss_a, loss_b):
    """losses, gradient and weights of the group against the single trainer; every replica's weights and momentum"""
    assert np.array_equal(loss_a.view(np.uint32), loss_b.view(np.uint32)), (step, loss_a, loss_b)
    assert np.array_equal(ref.last_grad().view(np.uint32), grp.last_grad().view(np.uint32)), step
    assert torch.equal(_bits(ref.blob_dev()), _bits(grp.blob_dev())), step
    w0, v0 = _state(ref, 0)
    for r in range(n):
        w, v = _state(grp, r)
        assert torch.equal(w, w0) and torch.equal(v, v0), (step, r)


def _compare(mc, max_batch, devices, batches, lrs, seed=17, data=None):
    data = data or _dataset()
    blob = _blob(mc)
    ref, grp = T.Trainer(mc, max_batch=max_batch), T.Trainer(mc, max_batch=max_batch, devices=devices)
    for tr in (ref, grp):
        tr.load_blob(blob)
    for s, (i, lr) in enumerate(zip(_indices(batches, seed), lrs)):
        a, b = ref.step(*data, i, lr).cpu().numpy(), grp.step(*data, i, lr).cpu().numpy()
        _check_equal(ref, grp, len(devices), s, a, b)
    ref.close()
    grp.close()


def _distinct_gpus():
    if torch.cuda.device_count() < 2:
        pytest.skip(f"needs two or more GPUs, {torch.cuda.device_count()} visible: the same cases run on repeats of device 0")


GROUPS = [[0] * 2, [0] * 3, [0] * 4, [0] * 8]


@pytest.mark.parametrize("name", list(SHAPES))
@pytest.mark.parametrize("devices", GROUPS, ids=lambda d: f"x{len(d)}")
def test_replicas_equal_the_single_trainer(name, devices):
    _, _, _, B, max_batch = SHAPES[name]
    _compare(_mc(name), max_batch, devices, [B] * len(LRS), LRS)


@pytest.mark.parametrize("batch", [1, 3])
@pytest.mark.parametrize("devices", [[0] * 4, [0] * 8], ids=lambda d: f"x{len(d)}")
def test_empty_shards(batch, devices):
    _compare(_mc("128x2"), 256, devices, [batch] * 3, LRS[:3])


def test_conv0_split_straddles_a_shard():
    """64 filters, batch 256, three replicas: the shard boundary at record 175 falls inside conv0's split 174-175"""
    _compare(M.ModelConfig(cnn_filter_num=64, res_layer_num=1, value_fc_size=64), 256, [0] * 3, [256] * 3, LRS[:3])


@pytest.mark.parametrize("devices", GROUPS, ids=lambda d: f"x{len(d)}")
def test_network_without_residual_blocks(devices):
    """208 x 0 with V = 4096: the shards sit on conv0's grid, and head_fc_kernel takes more than 48 KB of shared memory on
    every replica"""
    _compare(M.ModelConfig(cnn_filter_num=208, res_layer_num=0, value_fc_size=4096), 5, devices, [5] * 3, LRS[:3])


@pytest.mark.parametrize("devices", [[0] * 3, [0] * 4], ids=lambda d: f"x{len(d)}")
def test_epoch_tail(devices):
    _compare(M.ModelConfig(cnn_filter_num=64, res_layer_num=1, value_fc_size=64), 64, devices, [64, 64, 17], [0.05, 0.05, 0.01])


@pytest.mark.parametrize("devices", [[0] * 3, [0] * 8], ids=lambda d: f"x{len(d)}")
def test_batch_changes_every_step(devices):
    batches = [97, 1, 256, 33, 128, 5, 200, 64, 255, 17]
    _compare(_mc("128x2"), 256, devices, batches, [0.02 - 0.001 * k for k in range(10)])


def _out_of_range(devices):
    mc, data = _mc("128x2"), _dataset()
    ref, grp = T.Trainer(mc, max_batch=256), T.Trainer(mc, max_batch=256, devices=devices)
    for tr in (ref, grp):
        tr.load_blob(_blob(mc))
    good, bad = _indices([100, 100], 23)
    bad[-1] = N_RECORDS + 5   # in the last replica's shard
    for tr in (ref, grp):
        tr.step(*data, good, 0.02)
    before = [_state(grp, r) for r in range(len(devices))]
    a, b = ref.step(*data, bad, 0.02).cpu().numpy(), grp.step(*data, bad, 0.02).cpu().numpy()
    assert np.isnan(b).all()
    _check_equal(ref, grp, len(devices), 1, a, b)
    for r in range(len(devices)):
        w, v = _state(grp, r)
        assert torch.equal(w, before[r][0]) and torch.equal(v, before[r][1]), r
    ref.close()
    grp.close()


@pytest.mark.parametrize("devices", [[0] * 2, [0] * 4], ids=lambda d: f"x{len(d)}")
def test_out_of_range_index_in_the_last_shard(devices):
    _out_of_range(devices)


def test_non_default_stream_reruns_and_two_live_groups():
    """steps enqueued on a side stream of the primary, the loss read after that stream synchronises; two groups alive at
    once, interleaved, give the same bits as each other, as a rerun and as the single trainer"""
    mc, data = _mc("128x2"), _dataset()
    idxs, lrs = _indices([97, 256, 64], 31), [0.02, 0.01, 0.01]

    def run(trainers):
        for tr in trainers:
            tr.load_blob(_blob(mc))
        side = torch.cuda.Stream()
        out = [[] for _ in trainers]
        with torch.cuda.stream(side):
            for i, lr in zip(idxs, lrs):
                for k, tr in enumerate(trainers):
                    out[k].append(tr.step(*data, i, lr))
        side.synchronize()
        res = [(np.concatenate([l.cpu().numpy() for l in o]).view(np.uint32), tr.blob().view(np.uint32)) for o, tr in zip(out, trainers)]
        for tr in trainers:
            tr.close()
        return res

    (la, wa), (lb, wb) = run([T.Trainer(mc, max_batch=256, devices=[0] * 3), T.Trainer(mc, max_batch=256, devices=[0] * 4)])
    (lc, wc), = run([T.Trainer(mc, max_batch=256, devices=[0] * 3)])
    (ld, wd), = run([T.Trainer(mc, max_batch=256)])
    for l, w in ((lb, wb), (lc, wc), (ld, wd)):
        assert np.array_equal(l, la) and np.array_equal(w, wa)


def test_opt_worker_on_a_group(tmp_path):
    """the `opt` worker with b200.train_devices = [0, 0] saves the same next-generation blob as on one device, and the
    blob loads into Net"""
    from reversi_zero_b200.worker import optimize as O
    from reversi_zero_b200.worker.evaluate import NEXT_GENERATION_BLOB
    from reversi_zero_b200.worker.self_play import SelfPlayWorker
    from test_selfplay_worker_gpu import mini_config
    cfg = mini_config(tmp_path)
    cfg.b200.write_play_rows = True
    assert SelfPlayWorker(cfg).start(max_games=8) >= 8
    cfg.trainer = dict(batch_size=64, min_data_size_to_learn=256, save_model_steps=5, wait_after_save_model_ratio=0)
    blobs = []
    for k, devices in enumerate((None, [0, 0])):
        cfg.b200.train_devices = devices
        cfg.resource.next_generation_model_dir = str(tmp_path / f"next_generation_{k}")
        os.makedirs(cfg.resource.next_generation_model_dir)
        ow = O.OptimizeWorker(cfg, seed=7)
        ow.start(max_epochs=1)
        assert ow.saved_model_dirs
        blobs.append(np.load(os.path.join(ow.saved_model_dirs[-1], NEXT_GENERATION_BLOB)))
    assert np.array_equal(blobs[0].view(np.uint32), blobs[1].view(np.uint32))
    net = N.Net(cfg.model)
    net.load_blob(blobs[1])
    p, v = net.predict_planes(np.zeros((2, 2, 8, 8), np.float32))
    assert np.isfinite(p).all() and np.isfinite(v).all()
    net.close()


@pytest.mark.parametrize("devices", [[0, 1], [0, 1, 0, 1]], ids=["0-1", "0-1-0-1"])
def test_distinct_gpus(devices):
    _distinct_gpus()
    for name in ("16x1", "128x2", "ch5"):
        _, _, _, B, max_batch = SHAPES[name]
        _compare(_mc(name), max_batch, devices, [B] * len(LRS), LRS)
    _compare(_mc("128x2"), 256, devices, [1, 3, 97], LRS[:3])
    _out_of_range(devices)


# A small group under memcheck: mini (16 x 1, V 16) on [0, 0, 0] at batches 64, 1 (two empty shards) and 17, and the
# 64-filter network at batch 256, whose conv0 split 174-175 straddles the second shard boundary (the peer copy of layer
# 0's dy rows).  Only host <-> device copies of torch run, so the kernels under test are the trainer's.
MEMCHECK_CASE = """
import sys
sys.path[:0] = [{root!r}, {pkg!r}]
import numpy as np
import torch
from reversi_zero_b200 import train as T
from reversi_zero_b200.agent import model as M

try:  # before any trainer code: can CUDA start under the tool at all?
    torch.as_tensor(np.zeros(4, np.float32), device="cuda").cpu()
except Exception as e:
    print("NO_CUDA_UNDER_SANITIZER", repr(e))
    sys.exit(3)


def run(mc, max_batch, devices, batches):
    rng = np.random.default_rng(1)
    n = 300
    occ = rng.random((n, 64)) < 0.6
    own = occ & (rng.random((n, 64)) < 0.5)
    states = torch.as_tensor(np.stack([own, occ & ~own], 1).reshape(n, 2, 8, 8).astype(np.uint8), device="cuda")
    p = rng.random((n, 64)).astype(np.float32)
    policy = torch.as_tensor(p / p.sum(1, keepdims=True), device="cuda")
    z = torch.as_tensor(rng.choice([-1.0, 0.0, 1.0], n).astype(np.float32), device="cuda")
    idxs = [torch.as_tensor(rng.choice(n, b, replace=False).astype(np.int32), device="cuda") for b in batches]
    blob = M.weights_to_blob(mc, M.build_random_weights(mc, 3, perturb_bn=True))
    out = []
    for devs in (None, devices):
        tr = T.Trainer(mc, max_batch=max_batch, devices=devs)
        tr.load_blob(blob)
        losses = np.concatenate([tr.step(states, policy, z, i, 0.02).cpu().numpy() for i in idxs])
        w = tr.blob()
        out.append((losses.view(np.uint32), w.view(np.uint32)))
        for r in range(len(devs or [])):
            assert np.array_equal(tr.replica_state(r)[0].cpu().numpy().view(np.uint32), w.view(np.uint32)), r
        tr.close()
    assert all(np.array_equal(a, b) for a, b in zip(*out)), mc


run(M.ModelConfig(cnn_filter_num=16, res_layer_num=1, value_fc_size=16), 64, [0, 0, 0], [64, 1, 17])
run(M.ModelConfig(cnn_filter_num=64, res_layer_num=1, value_fc_size=64), 256, [0, 0, 0], [256])
print("group memcheck case ok")
"""


def test_group_step_is_clean_under_memcheck(tmp_path):
    tool = shutil.which("compute-sanitizer") or "/usr/local/cuda/bin/compute-sanitizer"
    if not os.path.exists(tool):
        pytest.skip("compute-sanitizer is not installed")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    script = tmp_path / "group_memcheck_case.py"
    script.write_text(MEMCHECK_CASE.format(root=root, pkg=os.path.join(root, "reversi-alpha-zero_b200")))
    r = subprocess.run([tool, "--tool", "memcheck", sys.executable, str(script)], capture_output=True, text=True, timeout=1200)
    out = r.stdout + r.stderr
    if "NO_CUDA_UNDER_SANITIZER" in out:  # the tool's own start-up failed before any trainer code ran
        pytest.skip("compute-sanitizer cannot run CUDA on this machine: a host-to-device copy fails under it before the "
                    "trainer runs (" + out[out.index("NO_CUDA_UNDER_SANITIZER"):][:200].strip() + ")")
    summary = re.search(r"ERROR SUMMARY: (\d+) error", out)
    assert summary is not None and int(summary.group(1)) == 0, out[-4000:]
    assert r.returncode == 0 and "group memcheck case ok" in out, out[-4000:]
