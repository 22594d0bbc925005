"""GPU suite for the device trainer (csrc/rz_train.cu): one step against the fp64 oracle and its TF32 format model
(oracle/train.py) on records that rz_ingest_dev expanded from real engine games; ragged batches and repeated indices;
five steps with learning-rate changes; bit-reproducibility; learning over 200 steps against the fp32 oracle; and the
hand-off of the trained blob to the inference network."""
import numpy as np
import pytest
import torch

from oracle import mcts, nn as onn, train as ot
from reversi_zero_b200 import engine as E, net as N, train as T
from reversi_zero_b200.agent import model as M
from reversi_zero_b200.worker import ingest as zi

pytestmark = pytest.mark.gpu

MINI = dict(cnn_filter_num=16, res_layer_num=1, value_fc_size=64)
TWO = dict(cnn_filter_num=256, res_layer_num=2, value_fc_size=256)
CH5 = dict(cnn_filter_num=256, res_layer_num=10, value_fc_size=256)
F32_EPS = 2.0 ** -23


@pytest.fixture(scope="module")
def records(tmp_path_factory):
    """training arrays of 24 self-play games of the engine (deterministic evaluator), expanded on the device"""
    pp = mcts.PlayParams(simulation_num_per_move=16, parallel_search_num=4, c_puct=5, noise_eps=0.25)
    eng = E.Engine(E.engine_cfg_from_play_config(pp, games=24, seed=11, eval_mode=E.EVAL_FAKE, max_games=24))
    eng.run(finished_target=24)
    G, ng, P, _ = eng.poll_raw()
    path = str(tmp_path_factory.mktemp("rows") / "play_x.rzrows")
    zi.write_play_rows(path, G, ng, P, True, 4)
    eng.close()
    rows, tau1, ctt = zi.read_play_rows(path)
    states, policy, z = zi.to_training_tensors(rows, tau1, ctt, 0)
    assert states.shape[0] >= 4096
    return states, policy, z


def _host(records, idx):
    s, p, z = records
    i = torch.as_tensor(idx, dtype=torch.long, device=s.device)
    return s[i].cpu().numpy(), p[i].cpu().numpy(), z[i].cpu().numpy()


def _weights(mc, kind, planes):
    if kind == "new":
        return M.build_random_weights(mc, 3)
    return onn.calibrate_bn(M.build_random_weights(mc, 3, perturb_bn=True), planes, mc.res_layer_num)


def _rel(a, b):
    return float(np.linalg.norm(np.asarray(a, np.float64) - b) / max(np.linalg.norm(b), 1e-30))


def _is_conv_bias(name):
    return name.endswith(".bias") and not name.startswith(("policy_fc", "value_fc"))


def _check_against_oracle(mc, w0, got_w, got_g, got_loss, o64, ofm, report=None):
    """o64 / ofm: (weights, losses, grads) of the fp64 oracle and of the format model, from the same start w0;
    got_loss None: the losses are checked by the caller.

    The kernel's own TF32 rounding is a different draw of the same noise as the format model's.  A tensor of one or two
    elements (the head BatchNorms' gamma / beta, the value output bias) has a relative error that is a single draw, so it
    is held to the format-model error of the whole layer it belongs to (kernel, bias and BN parameters together)."""
    (w64, l64, g64), (wfm, lfm, gfm) = o64, ofm
    for a, b, c in zip(got_loss or (), l64, lfm):
        assert abs(a - b) <= 1.5 * abs(c - b) + 1e-4 * abs(b), (got_loss, l64, lfm)

    def layer_rel(got, ref, fm, name):
        keys = [k for k in ref if k.rsplit(".", 2 if ".bn_" in k else 1)[0] == name.rsplit(".", 2 if ".bn_" in name else 1)[0]]
        flat = lambda d: np.concatenate([np.asarray(d[k], np.float64).ravel() for k in keys])
        return _rel(flat(got), flat(ref)), _rel(flat(fm), flat(ref))

    for name, shape in M.tensor_specs(mc):
        small = int(np.prod(shape)) <= 2
        if name in g64 and got_g is not None:
            if _is_conv_bias(name):
                assert np.abs(got_g[name]).max() <= 1e-6, name
            else:
                ek, ef = _rel(got_g[name], g64[name]), _rel(gfm[name], g64[name])
                if report is not None:
                    report.append((name, ek, ef))
                if small:
                    ef = max(ef, layer_rel(got_g, g64, gfm, name)[1])
                assert ek <= 1.5 * ef + 1e-6, (name, ek, ef)
        # weights after the update (trainables and moving statistics): error of the change, plus fp32 storage rounding
        ref = np.asarray(w64[name], np.float64)
        delta = np.linalg.norm(ref - np.asarray(w0[name], np.float64))
        efm = np.linalg.norm(np.asarray(wfm[name], np.float64) - ref)
        if small:
            efm = max(efm, delta * layer_rel({k: np.asarray(wfm[k], np.float64) - w0[k] for k in w64},
                                             {k: np.asarray(w64[k], np.float64) - w0[k] for k in w64},
                                             {k: np.asarray(wfm[k], np.float64) - w0[k] for k in w64}, name)[1])
        store = 4 * F32_EPS * np.linalg.norm(ref) + 1e-12
        err = np.linalg.norm(np.asarray(got_w[name], np.float64) - ref)
        assert err <= 1.5 * efm + 1e-6 * delta + store, (name, err, efm, delta)


def _oracle_steps(mc, w0, batches, lrs, dtype=torch.float64, tf32_convs=False):
    w, v, losses, grads = w0, None, [], None
    for (planes, policy, z), lr in zip(batches, lrs):
        w, v, l, grads = ot.step(w, v, planes, policy, z, lr, mc.res_layer_num, mc.l2_reg, dtype=dtype, tf32_convs=tf32_convs)
        losses.append(l)
    return w, losses, grads


def _trainer_steps(mc, w0, records, idxs, lrs):
    tr = T.Trainer(mc, max_batch=max(len(i) for i in idxs))
    tr.load_blob(M.weights_to_blob(mc, w0))
    losses = []
    for idx, lr in zip(idxs, lrs):
        loss = tr.step(*records, torch.as_tensor(np.asarray(idx, np.int32), device="cuda"), lr)
        losses.append(tuple(float(x) for x in loss.cpu().numpy()))
    w = M.blob_to_weights(mc, tr.blob())
    g = M.blob_to_weights(mc, tr.last_grad())
    tr.close()
    return w, losses, g


@pytest.mark.parametrize("cfg,batch,kind", [(MINI, 64, "new"), (MINI, 64, "calibrated"), (TWO, 256, "calibrated"),
                                            (TWO, 32, "new"), (CH5, 32, "calibrated")])
def test_one_step_matches_oracle(records, cfg, batch, kind):
    mc = M.ModelConfig(**cfg)
    rng = np.random.default_rng(batch)
    idx = rng.choice(records[0].shape[0], batch, replace=False)
    host = _host(records, idx)
    w0 = _weights(mc, kind, host[0])
    w, losses, g = _trainer_steps(mc, w0, records, [idx], [0.02])
    o64 = _oracle_steps(mc, w0, [host], [0.02])
    ofm = _oracle_steps(mc, w0, [host], [0.02], tf32_convs=True)
    report = []
    _check_against_oracle(mc, w0, w, g, losses[0], (o64[0], o64[1][0], o64[2]), (ofm[0], ofm[1][0], ofm[2]), report)
    worst = max(report, key=lambda r: r[1])
    print(f"\n{cfg} B={batch} {kind}: loss {losses[0]} fp64 {o64[1][0]}; worst gradient {worst[0]}: kernel {worst[1]:.2e} "
          f"format model {worst[2]:.2e}; median kernel/format {np.median([r[1] / r[2] for r in report]):.2f}")


@pytest.mark.parametrize("idx", [[5], [3, 9, 27, 81, 243, 729, 2187], list(range(100, 229)), [7, 7, 7, 12, 12, 40, 7, 3000]],
                         ids=["B1", "B7", "B129", "repeats"])
def test_ragged_batches_and_repeated_indices(records, idx):
    mc = M.ModelConfig(**MINI)
    host = _host(records, idx)
    w0 = _weights(mc, "calibrated", host[0] if len(idx) > 1 else _host(records, range(64))[0])
    w, losses, g = _trainer_steps(mc, w0, records, [idx], [0.05])
    o64 = _oracle_steps(mc, w0, [host], [0.05])
    ofm = _oracle_steps(mc, w0, [host], [0.05], tf32_convs=True)
    _check_against_oracle(mc, w0, w, g, losses[0], (o64[0], o64[1][0], o64[2]), (ofm[0], ofm[1][0], ofm[2]))


def test_five_steps_with_learning_rate_changes(records):
    mc = M.ModelConfig(**MINI)
    rng = np.random.default_rng(9)
    idxs = [rng.choice(records[0].shape[0], 48, replace=False) for _ in range(5)]
    lrs = [0.05, 0.05, 0.01, 0.01, 0.002]
    w0 = _weights(mc, "calibrated", _host(records, idxs[0])[0])
    w, losses, g = _trainer_steps(mc, w0, records, idxs, lrs)
    batches = [_host(records, i) for i in idxs]
    o64 = _oracle_steps(mc, w0, batches, lrs)
    ofm = _oracle_steps(mc, w0, batches, lrs, tf32_convs=True)
    for k in range(5):  # after the first step the runs differ by their own rounding: bound by the format model's distance
        for a, b, c in zip(losses[k], o64[1][k], ofm[1][k]):
            assert abs(a - b) <= 1.5 * abs(c - b) + 1e-4 * abs(b), (k, losses[k], o64[1][k], ofm[1][k])
    _check_against_oracle(mc, w0, w, None, None, (o64[0], o64[1][4], o64[2]), (ofm[0], ofm[1][4], ofm[2]))


def test_bad_index_leaves_weights_unchanged(records):
    mc = M.ModelConfig(**MINI)
    w0 = M.weights_to_blob(mc, M.build_random_weights(mc, 1))
    tr = T.Trainer(mc, max_batch=4)
    tr.load_blob(w0)
    loss = tr.step(*records, torch.tensor([0, 1, records[0].shape[0], 2], dtype=torch.int32, device="cuda"), 0.1)
    assert np.isnan(loss.cpu().numpy()).all() and np.array_equal(tr.blob(), w0)
    with pytest.raises(Exception):
        tr.step(*records, torch.zeros(5, dtype=torch.int32, device="cuda"), 0.1)  # more than max_batch


def test_ten_steps_are_bit_reproducible(records):
    mc = M.ModelConfig(**TWO)
    rng = np.random.default_rng(4)
    idxs = [rng.choice(records[0].shape[0], 256, replace=False) for _ in range(10)]
    w0 = _weights(mc, "new", None)
    runs = [_trainer_steps(mc, w0, records, idxs, [0.02] * 10) for _ in range(2)]
    assert runs[0][1] == runs[1][1]
    for name in runs[0][0]:
        assert np.array_equal(runs[0][0][name], runs[1][0][name]), name


def test_two_hundred_steps_learn_like_the_fp32_oracle(records):
    mc = M.ModelConfig(**MINI)
    rng = np.random.default_rng(2)
    n, batch = 2048, 128
    idxs = []
    while len(idxs) < 200:  # one permutation per epoch, as fit(shuffle=True) does
        perm = rng.permutation(n)
        idxs += [perm[i:i + batch] for i in range(0, n, batch)]
    idxs = idxs[:200]
    w0 = M.build_random_weights(mc, 5)
    _, losses, _ = _trainer_steps(mc, w0, records, idxs, [0.01] * 200)
    _, olosses, _ = _oracle_steps(mc, w0, [_host(records, i) for i in idxs], [0.01] * 200, dtype=torch.float32)
    first, last = np.mean([l[0] for l in losses[:10]]), np.mean([l[0] for l in losses[-10:]])
    print(f"\nloss: steps 1-10 {first:.4f}, 191-200 {last:.4f}; step 200 kernel {losses[-1][0]:.4f} fp32 oracle {olosses[-1][0]:.4f}")
    assert last < first
    assert abs(losses[-1][0] - olosses[-1][0]) <= 0.05 * olosses[-1][0]


@pytest.mark.parametrize("impl", [N.IMPL_TCGEN05, N.IMPL_GENERIC])
def test_trained_blob_loads_into_the_inference_network(records, impl):
    mc = M.ModelConfig(**TWO)
    rng = np.random.default_rng(8)
    idxs = [rng.choice(records[0].shape[0], 128, replace=False) for _ in range(3)]
    tr = T.Trainer(mc, max_batch=128)
    tr.load_blob(M.weights_to_blob(mc, M.build_random_weights(mc, 2)))
    for idx in idxs:
        tr.step(*records, torch.as_tensor(idx.astype(np.int32), device="cuda"), 0.05)
    blob_t = tr.blob_dev()
    net = N.Net(mc)
    net.load_blob_dev(blob_t)
    torch.cuda.synchronize()
    planes = _host(records, np.arange(0, 4000, 37))[0]
    p, v = net.predict_planes(planes, impl)
    p_ref, v_ref = onn.forward(M.blob_to_weights(mc, blob_t.cpu().numpy()), planes, mc.res_layer_num)
    assert np.abs(p - p_ref).max() < 1e-3 and np.abs(v - v_ref).max() < 1e-3
    net.close()
    tr.close()
