"""The play-JSON parser on the device (rz_ingest_json_dev, csrc/rz_ingest_json.cu): bit-identical to its host twin and
to the reference trainer's arrays, to rz_ingest_dev on the rows twin of this engine's own files at ragged sizes, the
same byte offsets for malformed text, repeatable on two streams, and the ``opt`` worker training from JSON alone."""
import glob
import json
import os

import numpy as np
import pytest
import torch

from reversi_zero_b200 import net as N
from reversi_zero_b200.agent import model as M
from reversi_zero_b200.worker import ingest as I
from reversi_zero_b200.worker import optimize as O
from reversi_zero_b200.worker.self_play import SelfPlayWorker, newest_next_generation_blob
from test_ingest_json import corpus, corpus_text, expected_f32, f32_bits, planes_of, small_text, REF_CASES
from test_selfplay_worker_gpu import mini_config

pytestmark = pytest.mark.gpu


def same(dev, host):
    for a, b in zip(dev, host):
        a = a.cpu().numpy()
        assert a.shape == b.shape and np.array_equal(a.view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


def test_device_equals_host_twin_and_python_on_the_corpus():
    text, toks, boards = corpus_text(corpus())
    dev = I.parse_play_json(text)
    host = I.parse_play_json_host(text)
    same(dev, host)
    exp = expected_f32(toks).reshape(-1, 65)
    assert np.array_equal(f32_bits(dev[1].cpu().numpy()), f32_bits(exp[:, :64]))
    assert np.array_equal(f32_bits(dev[2].cpu().numpy()), f32_bits(exp[:, 64]))
    assert np.array_equal(dev[0].cpu().numpy(), planes_of(boards))


@pytest.mark.parametrize("name", REF_CASES)
def test_device_gives_the_reference_trainers_arrays(golden_dir, name):
    g = np.load(os.path.join(golden_dir, "play_json_ref.npz"))
    states, policy, z = I.parse_play_json(g[name + "_text"].tobytes())
    ref_states = np.unpackbits(g[name + "_states_packed"], axis=1, bitorder="little").reshape(-1, 2, 8, 8)
    assert np.array_equal(states.cpu().numpy(), ref_states)
    assert np.array_equal(f32_bits(policy.cpu().numpy()), f32_bits(g[name + "_policy"].astype(np.float32)))
    assert np.array_equal(f32_bits(z.cpu().numpy()), f32_bits(g[name + "_z"].astype(np.float32)))


@pytest.fixture(scope="module")
def engine_files(tmp_path_factory):
    cfg = mini_config(tmp_path_factory.mktemp("selfplay"))
    cfg.b200.write_play_rows = True
    assert SelfPlayWorker(cfg).start(max_games=8) >= 8
    files = sorted(glob.glob(os.path.join(cfg.resource.play_data_dir, "play_*.json")))
    assert files
    return files


def rows_tensors(path):
    rows, tau1, ctt = I.read_play_rows(I.rows_path_of(path))
    return I.to_training_tensors(rows, tau1, ctt, 0)


def test_engine_json_equals_rz_ingest_dev_on_its_rows_twin(engine_files):
    parts = []
    for path in engine_files:
        got, ref = I.read_play_json(path), rows_tensors(path)
        for a, b in zip(got, ref):
            assert torch.equal(a.view(torch.uint8), b.view(torch.uint8))
        parts.append((path, ref))
    # ragged sizes: one record, 7 records, an empty array, and a multi-MB file of all records repeated
    recs = json.loads(open(engine_files[0]).read())
    ref = parts[0][1]
    for k in (1, 7, 8 * 5 + 3):
        got = I.parse_play_json(json.dumps(recs[:k]).encode())
        for a, b in zip(got, ref):
            assert torch.equal(a.view(torch.uint8), b[:k].view(torch.uint8))
    s, p, z = I.parse_play_json(b"[]")
    assert s.shape == (0, 2, 8, 8) and p.shape == (0, 64) and z.shape == (0,)
    all_recs = [r for path, _ in parts for r in json.loads(open(path).read())]
    text = json.dumps(all_recs)
    reps = max(1, -(-6_000_000 // len(text)))
    got = I.parse_play_json(json.dumps(all_recs * reps).encode())
    for i in range(3):
        ref_i = torch.cat([t[i] for _, t in parts] * reps)
        assert torch.equal(got[i].view(torch.uint8), ref_i.view(torch.uint8))


def test_malformed_text_gives_the_host_twins_offset():
    text = small_text()
    for k in list(range(0, 200)) + list(range(200, len(text), 7)):
        with pytest.raises(I.PlayJsonError) as d:
            I.parse_play_json(text[:k])
        with pytest.raises(I.PlayJsonError) as h:
            I.parse_play_json_host(text[:k])
        assert d.value.offset == h.value.offset, k
    for bad in (text + b"x", text.replace(b"]", b"]]", 3), text.replace(b", ", b', "', 40), text.replace(b"0.0", b"00", 1),
                b"[" + text + b"]", b'{"a": 1}', b""):
        with pytest.raises(I.PlayJsonError) as d:
            I.parse_play_json(bad)
        with pytest.raises(I.PlayJsonError) as h:
            I.parse_play_json_host(bad)
        assert d.value.offset == h.value.offset


def test_repeatable_and_two_streams():
    text, _, _ = corpus_text(corpus()[:30000], seed=3)
    first = I.parse_play_json(text)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    with torch.cuda.stream(s1):
        a = I.parse_play_json(text)
    with torch.cuda.stream(s2):
        b = I.parse_play_json(text)
    torch.cuda.synchronize()
    for x, y, f in zip(a, b, first):
        assert torch.equal(x.view(torch.uint8), f.view(torch.uint8)) and torch.equal(y.view(torch.uint8), f.view(torch.uint8))


def test_opt_trains_from_json_alone_and_the_blob_loads(tmp_path):
    cfg = mini_config(tmp_path)
    assert SelfPlayWorker(cfg).start(max_games=8) >= 8       # write_play_rows is off: JSON only
    play_dir = cfg.resource.play_data_dir
    assert glob.glob(os.path.join(play_dir, "play_*.json")) and not glob.glob(os.path.join(play_dir, "*.rzrows"))
    cfg.b200.train_from_json = True
    cfg.trainer = dict(batch_size=64, min_data_size_to_learn=256, save_model_steps=5, wait_after_save_model_ratio=0)
    ow = O.OptimizeWorker(cfg)
    total = ow.start(max_epochs=1)
    assert ow.dataset_size >= 256 and total == ow.dataset_size // 64 and ow.saved_model_dirs
    blob = np.load(newest_next_generation_blob(cfg))
    assert blob.size == M.blob_size(cfg.model) and M.blob_digest(blob) != M.blob_digest(np.load(cfg.resource.model_best_blob_path))
    net = N.Net(cfg.model)
    net.load_blob(blob)
    p, v = net.predict_planes(ow.dataset[0][:16].cpu().numpy())
    assert np.isfinite(p).all() and np.isfinite(v).all() and np.allclose(p.sum(axis=1), 1, atol=1e-4)
