"""CPU suite for the ``opt`` worker mirror (reversi_zero_b200/worker/optimize.py) with a stand-in trainer: every host
decision the unmodified reference trainer made in tests/golden/optimize_ref.json (tests/golden/make_golden_optimize.py),
the Keras batch count, the atomic and directory-clean model save, model loading and the rows-twin refusal."""
import json
import os
import sys
import types

import numpy as np
import pytest
import torch

from oracle import ingest as oi
from reversi_zero_b200.agent import model as M
from reversi_zero_b200.config import Config
from reversi_zero_b200.worker import optimize as O
from reversi_zero_b200.worker.evaluate import EvaluateWorker, NEXT_GENERATION_BLOB
from reversi_zero_b200.worker.self_play import newest_next_generation_blob

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_golden_optimize as G  # noqa: E402


@pytest.fixture(scope="module")
def golden(golden_dir):
    with open(os.path.join(golden_dir, "optimize_ref.json")) as f:
        return json.load(f)


class StandInTrainer:
    """The Trainer interface (load_blob / step / blob) without a device: every step adds 1 to the blob"""

    def __init__(self):
        self.steps, self.w = [], None

    def load_blob(self, blob):
        self.w = np.array(blob, np.float32)

    def step(self, states, policy, z, index, lr):
        assert index.dtype == torch.int32 and int(index.max()) < states.shape[0]
        self.steps.append((int(index.numel()), lr))
        self.w = self.w + 1
        return torch.zeros(3)

    def blob(self):
        return self.w.copy()


def host_tensors(rows, tau1, ctt):
    return tuple(torch.from_numpy(np.ascontiguousarray(a))
                 for a in oi.rows_to_training_arrays(rows["own"], rows["enemy"], rows["n_visit"], rows["z"], tau1, ctt))


class Clock:
    def __init__(self, t=1000.0):
        self.t, self.sleeps = t, []

    def __call__(self):
        return self.t

    def sleep(self, s):
        self.sleeps.append(s)
        self.t += s


def make_config(tmp_path, **trainer):
    cfg = Config(project_dir=str(tmp_path), data_dir=str(tmp_path / "data"))
    cfg.model.update(dict(cnn_filter_num=16, res_layer_num=1, value_fc_size=16))
    cfg.resource.create_directories()
    cfg.trainer = dict(trainer)   # the YAML section, kept as a plain dict
    return cfg


def make_worker(cfg, clock=None):
    clock = clock or Clock()
    return O.OptimizeWorker(cfg, trainer=StandInTrainer(), to_tensors=host_tensors, sleep=clock.sleep, clock=clock)


def save_best(cfg):
    blob = M.weights_to_blob(cfg.model, M.build_random_weights(cfg.model, 0))
    np.save(cfg.resource.model_best_blob_path, blob)
    return blob


def test_trainer_defaults_are_the_reference_trainer_config():
    import oracle.ref_shims.install as shims
    cfg = types.SimpleNamespace(trainer={"batch_size": 64})
    assert O.trainer_field(cfg, "batch_size") == 64 and O.trainer_field(cfg, "save_model_steps") == 200
    assert O.trainer_field(types.SimpleNamespace(), "min_data_size_to_learn") == 100000
    if shims.available():   # where the reference checkout exists: its TrainerConfig itself
        shims.install()
        from reversi_zero.config import TrainerConfig
        ref = vars(TrainerConfig())
        assert {k: (list(v) if isinstance(v, list) else v) for k, v in ref.items()} == O.TRAINER_DEFAULTS


def test_decide_learning_rate_matches_reference(tmp_path, golden):
    for name, sched in G.SCHEDULES.items():
        for text in G.FORCE_TEXTS:
            cfg = make_config(tmp_path, lr_schedules=sched)
            path = cfg.resource.force_learing_rate_file
            if os.path.exists(path):
                os.remove(path)
            if text is not None:
                with open(path, "wt") as f:
                    f.write(text)
            w = make_worker(cfg)
            assert [w.decide_learning_rate(s) for s in golden["lr_steps"]] == golden["lr"][f"{name}|{text!r}"], (name, text)


def test_train_epoch_steps_and_keras_batches(tmp_path, golden):
    for n, b, epochs, steps in golden["epochs"]:
        w = make_worker(make_config(tmp_path, batch_size=b))
        w.trainer.load_blob(np.zeros(4, np.float32))
        w.dataset = (torch.zeros((n, 2, 8, 8), dtype=torch.uint8), torch.zeros((n, 64)), torch.zeros(n))
        cb = O.PerStepCallback(10 ** 9, lambda: None)
        assert w.train_epoch(epochs, cb) == steps
        per_epoch = [b] * (n // b) + ([n % b] if n % b else [])   # fit runs ceil(N / B) batches, the last one partial
        assert [s for s, _ in w.trainer.steps] == per_epoch * epochs and cb.step == len(per_epoch) * epochs


def test_save_cadence_matches_reference(golden):
    c = G.CADENCE
    clock = Clock(100.0)
    saves, sleeps = [], []
    batch = [0]

    def sleep(s):
        sleeps.append([len(saves), s])

    cb = O.PerStepCallback(c["per_step"], lambda: saves.append(batch[0]), c["ratio"], sleep=sleep, clock=clock)
    for batch[0] in range(1, c["batches"] + 1):
        clock.t += c["tick"]
        cb.on_batch_end()
    assert saves == golden["cadence"]["saves"] and sleeps == golden["cadence"]["sleeps"]


def test_load_unload_delete_timeline_matches_reference(tmp_path, golden):
    cfg = make_config(tmp_path, delete_self_play_after_number_of_training=G.DELETE_LIMIT)
    play_dir = cfg.resource.play_data_dir
    w = make_worker(cfg)
    for (action, key), ref in zip(G.TIMELINE, golden["timeline"]):
        if action == "add":
            G.write_play_files(play_dir, key)
        elif action == "remove":
            for name in os.listdir(play_dir):
                if G.FILES[key] in name:
                    os.remove(os.path.join(play_dir, name))
        elif action == "load":
            w.load_play_data()
        else:
            w.count_up_training_count_and_delete_self_play_data_files()
        json_files = sorted(n for n in os.listdir(play_dir) if n.endswith(".json"))
        got = dict(loaded=sorted(os.path.basename(f) for f in w.loaded_filenames), dataset_size=w.dataset_size,
                   counts={os.path.basename(f): c for f, c in sorted(w.training_count_of_files.items())}, json_files=json_files)
        assert got == ref, (action, key)
        # a deleted JSON file takes its rows twin with it
        assert sorted(n for n in os.listdir(play_dir) if n.endswith(".rzrows")) == [n[:-5] + ".rzrows" for n in json_files]


def test_json_without_rows_twin_stops_the_worker_after_a_grace_period(tmp_path):
    cfg = make_config(tmp_path)
    clock = Clock()
    w = make_worker(cfg, clock)
    path = G.write_play_files(cfg.resource.play_data_dir, "a")
    os.remove(path[:-5] + ".rzrows")
    w.load_play_data()                       # self-play writes the twin right after the JSON file: wait for it
    assert w.dataset_size == 0
    clock.t += O.ROWS_GRACE_SEC
    with pytest.raises(RuntimeError, match="write_play_rows"):
        w.load_play_data()


def test_training_loop_waits_then_trains_and_saves_atomically(tmp_path):
    cfg = make_config(tmp_path, batch_size=256, min_data_size_to_learn=500, save_model_steps=3, wait_after_save_model_ratio=0)
    with pytest.raises(RuntimeError, match="Best model"):
        make_worker(cfg).load_model()
    best = save_best(cfg)
    clock = Clock()
    w = make_worker(cfg, clock)
    assert w.load_model() == cfg.resource.model_best_blob_path and np.array_equal(w.trainer.w, best)
    G.write_play_files(cfg.resource.play_data_dir, "a")      # 480 records: below min_data_size_to_learn
    real_sleep = w.sleep

    def sleep(s):
        real_sleep(s)
        if len(clock.sleeps) == 1:
            G.write_play_files(cfg.resource.play_data_dir, "b")
    w.sleep = sleep
    total = w.training(max_epochs=3)
    assert clock.sleeps[0] == O.WAIT_SEC
    assert total == (960 // 256) * 3 and len(w.trainer.steps) == 4 * 3          # 4 batches per epoch (the last one partial)
    assert all(lr == O.INITIAL_LR for _, lr in w.trainer.steps)
    ng = cfg.resource.next_generation_model_dir
    dirs = sorted(os.listdir(ng))
    assert len(dirs) == 4 and all(d.startswith("model_") for d in dirs)          # saves after batches 3, 6, 9, 12
    assert all(os.listdir(os.path.join(ng, d)) == [NEXT_GENERATION_BLOB] for d in dirs)
    newest = np.load(newest_next_generation_blob(cfg))
    assert np.allclose(newest, best + 12, atol=1e-5)
    # a new worker continues from the newest next-generation model
    w2 = make_worker(cfg)
    assert w2.load_model() == os.path.join(ng, dirs[-1], NEXT_GENERATION_BLOB)
    # the evaluator's remove_model leaves nothing behind
    for d in dirs:
        EvaluateWorker(cfg).remove_model(os.path.join(ng, d))
    assert os.listdir(ng) == []


def test_save_never_exposes_an_incomplete_model_directory(tmp_path, monkeypatch):
    cfg = make_config(tmp_path)
    w = make_worker(cfg)
    w.trainer.load_blob(save_best(cfg))
    seen = []
    real_save = np.save

    def save(path, arr):
        seen.append(sorted(os.listdir(cfg.resource.next_generation_model_dir)))   # while the blob is being written
        real_save(path, arr)
    monkeypatch.setattr(np, "save", save)
    final = w.save_current_model()
    assert seen and not any(n.startswith("model_") for n in seen[0])
    assert os.listdir(cfg.resource.next_generation_model_dir) == [os.path.basename(final)]
