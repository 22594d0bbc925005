"""Writes what the UNMODIFIED reference trainer's host logic (worker/optimize.py OptimizeWorker / PerStepCallback, imported
through oracle/ref_shims) decides, for tests/test_train_host.py:

  * decide_learning_rate over lr_schedules x total_steps x .force-lr contents (absent, valid, 0, garbage, empty)
  * the step count train_epoch returns for several dataset sizes, batch sizes and epoch counts
  * PerStepCallback's save cadence and the sleeps of wait_after_save_model_ratio under a scripted clock
  * load_play_data / unload / count_up_training_count_and_delete_self_play_data_files over a scripted timeline of
    play_*.json files appearing and vanishing

-> optimize_ref.json.  Run once where the reference checkout exists:

    python tests/golden/make_golden_optimize.py
"""
import json
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "reversi-alpha-zero_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

import oracle.ref_shims.install as shims  # noqa: E402

SCHEDULES = {"default": [(0, 0.01), (150000, 0.001), (300000, 0.0001)], "custom": [(0, 0.02), (10, 0.005)]}
LR_STEPS = [0, 1, 9, 10, 149999, 150000, 299999, 300000, 10 ** 7]
FORCE_TEXTS = [None, "0.005\n", "0", "garbage", "", " 1e-3 "]
EPOCH_CASES = [(1000, 256, 1), (256, 256, 1), (255, 256, 1), (100000, 256, 2), (513, 7, 3), (1, 256, 1)]
CADENCE = dict(per_step=3, ratio=0.5, batches=20, tick=1.5)
# timeline: (action, argument); files are named play_<FILES[k]>.json and hold the fixed games GAMES[k]
FILES = {"a": "20260101-000001.000000", "b": "20260101-000002.000000", "c": "20260101-000003.000000", "d": "20260101-000004.000000"}
GAMES = {"a": [0], "b": [1], "c": [0, 1], "d": [1]}
TIMELINE = [("add", "a"), ("add", "b"), ("load", None), ("count", None), ("add", "c"), ("remove", "a"), ("load", None),
            ("count", None), ("load", None), ("add", "d"), ("load", None), ("count", None), ("count", None), ("load", None)]
DELETE_LIMIT = 2


def write_play_files(play_dir, key):
    """the JSON file and its rows twin of the timeline's file `key` (the fixed games of tests/test_playdata_writer.py)"""
    import test_playdata_writer as T
    from reversi_zero_b200 import engine as E
    from reversi_zero_b200.worker import ingest
    games = [T.fixed_games()[i] for i in GAMES[key]]
    G, P = T.to_ctypes(games)
    path = os.path.join(play_dir, f"play_{FILES[key]}.json")
    E.write_play_data(path, G, len(games), P, True, 4)
    ingest.write_play_rows(ingest.rows_path_of(path), G, len(games), P, True, 4)
    return path


def lr_golden(tmp):
    from reversi_zero.worker.optimize import OptimizeWorker
    force = os.path.join(tmp, ".force-lr")
    out = {}
    for name, sched in SCHEDULES.items():
        for text in FORCE_TEXTS:
            if os.path.exists(force):
                os.remove(force)
            if text is not None:
                with open(force, "wt") as f:
                    f.write(text)
            w = types.SimpleNamespace(config=types.SimpleNamespace(resource=types.SimpleNamespace(force_learing_rate_file=force),
                                                                   trainer=types.SimpleNamespace(lr_schedules=sched)))
            out[f"{name}|{text!r}"] = [OptimizeWorker.decide_learning_rate(w, s) for s in LR_STEPS]
    return out


def epoch_golden():
    from reversi_zero.worker.optimize import OptimizeWorker
    out = []
    for n, b, epochs in EPOCH_CASES:
        w = types.SimpleNamespace(config=types.SimpleNamespace(trainer=types.SimpleNamespace(batch_size=b)),
                                  dataset=(np.zeros((n, 1)), np.zeros((n, 1)), np.zeros(n)),
                                  model=types.SimpleNamespace(model=types.SimpleNamespace(fit=lambda *a, **k: None)))
        out.append([n, b, epochs, OptimizeWorker.train_epoch(w, epochs, [])])
    return out


def cadence_golden():
    import reversi_zero.worker.optimize as ref
    clock = [100.0]
    sleeps, saves = [], []
    ref.time = lambda: clock[0]
    ref.sleep = lambda s: sleeps.append([len(saves), s])
    cb = ref.PerStepCallback(CADENCE["per_step"], lambda: saves.append(batch), CADENCE["ratio"])
    for batch in range(1, CADENCE["batches"] + 1):
        clock[0] += CADENCE["tick"]
        cb.on_batch_end(batch)
    return dict(saves=saves, sleeps=sleeps)


def timeline_golden(tmp):
    from reversi_zero.worker.optimize import OptimizeWorker
    play_dir = os.path.join(tmp, "play_data")
    os.makedirs(play_dir)
    cfg = types.SimpleNamespace(resource=types.SimpleNamespace(play_data_dir=play_dir, play_data_filename_tmpl="play_%s.json"),
                                trainer=types.SimpleNamespace(delete_self_play_after_number_of_training=DELETE_LIMIT))
    w = OptimizeWorker(cfg)
    out = []
    for action, key in TIMELINE:
        if action == "add":
            write_play_files(play_dir, key)
        elif action == "remove":
            for name in os.listdir(play_dir):
                if FILES[key] in name:
                    os.remove(os.path.join(play_dir, name))
        elif action == "load":
            w.load_play_data()
        else:
            w.count_up_training_count_and_delete_self_play_data_files()
        out.append(dict(loaded=sorted(os.path.basename(f) for f in w.loaded_filenames), dataset_size=w.dataset_size,
                        counts={os.path.basename(f): c for f, c in sorted(w.training_count_of_files.items())},
                        json_files=sorted(n for n in os.listdir(play_dir) if n.endswith(".json"))))
    return out


def main():
    assert shims.available(), "reference sources not present"
    shims.install()
    with tempfile.TemporaryDirectory() as tmp:
        golden = dict(lr=lr_golden(tmp), lr_steps=LR_STEPS, epochs=epoch_golden(), cadence=cadence_golden(),
                      timeline=timeline_golden(tmp))
    with open(os.path.join(HERE, "optimize_ref.json"), "w") as f:
        json.dump(golden, f, indent=1)


if __name__ == "__main__":
    main()
