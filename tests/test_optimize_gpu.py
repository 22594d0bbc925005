"""The AlphaZero loop on the device, mini configuration, bounded sizes: SelfPlayWorker (with play rows) -> OptimizeWorker
writes a next-generation blob with a new digest -> a running SelfPlayWorker reloads it at its next check ->
EvaluateWorker plays it and removes its directory."""
import glob
import os

import numpy as np
import pytest

from reversi_zero_b200.agent import model as M
from reversi_zero_b200.worker import optimize as O
from reversi_zero_b200.worker.evaluate import EvaluateWorker, NEXT_GENERATION_BLOB
from reversi_zero_b200.worker.self_play import SelfPlayWorker, newest_next_generation_blob
from test_selfplay_worker_gpu import mini_config

pytestmark = pytest.mark.gpu


def test_self_opt_eval_loop_on_the_device(tmp_path):
    cfg = mini_config(tmp_path)
    cfg.b200.write_play_rows = True
    sp = SelfPlayWorker(cfg)
    assert sp.start(max_games=8) >= 8
    best_digest = M.blob_digest(np.load(cfg.resource.model_best_blob_path))
    assert sp.net.digest == best_digest

    cfg.trainer = dict(batch_size=64, min_data_size_to_learn=256, save_model_steps=5, wait_after_save_model_ratio=0)
    ow = O.OptimizeWorker(cfg)
    total = ow.start(max_epochs=1)
    n = ow.dataset_size
    assert n >= 256 and total == n // 64
    assert len(ow.saved_model_dirs) == -(-n // 64) // 5                     # every 5th batch, the partial one included
    loss = ow.last_loss.cpu().numpy()
    assert np.isfinite(loss).all() and loss[0] > loss[1] > 0
    ng = cfg.resource.next_generation_model_dir
    assert sorted(glob.glob(os.path.join(ng, "*"))) == sorted(ow.saved_model_dirs)   # nothing but complete model_* directories
    newest = newest_next_generation_blob(cfg)
    blob = np.load(newest)
    assert blob.dtype == np.float32 and blob.size == M.blob_size(cfg.model) and M.blob_digest(blob) != best_digest

    assert sp.try_reload_model(force_check=True) and sp.net.digest == M.blob_digest(blob)

    cfg.eval = dict(game_num=4, replace_rate=0.55, play_config=dict(simulation_num_per_move=10, thinking_loop=1))
    assert EvaluateWorker(cfg).start(max_models=1) == 1
    assert not os.path.exists(os.path.dirname(newest))                       # played, then removed without leftovers
    assert all(os.listdir(d) == [NEXT_GENERATION_BLOB] for d in glob.glob(os.path.join(ng, "model_*")))
