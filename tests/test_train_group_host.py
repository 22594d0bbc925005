"""CPU suite for the data-parallel training group (rz_trainer_create_group, csrc/rz_train.cu): its ABI symbols, the shard
plan restated in Python against the library's host twin, the `b200.train_devices` knob from YAML to the trainer the
`opt` worker builds, and Trainer's argument checks."""
import ctypes as C

import numpy as np
import pytest
import yaml

from reversi_zero_b200 import _cabi, train as T
from reversi_zero_b200.agent import model as M
from reversi_zero_b200.config import create_config
from reversi_zero_b200.worker import optimize as O

NEW_SYMBOLS = ("rz_trainer_create_group", "rz_train_shard_plan_host", "rz_trainer_replica_state_dev")


def test_group_symbols_resolve():
    lib = C.CDLL(_cabi.LIB_PATH)
    for name in NEW_SYMBOLS:
        assert getattr(lib, name, None) is not None, name
        assert name in _cabi.SIGNATURES


def wgrad_per(cin, F, batch):
    """records per weight-gradient split of a convolution with cin input channels (wgrad_splits / launch_wgrad)"""
    tiles = -(-9 * cin // 128) * -(-F // 128)
    return -(-batch // min(-(-264 // tiles), batch))


def shard_plan(F, R, batch, n):
    """the grid of the F->F convolutions' weight-gradient splits (conv0's without residual blocks), its cells dealt out
    as evenly as possible with the larger shares first"""
    per = wgrad_per(F if R else 16, F, batch)
    cells = -(-batch // per)
    q, rem = divmod(cells, n)
    return [min(batch, per * (r * q + min(r, rem))) for r in range(n + 1)], per


_PLAN_OUT = (C.c_int32 * 65)()


def host_plan(F, R, batch, n):
    _cabi.check(_cabi.lib().rz_train_shard_plan_host(F, R, batch, n, _PLAN_OUT), "rz_train_shard_plan_host")
    return _PLAN_OUT[:n + 1]


@pytest.mark.parametrize("R", [0, 1])
def test_shard_plan(R):
    """the library's plan: every batch position in exactly one shard, boundaries on the split grid, cell counts within
    one of each other (the larger first), and equal to this restatement: every B <= 2048, group size <= 8 and trainer
    width"""
    for F in range(16, 257, 16):
        for batch in range(1, 2049):
            for n in range(1, 9):
                b, per = shard_plan(F, R, batch, n)
                assert host_plan(F, R, batch, n) == b, (F, R, batch, n)
                assert b[0] == 0 and b[-1] == batch and all(x <= y for x, y in zip(b, b[1:])), (F, batch, n, b)
                assert all(x % per == 0 or x == batch for x in b), (F, batch, n, b)
                cells = [-(-(y - x) // per) for x, y in zip(b, b[1:])]
                assert max(cells) - min(cells) <= 1 and cells == sorted(cells, reverse=True), (F, batch, n, b)


def test_conv0_split_straddles_a_shard_in_the_documented_case():
    """64 filters, batch 256, three replicas: tower splits of 5 records (52 cells: 18, 17, 17) put a boundary at 175,
    inside conv0's split of records 174-175"""
    b, per = shard_plan(64, 1, 256, 3)
    assert per == 5 and b == [0, 90, 175, 256] and host_plan(64, 1, 256, 3) == b
    assert wgrad_per(16, 64, 256) == 2


class RecordingTrainer:
    made = []

    def __init__(self, model_config, max_batch, device=0, devices=None):
        RecordingTrainer.made.append(dict(max_batch=max_batch, device=device, devices=devices))

    def load_blob(self, blob):
        pass


def test_train_devices_from_yaml_reach_the_trainer(tmp_path):
    cfg = create_config(yaml.safe_load("model: {cnn_filter_num: 16, res_layer_num: 1, value_fc_size: 16}\n"
                                       "trainer: {batch_size: 64}\nb200: {train_devices: [2, 0, 2]}\n"),
                        project_dir=str(tmp_path), data_dir=str(tmp_path / "data"))
    assert cfg.b200.train_devices == [2, 0, 2] and create_config().b200.train_devices is None
    cfg.resource.create_directories()
    np.save(cfg.resource.model_best_blob_path, M.weights_to_blob(cfg.model, M.build_random_weights(cfg.model, 0)))
    RecordingTrainer.made.clear()
    w = O.OptimizeWorker(cfg, trainer_cls=RecordingTrainer)
    w.load_model()
    assert RecordingTrainer.made == [dict(max_batch=64, device=2, devices=[2, 0, 2])]
    assert w.device == 2   # the dataset goes to the primary
    RecordingTrainer.made.clear()
    O.OptimizeWorker(create_config(dict(model=vars(cfg.model), trainer=dict(batch_size=8)), project_dir=str(tmp_path),
                                   data_dir=str(tmp_path / "data")), trainer_cls=RecordingTrainer).load_model()
    assert RecordingTrainer.made == [dict(max_batch=8, device=0, devices=None)]


@pytest.mark.parametrize("devices", [[0, "1"], [0, 1.0], [True], [None]])
def test_trainer_refuses_non_integer_devices(devices):
    with pytest.raises(TypeError, match="CUDA ordinals"):
        T.Trainer(M.ModelConfig(cnn_filter_num=16, res_layer_num=1, value_fc_size=16), max_batch=4, devices=devices)


@pytest.mark.parametrize("devices", [[], [0, 4096], [-1]])
def test_library_refuses_empty_and_invisible_devices(devices):
    with pytest.raises(_cabi.RzError, match="rz_trainer_create_group"):
        T.Trainer(M.ModelConfig(cnn_filter_num=16, res_layer_num=1, value_fc_size=16), max_batch=4, devices=devices)
