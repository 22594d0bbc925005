"""Mirror of the reference's trainer (worker/optimize.py:25-255, the ``opt`` worker) on the device trainer
(``reversi_zero_b200.train.Trainer``, csrc/rz_train.cu).

Same host decisions as ``OptimizeWorker`` / ``PerStepCallback``: which play-data files are loaded and unloaded, the
``min_data_size_to_learn`` wait, ``decide_learning_rate`` (``lr_schedules`` and the ``.force-lr`` file), the step count
``(N // batch_size) * epochs`` per ``train_epoch``, the save cadence (every ``save_model_steps`` batches, partial ones
included, then a sleep of ``wait_after_save_model_ratio`` x the time since the last one) and the deletion of trained files.

Differences, all on the data path:
  * the training data comes from the ``play_*.rzrows`` twin of every ``play_*.json`` (``b200.write_play_rows``), expanded
    on the device by ``rz_ingest_dev``; the JSON files hold policies rather than visit counts and cannot be converted, so
    a JSON file whose twin does not appear stops the worker with a hint.  With ``b200.train_from_json`` the worker
    instead parses every ``play_*.json`` itself on the device (``rz_ingest_json_dev``) and ignores the twins; as in the
    reference, a file that does not parse (one still being written) is logged and retried at the next load;
  * each epoch runs ceil(N / batch_size) batches of a permutation drawn from the worker's own seeded generator (Keras uses
    numpy's global RNG);
  * a model is saved as ``next_generation/model_<ts>/model_weight.rzblob.npy`` only, built in a directory whose name does
    not match ``model_*`` and renamed into place, so self-play's reload and the evaluator never see a half-written model;
  * momentum lives in device memory only (the reference does not persist it either);
  * with ``b200.train_devices`` (a list of CUDA ordinals) each batch is trained across those devices by one data-parallel
    trainer, bit for bit as on one device; the dataset lives on the first of them.
"""
import os
import time
from collections import Counter
from datetime import datetime
from glob import glob
from logging import getLogger

from . import ingest
from .self_play import NEXT_GENERATION_BLOB, blob_path_of

logger = getLogger(__name__)

# TrainerConfig (config.py:169-184)
TRAINER_DEFAULTS = dict(wait_after_save_model_ratio=1, batch_size=256, min_data_size_to_learn=100000, epoch_to_checkpoint=1,
                        start_total_steps=0, save_model_steps=200, use_tensorboard=True, logging_per_steps=100,
                        delete_self_play_after_number_of_training=0,
                        lr_schedules=[(0, 0.01), (150000, 0.001), (300000, 0.0001)])
INITIAL_LR = 1e-2        # SGD(lr=1e-2, momentum=0.9), worker/optimize.py:84
WAIT_SEC = 10            # sleep while the dataset is too small, :63
ROWS_GRACE_SEC = 60      # self-play writes the JSON file first and its rows twin right after it


def trainer_field(config, name):
    """``config.trainer.<name>`` with the reference's default; ``config.trainer`` may be a dict (the YAML section kept as
    it is), an object with attributes (the reference's own Config) or absent."""
    tr = getattr(config, "trainer", None)
    default = TRAINER_DEFAULTS[name]
    if isinstance(tr, dict):
        return tr.get(name, default)
    return getattr(tr, name, default) if tr is not None else default


def start(config):
    return OptimizeWorker(config).start()


class PerStepCallback:
    """worker/optimize.py:238-255: ``callback`` after every ``per_step``-th batch, then a sleep of
    ``wait_after_save_model_ratio`` x the time since the previous sleep."""

    def __init__(self, per_step, callback, wait_after_save_model_ratio=None, sleep=time.sleep, clock=time.time):
        self.per_step = per_step
        self.step = 0
        self.callback = callback
        self.wait_after_save_model_ratio = wait_after_save_model_ratio
        self.sleep, self.clock = sleep, clock
        self.last_wait_time = clock()

    def on_batch_end(self, batch=None, logs=None):
        self.step += 1
        if self.step % self.per_step == 0:
            self.callback()
            self.wait()

    def wait(self):
        if self.wait_after_save_model_ratio:
            time_spent = self.clock() - self.last_wait_time
            self.sleep(time_spent * self.wait_after_save_model_ratio)
            self.last_wait_time = self.clock()


class OptimizeWorker:
    def __init__(self, config, device=0, trainer=None, to_tensors=None, sleep=time.sleep, clock=time.time, seed=0,
                 read_json=None, trainer_cls=None):
        """``trainer`` (an object with load_blob / step / blob, default ``trainer_cls(model_config, max_batch=...,
        device=..., devices=b200.train_devices)`` with ``trainer_cls`` = ``train.Trainer``), ``to_tensors`` (rows ->
        (states, policy, z) tensors, default ``ingest.to_training_tensors`` on ``device``) and ``read_json`` (a
        play_*.json path -> the same tensors, default ``ingest.read_play_json`` on ``device``) can be replaced, e.g. by
        stand-ins in host-only tests."""
        self.config = config
        # a data-parallel trainer's dataset lives on its primary, devices[0]
        self.train_devices = getattr(getattr(config, "b200", None), "train_devices", None)
        self.device = self.train_devices[0] if self.train_devices else device
        self.trainer = trainer
        self.trainer_cls = trainer_cls
        self.to_tensors = to_tensors or (lambda rows, tau1, ctt: ingest.to_training_tensors(rows, tau1, ctt, self.device))
        self.read_json = read_json or (lambda path: ingest.read_play_json(path, self.device))
        # the source of the training data: JSON can come from writers whose config this process cannot see
        self.train_from_json = bool(getattr(getattr(config, "b200", None), "train_from_json", False))
        self.sleep, self.clock = sleep, clock
        self.seed = seed
        self.generator = None
        self.loaded_filenames = set()
        self.loaded_data = {}
        self.training_count_of_files = Counter()
        self.missing_rows_since = {}
        self.dataset = None
        self.lr = INITIAL_LR
        self.last_loss = None
        self.saved_model_dirs = []

    def start(self, max_epochs=None):
        self.load_model()
        return self.training(max_epochs)

    def training(self, max_epochs=None):
        """worker/optimize.py:43-67; returns total_steps after ``max_epochs`` calls of train_epoch (None = forever)"""
        total_steps = trainer_field(self.config, "start_total_steps")
        callback = PerStepCallback(trainer_field(self.config, "save_model_steps"), self.save_current_model,
                                   trainer_field(self.config, "wait_after_save_model_ratio"), self.sleep, self.clock)
        epochs_done = 0
        while max_epochs is None or epochs_done < max_epochs:
            self.load_play_data()
            if self.dataset_size < trainer_field(self.config, "min_data_size_to_learn"):
                logger.info(f"dataset_size={self.dataset_size} is less than {trainer_field(self.config, 'min_data_size_to_learn')}")
                self.sleep(WAIT_SEC)
                continue
            self.update_learning_rate(total_steps)
            total_steps += self.train_epoch(trainer_field(self.config, "epoch_to_checkpoint"), callback)
            self.count_up_training_count_and_delete_self_play_data_files()
            epochs_done += 1
        return total_steps

    def train_epoch(self, epochs, callback):
        """Keras fit(shuffle=True): every epoch a permutation, ceil(N / B) batches, the last one partial"""
        import torch
        batch_size = trainer_field(self.config, "batch_size")
        states, policy, z = self.dataset
        n = states.shape[0]
        if self.generator is None:
            self.generator = torch.Generator(device=states.device).manual_seed(self.seed)
        for _ in range(epochs):
            perm = torch.randperm(n, generator=self.generator, device=states.device).to(torch.int32)
            for i in range(0, n, batch_size):
                self.last_loss = self.trainer.step(states, policy, z, perm[i:i + batch_size], self.lr)
                callback.on_batch_end()
        return (n // batch_size) * epochs

    def update_learning_rate(self, total_steps):
        lr = self.decide_learning_rate(total_steps)
        if lr:
            self.lr = lr

    def decide_learning_rate(self, total_steps):
        """worker/optimize.py:100-116"""
        ret = None
        path = self.config.resource.force_learing_rate_file
        if os.path.exists(path):
            try:
                with open(path, "rt") as f:
                    ret = float(str(f.read()).strip())
                    if ret:
                        return ret
            except ValueError:
                pass
        for step, lr in trainer_field(self.config, "lr_schedules"):
            if total_steps >= step:
                ret = lr
        return ret

    # -- model files ------------------------------------------------------------------------------------------------
    def _next_generation_dirs(self):
        rc = self.config.resource
        return sorted(glob(os.path.join(rc.next_generation_model_dir, rc.next_generation_model_dirname_tmpl % "*")))

    def load_model(self):
        """worker/optimize.py:147-163: the newest next-generation model, else the best model, else an error"""
        import numpy as np
        dirs = self._next_generation_dirs()
        if dirs:
            path = os.path.join(dirs[-1], NEXT_GENERATION_BLOB)
            if not os.path.exists(path):
                raise RuntimeError(f"{dirs[-1]} has no {NEXT_GENERATION_BLOB}: export its Keras weights with "
                                   f"tools/export_keras_weights.py (INTEGRATION.md section 4)")
        else:
            path = blob_path_of(self.config)
            if not os.path.exists(path):
                raise RuntimeError(f"Best model can not loaded! ({path} does not exist)")
        if self.trainer is None:
            from ..train import Trainer
            self.trainer = (self.trainer_cls or Trainer)(self.config.model, max_batch=trainer_field(self.config, "batch_size"),
                                                         device=self.device, devices=self.train_devices)
        self.trainer.load_blob(np.load(path))
        logger.debug(f"loaded model from {path}")
        return path

    def save_current_model(self):
        """worker/optimize.py:118-125, blob only: written into a directory that no ``model_*`` glob matches, then renamed"""
        import numpy as np
        rc = self.config.resource
        model_id = datetime.now().strftime("%Y%m%d-%H%M%S.%f")
        final = os.path.join(rc.next_generation_model_dir, rc.next_generation_model_dirname_tmpl % model_id)
        tmp = os.path.join(rc.next_generation_model_dir, f".incomplete-{model_id}")
        os.makedirs(tmp)
        np.save(os.path.join(tmp, NEXT_GENERATION_BLOB), self.trainer.blob())
        os.rename(tmp, final)
        self.saved_model_dirs.append(final)
        logger.debug(f"saved model to {final}")
        return final

    # -- play data --------------------------------------------------------------------------------------------------
    def _game_data_filenames(self):
        rc = self.config.resource
        return sorted(glob(os.path.join(rc.play_data_dir, rc.play_data_filename_tmpl % "*")))

    @property
    def dataset_size(self):
        return 0 if self.dataset is None else int(self.dataset[0].shape[0])

    def load_play_data(self):
        """worker/optimize.py:165-180"""
        filenames = self._game_data_filenames()
        updated = False
        for filename in filenames:
            if filename in self.loaded_filenames:
                continue
            self.load_data_from_file(filename)
            updated = True
        for filename in self.loaded_filenames - set(filenames):
            self.unload_data_of_file(filename)
            updated = True
        if updated:
            self.dataset = self.collect_all_loaded_data()

    def load_data_from_file(self, filename):
        if self.train_from_json:  # worker/optimize.py:182-189: a file that does not parse stays unloaded and is retried
            try:
                self.loaded_data[filename] = self.read_json(filename)
                self.loaded_filenames.add(filename)
            except Exception as e:
                logger.warning(str(e))
            return
        rows_path = ingest.rows_path_of(filename)
        if not os.path.exists(rows_path):
            first = self.missing_rows_since.setdefault(filename, self.clock())
            if self.clock() - first >= ROWS_GRACE_SEC:
                raise RuntimeError(f"{filename} has no {os.path.basename(rows_path)} next to it: the device trainer reads the "
                                   f"compact play rows, which self-play writes with b200.write_play_rows = True "
                                   f"(INTEGRATION.md section 3b); JSON play data holds policies, not visit counts")
            return
        self.missing_rows_since.pop(filename, None)
        try:
            rows, tau1, ctt = ingest.read_play_rows(rows_path)
            self.loaded_data[filename] = self.to_tensors(rows, tau1, ctt)
            self.loaded_filenames.add(filename)
        except Exception as e:
            logger.warning(str(e))

    def unload_data_of_file(self, filename):
        self.loaded_filenames.remove(filename)
        self.loaded_data.pop(filename, None)
        self.training_count_of_files.pop(filename, None)

    def collect_all_loaded_data(self):
        import torch
        parts = [d for d in self.loaded_data.values() if d[0].shape[0]]
        if not parts:
            return None
        return tuple(torch.cat([p[i] for p in parts]) for i in range(3))

    def count_up_training_count_and_delete_self_play_data_files(self):
        """worker/optimize.py:199-213; the rows twin goes with its JSON file"""
        limit = trainer_field(self.config, "delete_self_play_after_number_of_training")
        if not limit:
            return
        for filename in self.loaded_filenames:
            self.training_count_of_files[filename] += 1
            if self.training_count_of_files[filename] >= limit:
                for victim in (filename, ingest.rows_path_of(filename)):
                    if os.path.exists(victim):
                        try:
                            os.remove(victim)
                        except OSError as e:
                            logger.warning(e)
