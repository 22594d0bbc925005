"""Handle of the device trainer (rz_trainer_* in include/rz_engine.h): one SGD step of the policy/value network per call
on a device-resident dataset (what ``worker.ingest.to_training_tensors`` returns), in the reference's Keras semantics
(worker/optimize.py:73-86, agent/model.py:28-72,104-110).  The weights exchanged are the float32 blob ``Net`` loads.

    tr = Trainer(model_config, max_batch=256)
    tr.load_blob(blob)
    loss = tr.step(states, policy, z, index, lr)   # index: int32 CUDA tensor of record numbers (a slice of a permutation)
    net.load_blob_dev(tr.blob_dev())

``Trainer(model_config, max_batch, devices=[0, 1, 2, 3])`` trains one batch across several devices (a data-parallel
group, rz_trainer_create_group): the same calls, the dataset and index on ``devices[0]``, and exactly the bits of the
one-device step.
"""
import ctypes as C

import numpy as np

from . import _cabi
from .agent import model as M

MOMENTUM = 0.9      # SGD(momentum=0.9), worker/optimize.py:84
BN_MOMENTUM = 0.99  # Keras BatchNormalization default
# ops of Trainer.debug_conv (RZ_TRAIN_CONV* in include/rz_engine.h)
CONV0_FWD, CONV_FWD, CONV_DGRAD, CONV_WGRAD, CONV0_WGRAD = 0, 1, 2, 3, 4
# tensors of Trainer.debug_tensor, in RZ_TRAIN_T_* order (include/rz_engine.h)
DEBUG_TENSORS = ("x0", "y", "a", "stats", "stat", "hc", "ah", "dh", "dyh", "hp", "hv", "dl", "h1", "dh1", "dv", "lp", "lv",
                 "loss_pv", "g", "dy", "dz")


class Trainer:
    def __init__(self, model_config, max_batch, device=0, devices=None, momentum=MOMENTUM, bn_momentum=BN_MOMENTUM, l2_reg=None):
        """``devices``: a list of CUDA ordinals (repeats allowed) builds a data-parallel group whose primary is
        ``devices[0]``; ``device`` is then ignored.  None trains on ``device`` alone."""
        import torch
        if devices is not None:
            devices = list(devices)
            if not all(isinstance(d, (int, np.integer)) and not isinstance(d, bool) for d in devices):
                raise TypeError(f"devices must be a list of CUDA ordinals, got {devices!r}")
            devices = [int(d) for d in devices]
        self.mc = model_config
        self.devices = devices
        self.max_batch = int(max_batch)
        self._last_batch = None
        self._h = C.c_void_p()
        ncfg = _cabi.NetCfg(model_config.cnn_filter_num, model_config.res_layer_num, model_config.value_fc_size,
                            model_config.cnn_filter_size)
        tcfg = _cabi.TrainCfg(self.max_batch, momentum, model_config.l2_reg if l2_reg is None else l2_reg, bn_momentum)
        if devices is None:
            _cabi.check(_cabi.lib().rz_trainer_create(C.byref(ncfg), C.byref(tcfg), device, C.byref(self._h)), "rz_trainer_create")
        else:
            ords = (C.c_int32 * max(len(devices), 1))(*devices)
            _cabi.check(_cabi.lib().rz_trainer_create_group(C.byref(ncfg), C.byref(tcfg), ords, len(devices), C.byref(self._h)),
                        "rz_trainer_create_group")
        self.device = torch.device("cuda", devices[0] if devices else device)
        n = C.c_size_t()
        _cabi.check(_cabi.lib().rz_trainer_blob_size(self._h, C.byref(n)), "rz_trainer_blob_size")
        self.blob_floats = n.value
        assert self.blob_floats == M.blob_size(model_config)

    def _stream(self):
        import torch
        return torch.cuda.current_stream(self.device).cuda_stream

    def load_blob(self, blob):
        """host float32 blob; also zeroes the momentum"""
        blob = np.ascontiguousarray(blob, dtype=np.float32)
        _cabi.check(_cabi.lib().rz_trainer_load_weights(self._h, blob.ctypes.data_as(_cabi.f32p), blob.size), "rz_trainer_load_weights")

    def load_blob_dev(self, tensor):
        """float32 CUDA tensor holding the blob; also zeroes the momentum"""
        _cabi.check(_cabi.lib().rz_trainer_load_weights_dev(self._h, C.c_void_p(tensor.data_ptr()), tensor.numel(), self._stream()),
                    "rz_trainer_load_weights_dev")

    def blob_dev(self):
        """current weights as a float32 CUDA tensor (blob layout)"""
        import torch
        out = torch.empty(self.blob_floats, dtype=torch.float32, device=self.device)
        _cabi.check(_cabi.lib().rz_trainer_weights_dev(self._h, C.c_void_p(out.data_ptr()), out.numel(), self._stream()),
                    "rz_trainer_weights_dev")
        return out

    def blob(self):
        return self.blob_dev().cpu().numpy()

    def step(self, states, policy, z, index, lr):
        """One step on records ``index`` of (states uint8 [N,2,8,8], policy float32 [N,64], z float32 [N]), all CUDA tensors.
        Returns a new device tensor [total, policy, value] with this batch's loss (NaN and no update if an index is out of
        range); reading it is the only synchronisation."""
        import torch
        for t, dt in ((states, torch.uint8), (policy, torch.float32), (z, torch.float32), (index, torch.int32)):
            if t.dtype != dt or not t.is_cuda or not t.is_contiguous():
                raise ValueError(f"expected a contiguous CUDA tensor of {dt}, got {t.dtype} on {t.device}")
        n = states.shape[0]
        if policy.shape != (n, 64) or z.shape != (n,) or tuple(states.shape[1:]) != (2, 8, 8) or index.dim() != 1:
            raise ValueError("expected states [N,2,8,8], policy [N,64], z [N], index [B]")
        loss = torch.empty(3, dtype=torch.float32, device=self.device)
        _cabi.check(_cabi.lib().rz_trainer_step_dev(self._h, C.c_void_p(states.data_ptr()), C.c_void_p(policy.data_ptr()),
                                                     C.c_void_p(z.data_ptr()), n, C.c_void_p(index.data_ptr()), index.numel(),
                                                     float(lr), C.c_void_p(loss.data_ptr()), self._stream()),
                    "rz_trainer_step_dev")
        self._last_batch = index.numel()
        return loss

    def last_grad(self):
        """gradient of the last step's total loss, host float32 blob layout (0 in the moving-statistics slots)"""
        import torch
        out = torch.empty(self.blob_floats, dtype=torch.float32, device=self.device)
        _cabi.check(_cabi.lib().rz_trainer_last_grad_dev(self._h, C.c_void_p(out.data_ptr()), out.numel(), self._stream()),
                    "rz_trainer_last_grad_dev")
        return out.cpu().numpy()

    def replica_state(self, r):
        """test hook: (weights, momentum) of replica ``r`` (0 = the primary) as float32 CUDA tensors on the primary"""
        import torch
        w = torch.empty(self.blob_floats, dtype=torch.float32, device=self.device)
        v = torch.empty_like(w)
        _cabi.check(_cabi.lib().rz_trainer_replica_state_dev(self._h, r, C.c_void_p(w.data_ptr()), C.c_void_p(v.data_ptr()), w.numel(),
                                                             self._stream()), "rz_trainer_replica_state_dev")
        return w, v

    def debug_conv(self, op, x, batch, kernel=None, bias=None, add=None):
        """test hook (rz_trainer_debug_conv_dev): one of the step's convolution GEMMs, CONV_* below, on float32 CUDA
        tensors; x and add are [64 * batch][C], kernel [9][Cin][Cout].  Returns a new tensor: [64 * batch][F] for the
        forward and input-gradient ops, the weight gradient [9][Cin][F] for the two WGRAD ops."""
        import torch
        F = self.mc.cnn_filter_num
        for t in (x, kernel, bias, add):
            if t is not None and (t.dtype != torch.float32 or not t.is_cuda or not t.is_contiguous()):
                raise ValueError(f"expected a contiguous float32 CUDA tensor, got {t.dtype} on {t.device}")
        shape = {CONV_WGRAD: (9, F, F), CONV0_WGRAD: (9, 2, F)}.get(op, (64 * batch, F))
        out = torch.empty(shape, dtype=torch.float32, device=self.device)
        ptr = lambda t: C.c_void_p(t.data_ptr()) if t is not None else None
        _cabi.check(_cabi.lib().rz_trainer_debug_conv_dev(self._h, op, ptr(x), ptr(kernel), ptr(bias), ptr(add), batch, ptr(out),
                                                          self._stream()), "rz_trainer_debug_conv_dev")
        return out

    def debug_keep_backward(self, on):
        """test hook (rz_trainer_debug_keep_backward, single trainers): make the following steps keep every tower layer's
        backward tensors "g", "dy" and "dz" for debug_tensor"""
        _cabi.check(_cabi.lib().rz_trainer_debug_keep_backward(self._h, int(bool(on))), "rz_trainer_debug_keep_backward")

    def debug_tensor(self, name, layer=0):
        """test hook (rz_trainer_debug_tensor_dev, single trainers): a new float32 CUDA tensor holding one intermediate
        tensor of the last step, one of DEBUG_TENSORS, in its natural shape: [64 * B][16] for x0, [64 * B][F] for the
        tower's y, a, g, dy, dz (``layer`` l), [4][F] for stats (slot ``layer``), [blob floats] for stat, [64 * B][3] for
        hc, ah, dh, dyh, [B][128 | 64 | V] for hp, hv, dl, h1, dh1, [B] for dv, lp, lv and [2] for loss_pv."""
        import torch
        if self._last_batch is None:
            raise RuntimeError("debug_tensor: no step has run")
        F, V, B = self.mc.cnn_filter_num, self.mc.value_fc_size, self._last_batch
        shape = {"x0": (64 * B, 16), "stats": (4, F), "stat": (self.blob_floats,), "hp": (B, 128), "hv": (B, 64), "dl": (B, 64),
                 "h1": (B, V), "dh1": (B, V), "dv": (B,), "lp": (B,), "lv": (B,), "loss_pv": (2,)}.get(name)
        if shape is None:
            shape = (64 * B, 3) if name in ("hc", "ah", "dh", "dyh") else (64 * B, F)
        out = torch.empty(shape, dtype=torch.float32, device=self.device)
        _cabi.check(_cabi.lib().rz_trainer_debug_tensor_dev(self._h, DEBUG_TENSORS.index(name), layer, C.c_void_p(out.data_ptr()),
                                                            out.numel(), self._stream()), "rz_trainer_debug_tensor_dev")
        return out

    def close(self):
        if self._h:
            _cabi.lib().rz_trainer_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
