"""Trainer-side ingest (SURVEY 8(f).4): what ``OptimizeWorker.load_play_data`` / ``convert_to_training_data``
(worker/optimize.py:165-231) do with ``play_*.json`` -- here from the compact row files the self-play worker can
write next to them (``play_*.rzrows``, 280 bytes per recorded ply instead of ~5 KB of JSON per ply), expanded to
training arrays on the device by ``rz_ingest`` (csrc/rz_ingest.cu).  No CPU fallback.

    rows, tau1, ctt = read_play_rows("data/play_data/play_20260922-101500.123456.rzrows")
    states, policy, z = to_training_arrays(rows, tau1, ctt)              # numpy, as the reference trainer holds them
    states_d, policy_d, z_d = to_training_tensors(rows, tau1, ctt, 0)    # torch tensors on cuda:0 for a device-side trainer

and from the ``play_*.json`` text itself, parsed on the device by ``rz_ingest_json_dev`` (csrc/rz_ingest_json.cu), for
play data without a rows twin (the reference's own self-play, or this engine with write_play_rows off):

    states_d, policy_d, z_d = read_play_json("data/play_data/play_20260922-101500.123456.json", 0)
    states, policy, z = read_play_json_host(path)                       # numpy, through the host twin of the parser
"""
import ctypes as C
import os
from glob import glob

import numpy as np

from .. import _cabi

ROW_DTYPE = np.dtype([("own", "<u8"), ("enemy", "<u8"), ("n_visit", "<i4", (64,)), ("z", "<i4"), ("pad", "<i4")])
assert ROW_DTYPE.itemsize == C.sizeof(_cabi.PlayRow) == 280

ROWS_SUFFIX = ".rzrows"
RZ_EINVAL, RZ_ECAPACITY = -1, -5   # include/rz_engine.h


def rows_path_of(json_path):
    """play_<ts>.json -> play_<ts>.rzrows (not matched by the trainer's ``play_*.json`` glob, lib/data_helper.py:11-14)."""
    return os.path.splitext(json_path)[0] + ROWS_SUFFIX


def write_play_rows(path, games, n_games, plies, save_policy_of_tau_1=True, change_tau_turn=4):
    """games / plies: ctypes arrays as returned by Engine.poll_raw(); same games and order as write_play_data."""
    n = C.c_size_t()
    _cabi.check(_cabi.lib().rz_write_play_rows(path.encode(), games, n_games, plies, int(bool(save_policy_of_tau_1)),
                                                int(change_tau_turn), C.byref(n)), "rz_write_play_rows")
    return n.value


def read_play_rows(path):
    """-> (rows: structured numpy array of ROW_DTYPE, save_policy_of_tau_1: bool, change_tau_turn: int)"""
    L = _cabi.lib()
    n, tau1, ctt = C.c_size_t(), C.c_int(), C.c_int()
    _cabi.check(L.rz_read_play_rows(path.encode(), None, 0, C.byref(n), C.byref(tau1), C.byref(ctt)), "rz_read_play_rows")
    rows = np.zeros(n.value, ROW_DTYPE)
    if n.value:
        _cabi.check(L.rz_read_play_rows(path.encode(), rows.ctypes.data_as(C.c_void_p), n.value, C.byref(n), None, None), "rz_read_play_rows")
    return rows, bool(tau1.value), int(ctt.value)


def make_rows(own, enemy, n_visit, z):
    rows = np.zeros(len(own), ROW_DTYPE)
    rows["own"], rows["enemy"], rows["n_visit"], rows["z"] = own, enemy, n_visit, z
    return rows


def to_training_arrays(rows, save_policy_of_tau_1=True, change_tau_turn=4):
    """numpy twin of convert_to_training_data: (states uint8 [N,2,8,8], policy float32 [N,64], z float32 [N]), N = 8 * rows."""
    rows = np.ascontiguousarray(rows, ROW_DTYPE)
    n = len(rows)
    states = np.empty((8 * n, 2, 8, 8), np.uint8)
    policy = np.empty((8 * n, 64), np.float32)
    z = np.empty((8 * n,), np.float32)
    _cabi.check(_cabi.lib().rz_ingest(rows.ctypes.data_as(C.c_void_p), n, int(bool(save_policy_of_tau_1)), int(change_tau_turn),
                                       states.ctypes.data_as(_cabi.u8p), policy.ctypes.data_as(_cabi.f32p), z.ctypes.data_as(_cabi.f32p)),
                "rz_ingest")
    return states, policy, z


def to_training_tensors(rows, save_policy_of_tau_1=True, change_tau_turn=4, device=0):
    """Rows -> torch tensors that stay on the device (one H2D copy of the compact rows, the expansion happens in HBM)."""
    import torch
    dev = torch.device("cuda", device)
    rows = np.ascontiguousarray(rows, ROW_DTYPE)
    n = len(rows)
    with torch.cuda.device(dev):
        d_rows = torch.from_numpy(rows.view(np.uint8).reshape(-1)).to(dev)
        states = torch.empty((8 * n, 2, 8, 8), dtype=torch.uint8, device=dev)
        policy = torch.empty((8 * n, 64), dtype=torch.float32, device=dev)
        z = torch.empty((8 * n,), dtype=torch.float32, device=dev)
        _cabi.check(_cabi.lib().rz_ingest_dev(d_rows.data_ptr(), n, int(bool(save_policy_of_tau_1)), int(change_tau_turn), states.data_ptr(),
                                               policy.data_ptr(), z.data_ptr(), torch.cuda.current_stream().cuda_stream), "rz_ingest_dev")
    return states, policy, z


class PlayJsonError(_cabi.RzError):
    """A play_*.json file that is not an array of [[own, enemy], [p0..p63], z] records (truncated, for instance: the
    reference's self-play writes its files in place); ``offset`` is the byte offset of the first error."""

    def __init__(self, msg, offset):
        super().__init__(msg)
        self.offset = offset


def _ingest_json(call, outputs, what):
    """Runs ``call(capacity, pointers, n, off)`` twice -- once to count the records, once into outputs of that size --
    and returns the three arrays; ``outputs(n)`` allocates them and returns (arrays, pointers)."""
    n, off = C.c_size_t(), C.c_size_t()
    rc = call(0, (None, None, None), n, off)
    arrays = None
    if rc == RZ_ECAPACITY:
        arrays, ptrs = outputs(n.value)
        rc = call(n.value, ptrs, n, off)
    if rc == RZ_EINVAL and off.value != C.c_size_t(-1).value:
        msg = _cabi.lib().rz_last_error()
        raise PlayJsonError(f"{what}: {msg.decode() if msg else ''}", off.value)
    _cabi.check(rc, what)
    return arrays if arrays is not None else outputs(0)[0]


def parse_play_json_host(text):
    """Host twin of the device parser (same grammar and conversion, csrc/rz_json_parse.cuh): play_*.json bytes ->
    (states uint8 [N,2,8,8], policy float32 [N,64], z float32 [N]) numpy arrays, one row per JSON record."""
    text = bytes(text)
    buf = C.create_string_buffer(text, len(text))

    def outputs(n):
        arrays = (np.empty((n, 2, 8, 8), np.uint8), np.empty((n, 64), np.float32), np.empty((n,), np.float32))
        return arrays, tuple(a.ctypes.data for a in arrays)

    def call(cap, ptrs, n, off):
        return _cabi.lib().rz_ingest_json_host(buf, len(text), cap, *ptrs, C.byref(n), C.byref(off))

    return _ingest_json(call, outputs, "rz_ingest_json_host")


def read_play_json_host(path):
    with open(path, "rb") as f:
        return parse_play_json_host(f.read())


def parse_play_json(text, device=0):
    """play_*.json bytes -> (states, policy, z) torch tensors on cuda:``device``, parsed on the device by
    rz_ingest_json_dev (csrc/rz_ingest_json.cu); what json.load + convert_to_training_data give, rounded to float32."""
    import torch
    dev = torch.device("cuda", device)
    text = bytes(text)
    with torch.cuda.device(dev):
        d_text = torch.frombuffer(bytearray(text), dtype=torch.uint8).to(dev) if text else torch.empty(0, dtype=torch.uint8, device=dev)
        stream = torch.cuda.current_stream().cuda_stream

        def outputs(n):
            arrays = (torch.empty((n, 2, 8, 8), dtype=torch.uint8, device=dev), torch.empty((n, 64), dtype=torch.float32, device=dev),
                      torch.empty((n,), dtype=torch.float32, device=dev))
            return arrays, tuple(a.data_ptr() for a in arrays)

        def call(cap, ptrs, n, off):
            return _cabi.lib().rz_ingest_json_dev(d_text.data_ptr() if len(text) else None, len(text), cap, *ptrs, C.byref(n),
                                                  C.byref(off), stream)

        return _ingest_json(call, outputs, "rz_ingest_json_dev")


def read_play_json(path, device=0):
    """A play_*.json file -> (states uint8 [N,2,8,8], policy float32 [N,64], z float32 [N]) tensors on cuda:``device``;
    raises PlayJsonError (with the byte offset) if the file is malformed or incomplete."""
    with open(path, "rb") as f:
        return parse_play_json(f.read(), device)


def load_play_data_dir(play_data_dir, device=0):
    """All row files of a play_data directory (the trainer's ``load_play_data``, worker/optimize.py:165-180) as one
    device-resident dataset: (states, policy, z) torch tensors, files in sorted order like get_game_data_filenames."""
    import torch
    parts = []
    for path in sorted(glob(os.path.join(play_data_dir, "play_*" + ROWS_SUFFIX))):
        rows, tau1, ctt = read_play_rows(path)
        if len(rows):
            parts.append(to_training_tensors(rows, tau1, ctt, device))
    if not parts:
        return None
    return tuple(torch.cat([p[i] for p in parts]) for i in range(3))
