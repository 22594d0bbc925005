"""Mirror of the reference's ``ReversiSolver`` (lib/alt/reversi_solver_cython.pyx:32-61, imported by
agent/player.py:15) over the device solvers: ``solve(black, white, next_player, timeout, exactly) -> (move, score)`` or
``(None, None)``.  ``solve_batch`` solves many positions in one launch of the lane solver (csrc/rz_solver.cuh, up to 12
empties); ``solve_deep_batch`` solves exact positions up to 30 empties one after another, each with the whole device
(csrc/rz_solver_deep.cu), which keeps a transposition table of proven bounds on the device across calls."""
import ctypes as C

import numpy as np

from .. import _cabi

LANE_MAX_EMPTIES = 12   # the lane solver refuses larger positions
DEEP_MAX_EMPTIES = 30   # ... and the deep solver


def solve_batch(own, enemy, exactly):
    """own / enemy: uint64 arrays in the mover's frame; exactly: bool array.  -> (move int8[], score int8[]), move -1 = none."""
    own = np.ascontiguousarray(own, dtype=np.uint64)
    enemy = np.ascontiguousarray(enemy, dtype=np.uint64)
    ex = np.ascontiguousarray(np.broadcast_to(np.asarray(exactly, dtype=np.uint8), own.shape))
    move = np.empty(own.shape, np.int8)
    score = np.empty(own.shape, np.int8)
    _cabi.check(_cabi.lib().rz_solve(own.ctypes.data_as(_cabi.u64p), enemy.ctypes.data_as(_cabi.u64p), ex.ctypes.data_as(_cabi.u8p),
                                      move.ctypes.data_as(_cabi.i8p), score.ctypes.data_as(_cabi.i8p), own.size), "rz_solve")
    return move, score


def solve_deep_batch(own, enemy, timeout=30.0, stats=False, stop=None):
    """Exact solve of each position (uint64 arrays in the mover's frame) with the whole device, one after another;
    `timeout` seconds per position.  -> (move int8[], score int8[]) with move -1 = no legal move, more than 30 empties,
    timed out or stopped; with stats=True also a list of dicts (probes, slices, resplits, leaves, node_steps, seconds).
    stop: a ``ctypes.c_int32`` another thread may set to nonzero to end the call within one slice
    (rz_solve_deep_with_stop); the positions not finished by then answer like a timeout."""
    own = np.ascontiguousarray(own, dtype=np.uint64).reshape(-1)
    enemy = np.ascontiguousarray(enemy, dtype=np.uint64).reshape(-1)
    move = np.empty(own.shape, np.int8)
    score = np.empty(own.shape, np.int8)
    st = (_cabi.DeepSolveStats * max(1, own.size))()
    if stop is None:
        _cabi.check(_cabi.lib().rz_solve_deep(own.ctypes.data_as(_cabi.u64p), enemy.ctypes.data_as(_cabi.u64p),
                                               move.ctypes.data_as(_cabi.i8p), score.ctypes.data_as(_cabi.i8p), own.size,
                                               float(timeout), st), "rz_solve_deep")
    else:
        _cabi.check(_cabi.lib().rz_solve_deep_with_stop(own.ctypes.data_as(_cabi.u64p), enemy.ctypes.data_as(_cabi.u64p),
                                                         move.ctypes.data_as(_cabi.i8p), score.ctypes.data_as(_cabi.i8p), own.size,
                                                         float(timeout), C.byref(stop), st), "rz_solve_deep_with_stop")
    if not stats:
        return move, score
    names = [f for f, _ in _cabi.DeepSolveStats._fields_ if f != "pad"]
    return move, score, [{k: getattr(st[i], k) for k in names} for i in range(own.size)]


def tune_deep(slice_us=0, leaf_target=0, leaf_floor=0):
    """Slice length (us), split leaf target and leaf floor (empties) of the deep solver; 0 restores a default.  The next
    solve starts from an empty transposition table."""
    _cabi.check(_cabi.lib().rz_solve_deep_tune(int(slice_us), int(leaf_target), int(leaf_floor)), "rz_solve_deep_tune")


def deep_table_bytes(nbytes=0):
    """Size of the deep solver's transposition table from its next call on (which starts empty); 0: the default 1 GiB."""
    _cabi.check(_cabi.lib().rz_solve_deep_table(int(nbytes)), "rz_solve_deep_table")


def clear_deep_table():
    """Empty the deep solver's transposition table on the current device and zero its counts."""
    _cabi.check(_cabi.lib().rz_solve_deep_clear(), "rz_solve_deep_clear")


def deep_table_stats():
    """Counts of the transposition table since the last clear: lookups, cutoffs, hints, stores, replaced, merges,
    dropped, occupied (entries now) and bytes."""
    st = _cabi.DeepTableStats()
    _cabi.check(_cabi.lib().rz_solve_deep_table_stats(C.byref(st)), "rz_solve_deep_table_stats")
    return {k: getattr(st, k) for k, _ in _cabi.DeepTableStats._fields_}


class ReversiSolver:
    def __init__(self, max_empties=LANE_MAX_EMPTIES):
        """max_empties: exact requests with 13..max_empties empty squares go to the deep solver with the caller's
        timeout; at the default 12 every request goes to the lane solver, which refuses larger positions."""
        if not LANE_MAX_EMPTIES <= int(max_empties) <= DEEP_MAX_EMPTIES:
            raise ValueError(f"max_empties must be in {LANE_MAX_EMPTIES}..{DEEP_MAX_EMPTIES}, got {max_empties}")
        self.max_empties = int(max_empties)

    def solve(self, black, white, next_player, timeout=30, exactly=False):
        """next_player: Player enum (or its value: 1 black, 2 white).  The lane solver refuses positions with more than
        12 empty squares and ignores `timeout`; the deep solver (exact requests up to `max_empties`) gives up after
        `timeout` seconds.  Both answer a refusal or a timeout with (None, None), like the reference's timeout."""
        p = getattr(next_player, "value", next_player)
        own, enemy = (black, white) if p == 1 else (white, black)
        empties = 64 - bin(int(own) | int(enemy)).count("1")
        if exactly and LANE_MAX_EMPTIES < empties <= self.max_empties:
            mv, sc = solve_deep_batch([own], [enemy], timeout)
        else:
            mv, sc = solve_batch([own], [enemy], [exactly])
        if mv[0] < 0:
            return None, None
        return int(mv[0]), int(sc[0])
