"""Mirror of the reference's ``ReversiSolver`` (lib/alt/reversi_solver_cython.pyx:32-61, imported by
agent/player.py:15) over the device solvers: ``solve(black, white, next_player, timeout, exactly) -> (move, score)`` or
``(None, None)``.  ``solve_batch`` solves many positions in one launch of the lane solver (csrc/rz_solver.cuh, up to 12
empties); ``solve_deep_batch`` solves exact positions up to 30 empties one after another, each with the whole device
(csrc/rz_solver_deep.cu), which keeps a transposition table of proven bounds on the device across calls.
``ReversiSolver.solve_moves`` gives the value of every root move (NBoard's exact hints): ``lane_move_values`` up to 12
empties, ``solve_moves`` (one forest per round over all open moves) beyond."""
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


def solve_moves(own, enemy, n_best=0, timeout=30.0, stop=None, on_bounds=None, stats=False):
    """Bounds on the value of every legal move of (own, enemy) (own to move, up to 30 empties) with the whole device
    (rz_solve_deep_moves) -> {square: (lo, hi)} in the mover's frame, {} with no legal move or more than 30 empties; with
    stats=True also the stats dict of solve_deep_batch (`probes` counts forests).  On return every move whose value is
    at least the n_best-th best value (n_best 0: every move) has lo == hi, and every other move has hi below that value.
    A timeout (seconds) or `stop` (a ``ctypes.c_int32`` another thread may set to nonzero) ends the call within one slice
    with the bounds proven so far, which always hold.  on_bounds({square: (lo, hi)}) is called on this thread after
    every round of the solve."""
    lo, hi = np.zeros(64, np.int8), np.zeros(64, np.int8)
    legal = C.c_uint64(0)
    st = _cabi.DeepSolveStats()

    def as_dict(lo_p, hi_p):
        return {s: (int(lo_p[s]), int(hi_p[s])) for s in range(64) if legal.value >> s & 1}

    # the callback object lives until the call returns
    cb = _cabi.DeepMovesCallback(lambda lo_p, hi_p, _user: on_bounds(as_dict(lo_p, hi_p))) if on_bounds else \
        _cabi.DeepMovesCallback()
    # `legal` is written before the first round, so the callback can read it
    _cabi.check(_cabi.lib().rz_solve_deep_moves(int(own), int(enemy), int(n_best), float(timeout),
                                                 C.byref(stop) if stop is not None else None, lo.ctypes.data_as(_cabi.i8p),
                                                 hi.ctypes.data_as(_cabi.i8p), C.byref(legal), cb, None, C.byref(st)),
                "rz_solve_deep_moves")
    out = as_dict(lo, hi)
    if not stats:
        return out
    return out, {k: getattr(st, k) for k, _ in _cabi.DeepSolveStats._fields_ if k != "pad"}


def lane_move_values(own, enemy):
    """The exact value of every legal move of (own, enemy) (own to move, at most 12 empties) from one lane-solver launch
    over the children -> {square: (value, value)} in the mover's frame.  A child whose mover (the opponent) has a move
    is solved in its frame and negated; after a forced pass of the opponent the position after the pass is solved; a
    move that ends the game is worth its disc difference (empties not awarded)."""
    from .bitboard import find_correct_moves, calc_flip, bit_count
    legal = find_correct_moves(own, enemy)
    out, kids = {}, []   # kids: (square, sign, own, enemy) to solve
    for s in range(64):
        if not legal >> s & 1:
            continue
        fl = calc_flip(s, own, enemy)
        o2, e2 = own | fl | (1 << s), enemy ^ fl
        if find_correct_moves(e2, o2):
            kids.append((s, -1, e2, o2))
        elif find_correct_moves(o2, e2):
            kids.append((s, 1, o2, e2))
        else:
            v = bit_count(o2) - bit_count(e2)
            out[s] = (v, v)
    if kids:
        _, score = solve_batch(np.array([k[2] for k in kids], np.uint64), np.array([k[3] for k in kids], np.uint64), True)
        for (s, sign, _, _), sc in zip(kids, score):
            out[s] = (sign * int(sc), sign * int(sc))
    return dict(sorted(out.items()))


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

    def solve_moves(self, black, white, next_player, n_best=0, timeout=30, stop=None, on_bounds=None):
        """The value of every legal move -> {square: (lo, hi)} in the mover's frame, routed like `solve`'s exact
        requests: up to 12 empties every move exact from one lane-solver launch (`timeout`, `stop` and `on_bounds` unused),
        13..max_empties the deep solver's solve_moves with its n_best contract; None beyond max_empties."""
        p = getattr(next_player, "value", next_player)
        own, enemy = (black, white) if p == 1 else (white, black)
        empties = 64 - bin(int(own) | int(enemy)).count("1")
        if empties <= LANE_MAX_EMPTIES:
            return lane_move_values(own, enemy)
        if empties <= self.max_empties:
            return solve_moves(own, enemy, n_best, timeout, stop, on_bounds)
        return None
