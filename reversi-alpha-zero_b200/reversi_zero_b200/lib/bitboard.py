"""Mirror of the reference's ``reversi_zero.lib.bitboard`` free functions (lib/bitboard.py) over the
C ABI.  Scalar calls use the host twins of the device code (csrc/rz_bitboard.cuh compiled for the
host); the ``*_batch`` functions run the sm_90a K1 kernels on numpy arrays (host buffers) and are
what the parity tests and the microbenchmark exercise."""
import ctypes as C

import numpy as np

from .. import _cabi

BLACK_CHR, WHITE_CHR, EXTRA_CHR = "O", "X", "*"  # lib/bitboard.py:4-6


def find_correct_moves(own, enemy):
    """lib/bitboard.py:53-67"""
    return int(_cabi.lib().rz_find_correct_moves_host(int(own), int(enemy)))


def calc_flip(pos, own, enemy):
    """lib/bitboard.py:70-81"""
    assert 0 <= pos <= 63, f"pos={pos}"
    return int(_cabi.lib().rz_calc_flip_host(int(pos), int(own), int(enemy)))


def flip_vertical(x):
    """lib/bitboard.py:119-125"""
    return int(_cabi.lib().rz_dihedral_host(int(x), 4))


def rotate90(x):
    """lib/bitboard.py:154 (clockwise)"""
    return int(_cabi.lib().rz_dihedral_host(int(x), 1))


def rotate180(x):
    """lib/bitboard.py:158"""
    return int(_cabi.lib().rz_dihedral_host(int(x), 2))


def flip_diag_a1h8(x):
    """lib/bitboard.py:141-151 == rotate90(flip_vertical(x))"""
    return int(_cabi.lib().rz_dihedral_host(int(x), 5))


def dihedral(x, t):
    """flip_vertical if t & 4, then (t & 3) x rotate90 (agent/player.py:166-179, :300-305)."""
    return int(_cabi.lib().rz_dihedral_host(int(x), int(t)))


def bit_count(x):
    """lib/bitboard.py:132"""
    return int(x).bit_count()


def bit_to_array(x, size):
    """lib/bitboard.py:136-138: bit i -> array[i] (uint8)"""
    x = int(x)
    return np.array([(x >> i) & 1 for i in range(size)], dtype=np.uint8)


def dirichlet_noise_of_mask(mask, alpha):
    """lib/bitboard.py:162-171 (host-side helper; the engine draws its root noise on the device)."""
    idx = [i for i in range(64) if (int(mask) >> i) & 1]
    out = np.zeros(64)
    out[idx] = np.random.dirichlet([alpha] * len(idx))
    return out


def board_to_string(black, white, with_edge=True, extra=None):
    """lib/bitboard.py:9-50"""
    extra = extra or 0
    cells = []
    for i in range(64):
        cells.append(BLACK_CHR if (black >> i) & 1 else WHITE_CHR if (white >> i) & 1 else EXTRA_CHR if (extra >> i) & 1 else " ")
    rows = ["".join(cells[y * 8:y * 8 + 8]) for y in range(8)]
    if with_edge:
        return "#" * 10 + "\n" + "".join(f"#{r}#\n" for r in rows) + "#" * 10 + "\n"
    return "".join(r + "\n" for r in rows)


# ---- batched GPU operators (host numpy buffers in / out through the C ABI) -------------------------
def _u64(a):
    return np.ascontiguousarray(a, dtype=np.uint64)


def find_correct_moves_batch(own, enemy):
    own, enemy = _u64(own), _u64(enemy)
    out = np.empty_like(own)
    _cabi.check(_cabi.lib().rz_find_correct_moves(own.ctypes.data_as(_cabi.u64p), enemy.ctypes.data_as(_cabi.u64p),
                                                   out.ctypes.data_as(_cabi.u64p), own.size), "rz_find_correct_moves")
    return out


def calc_flip_batch(pos, own, enemy):
    pos = np.ascontiguousarray(pos, dtype=np.uint8)
    own, enemy = _u64(own), _u64(enemy)
    out = np.empty_like(own)
    _cabi.check(_cabi.lib().rz_calc_flip(pos.ctypes.data_as(_cabi.u8p), own.ctypes.data_as(_cabi.u64p),
                                          enemy.ctypes.data_as(_cabi.u64p), out.ctypes.data_as(_cabi.u64p), own.size),
                "rz_calc_flip")
    return out


def bitsliced_host(own, enemy, pos=None):
    """Host twin of the bit-sliced formulation the batched GPU operators use (rz_bitsliced_host): legal-move masks when
    ``pos`` is None, flip masks otherwise.  For tests; the product path is the GPU."""
    own, enemy = _u64(own), _u64(enemy)
    out = np.empty_like(own)
    p = None if pos is None else np.ascontiguousarray(pos, dtype=np.uint8)
    _cabi.check(_cabi.lib().rz_bitsliced_host(None if p is None else p.ctypes.data_as(_cabi.u8p), own.ctypes.data_as(_cabi.u64p),
                                              enemy.ctypes.data_as(_cabi.u64p), out.ctypes.data_as(_cabi.u64p), own.size),
                "rz_bitsliced_host")
    return out


def dihedral_batch(x, t, device="cuda:0"):
    """rz_dihedral_dev over arrays: out[i] = flip_vertical if t[i] & 4, then (t[i] & 3) x rotate90 of x[i]
    (lib/bitboard.py:119-159 in the order of agent/player.py:166-179,300-305) -- the device code the engine's leaf
    gather and the ingest kernel use.  Device buffers through torch (plumbing); host arrays in / out."""
    import torch
    from .. import device as D
    x = _u64(x)
    t = np.ascontiguousarray(np.broadcast_to(np.asarray(t, dtype=np.uint8), x.shape))
    dx, dt = D.to_device(x, device), D.to_device(t, device)
    out = D.empty(x.size, np.uint64, device)
    _cabi.check(_cabi.lib().rz_dihedral_dev(D.ptr(dx), D.ptr(dt), D.ptr(out), x.size, D.stream_ptr()), "rz_dihedral_dev")
    torch.cuda.synchronize()
    return D.to_numpy_u64(out)


def step_batch(black, white, next_player, turn, done, winner, action, want_legal=False):
    """In place on contiguous uint64 / uint8 arrays; action int8 with -1 = resign.  Returns legal masks or None."""
    n = black.size
    legal = np.empty(n, dtype=np.uint64) if want_legal else None
    p = lambda a, t: a.ctypes.data_as(t)
    _cabi.check(_cabi.lib().rz_step(p(black, _cabi.u64p), p(white, _cabi.u64p), p(next_player, _cabi.u8p), p(turn, _cabi.u8p),
                                     p(done, _cabi.u8p), p(winner, _cabi.u8p), p(action, _cabi.i8p),
                                     p(legal, _cabi.u64p) if want_legal else None, n), "rz_step")
    return legal
