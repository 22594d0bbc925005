"""The reference's OWN compiled code (lib/alt/bitboard_cython.pyx, lib/alt/reversi_solver_cython.pyx) against
  * the oracle restatements (CPU), and
  * the CUDA operators through the C ABI (GPU): K1 move generation / flips on 1 M seeded positions of the
    SURVEY 8(d) config-5 recipe, and the batched endgame solver.
The reference's outputs on these seeded inputs are stored under tests/golden (ref_native.npz: a fixed sample of the 1 M
positions; ref_native_solver.json: every endgame), written by tests/golden/make_golden_ref_native.py from the compiled
reference modules."""
import json
import os

import numpy as np
import pytest

from oracle import bitboard as ob
from oracle.solver import Solver

U64 = np.uint64
N_POSITIONS = 1_000_000
GOLDEN_SAMPLE = 32_768
ENDGAME_SETS = dict(oracle=(120, 41), device=(200, 43))


def config5_positions(n, seed=20260922):
    """SURVEY 8(d) config 5: thirds of the set with occupancy a & b / a / a | b (densities 1/4, 1/2, 3/4), disjoint own/enemy."""
    rng = np.random.default_rng(seed)
    a = rng.integers(0, 2 ** 64, size=n, dtype=U64)
    b = rng.integers(0, 2 ** 64, size=n, dtype=U64)
    r = rng.integers(0, 2 ** 64, size=n, dtype=U64)
    occ = a.copy()
    third = n // 3
    occ[:third] = a[:third] & b[:third]
    occ[2 * third:] = a[2 * third:] | b[2 * third:]
    pos = rng.integers(0, 64, size=n, dtype=np.uint8)
    return occ & r, occ & ~r, pos


def golden_sample_indices():
    """the positions of the 1 M set whose reference outputs are stored: a fixed seeded sample across all three thirds"""
    return np.sort(np.random.default_rng(7).choice(N_POSITIONS, GOLDEN_SAMPLE, replace=False))


def random_endgames(n, seed, max_empties=10):
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        empties = int(rng.integers(1, max_empties + 1))
        e = ob.Env().reset()
        while not e.done and 60 - e.turn > empties:
            o, en = e.own_enemy()
            legal = ob.find_correct_moves(o, en)
            ms = [i for i in range(64) if legal >> i & 1]
            e.step(ms[rng.integers(len(ms))])
        if not e.done:
            out.append(e.own_enemy())
    return out


def reference_outputs(golden_dir):
    """(indices, legal, flip) of the compiled reference on the stored sample of the 1 M positions"""
    z = np.load(os.path.join(golden_dir, "ref_native.npz"))
    return golden_sample_indices(), z["legal"], z["flip"]


def reference_solves(golden_dir, name):
    """{exactly: [(move, score)] } of ReversiSolver.solve(black, white, next_player, exactly) of the compiled reference,
    positions given in the mover's frame, move -1 / score 0 where it returns no move"""
    with open(os.path.join(golden_dir, "ref_native_solver.json")) as f:
        d = json.load(f)[name]
    return {ex: [tuple(x) for x in d[str(ex)]] for ex in (True, False)}


def test_oracle_bitboard_matches_compiled_reference(golden_dir):
    own, enemy, pos = config5_positions(N_POSITIONS)
    idx, legal, flip = reference_outputs(golden_dir)
    assert np.array_equal(ob.find_correct_moves_batch(own[idx], enemy[idx]), legal)
    assert np.array_equal(ob.calc_flip_batch(pos[idx], own[idx], enemy[idx]), flip)


def test_oracle_solver_matches_compiled_reference(golden_dir):
    ref = reference_solves(golden_dir, "oracle")
    for i, (own, enemy) in enumerate(random_endgames(*ENDGAME_SETS["oracle"])):
        for exactly in (True, False):
            mv, sc = Solver().solve(own, enemy, exactly)
            assert ((-1, 0) if mv is None else (mv, sc)) == ref[exactly][i]


@pytest.mark.gpu
def test_k1_kernels_match_compiled_reference_1m(golden_dir):
    from reversi_zero_b200.lib import bitboard as zb
    own, enemy, pos = config5_positions(N_POSITIONS)
    legal, flip = zb.find_correct_moves_batch(own, enemy), zb.calc_flip_batch(pos, own, enemy)   # 1 M positions
    idx, ref_legal, ref_flip = reference_outputs(golden_dir)
    assert np.array_equal(legal[idx], ref_legal)      # bit-exact against the reference on the stored sample
    assert np.array_equal(flip[idx], ref_flip)        # including occupied / illegal squares
    assert np.array_equal(legal, ob.find_correct_moves_batch(own, enemy))   # and against the oracle on all 1 M
    assert np.array_equal(flip, ob.calc_flip_batch(pos, own, enemy))


@pytest.mark.gpu
def test_device_solver_matches_compiled_reference(golden_dir):
    from reversi_zero_b200.lib import reversi_solver as zs
    ref = reference_solves(golden_dir, "device")
    cases = random_endgames(*ENDGAME_SETS["device"])
    own = [c[0] for c in cases]
    enemy = [c[1] for c in cases]
    for exactly in (True, False):
        mv, sc = zs.solve_batch(own, enemy, [exactly] * len(cases))
        assert [(int(m), int(s)) for m, s in zip(mv, sc)] == ref[exactly]
