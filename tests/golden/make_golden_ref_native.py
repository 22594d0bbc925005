"""Writes tests/golden/ref_native.npz and tests/golden/ref_native_solver.json: the outputs of the reference's own compiled
Cython modules (lib/alt/bitboard_cython.pyx, lib/alt/reversi_solver_cython.pyx, built by oracle/build_ref.py into
oracle/_ref) on the seeded inputs of tests/test_ref_native.py, so that the tests compare against the reference without
needing its checkout.  Run once where oracle/_ref has been built:

    python tests/golden/make_golden_ref_native.py
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle import ref_native  # noqa: E402
import test_ref_native as T  # noqa: E402


def main():
    assert ref_native.available(), "oracle/_ref is not built"
    bb, sv = ref_native.load()
    own, enemy, pos = T.config5_positions(T.N_POSITIONS)
    idx = T.golden_sample_indices()
    o, e, p = own[idx], enemy[idx], pos[idx]
    legal = np.fromiter((bb.find_correct_moves(int(a), int(b)) for a, b in zip(o, e)), dtype=np.uint64, count=len(idx))
    flip = np.fromiter((bb.calc_flip(int(q), int(a), int(b)) for q, a, b in zip(p, o, e)), dtype=np.uint64, count=len(idx))
    np.savez_compressed(os.path.join(HERE, "ref_native.npz"), legal=legal, flip=flip)

    def solve(a, b, exactly):
        mv, sc = sv.ReversiSolver().solve(a, b, ref_native.player_enum().black, exactly=exactly)
        return [-1, 0] if mv is None else [int(mv), int(sc)]

    out = {}
    for name, (n, seed) in T.ENDGAME_SETS.items():
        cases = T.random_endgames(n, seed)
        out[name] = {str(ex): [solve(a, b, ex) for a, b in cases] for ex in (True, False)}
    with open(os.path.join(HERE, "ref_native_solver.json"), "w") as f:
        json.dump(out, f)


if __name__ == "__main__":
    main()
