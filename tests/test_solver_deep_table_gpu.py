"""GPU suite of the deep solver's transposition table (rz_solve_deep, csrc/rz_solver_deep.cuh): the fixture
tests/golden/deep_solver.json is reproduced from an empty table, again from a warm one (with bound cutoffs), with a tiny
table that keeps evicting and under 300 us slices with re-splits; the deep solver still equals the lane solver up to 12
empties and is self-consistent at 22 empties with a warm table; a seeded game solved in order with the table kept equals
the same positions solved cold; the timeout still holds; and the clear / size / stats calls."""
import json
import os
import time

import numpy as np
import pytest

from oracle import bitboard as ob
from reversi_zero_b200.lib import reversi_solver as zs

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fixture(golden_dir):
    with open(os.path.join(golden_dir, "deep_solver.json")) as f:
        return json.load(f)["positions"]


@pytest.fixture(autouse=True)
def defaults():
    zs.tune_deep()
    zs.deep_table_bytes(0)
    yield
    zs.tune_deep()
    zs.deep_table_bytes(0)


def random_positions(seed, n, lo, hi):
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        empties = int(rng.integers(lo, hi + 1))
        e = ob.Env().reset()
        while not e.done and 60 - e.turn > empties:
            o, en = e.own_enemy()
            legal = ob.find_correct_moves(o, en)
            ms = [i for i in range(64) if legal >> i & 1]
            e.step(ms[rng.integers(len(ms))])
        if not e.done and 60 - e.turn == empties:
            out.append(e.own_enemy())
    return out


def solve_fixture(pos, timeout=120):
    mv, sc, st = zs.solve_deep_batch([p["own"] for p in pos], [p["enemy"] for p in pos], timeout=timeout, stats=True)
    for p, m, s, t in zip(pos, mv, sc, st):
        assert (int(m), int(s)) == (p["move"], p["score"]), (p["empties"], hex(p["own"]), hex(p["enemy"]), t)
    return st


def test_fixture_cold_then_warm(fixture):
    zs.solve_deep_batch([fixture[0]["own"]], [fixture[0]["enemy"]])  # the default table exists
    zs.clear_deep_table()
    t = zs.deep_table_stats()
    assert t["bytes"] == 1 << 30 and all(t[k] == 0 for k in t if k != "bytes")
    cold = solve_fixture(fixture)
    t_cold = zs.deep_table_stats()
    assert t_cold["lookups"] > 0 and t_cold["stores"] > 0 and t_cold["occupied"] > 0 and t_cold["hints"] > 0
    warm = solve_fixture(fixture)
    t_warm = zs.deep_table_stats()
    assert t_warm["cutoffs"] > t_cold["cutoffs"]
    assert sum(s["node_steps"] for s in warm) < sum(s["node_steps"] for s in cold)


def test_fixture_with_a_tiny_table(fixture):
    zs.deep_table_bytes(16 << 20)  # 131 072 buckets of 4 entries, against millions of stores at 18..20 empties
    solve_fixture(fixture)
    t = zs.deep_table_stats()
    assert t["bytes"] == 16 << 20 and t["occupied"] <= 524288
    assert t["replaced"] > 0


def test_fixture_under_tiny_slices_and_resplits(fixture):
    pick = [p for p in fixture if 14 <= p["empties"] <= 16][:6]
    assert len(pick) >= 4
    zs.tune_deep(slice_us=300, leaf_target=48, leaf_floor=5)
    zs.solve_deep_batch([pick[0]["own"]], [pick[0]["enemy"]])
    zs.clear_deep_table()
    st = solve_fixture(pick, timeout=300)  # from an empty table
    assert all(t["slices"] > 1 for t in st) and sum(t["resplits"] for t in st) > 0
    st = solve_fixture(pick, timeout=300)  # warm: the leaves are answered from the table, so nothing is re-split
    assert all(t["slices"] > 1 for t in st)
    assert zs.deep_table_stats()["cutoffs"] > 0


def test_equals_lane_solver_up_to_12_empties_warm(golden_dir):
    g = json.load(open(os.path.join(golden_dir, "solver.json")))["positions"]
    pos = [(c["black"], c["white"]) if c["next_player"] == 1 else (c["white"], c["black"]) for c in g]
    pos = [p for p in pos if 64 - bin(p[0] | p[1]).count("1") <= 12]
    assert pos
    pos += random_positions(53, 2000, 6, 12)
    own, enemy = np.array([p[0] for p in pos], np.uint64), np.array([p[1] for p in pos], np.uint64)
    mv_l, sc_l = zs.solve_batch(own, enemy, [True] * len(pos))
    for n in (len(pos), 400):  # the table kept over the positions, then the first 400 again
        mv_d, sc_d = zs.solve_deep_batch(own[:n], enemy[:n], timeout=60)
        bad = [(hex(int(o)), hex(int(e)), (int(a), int(b)), (int(c), int(d)))
               for o, e, a, b, c, d in zip(own, enemy, mv_l, sc_l, mv_d, sc_d) if (a, b) != (c, d)]
        assert not bad, bad[:10]
    assert zs.deep_table_stats()["cutoffs"] > 0


def _children(own, enemy):
    """root moves ascending -> (square, own', enemy', negate) or (square, None, final diff, None)"""
    out = []
    legal = ob.find_correct_moves(own, enemy)
    for a in range(64):
        if legal >> a & 1:
            fl = ob.calc_flip(a, own, enemy)
            o2, e2 = (own ^ fl) | (1 << a), enemy ^ fl
            if ob.find_correct_moves(e2, o2):
                out.append((a, e2, o2, True))
            elif ob.find_correct_moves(o2, e2):
                out.append((a, o2, e2, False))
            else:
                out.append((a, None, ob.bit_count(o2) - ob.bit_count(e2), None))
    return out


def test_self_consistent_22_empties_warm():
    own, enemy = min(random_positions(62, 40, 22, 22), key=lambda p: bin(ob.find_correct_moves(*p)).count("1"))
    kids = _children(own, enemy)
    need = [(o2, e2) for _, o2, e2, neg in kids if neg is not None]
    zs.clear_deep_table()
    km, ks = zs.solve_deep_batch([o for o, _ in need], [e for _, e in need], timeout=600)  # warms the root's subtrees
    (mv,), (sc,) = zs.solve_deep_batch([own], [enemy], timeout=600)
    assert all(m >= 0 for m in km)
    vals, it = {}, iter(ks)
    for a, o2, e2, neg in kids:
        vals[a] = e2 if neg is None else (-int(next(it)) if neg else int(next(it)))
    v = max(vals.values())
    assert int(sc) == v and int(mv) == min(a for a, x in vals.items() if x == v), (hex(own), hex(enemy), vals)
    assert zs.deep_table_stats()["cutoffs"] > 0


def game_positions(seed, start):
    """one seeded random game's positions from `start` empties down to 13"""
    rng = np.random.default_rng(seed)
    e, out = ob.Env().reset(), []
    while not e.done:
        o, en = e.own_enemy()
        if 13 <= 64 - bin(o | en).count("1") <= start:
            out.append((o, en))
        legal = ob.find_correct_moves(o, en)
        ms = [i for i in range(64) if legal >> i & 1]
        e.step(ms[rng.integers(len(ms))])
    return out


def test_game_in_order_with_the_table_kept_equals_cold():
    pos = game_positions(7, 18)
    assert len(pos) >= 5 and 64 - bin(pos[0][0] | pos[0][1]).count("1") == 18
    cold = []
    for o, e in pos:
        zs.clear_deep_table()
        mv, sc = zs.solve_deep_batch([o], [e], timeout=120)
        cold.append((int(mv[0]), int(sc[0])))
    assert all(m >= 0 for m, _ in cold)
    zs.clear_deep_table()
    kept = [(int(m), int(s)) for o, e in pos for m, s in zip(*zs.solve_deep_batch([o], [e], timeout=120))]
    assert kept == cold
    assert zs.deep_table_stats()["cutoffs"] > 0


def test_timeout_with_a_warm_table(fixture):
    p = next(p for p in fixture if p["empties"] == 16)
    assert zs.solve_deep_batch([p["own"]], [p["enemy"]])[0][0] == p["move"]
    (o28, e28), = random_positions(71, 1, 28, 28)
    t0 = time.perf_counter()
    mv, sc, st = zs.solve_deep_batch([o28], [e28], timeout=0.05, stats=True)
    took = time.perf_counter() - t0
    assert (int(mv[0]), int(sc[0])) == (-1, 0)
    assert took < 0.05 + 0.004 + 0.5, (took, st)
    assert zs.solve_deep_batch([p["own"]], [p["enemy"]])[0][0] == p["move"]


def test_table_size_and_clear(fixture):
    p = next(p for p in fixture if p["empties"] == 14)
    zs.deep_table_bytes(100)  # below one bucket: one bucket
    assert zs.solve_deep_batch([p["own"]], [p["enemy"]])[0][0] == p["move"]
    t = zs.deep_table_stats()
    assert t["bytes"] == 128 and 0 < t["occupied"] <= 4
    zs.deep_table_bytes((3 << 20) + 5)  # rounded down to 2 MiB
    assert zs.solve_deep_batch([p["own"]], [p["enemy"]])[0][0] == p["move"]
    t = zs.deep_table_stats()
    assert t["bytes"] == 2 << 20 and t["occupied"] == t["stores"] - t["replaced"] > 0  # resized: a fresh table
    zs.clear_deep_table()
    assert all(v == 0 for k, v in zs.deep_table_stats().items() if k != "bytes")
    with pytest.raises(zs._cabi.RzError):
        zs.deep_table_bytes(-1)
