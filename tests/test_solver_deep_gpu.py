"""GPU suite of the deep exact endgame solver (rz_solve_deep): equal to the lane solver's exact mode up to 12 empties,
equal to the host oracle's fixture (tests/golden/deep_solver.json) at 13..20 empties, self-consistent at 21..24 empties
(value = pass-aware max over the children solved through the same ABI, move = lowest argmax), invariant under tiny slices
and small leaf targets, the timeout and the refusals, the Python mirror and the NBoard engine."""
import io
import json
import os
import time

import numpy as np
import pytest

from oracle import bitboard as ob
from reversi_zero_b200.config import create_config
from reversi_zero_b200.env.reversi_env import Player
from reversi_zero_b200.lib import reversi_solver as zs
from reversi_zero_b200.lib.ggf import convert_action_to_move
from reversi_zero_b200.play_game import nboard as NB

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fixture(golden_dir):
    with open(os.path.join(golden_dir, "deep_solver.json")) as f:
        return json.load(f)["positions"]


@pytest.fixture(autouse=True)
def default_tuning():
    zs.tune_deep()
    yield
    zs.tune_deep()


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


def test_equals_lane_solver_up_to_12_empties(golden_dir):
    g = json.load(open(os.path.join(golden_dir, "solver.json")))["positions"]
    pos = [(c["black"], c["white"]) if c["next_player"] == 1 else (c["white"], c["black"]) for c in g]
    pos = [p for p in pos if 64 - bin(p[0] | p[1]).count("1") <= 12]
    assert pos
    pos += random_positions(53, 2000, 6, 12)
    own, enemy = np.array([p[0] for p in pos], np.uint64), np.array([p[1] for p in pos], np.uint64)
    mv_l, sc_l = zs.solve_batch(own, enemy, [True] * len(pos))
    mv_d, sc_d = zs.solve_deep_batch(own, enemy, timeout=60)
    bad = [(hex(int(o)), hex(int(e)), (int(a), int(b)), (int(c), int(d)))
           for o, e, a, b, c, d in zip(own, enemy, mv_l, sc_l, mv_d, sc_d) if (a, b) != (c, d)]
    assert not bad, bad[:10]


def test_equals_fixture_13_to_20_empties(fixture):
    own = np.array([p["own"] for p in fixture], np.uint64)
    enemy = np.array([p["enemy"] for p in fixture], np.uint64)
    mv, sc, st = zs.solve_deep_batch(own, enemy, timeout=120, stats=True)
    for p, m, s, t in zip(fixture, mv, sc, st):
        assert (int(m), int(s)) == (p["move"], p["score"]), (p["empties"], hex(p["own"]), hex(p["enemy"]), t)
        assert t["probes"] >= 2 and t["slices"] >= 1 and t["node_steps"] > 0


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


def test_self_consistent_22_empties():
    # the seeded position with the fewest root moves (three) keeps the number of child solves (21 empties each) small
    for empties, seed in ((22, 62),):
        own, enemy = min(random_positions(seed, 40, empties, empties), key=lambda p: bin(ob.find_correct_moves(*p)).count("1"))
        (mv,), (sc,) = zs.solve_deep_batch([own], [enemy], timeout=600)
        kids = _children(own, enemy)
        need = [(o2, e2) for _, o2, e2, neg in kids if neg is not None]
        km, ks = zs.solve_deep_batch([o for o, _ in need], [e for _, e in need], timeout=600)
        assert all(m >= 0 for m in km)
        vals, it = {}, iter(ks)
        for a, o2, e2, neg in kids:
            vals[a] = e2 if neg is None else (-int(next(it)) if neg else int(next(it)))
        v = max(vals.values())
        assert int(sc) == v and int(mv) == min(a for a, x in vals.items() if x == v), (empties, hex(own), hex(enemy), vals)


def test_invariant_under_tiny_slices_and_resplits(fixture):
    pick = [p for p in fixture if 14 <= p["empties"] <= 16][:6]
    assert len(pick) >= 4
    zs.tune_deep(slice_us=300, leaf_target=48, leaf_floor=5)
    own = [p["own"] for p in pick]
    enemy = [p["enemy"] for p in pick]
    mv, sc, st = zs.solve_deep_batch(own, enemy, timeout=300, stats=True)
    for p, m, s in zip(pick, mv, sc):
        assert (int(m), int(s)) == (p["move"], p["score"])
    assert sum(t["slices"] for t in st) > len(pick) * 10
    assert all(t["slices"] > 1 for t in st) and sum(t["resplits"] for t in st) > 0


def test_timeout_and_refusals(fixture):
    p = fixture[0]
    assert zs.solve_deep_batch([p["own"]], [p["enemy"]])[0][0] == p["move"]   # workspace allocated
    (o28, e28), = random_positions(71, 1, 28, 28)
    t0 = time.perf_counter()
    mv, sc, st = zs.solve_deep_batch([o28], [e28], timeout=0.05, stats=True)
    took = time.perf_counter() - t0
    assert (int(mv[0]), int(sc[0])) == (-1, 0)
    # the timeout is checked between slices (4 ms) and between split levels; 0.5 s of margin for the host's split
    assert took < 0.05 + 0.004 + 0.5, (took, st)
    # the device is usable right after
    q = next(p for p in fixture if p["empties"] == 15)
    mv, sc = zs.solve_deep_batch([q["own"]], [q["enemy"]])
    assert (int(mv[0]), int(sc[0])) == (q["move"], q["score"])
    # no legal move; a finished game; too many empties
    mv, sc = zs.solve_deep_batch([0xFFFFFFFFFFFFFF00, 0xFFFFFFFF00000000, 0x0000000810000000],
                                 [0x00000000000000FE, 0x00000000FFFFFFFF, 0x0000001008000000])
    assert list(mv) == [-1, -1, -1] and list(sc) == [0, 0, 0]
    (o31, e31), = random_positions(72, 1, 31, 31)
    mv, sc = zs.solve_deep_batch([o31], [e31])
    assert (int(mv[0]), int(sc[0])) == (-1, 0)


def test_python_mirror(fixture):
    p = next(p for p in fixture if p["empties"] == 16)
    assert zs.ReversiSolver(max_empties=20).solve(p["own"], p["enemy"], Player.black, exactly=True) == (p["move"], p["score"])
    assert zs.ReversiSolver(max_empties=20).solve(p["enemy"], p["own"], Player.white, exactly=True) == (p["move"], p["score"])
    assert zs.ReversiSolver().solve(p["own"], p["enemy"], Player.black, exactly=True) == (None, None)


def _go(cfg, own, enemy, monkeypatch):
    """`set game` at (own to move as black) and `go` through the NBoard engine with the deterministic evaluator"""
    board = "".join("*" if own >> i & 1 else "O" if enemy >> i & 1 else "-" for i in range(64))
    monkeypatch.setattr(NB, "load_model", lambda config: None)
    out = io.StringIO()
    eng = NB.NBoardEngine(cfg, stdin=io.StringIO(), stdout=out)
    try:
        eng.handler.handle_message(f"set game (;GM[Othello]PC[NBoard]BO[8 {board} *];)")
        eng.handler.handle_message("go")
    finally:
        eng.player.engine.close()
    return [l for l in out.getvalue().splitlines() if l.startswith("=== ")][-1]


def test_nboard_plays_the_deep_solvers_move(fixture, golden_dir, monkeypatch):
    with open(os.path.join(golden_dir, "nboard_ref.json")) as f:
        base = json.load(f)["config"]
    p = next(p for p in fixture if 18 <= p["empties"] <= 20 and p["move"] != min(
        int(a) for a in p["move_values"]))   # a position where the lowest legal square is not the answer
    cfg = create_config(dict(base, b200={"solver_max_empties": 20}))
    cfg.play.use_solver_turn = 40
    cfg.play_with_human.update_play_config(cfg.play)
    reply = _go(cfg, p["own"], p["enemy"], monkeypatch)
    assert reply.split("/")[0] == "=== " + convert_action_to_move(p["move"]), reply
    # without the knob: the lane solver refuses, the search plays, and the deep solver is never asked
    cfg = create_config(base)
    cfg.play.use_solver_turn = 40
    cfg.play_with_human.update_play_config(cfg.play)
    monkeypatch.setattr(zs, "solve_deep_batch", lambda *a, **k: pytest.fail("deep solver called at the default"))
    before = _go(cfg, p["own"], p["enemy"], monkeypatch)
    again = _go(cfg, p["own"], p["enemy"], monkeypatch)
    assert before.split("/")[0] == again.split("/")[0]
    legal = ob.find_correct_moves(p["own"], p["enemy"])
    assert any(before.split("/")[0] == "=== " + convert_action_to_move(a) for a in range(64) if legal >> a & 1), before
