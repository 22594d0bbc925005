"""GPU suite of the per-move endgame solve (rz_solve_deep_moves, lib/reversi_solver.solve_moves) and NBoard's exact
hints: every move's value against tests/golden/deep_solver.json, the n_best contract, the table and slicing left free,
the lane path against the deep path, a 22-empty position against solves of its children, the stop flag, and the
engine as NBoard runs it."""
import ctypes as C
import json
import os
import sys
import threading
import time

import numpy as np
import pytest

from oracle import bitboard as ob
from reversi_zero_b200.agent import model as M
from reversi_zero_b200.config import load_yaml
from reversi_zero_b200.lib import reversi_solver as zs
from reversi_zero_b200.lib.ggf import convert_action_to_move

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_exact_hint_host import check_contract, random_positions  # noqa: E402
from test_nboard_gpu import Session  # noqa: E402

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def fixture(golden_dir):
    with open(os.path.join(golden_dir, "deep_solver.json")) as f:
        return json.load(f)["positions"]


@pytest.fixture(autouse=True)
def default_tuning():
    zs.tune_deep()
    zs.deep_table_bytes()
    yield
    zs.tune_deep()
    zs.deep_table_bytes()


def values_of(p):
    return {int(a): int(v) for a, v in p["move_values"].items()}


def check(p, got, n_best):
    mv = values_of(p)
    assert set(got) == set(mv), (hex(p["own"]), hex(p["enemy"]))
    sq = sorted(mv)
    check_contract([mv[s] for s in sq], n_best, [got[s] for s in sq])


def test_every_move_of_every_fixture_position(fixture):
    zs.clear_deep_table()
    for p in fixture:
        got, st = zs.solve_moves(p["own"], p["enemy"], 0, 60, stats=True)
        assert got == {a: (v, v) for a, v in values_of(p).items()}, (hex(p["own"]), hex(p["enemy"]))
        assert 1 <= st["probes"] <= 8 and st["node_steps"] >= 0
        # the best move and value are rz_solve_deep's
        best = max(v for v, _ in got.values())
        assert best == p["score"] and min(a for a, (v, _) in got.items() if v == best) == p["move"]
    for nb in (1, 2, 3):
        for p in fixture:
            check(p, zs.solve_moves(p["own"], p["enemy"], nb, 60), nb)


def test_best_move_matches_solve_deep(fixture):
    pos = [p for p in fixture if p["empties"] >= 17][:6]
    mv, sc = zs.solve_deep_batch([p["own"] for p in pos], [p["enemy"] for p in pos], 60)
    for p, m, s in zip(pos, mv, sc):
        got = zs.solve_moves(p["own"], p["enemy"], 1, 60)
        best = max(lo for lo, hi in got.values() if lo == hi)
        assert (int(m), int(s)) == (min(a for a, (lo, hi) in got.items() if lo == hi == best), best)


@pytest.mark.parametrize("mode", ["cold", "warm", "evicting", "sliced"])
def test_table_and_slices_change_no_answer(fixture, mode):
    pos = [p for p in fixture if p["empties"] in (14, 16, 18)][:9]
    if mode == "evicting":
        zs.deep_table_bytes(16 << 20)
    if mode == "sliced":
        zs.tune_deep(slice_us=300, leaf_target=64)
    zs.clear_deep_table()
    for nb in (0, 2):
        for p in pos:
            if mode == "cold":
                zs.clear_deep_table()
            got = zs.solve_moves(p["own"], p["enemy"], nb, 60, stats=True)
            check(p, got[0], nb)
            if mode == "sliced":
                assert got[1]["slices"] > 0
    if mode == "evicting":
        assert zs.deep_table_stats()["bytes"] == 16 << 20


def test_lane_path_equals_deep_path():
    pos = random_positions(77, 2000, 6, 12)
    s = zs.ReversiSolver(max_empties=20)
    for own, enemy in pos:
        lane = s.solve_moves(own, enemy, 1)
        deep = zs.solve_moves(own, enemy, 0, 60)
        assert lane == deep, (hex(own), hex(enemy))


def test_22_empties_against_the_children():
    own, enemy = random_positions(2222, 1, 22, 22)[0]
    got, st = zs.solve_moves(own, enemy, 1, 600, stats=True)
    legal = ob.find_correct_moves(own, enemy)
    assert set(got) == {a for a in range(64) if legal >> a & 1}
    kids = []
    for a in sorted(got):
        fl = ob.calc_flip(a, own, enemy)
        o2, e2 = own | fl | (1 << a), enemy ^ fl
        kids.append((a, -1, e2, o2) if ob.find_correct_moves(e2, o2) else (a, 1, o2, e2))
    mv, sc = zs.solve_deep_batch([k[2] for k in kids], [k[3] for k in kids], 600)
    vals = {}
    for (a, sign, o2, e2), m, v in zip(kids, mv, sc):
        if m < 0:   # the game ended with the move
            assert not ob.find_correct_moves(o2, e2) and not ob.find_correct_moves(e2, o2)
            vals[a] = bin(o2).count("1") - bin(e2).count("1")
        else:
            vals[a] = sign * int(v)
    sq = sorted(got)
    check_contract([vals[a] for a in sq], 1, [got[a] for a in sq])
    assert sum(lo == hi for lo, hi in got.values()) >= 1


def test_stop_before_and_during(fixture):
    p = max(fixture, key=lambda p: p["empties"])
    mv = values_of(p)
    flag = C.c_int32(1)
    t0 = time.perf_counter()
    got = zs.solve_moves(p["own"], p["enemy"], 0, 60, stop=flag)
    assert time.perf_counter() - t0 < 0.5
    assert set(got) == set(mv) and all(lo <= mv[a] <= hi for a, (lo, hi) in got.items())
    zs.clear_deep_table()
    flag = C.c_int32(0)
    rounds = []
    timer = threading.Timer(0.05, lambda: setattr(flag, "value", 1))
    timer.start()
    t0 = time.perf_counter()
    got = zs.solve_moves(p["own"], p["enemy"], 0, 60, stop=flag, on_bounds=rounds.append)
    took = time.perf_counter() - t0
    timer.join()
    assert took < 0.05 + 1.5, took   # one 4 ms slice plus the host's split work
    assert all(lo <= mv[a] <= hi for a, (lo, hi) in got.items())
    assert any(lo < hi for lo, hi in got.values())
    for r in rounds:
        assert all(lo <= mv[a] <= hi for a, (lo, hi) in r.items())


def _ggf_position(own, enemy):
    """a GGF game whose start position is (own = black, enemy = white) with black to move, and no moves"""
    sq = "".join("*" if own >> i & 1 else "O" if enemy >> i & 1 else "-" for i in range(64))
    return f"(;GM[Othello]PC[NBoard]BO[8 {sq} *];)"


def test_nboard_exact_hint_subprocess(fixture, tmp_path):
    import yaml
    base = os.path.join(ROOT, "tests", "golden", "ref_config", "ch5.yml")
    with open(base) as f:
        d = yaml.safe_load(f)
    d.setdefault("play", {})["use_solver_turn"] = 40
    d.setdefault("b200", {}).update(nboard_exact_hint=True, solver_max_empties=20)
    yml = str(tmp_path / "c.yml")
    with open(yml, "w") as f:
        yaml.safe_dump(d, f)
    cfg = load_yaml(yml, project_dir=str(tmp_path))
    cfg.resource.create_directories()
    np.save(cfg.resource.model_best_blob_path, M.weights_to_blob(cfg.model, M.build_random_weights(cfg.model, 5)))
    env = dict(os.environ, PROJECT_DIR=str(tmp_path), PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "reversi-alpha-zero_b200"), ROOT]))
    env.pop("DATA_DIR", None)
    env.pop("MODEL_DIR", None)
    s = Session([sys.executable, "-m", "reversi_zero_b200.run", "nboard", "-c", yml], str(tmp_path), env)
    try:
        s.send("nboard 2")
        s.until(lambda l: l.startswith("status"))
        p = next(p for p in fixture if p["empties"] == 16 and len(p["move_values"]) >= 3)
        mv = values_of(p)
        top = sorted(mv, key=lambda a: (-mv[a], a))[:3]
        s.send(f"set game {_ggf_position(p['own'], p['enemy'])}")
        s.send("hint 3")
        got = s.until(lambda l: l == "status waiting", timeout=300)
        exact = [l for l in got if l.endswith(" 100%")]
        assert exact[-3:] == [f"search {convert_action_to_move(a)} {mv[a]} 0 100%" for a in reversed(top)], got
        assert exact[-1].split(" ")[1] == convert_action_to_move(p["move"])
        assert all(l.startswith("status") or l.endswith("100%") or l.endswith("100%W") for l in got), got
        # a ping during a deep hint: the pong after `status waiting`, and no search line after it
        q = next(p for p in fixture if p["empties"] == 20)
        s.send(f"set game {_ggf_position(q['own'], q['enemy'])}")
        s.send("hint 8")
        s.until(lambda l: l.startswith("status thinkng"))
        s.send("ping 5")
        got = s.until(lambda l: l.startswith("pong"), timeout=120)
        assert got[-1] == "pong 5" and got[-2] == "status waiting", got
        s.send("learn")
        tail = s.until(lambda l: l == "learned")
        assert not [l for l in tail if l.startswith("search")], tail
        s.p.stdin.close()
        s.p.wait(timeout=60)
        assert s.p.returncode == 0, "".join(s.err)[-3000:]
    finally:
        if s.p.poll() is None:
            s.p.kill()
        s.p.wait(timeout=30)
