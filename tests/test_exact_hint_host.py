"""CPU suite of the per-move endgame solve behind NBoard's exact hints: the forest's two questions and the round plan of
rz_solve_deep_moves compiled for the host (tests/support/deep_roots_check.cu); the lane path's construction of every
move's child; the NBoard `hint` lines with stand-in solvers; the knob; the C ABI.  No GPU needed."""
import ctypes as C
import io
import json
import os
import re
import shutil
import subprocess
import types

import numpy as np
import pytest

from oracle import bitboard as ob
from oracle.solver import Solver
from reversi_zero_b200 import _cabi
from reversi_zero_b200.config import Config, create_config
from reversi_zero_b200.env.reversi_env import ReversiEnv, Player
from reversi_zero_b200.lib import reversi_solver as zs
from reversi_zero_b200.lib.ggf import convert_action_to_move
from reversi_zero_b200.play_game import nboard as NB

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "reversi-alpha-zero_b200", "csrc")
OPEN, TRUE, FALSE, EVERY = 0, 1, 2, 2


@pytest.fixture(scope="module")
def roots_exe(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("deep_roots_check") / "deep_roots_check")
    subprocess.run([nvcc, "-O2", "-std=c++17", "--expt-relaxed-constexpr", "-Wno-deprecated-gpu-targets", "-I", CSRC,
                    os.path.join(ROOT, "tests", "support", "deep_roots_check.cu"), "-o", exe], check=True)
    return exe


@pytest.fixture(scope="module")
def fixture(golden_dir):
    with open(os.path.join(golden_dir, "deep_solver.json")) as f:
        return json.load(f)["positions"]


def test_roots_answered_both_questions(roots_exe):
    out = subprocess.run([roots_exe, "roots"], capture_output=True, text=True, check=True).stdout.split("\n")
    seen = {"lowest": 0, "every": 0}
    for line in filter(None, out):
        v = [int(x) for x in line.split()]
        n, status, flip, got = v[0], v[1:1 + v[0]], v[1 + v[0]:1 + 2 * v[0]], v[-1]
        if all(f == EVERY for f in flip):
            want = all(s != OPEN for s in status)   # every root decided
            seen["every"] += 1
        else:   # the lowest root with its wanted answer, every root below it decided the other way; or all decided
            want = True
            for s, f in zip(status, flip):
                if s == OPEN:
                    want = False
                    break
                if (s == TRUE) == (f != 0):
                    break
            seen["lowest"] += 1
        assert bool(got) == want, line
    assert seen == {"lowest": sum(3 ** n * 2 ** n for n in range(1, 5)), "every": sum(3 ** n for n in range(1, 5))}


def run_rounds(exe, cases):
    """cases: (n_best, values) -> list of (rounds, [(lo, hi)])"""
    text = "".join(f"{nb} {len(v)} {' '.join(map(str, v))}\n" for nb, v in cases)
    out = subprocess.run([exe, "moves"], input=text, capture_output=True, text=True, check=True).stdout.split("\n")
    res = []
    for line in filter(None, out):
        w = [int(x) for x in line.split()]
        res.append((w[0], list(zip(w[1::2], w[2::2]))))
    return res


def check_contract(values, n_best, bounds):
    """lo <= value <= hi; moves at least the n_best-th best value (ties included) exact; every other one below it"""
    vn = sorted(values, reverse=True)[n_best - 1] if 0 < n_best <= len(values) else min(values)
    for v, (lo, hi) in zip(values, bounds):
        assert lo <= v <= hi
        if v >= vn:
            assert lo == hi
        else:
            assert hi < vn


def test_rounds_meet_the_n_best_contract(roots_exe, fixture):
    rng = np.random.default_rng(5)
    cases = [(nb, [int(v) for v in p["move_values"].values()]) for p in fixture for nb in range(0, 5)]
    for _ in range(400):   # extreme and tied values
        k = int(rng.integers(1, 16))
        vals = [int(x) for x in rng.choice([-64, -63, -2, -1, 0, 1, 2, 63, 64, int(rng.integers(-64, 65))], k)]
        cases.append((int(rng.integers(0, 6)), vals))
    for (nb, vals), (rounds, bounds) in zip(cases, run_rounds(roots_exe, cases)):
        assert 0 <= rounds <= 8, (nb, vals)
        check_contract(vals, nb, bounds)
    # n_best prunes: the best of the fixture's moves alone takes fewer probes than all of them
    full = run_rounds(roots_exe, [(0, [int(v) for v in p["move_values"].values()]) for p in fixture])
    best = run_rounds(roots_exe, [(1, [int(v) for v in p["move_values"].values()]) for p in fixture])
    assert sum(sum(lo == hi for lo, hi in b) for _, b in best) < sum(sum(lo == hi for lo, hi in b) for _, b in full)


# ---------------------------------------------------------------------------------------------------------- lane path

def negamax(own, enemy, alpha=-65, beta=65):
    """exact value for own to move (empties not awarded), alpha-beta over the oracle's move generator"""
    moves = ob.find_correct_moves(own, enemy)
    if not moves:
        if not ob.find_correct_moves(enemy, own):
            return bin(own).count("1") - bin(enemy).count("1")
        return -negamax(enemy, own, -beta, -alpha)
    best = -65
    for a in range(64):
        if moves >> a & 1:
            fl = ob.calc_flip(a, own, enemy)
            v = -negamax(enemy ^ fl, own | fl | (1 << a), -beta, -max(alpha, best))
            best = max(best, v)
            if best >= beta:
                break
    return best


def child_value(own, enemy, a):
    fl = ob.calc_flip(a, own, enemy)
    return -negamax(enemy ^ fl, own | fl | (1 << a))


def random_positions(seed, n, lo, hi):
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        empties = int(rng.integers(lo, hi + 1))
        e = ob.Env().reset()
        while not e.done and 60 - e.turn > empties:
            o, en = e.own_enemy()
            legal = ob.find_correct_moves(o, en)
            e.step([i for i in range(64) if legal >> i & 1][rng.integers(len([i for i in range(64) if legal >> i & 1]))])
        if not e.done:
            out.append(e.own_enemy())
    return out


def oracle_solve_batch(own, enemy, exactly):
    mv, sc = [], []
    for o, e in zip(own, enemy):
        m, s = Solver().solve(int(o), int(e), True)
        mv.append(-1 if m is None else m)
        sc.append(0 if m is None else s)
    return np.array(mv, np.int8), np.array(sc, np.int8)


def test_lane_path_builds_every_child(monkeypatch):
    calls = []
    monkeypatch.setattr(zs, "solve_batch", lambda o, e, x: calls.append(len(o)) or oracle_solve_batch(o, e, x))
    pos = random_positions(61, 40, 6, 10)
    for own, enemy in pos:
        got = zs.lane_move_values(own, enemy)
        legal = ob.find_correct_moves(own, enemy)
        assert set(got) == {a for a in range(64) if legal >> a & 1}
        for a, (lo, hi) in got.items():
            assert lo == hi == child_value(own, enemy, a), (hex(own), hex(enemy), a)
    assert len(calls) == len(pos)   # one launch per position


def test_lane_path_after_a_pass_and_at_the_end(monkeypatch):
    monkeypatch.setattr(zs, "solve_batch", oracle_solve_batch)
    rng = np.random.default_rng(7)
    found = {"pass": 0, "over": 0}
    tried = 0
    while min(found.values()) < 3 and tried < 4000:
        tried += 1
        o, e = random_positions(int(rng.integers(1 << 30)), 1, 2, 8)[0]
        legal = ob.find_correct_moves(o, e)
        for a in range(64):
            if legal >> a & 1:
                fl = ob.calc_flip(a, o, e)
                o2, e2 = o | fl | (1 << a), e ^ fl
                if ob.find_correct_moves(e2, o2):
                    continue
                kind = "pass" if ob.find_correct_moves(o2, e2) else "over"
                found[kind] += 1
                assert zs.lane_move_values(o, e)[a] == (child_value(o, e, a),) * 2
    assert min(found.values()) >= 3, found


def test_solver_routes_solve_moves(monkeypatch):
    calls = []
    monkeypatch.setattr(zs, "lane_move_values", lambda o, e: calls.append(("lane", o, e)) or {1: (2, 2)})
    monkeypatch.setattr(zs, "solve_moves", lambda o, e, nb, t, s, cb: calls.append(("deep", o, e, nb, t)) or {3: (4, 4)})
    e12 = (0x00FFFFFFFFFF0000 | 0xF0, 0x000000000000FF00)        # 12 empties
    e16 = (0x00FFFFFFFFFF0000, 0x000000000000FF00)               # 16 empties
    s = zs.ReversiSolver(max_empties=20)
    assert s.solve_moves(*e12, 1) == {1: (2, 2)}
    assert s.solve_moves(*e16, 2, n_best=3, timeout=7) == {3: (4, 4)}
    assert zs.ReversiSolver().solve_moves(*e16, 1) is None          # beyond max_empties
    assert calls == [("lane", *e12), ("deep", e16[1], e16[0], 3, 7)]


# ------------------------------------------------------------------------------------------------------------ NBoard

class StandInSolver:
    """ReversiSolver.solve_moves revealing `rounds` of bounds through on_bounds, then returning the last; `on_round(i)`
    runs before round i is revealed (a ping, say)"""

    def __init__(self, rounds, on_round=None):
        self.rounds, self.on_round, self.calls = rounds, on_round, []

    def solve_moves(self, black, white, next_player, n_best=0, timeout=30, stop=None, on_bounds=None):
        self.calls.append((black, white, next_player, n_best, timeout))
        last = {}
        for i, b in enumerate(self.rounds):
            if self.on_round:
                self.on_round(i)
            if stop is not None and stop.value:
                return last
            last = b
            if on_bounds:
                on_bounds(b)
        return last


def _engine(exact_hint=True, solver_max_empties=20, solver=None):
    eng = NB.NBoardEngine.__new__(NB.NBoardEngine)
    eng.config = Config()
    eng.config.b200.nboard_exact_hint = exact_hint
    eng.config.b200.solver_max_empties = solver_max_empties
    eng.config.play.use_solver_turn = 40
    eng.nc = eng.config.nboard
    eng.play_config = eng.config.play
    eng.stdout = io.StringIO()
    eng.handler = NB.NBoardProtocolVersion2(eng.config, eng)
    eng.env = ReversiEnv().reset()
    eng.player = types.SimpleNamespace(calls=[], stopped=0)

    def action(own, enemy, callback_in_mtcs=None, solve=True):
        eng.player.calls.append(("action", solve))
        values, visits = [0.0] * 64, [0] * 64
        values[19], visits[19] = 0.25, 9
        callback_in_mtcs.callback(values, visits)
        return 19

    eng.player.action = action
    eng.player.ask_thought_about = lambda own, enemy: types.SimpleNamespace(values=[0.25 if i == 19 else 0.0 for i in range(64)],
                                                                           visit=[9 if i == 19 else 0 for i in range(64)])
    eng.player.stop_thinking = lambda: setattr(eng.player, "stopped", eng.player.stopped + 1)
    if solver is not None:
        eng.hint_solver, eng.hint_stop = solver, C.c_int32(0)
    return eng


def _set_position(eng, fixture, empties):
    p = next(p for p in fixture if p["empties"] == empties)
    eng.env.update(p["own"], p["enemy"], Player.black)   # own = black, to move
    return p


def _lines(eng):
    return eng.stdout.getvalue().splitlines()


def _m(a):
    return convert_action_to_move(a)


def test_exact_hint_lines_and_order(fixture):
    eng = _engine()
    p = _set_position(eng, fixture, 16)
    mv = {int(a): v for a, v in p["move_values"].items()}
    order = sorted(mv, key=lambda a: (-mv[a], a))
    a0, a1, a2 = order[0], order[1], order[2]
    # round 1: signs of some moves; round 2: everything exact
    r1 = {a: (-64, 64) for a in mv}
    wins = [a for a in mv if mv[a] >= 1]
    losses = [a for a in mv if mv[a] <= -1]
    for a in wins:
        r1[a] = (1, 64)
    for a in losses:
        r1[a] = (-64, -1)
    r2 = {a: (v, v) for a, v in mv.items()}
    eng.hint_solver, eng.hint_stop = StandInSolver([r1, r2]), C.c_int32(0)
    eng.handler.handle_message("hint 3")
    lines = _lines(eng)
    assert lines[0] == "status thinkng hint..." and lines[-1] == "status waiting"
    body = lines[1:-1]
    wld = [l for l in body if l.endswith(" 100%W")]
    exact = [l for l in body if l.endswith(" 100%")]
    assert len(wld) == len(wins) + len(losses) and body[:len(wld)] == wld
    for l in wld:   # lo of a proven win, hi of a proven loss, ascending
        _, m, v, _, _ = l.split(" ")
        assert int(v) in (1, -1)
    assert [int(l.split(" ")[2]) for l in wld] == sorted(int(l.split(" ")[2]) for l in wld)
    assert exact == [f"search {_m(a)} {mv[a]} 0 100%" for a in (a2, a1, a0)]
    assert exact[-1].split(" ")[1] == _m(p["move"])   # the last line is go's move
    assert eng.hint_solver.calls[0][3:] == (3, 30) and eng.player.calls == []
    assert all(re.match(r"^search [A-H][1-8] -?\d+ 0 100%W?$", l) for l in body)


def test_exact_hint_ties_put_the_lowest_square_last():
    eng = _engine(solver=StandInSolver([{44: (2, 2), 19: (2, 2), 37: (-4, -4), 26: (2, 2)}]))
    eng.env.update(0x00FFFFFFFFFF0000, 0x000000000000FF00, Player.black)
    eng.hint(2)
    assert _lines(eng) == [f"search {_m(26)} 2 0 100%", f"search {_m(19)} 2 0 100%"]


def test_timeout_reports_what_is_proven_and_falls_back_without_solving(fixture):
    # a timeout after one round: the proven moves, best n of them
    eng = _engine(solver=StandInSolver([{19: (3, 3), 26: (1, 64), 37: (-64, 64), 44: (-64, -2)}]))
    eng.env.update(0x00FFFFFFFFFF0000, 0x000000000000FF00, Player.black)
    eng.hint(3)
    lines = _lines(eng)
    # the round's WLD lines, then the final list
    assert lines[:2] == [f"search {_m(44)} -2 0 100%W", f"search {_m(26)} 1 0 100%W"]
    assert lines[2:] == [f"search {_m(44)} -2 0 100%W", f"search {_m(26)} 1 0 100%W", f"search {_m(19)} 3 0 100%"]
    assert eng.player.calls == []
    # nothing proven at all: the search hint, with the player's solver skipped
    eng = _engine(solver=StandInSolver([{19: (-64, 64), 26: (-64, 64)}]))
    eng.env.update(0x00FFFFFFFFFF0000, 0x000000000000FF00, Player.black)
    eng.hint(3)
    assert _lines(eng) == [f"search {_m(19)} 0.25 0 9"] * 2
    assert eng.player.calls == [("action", False)]


def test_ping_stops_the_exact_hint_and_nothing_follows():
    eng = _engine()
    rounds = [{19: (1, 64), 26: (-64, -1)}, {19: (5, 5), 26: (-3, -3)}]
    eng.hint_solver, eng.hint_stop = StandInSolver(rounds, on_round=lambda i: i == 1 and eng.push_callback("ping 3")), C.c_int32(0)
    eng.env.update(0x00FFFFFFFFFF0000, 0x000000000000FF00, Player.black)
    eng.handler.handle_message("hint 2")
    eng.handler.handle_message("ping 3")
    lines = _lines(eng)
    assert lines == ["status thinkng hint...", f"search {_m(26)} -1 0 100%W", f"search {_m(19)} 1 0 100%W",
                     "status waiting", "pong 3"]
    assert eng.player.calls == [] and eng.player.stopped == 1
    # a stop before the solve: no line at all; the next hint starts with the flag cleared
    eng.stdout = io.StringIO()
    eng.hint_solver = StandInSolver(rounds, on_round=lambda i: eng.push_callback("ping 4"))
    eng.hint(2)
    assert _lines(eng) == []
    eng.stdout = io.StringIO()
    eng.hint_solver = StandInSolver(rounds)
    eng.hint(2)
    assert _lines(eng)[-2:] == [f"search {_m(26)} -3 0 100%", f"search {_m(19)} 5 0 100%"]


def test_knob_off_or_out_of_range_keeps_the_search_hint():
    for eng in (_engine(exact_hint=False, solver=StandInSolver([{19: (1, 1)}])),
                _engine(solver_max_empties=12, solver=StandInSolver([{19: (1, 1)}]))):
        eng.env.update(0x00FFFFFFFFFF0000, 0x000000000000FF00, Player.black)   # 16 empties, turn 44
        eng.handler.handle_message("hint 2")
        assert _lines(eng) == ["status thinkng hint...", f"search {_m(19)} 0.25 0 9", f"search {_m(19)} 0.25 0 9", "status waiting"]
        assert eng.hint_solver.calls == [] and eng.player.calls == [("action", True)]
    eng = _engine(solver=StandInSolver([{19: (1, 1)}]))
    eng.config.play.use_solver_turn = 50   # before the solver's turn
    eng.env.update(0x00FFFFFFFFFF0000, 0x000000000000FF00, Player.black)
    eng.hint(2)
    assert eng.hint_solver.calls == [] and eng.player.calls == [("action", True)]


def test_knob_from_yaml(tmp_path):
    import yaml
    from reversi_zero_b200.config import load_yaml
    assert Config().b200.nboard_exact_hint is False and create_config({}).b200.nboard_exact_hint is False
    yml = tmp_path / "c.yml"
    yml.write_text(yaml.safe_dump({"b200": {"nboard_exact_hint": True, "solver_max_empties": 20}}))
    cfg = load_yaml(str(yml), project_dir=str(tmp_path))
    assert cfg.b200.nboard_exact_hint is True and cfg.b200.nboard_analyze is False


def test_solvable_rule_is_shared():
    from reversi_zero_b200.agent.player import solves_exactly
    pc = types.SimpleNamespace(use_solver_turn=40)
    own, enemy = 0x00FFFFFFFFFF0000, 0x000000000000FF00   # 48 discs: turn 44, 16 empties
    assert solves_exactly(pc, own, enemy) and solves_exactly(pc, own, enemy, 16) and not solves_exactly(pc, own, enemy, 15)
    assert not solves_exactly(types.SimpleNamespace(use_solver_turn=45), own, enemy)
    assert not solves_exactly(types.SimpleNamespace(use_solver_turn=None), own, enemy)
    assert not solves_exactly(types.SimpleNamespace(), own, enemy)


def test_deep_moves_prototype():
    hdr = open(os.path.join(ROOT, "include", "rz_engine.h")).read()
    assert "typedef void (*rz_deep_moves_cb)(const int8_t* lo, const int8_t* hi, void* user);" in hdr
    proto = re.search(r"int rz_solve_deep_moves\((.*?)\);", hdr, re.S).group(1)
    assert len(proto.split(",")) == 11 and "rz_deep_moves_cb on_round" in proto
    res, args = _cabi.SIGNATURES["rz_solve_deep_moves"]
    assert res is C.c_int and len(args) == 11 and args[8] is _cabi.DeepMovesCallback
    lib = C.CDLL(_cabi.LIB_PATH)
    assert getattr(lib, "rz_solve_deep_moves", None) is not None
