"""CPU suite for NBoard's retrograde analysis (reversi_zero_b200/play_game/analysis.py, the `analyze` command of
play_game/nboard.py): the positions of a game and their numbering, the split into solved and searched positions with
stand-in solvers and search, the report order, stopping, the protocol lines and the config knob."""
import json
import os
import re

import pytest

from reversi_zero_b200 import _cabi
from reversi_zero_b200.config import Config, create_config, load_yaml
from reversi_zero_b200.env.reversi_env import Player
from reversi_zero_b200.lib.bitboard import bit_count
from reversi_zero_b200.lib.ggf import convert_to_bitboard_and_actions, parse_ggf
from reversi_zero_b200.play_game import analysis as A, nboard as NB

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
START_B, START_W = 1 << 28 | 1 << 35, 1 << 27 | 1 << 36
# seeded random games from the standard start: a wipeout after 9 moves, and a full game with a pass at move 59 that
# ends with one square empty
WIPEOUT = [19, 18, 37, 29, 21, 11, 3, 20, 17]
PASS_GAME = [37, 45, 19, 20, 13, 29, 21, 5, 54, 42, 38, 12, 11, 34, 43, 47, 33, 18, 30, 32, 25, 9, 0, 39, 10, 1, 22, 4, 6, 63,
             3, 26, 16, 50, 57, 58, 46, 41, 49, 51, 44, 24, 59, 52, 2, 17, 60, 61, 40, 56, 53, 15, 31, 48, 8, 62, 55, 23, None, 14]


@pytest.fixture(scope="module")
def golden(golden_dir):
    with open(os.path.join(golden_dir, "nboard_ref.json")) as f:
        return json.load(f)


def golden_pass_game(golden):
    """the golden `pass` session's game: `set game`, then `move PA`"""
    line = next(t["line"] for t in golden["sessions"]["pass"]["transcript"] if t["line"].startswith("set game "))
    ggf = parse_ggf(line[len("set game "):])
    black, white, actions = convert_to_bitboard_and_actions(ggf)
    return black, white, Player.black if ggf.BO.color == "*" else Player.white, actions + [None]


def test_positions_of_the_golden_pass_game(golden):
    black, white, player, actions = golden_pass_game(golden)
    pos = A.enumerate_positions(black, white, player, actions)
    assert [p.moves_made for p in pos] == list(range(len(actions) + 1))
    assert pos[0].player == 1 and [p.player for p in pos[1:]] == [2 if k % 2 == 0 else 1 for k in range(len(actions))]
    kinds = A.classify(pos)
    # before `move PA` the mover must pass: its value is the negated value of the position after the pass
    assert kinds[-2][:2] == ("pass", -1) and kinds[-2][2:] == (pos[-1].own, pos[-1].enemy)
    assert kinds[-1][0] == "move" and all(k[0] == "move" for k in kinds[:-2])
    assert pos[-1].own == pos[-2].enemy and pos[-1].enemy == pos[-2].own


def test_positions_of_games_that_end():
    pos = A.enumerate_positions(START_B, START_W, 1, WIPEOUT)
    kinds = A.classify(pos)
    assert kinds[-1][0] == "over" and bit_count(pos[-1].own) == 0 and bit_count(pos[-1].enemy) == 13
    assert all(k[0] == "move" for k in kinds[:-1])
    pos = A.enumerate_positions(START_B, START_W, Player.black, PASS_GAME)
    kinds = A.classify(pos)
    assert len(pos) == 61 and [k[0] for k in kinds[-4:]] == ["move", "pass", "move", "over"]
    assert 64 - bit_count(pos[-1].own | pos[-1].enemy) == 1
    # the record's side to move alternates with every action, passes included
    assert [p.player for p in pos] == [1 + k % 2 for k in range(61)]
    # a move the record's mover cannot play is the other side's after an unrecorded pass
    no_pass = PASS_GAME[:58] + PASS_GAME[59:]
    pos2 = A.enumerate_positions(START_B, START_W, 1, no_pass)
    assert (pos2[-1].own, pos2[-1].enemy) == (pos[-1].own, pos[-1].enemy) and len(pos2) == 60
    with pytest.raises(ValueError):
        A.enumerate_positions(START_B, START_W, 1, [0])


class StandIns:
    """solvers and search that record their calls and answer with recognisable values: 200 + empties from the lane
    solver, 100 + empties from the deep solver, disc difference / 8 from the search"""

    def __init__(self, deep_fails=()):
        self.calls, self.out, self.deep_fails = [], [], set(deep_fails)

    def solve_lane(self, own, enemy):
        self.calls.append(("lane", [64 - bit_count(o | e) for o, e in zip(own, enemy)]))
        return [200 + 64 - bit_count(o | e) for o, e in zip(own, enemy)]

    def solve_deep(self, own, enemy):
        empties = 64 - bit_count(own | enemy)
        self.calls.append(("deep", empties))
        return None if empties in self.deep_fails else 100 + empties   # a recognisable stand-in value

    def search(self, own, enemy):
        self.calls.append(("search", len(own)))
        return [(bit_count(o) - bit_count(e)) / 8 for o, e in zip(own, enemy)]

    def report(self, moves_made, value, exact):
        self.out.append((moves_made, value, exact))


def _run(actions, use_solver_turn, max_empties, si, stopped=lambda: False):
    pc = Config().play
    pc.use_solver_turn = use_solver_turn
    pos = A.enumerate_positions(START_B, START_W, 1, actions)
    return pos, A.analyse(pos, pc, max_empties, si.report, stopped, si.solve_lane, si.solve_deep, si.search)


def test_split_follows_use_solver_turn_and_solver_max_empties():
    si = StandIns(deep_fails={15})
    pos, done = _run(PASS_GAME, 40, 16, si)
    assert done
    empties = [64 - bit_count(p.own | p.enemy) for p in pos]
    # one lane batch (<= 12 empties, the pass position shares its successor's solve), then 13..16 one at a time in
    # ascending order of empties, then one search of everything else (the failed 15-empty solve included)
    lane = si.calls[0]
    assert lane[0] == "lane" and sorted(lane[1]) == sorted(e for m, e in enumerate(empties) if e <= 12 and m not in (58, 60))
    assert [c for c in si.calls[1:-1]] == [("deep", 13), ("deep", 14), ("deep", 15), ("deep", 16)]
    n_searched = sum(1 for p, e in zip(pos, empties) if e > 16 or e == 15)
    assert si.calls[-1] == ("search", n_searched)
    got = {m: (v, ex) for m, v, ex in si.out}
    assert sorted(got) == list(range(61)) and len(si.out) == 61
    for p, e in zip(pos, empties):
        v, ex = got[p.moves_made]
        if p.moves_made == 60:
            assert (v, ex) == (bit_count(p.own) - bit_count(p.enemy), True)
        elif e <= 12:
            # the pass position (58) is worth its successor's value negated
            assert (v, ex) == ((-(200 + empties[59]) if p.moves_made == 58 else 200 + e), True)
        elif e in (13, 14, 16):
            assert (v, ex) == (100 + e, True)
        else:
            assert (v, ex) == ((bit_count(p.own) - bit_count(p.enemy)) / 8, False)
    # report order: exact values from the end backwards as they are proven, then the searched ones from the end backwards
    exact = [m for m, _, ex in si.out if ex]
    searched = [m for m, _, ex in si.out if not ex]
    assert si.out[:len(exact)] == [x for x in si.out if x[2]]
    assert exact == sorted(exact, reverse=True) and searched == sorted(searched, reverse=True)


def test_no_solver_turn_searches_everything_and_game_over_stays_exact():
    si = StandIns()
    pos, _ = _run(WIPEOUT, 0, 20, si)
    assert si.calls == [("search", 9)]
    assert si.out[0] == (9, -13, True) and [m for m, _, _ in si.out[1:]] == list(range(8, -1, -1))
    assert all(not ex for _, _, ex in si.out[1:])


def test_stop_sends_nothing_more():
    si = StandIns()
    _, done = _run(PASS_GAME, 40, 16, si, stopped=lambda: len(si.out) >= 3)
    assert not done and len(si.out) == 3 and ("search", 1) not in si.calls
    # a search that reports a stop (None) drops everything it would have given
    si = StandIns()
    si.search = lambda own, enemy: None
    _, done = _run(WIPEOUT, 0, 20, si)
    assert not done and si.out == [(9, -13, True)]


def test_search_value_and_chunks():
    import numpy as np
    n = np.zeros(64, np.int32)
    w = np.zeros(64, np.float32)
    n[[3, 10]] = 7
    w[3], w[10] = 2.5, -1.0
    assert A.search_value(n, w) == float(np.float64(2.5) / (7 + 1e-5)) * 10     # first index of the most visits
    assert A.chunk_steps(25, 10) == [5, 10, 10] and A.chunk_steps(20, 10) == [10, 10] and A.chunk_steps(20, 0) == [20]


class AnalysisStandIn:
    def __init__(self, cfg):
        self.out, self.calls = [], []
        self.handler = NB.NBoardProtocolVersion2(cfg, self)

    def reply(self, message):
        self.out.append(message)

    def begin_analysis(self):
        self.calls.append("begin")

    def analyze(self, report):
        self.calls.append("analyze")
        report(60, -1, True)
        report(58, 3, True)
        report(12, 9.999999899899901, False)
        report(11, -0.25, False)


def test_protocol_analyze_is_ignored_by_default_and_answers_with_the_knob():
    e = AnalysisStandIn(Config())
    e.handler.handle_message("analyze")
    assert e.out == [] and e.calls == []
    cfg = Config()
    cfg.b200.nboard_analyze = True
    e = AnalysisStandIn(cfg)
    e.handler.handle_message("analyze")
    assert e.calls == ["begin", "analyze"]
    assert e.out == ["status analyzing...", "analysis 60 -1", "analysis 58 3", "analysis 12 9.999999899899901",
                     "analysis 11 -0.25", "status waiting"]


def test_knob_reaches_the_engine_from_yaml(tmp_path):
    assert Config().b200.nboard_analyze is False
    assert create_config({"b200": {"nboard_analyze": True}}).b200.nboard_analyze is True
    p = tmp_path / "c.yml"
    p.write_text("type: x\nb200:\n  nboard_analyze: true\n")
    cfg = load_yaml(str(p), project_dir=str(tmp_path))
    e = AnalysisStandIn(cfg)
    e.handler.handle_message("analyze")
    assert e.out[0] == "status analyzing..." and e.out[-1] == "status waiting"


def test_new_abi_symbols_have_prototypes():
    with open(os.path.join(ROOT, "include", "rz_engine.h")) as f:
        header = re.sub(r"\s+", " ", f.read())
    assert ("int rz_engine_search_roots(rz_engine* e, const uint64_t* own, const uint64_t* enemy, const uint8_t* player, "
            "int n, int keep_tree, int32_t* n_visit, float* w_sum);") in header
    assert ("int rz_solve_deep_with_stop(const uint64_t* own, const uint64_t* enemy, int8_t* move, int8_t* score, size_t n, "
            "double timeout_s, const volatile int32_t* stop, rz_deep_solve_stats* stats);") in header
    import ctypes as C
    res, args = _cabi.SIGNATURES["rz_engine_search_roots"]
    assert res is C.c_int and args == [C.c_void_p, _cabi.u64p, _cabi.u64p, _cabi.u8p, C.c_int, C.c_int, _cabi.i32p, _cabi.f32p]
    res, args = _cabi.SIGNATURES["rz_solve_deep_with_stop"]
    assert res is C.c_int and args[:6] == _cabi.SIGNATURES["rz_solve_deep"][1][:6]
    assert args[6] == C.POINTER(C.c_int32) and args[7] == C.POINTER(_cabi.DeepSolveStats)
    lib = _cabi.lib()
    assert hasattr(lib, "rz_engine_search_roots") and hasattr(lib, "rz_solve_deep_with_stop")
