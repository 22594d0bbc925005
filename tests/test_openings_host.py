"""CPU suite of opening suites: the enumerator's expansion step compiled for the host (tests/support/openings_check.cu)
against a Python restatement over lib/bitboard.py; suite files and their refusals; how eval and league assign openings
to games; the YAML keys and the command; oracle games from an opening; the C ABI.  No GPU needed."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

from oracle import bitboard as ob, mcts, nn as onn
from reversi_zero_b200 import _cabi, engine as E
from reversi_zero_b200.config import create_config
from reversi_zero_b200.lib import bitboard as bb, openings as OP
from reversi_zero_b200.lib.ggf import convert_action_to_move
from reversi_zero_b200.worker import evaluate as EV, league as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "reversi-alpha-zero_b200", "csrc")
START = (0x10 << 24) | (0x08 << 32), (0x08 << 24) | (0x10 << 32)


@pytest.fixture(scope="module")
def check_exe(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("openings_check") / "openings_check")
    subprocess.run([nvcc, "-O2", "-std=c++17", "--expt-relaxed-constexpr", "-Wno-deprecated-gpu-targets", "-I", CSRC,
                    os.path.join(ROOT, "tests", "support", "openings_check.cu"), "-o", exe], check=True)
    return exe


def run_check(exe, plies):
    """-> (level counts, [(own, enemy, moves)]) as the host twin prints them"""
    lines = subprocess.run([exe, str(plies)], capture_output=True, text=True, check=True).stdout.split("\n")
    counts = [int(x) for x in lines[0].split()[1:]]
    out = []
    for line in filter(None, lines[1:]):
        v = [int(x) for x in line.split()]
        out.append((v[0], v[1], v[2:]))
    return counts, out


def py_enumerate(plies):
    """the enumerator restated: children in (parent, square) order, dropped when their mover has no move; per canonical
    key the first child; the next level in ascending key order"""
    frontier = [(START[0], START[1], [])]
    counts = [1]
    for _ in range(plies):
        best = {}
        for own, enemy, moves in frontier:
            legal = bb.find_correct_moves(own, enemy)
            for sq in range(64):
                if not (legal >> sq) & 1:
                    continue
                fl = bb.calc_flip(sq, own, enemy)
                co, ce = enemy ^ fl, own | fl | (1 << sq)
                if not bb.find_correct_moves(co, ce):
                    continue
                best.setdefault(OP.canonical_key(co, ce), (co, ce, moves + [sq]))
        frontier = [best[k] for k in sorted(best)]
        counts.append(len(frontier))
    return counts, frontier


@pytest.mark.parametrize("plies", range(1, 8))
def test_expand_step_matches_python(check_exe, plies):
    counts, out = run_check(check_exe, plies)
    want_counts, want = py_enumerate(plies)
    assert counts == want_counts
    assert [OP.canonical_key(o, e) for o, e, _ in out] == sorted({OP.canonical_key(o, e) for o, e, _ in want})
    assert out == [(o, e, m) for o, e, m in want]   # the same representative, orientation and moves for every class
    for own, enemy, moves in out:
        assert len(moves) == plies and OP.replay(moves) == (own, enemy)   # legal, no pass, not finished
        assert bb.find_correct_moves(own, enemy)


def test_first_moves_are_one_opening(check_exe):
    counts, out = run_check(check_exe, 1)
    assert counts == [1, 1] and out[0][2] == [min(sq for sq in range(64) if (bb.find_correct_moves(*START) >> sq) & 1)]


def test_known_counts(check_exe):
    assert run_check(check_exe, 8)[0] == [1, 1, 3, 14, 60, 322, 1773, 10649, 67239]


def line_of(moves):
    return " ".join(convert_action_to_move(a) for a in moves)


def test_suite_round_trip(tmp_path):
    suite = [[19, 18, 17], [37, 43], [26, 20, 29, 34]]
    p = str(tmp_path / "s" / "suite.txt")
    OP.save_suite(p, suite, header=["three openings"])
    assert OP.load_suite(p) == suite
    OP.save_suite(p, [OP.SuiteEntry(m, 0.125) for m in suite])
    assert OP.load_suite(p) == suite and "# v=+0.1250" in open(p).read()
    (tmp_path / "c.txt").write_text("# comment\n\n  d3 c5   # lower case, trailing comment\n")
    assert OP.load_suite(str(tmp_path / "c.txt")) == [[26, 20]]   # letter = row, digit = column (lib/ggf.py)


def forcing_pass_sequence():
    """the shortest move sequence found by breadth-first search after which the side to move must pass"""
    frontier = [(START[0], START[1], [])]
    while True:
        nxt = []
        for own, enemy, moves in frontier:
            for sq in range(64):
                if (bb.find_correct_moves(own, enemy) >> sq) & 1:
                    fl = bb.calc_flip(sq, own, enemy)
                    co, ce = enemy ^ fl, own | fl | (1 << sq)
                    if not bb.find_correct_moves(co, ce):
                        return moves + [sq], bool(bb.find_correct_moves(ce, co))
                    nxt.append((co, ce, moves + [sq]))
        frontier = nxt[:4000]


def test_suite_refusals(tmp_path):
    seq, passes = forcing_pass_sequence()
    ok = "F5 D6\n"
    cases = {
        "J1": "is not a square", "F9": "is not a square", "F5x": "is not a square",
        "F5 A1": "illegal", "F5 PA": "a pass",
        line_of(seq): "must pass" if passes else "ends the game",
        " ".join(["F5"] * 21): "at most 20",
    }
    for bad, why in cases.items():
        p = tmp_path / "bad.txt"
        p.write_text("# header\n" + ok + bad + "\n")
        with pytest.raises(ValueError, match=rf"bad.txt:3: .*{why}"):
            OP.load_suite(str(p))
    (tmp_path / "empty.txt").write_text("# nothing\n\n")
    with pytest.raises(ValueError, match="no opening"):
        OP.load_suite(str(tmp_path / "empty.txt"))


def test_match_openings_pairs_with_swapped_colours():
    suite = [[19], [37], [26]]
    got = EV.match_openings(8, suite)
    assert got == [[19], [19], [37], [37], [26], [26], [19], [19]]
    # colours alternate with the game index (rz_engine_set_second_net): each opening once with each colour
    assert all(got[i] == got[i + 1] for i in range(0, 8, 2))
    assert EV.match_openings(5, suite)[4] == [26]


@pytest.mark.parametrize("n_models,games_per_pair", [(2, 4), (3, 5), (4, 6)])
def test_league_openings_pairs_with_swapped_colours(n_models, games_per_pair):
    suite = [[19], [37], [26], [44]]
    black, white = L.schedule(n_models, games_per_pair)
    got = L.league_openings(n_models, games_per_pair, suite)
    assert len(got) == black.size
    per = {}
    for k, op in enumerate(got):
        pair = (min(black[k], white[k]), max(black[k], white[k]))
        per.setdefault((pair, tuple(op)), []).append(int(black[k]))
    n_ops = (games_per_pair + 1) // 2
    for (pair, op), blacks in per.items():
        if games_per_pair % 2 and op == tuple(suite[(n_ops - 1) % len(suite)]) and n_ops <= len(suite):
            assert len(blacks) == 1   # the odd last round: that opening once
        else:
            assert sorted(blacks) == sorted(pair)   # once with each colour
    assert len({op for _, op in per}) == min(n_ops, len(suite))


def test_yaml_keys_reach_workers(tmp_path):
    import yaml
    p = tmp_path / "c.yml"
    p.write_text(yaml.safe_dump(dict(openings=dict(plies=6, count=7, max_abs_value=0.3, seed=5, model="m.npy", path="o.txt"),
                                     eval=dict(openings="o.txt"), league=dict(openings="o.txt"))))
    from reversi_zero_b200.config import load_yaml
    cfg = load_yaml(str(p), project_dir=str(tmp_path))
    assert [OP._field(cfg, k, None) for k in ("plies", "count", "max_abs_value", "seed", "model", "path")] == [6, 7, 0.3, 5, "m.npy", "o.txt"]
    assert L._field(cfg, "openings", None) == "o.txt" and EV._eval_field(cfg, "openings", None) == "o.txt"
    OP.save_suite(str(tmp_path / "o.txt"), [[19, 18]])
    assert EV.EvaluateWorker(cfg).load_openings() == [[19, 18]]
    d = create_config(project_dir=str(tmp_path))
    assert (d.openings.plies, d.openings.count, d.openings.max_abs_value, d.openings.seed, d.openings.model) == (8, 500, 0.2, None, None)
    assert d.openings.path == os.path.join("data", "openings", "openings.txt") and d.league.openings is None
    assert EV.EvaluateWorker(d).load_openings() is None


def test_openings_command_parses():
    from reversi_zero_b200 import run
    assert run.create_parser().parse_args(["openings", "-c", "x.yml"]).cmd == "openings"


def oracle_game(pp, opening, seed, game_id, api_b=None):
    g = mcts.SelfPlayGame(pp, onn.FakeNetAPI(), seed=seed, game_id=game_id, api_b=api_b, black_net=0)
    for a in opening:
        g.env.step(a)
    return g.play()


def test_oracle_game_from_opening():
    pp = mcts.PlayParams(simulation_num_per_move=12, parallel_search_num=4, noise_eps=0.0, change_tau_turn=0, c_puct=5,
                         thinking_loop=1, resign_threshold=None, share_mtcs_info_in_self_play=False)
    opening = [37, 43, 34]
    g = oracle_game(pp, opening, 3, 0)
    env = ob.Env().reset()
    for a in opening:
        env.step(a)
    first = g.plies[0]
    assert (first["own"], first["enemy"], first["pid"]) == (*env.own_enemy(), env.next_player)
    assert len(g.plies) + len(opening) >= 4 and g.env.done
    # without the opening the first move is the forced lowest square
    assert oracle_game(pp, [], 3, 0).actions[0] == min(sq for sq in range(64) if (bb.find_correct_moves(*START) >> sq) & 1)


def test_abi():
    hdr = open(os.path.join(ROOT, "include", "rz_engine.h")).read()
    assert "#define RZ_MAX_OPENING_PLIES 20" in hdr and E.MAX_OPENING_PLIES == OP.MAX_OPENING_PLIES == 20
    assert re.search(r"int rz_engine_set_openings\(rz_engine\* e, const uint8_t\* moves, const uint8_t\* n_moves, uint64_t n_games\);", hdr)
    assert re.search(r"int rz_openings_enumerate\(int plies, uint64_t\* own, uint64_t\* enemy, uint8_t\* moves, size_t cap, size_t\* n_out,\s+uint64_t\* level_counts\);", hdr)
    for name in ("rz_engine_set_openings", "rz_openings_enumerate"):
        assert name in _cabi.SIGNATURES and hasattr(_cabi.lib(), name)
    assert C.sizeof(_cabi.Game) == 56 and _cabi.Game.opening_plies.offset == _cabi.Game.white_net.offset + 1
    assert _cabi.Game.table_nodes.offset == 48
    assert _cabi.lib().rz_openings_enumerate(0, None, None, None, 0, C.byref(C.c_size_t()), None) == -1
    assert _cabi.lib().rz_openings_enumerate(13, None, None, None, 0, C.byref(C.c_size_t()), None) == -1
