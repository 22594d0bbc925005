"""CPU suite of the deep exact endgame solver (csrc/rz_solver_deep.cu): the independent host oracle
(tests/support/endgame_oracle.cu) against the reference restatement and the reference's exact golden cases; the leaf
machine (csrc/rz_solver_deep.cuh) compiled for the host, whole and time-sliced, against the oracle at thresholds around
the value; the fixture tests/golden/deep_solver.json (coverage, and its entries up to 16 empties re-derived); the
configuration plumbing up to the player's solver; the C ABI.  No GPU needed."""
import ctypes as C
import json
import os
import shutil
import subprocess
from types import SimpleNamespace

import numpy as np
import pytest

from oracle import bitboard as ob
from oracle.solver import Solver
from reversi_zero_b200 import _cabi
from reversi_zero_b200.agent import player as P
from reversi_zero_b200.config import create_config
from reversi_zero_b200.lib import reversi_solver as zs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "reversi-alpha-zero_b200", "csrc")
REQUIRED_TAGS = ("tie", "zero", "single", "pass_child", "pass_deep", "wipeout")


def _compile(tmp_path_factory, src, name):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp(name) / name)
    subprocess.run([nvcc, "-O2", "-std=c++17", "--expt-relaxed-constexpr", "-Wno-deprecated-gpu-targets", "-I", CSRC,
                    os.path.join(ROOT, "tests", "support", src), "-o", exe], check=True)
    return exe


@pytest.fixture(scope="module")
def oracle_exe(tmp_path_factory):
    return _compile(tmp_path_factory, "endgame_oracle.cu", "endgame_oracle")


@pytest.fixture(scope="module")
def leaf_exe(tmp_path_factory):
    return _compile(tmp_path_factory, "deep_leaf_check.cu", "deep_leaf_check")


@pytest.fixture(scope="module")
def fixture(golden_dir):
    with open(os.path.join(golden_dir, "deep_solver.json")) as f:
        return json.load(f)["positions"]


def oracle_solve(exe, positions):
    text = "".join(f"{o:x} {e:x}\n" for o, e in positions)
    r = subprocess.run([exe], input=text, capture_output=True, text=True, check=True)
    return [tuple(int(v) for v in line.split()) for line in r.stdout.strip().split("\n")]


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
        if not e.done:
            out.append(e.own_enemy())
    return out


def test_oracle_matches_reference_restatement(oracle_exe):
    pos = random_positions(41, 200, 1, 10)
    pos.append((0xFFFFFFFFFFFFFF00, 0x00000000000000FE))  # no legal move
    for (o, e), got in zip(pos, oracle_solve(oracle_exe, pos)):
        mv, sc = Solver().solve(o, e, True)
        assert got == ((-1, 0) if mv is None else (mv, sc)), (hex(o), hex(e))


def test_oracle_matches_reference_golden_exact_cases(oracle_exe, golden_dir):
    g = [c for c in json.load(open(os.path.join(golden_dir, "solver.json")))["positions"] if c["exactly"]]
    assert g
    pos = [(c["black"], c["white"]) if c["next_player"] == 1 else (c["white"], c["black"]) for c in g]
    for c, got in zip(g, oracle_solve(oracle_exe, pos)):
        assert got == (c["move"], c["score"]), c["tag"]


@pytest.mark.parametrize("every", [0, 7])
def test_leaf_machine_thresholds(oracle_exe, leaf_exe, every):
    pos = random_positions(43, 60, 4, 14)
    vals = oracle_solve(oracle_exe, pos)
    qs = [(o, e, v + d) for (o, e), (m, v) in zip(pos, vals) if m >= 0 for d in range(-2, 3)]
    text = "".join(f"{o:x} {e:x} {t}\n" for o, e, t in qs)
    r = subprocess.run([leaf_exe, str(every)], input=text, capture_output=True, text=True, check=True)
    got = [int(x) for x in r.stdout.split()]
    assert len(got) == len(qs)
    for (o, e, t), g in zip(qs, got):
        v = next(v for (o2, e2), (_, v) in zip(pos, vals) if (o2, e2) == (o, e))
        assert g == int(v >= t), (hex(o), hex(e), t, v)
    suspensions = int(r.stderr.split()[-1])
    assert (suspensions > 1000) if every else suspensions == 0


def test_fixture_coverage(fixture):
    assert len(fixture) >= 55
    assert {p["empties"] for p in fixture} == set(range(13, 21))
    tags = {t for p in fixture for t in p["tags"]}
    assert tags >= set(REQUIRED_TAGS), set(REQUIRED_TAGS) - tags
    for p in fixture:  # each entry is consistent: move = lowest root move reaching the value
        mv = {int(a): v for a, v in p["move_values"].items()}
        assert max(mv.values()) == p["score"]
        assert p["move"] == min(a for a, v in mv.items() if v == p["score"])
        legal = ob.find_correct_moves(p["own"], p["enemy"])
        assert set(mv) == {i for i in range(64) if legal >> i & 1}


def test_fixture_rederived_up_to_16_empties(oracle_exe, fixture):
    small = [p for p in fixture if p["empties"] <= 16]
    assert len(small) >= 25
    got = oracle_solve(oracle_exe, [(p["own"], p["enemy"]) for p in small])
    for p, g in zip(small, got):
        assert g == (p["move"], p["score"]), (hex(p["own"]), hex(p["enemy"]))


class _StandIn:
    made = []

    def __init__(self, max_empties=12):
        _StandIn.made.append(max_empties)

    def solve(self, own, enemy, next_player, timeout=30, exactly=False):
        return 19, 4


def _bare_player(config):
    """a ReversiPlayer without its engine: the solver branch of action_with_evaluation needs none"""
    p = P.ReversiPlayer.__new__(P.ReversiPlayer)
    p.config, p.play_config, p.solver, p.thinking_history = config, config.play, None, {}
    return p


def test_config_reaches_the_players_solver(tmp_path, monkeypatch):
    import yaml
    yml = tmp_path / "c.yml"
    yml.write_text(yaml.safe_dump({"play": {"use_solver_turn": 40}, "b200": {"solver_max_empties": 20}}))
    from reversi_zero_b200.config import load_yaml
    cfg = load_yaml(str(yml), project_dir=str(tmp_path))
    assert cfg.b200.solver_max_empties == 20 and cfg.b200.games_per_gpu == 4096
    monkeypatch.setattr(zs, "ReversiSolver", _StandIn)
    _StandIn.made.clear()
    own, enemy = 0xFF00FFFFFFFF0000, 0x00000000000000FF  # 48 discs: turn 44, past use_solver_turn
    act = _bare_player(cfg).action_with_evaluation(own, enemy)
    assert act.action == 19 and _StandIn.made == [20]
    # the default, and a reference Config without b200: the lane solver alone
    _StandIn.made.clear()
    _bare_player(create_config({"play": {"use_solver_turn": 40}})).action_with_evaluation(own, enemy)
    ref_like = SimpleNamespace(play=create_config({"play": {"use_solver_turn": 40}}).play)
    assert P.solver_max_empties(ref_like) == 12
    _bare_player(ref_like).action_with_evaluation(own, enemy)
    assert _StandIn.made == [12, 12]


def test_default_solver_makes_todays_calls(monkeypatch):
    calls = []
    monkeypatch.setattr(zs, "solve_batch", lambda o, e, x: calls.append(("lane", list(o), list(e), list(x))) or
                        (np.array([-1], np.int8), np.array([0], np.int8)))
    monkeypatch.setattr(zs, "solve_deep_batch", lambda *a, **k: calls.append(("deep",)) or
                        (np.array([-1], np.int8), np.array([0], np.int8)))
    own, enemy = 0x0000000810000000, 0x0000001008000000      # 60 empties
    mid_o, mid_e = 0x00FFFFFFFFFF0000, 0x000000000000FF00   # 16 empties
    assert zs.ReversiSolver().solve(own, enemy, 1, exactly=True) == (None, None)
    assert zs.ReversiSolver().solve(mid_o, mid_e, 2, timeout=5, exactly=True) == (None, None)
    assert calls == [("lane", [own], [enemy], [True]), ("lane", [mid_e], [mid_o], [True])]
    calls.clear()
    s = zs.ReversiSolver(max_empties=20)
    s.solve(mid_o, mid_e, 1, exactly=True)     # 16 empties, exact: the deep solver
    s.solve(mid_o, mid_e, 1, exactly=False)    # WLD: the lane solver
    s.solve(own, enemy, 1, exactly=True)       # 60 empties: beyond max_empties, the lane solver (which refuses)
    assert [c[0] for c in calls] == ["deep", "lane", "lane"]
    with pytest.raises(ValueError):
        zs.ReversiSolver(max_empties=31)


def test_deep_symbols_resolve():
    lib = C.CDLL(_cabi.LIB_PATH)
    for name in ("rz_solve_deep", "rz_solve_deep_tune"):
        assert getattr(lib, name, None) is not None, name
        assert name in _cabi.SIGNATURES
    assert C.sizeof(_cabi.DeepSolveStats) == 40
