"""CPU suite of the deep solver's transposition table (csrc/rz_solver_deep.cuh), with the leaf machine and the table
compiled for the host (tests/support/deep_table_check.cu): the thresholds v-2..v+2 of the fixture's 13..16-empty
positions give the same booleans with an empty table, a warm one, a single bucket that keeps evicting and under time
slicing; the warm table takes fewer node steps than none; merging only tightens bounds; and a deliberately wrong bound
changes the answer, so the table is consulted both at a leaf's root and below it.  No GPU needed."""
import json
import os
import shutil
import subprocess

import numpy as np
import pytest

from oracle import bitboard as ob

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "reversi-alpha-zero_b200", "csrc")


@pytest.fixture(scope="module")
def table_exe(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("deep_table_check") / "deep_table_check")
    subprocess.run([nvcc, "-O2", "-std=c++17", "--expt-relaxed-constexpr", "-Wno-deprecated-gpu-targets", "-I", CSRC,
                    os.path.join(ROOT, "tests", "support", "deep_table_check.cu"), "-o", exe], check=True)
    return exe


@pytest.fixture(scope="module")
def positions(golden_dir):
    with open(os.path.join(golden_dir, "deep_solver.json")) as f:
        pos = [p for p in json.load(f)["positions"] if 13 <= p["empties"] <= 16]
    assert len(pos) >= 25
    return pos


def run(exe, commands, buckets, every=0):
    """-> (printed lines other than the P lines, list of the P lines' counts as dicts)"""
    r = subprocess.run([exe, str(buckets), str(every)], input="".join(c + "\n" for c in commands), capture_output=True,
                       text=True, check=True)
    out, counts = [], []
    for line in r.stdout.splitlines():
        if line.startswith("steps "):
            w = line.split()
            counts.append({w[i]: int(w[i + 1]) for i in range(0, len(w), 2)})
        else:
            out.append(line)
    return out, counts


def questions(pos):
    return [(p["own"], p["enemy"], p["score"] + d, int(d <= 0)) for p in pos for d in range(-2, 3)]


def q(o, e, t):
    return f"Q {o:x} {e:x} {t}"


@pytest.mark.parametrize("condition", ["empty", "warm", "single_bucket", "sliced"])
def test_same_booleans(table_exe, positions, condition):
    qs = questions(positions)
    want = [str(w) for *_, w in qs]
    if condition == "empty":  # every question starts from an empty table
        out, counts = run(table_exe, [c for o, e, t, _ in qs for c in ("X", q(o, e, t))] + ["P"], 1 << 16)
        assert out == want
    elif condition == "warm":  # the table kept over all questions, then every question again
        cmds = [q(o, e, t) for o, e, t, _ in qs]
        out, counts = run(table_exe, cmds + ["P"] + cmds + ["P"], 1 << 16)
        assert out == want + want
        assert counts[1]["cutoffs"] - counts[0]["cutoffs"] == len(qs)  # the second pass is answered from the table alone
    elif condition == "single_bucket":
        out, counts = run(table_exe, [q(o, e, t) for o, e, t, _ in qs] + ["P"], 1)
        assert out == want
        assert counts[0]["replaced"] > 1000
    else:  # parked and resumed every 7 node steps, warm table
        out, counts = run(table_exe, [q(o, e, t) for o, e, t, _ in qs] + ["P"], 1 << 16, every=7)
        assert out == want
        assert counts[0]["suspensions"] > 10000
    assert counts[-1]["lookups"] > 0 and counts[-1]["stores"] > 0 and counts[-1]["dropped"] == 0


def test_warm_table_takes_fewer_node_steps(table_exe, positions):
    cmds = [q(o, e, t) for o, e, t, _ in questions(positions)]
    _, (none,) = run(table_exe, cmds + ["P"], 0)
    _, (first, second) = run(table_exe, cmds + ["P"] + cmds + ["P"], 1 << 16)
    warmed = second["steps"] - first["steps"]
    assert none["lookups"] == 0
    assert first["steps"] < none["steps"]  # warmed question by question
    assert warmed < first["steps"]         # warm from the start
    assert first["hints"] > 0 and first["cutoffs"] > 0 and first["merges"] > 0


def test_merging_only_tightens_bounds(table_exe, positions):
    rng = np.random.default_rng(5)
    for p in positions[:6]:
        o, e, v = p["own"], p["enemy"], p["score"]
        legal = [a for a in range(64) if ob.find_correct_moves(o, e) >> a & 1]
        facts = []
        for _ in range(40):  # true facts in random order: "value >= t" is (v >= t)
            t = int(rng.integers(-64, 66))
            facts.append((t, int(v >= t), int(rng.choice(legal)) if v >= t else -1))
        cmds = []
        for t, r, mv in facts:
            cmds += [f"S {o:x} {e:x} {t} {r} {mv}", f"L {o:x} {e:x}"]
        out, _ = run(table_exe, cmds, 1)
        lo, hi, hint = -64, 64, -1
        for (t, r, mv), line in zip(facts, out):
            if r:
                lo, hint = max(lo, t), mv
            else:
                hi = min(hi, t - 1)
            assert line.split() == [str(lo), str(hi), str(hint)], (t, r, mv)
            assert lo <= v <= hi


def test_a_wrong_bound_changes_the_answer(table_exe, positions):
    p = next(p for p in positions if p["empties"] == 14)
    o, e, v = p["own"], p["enemy"], p["score"]
    truth, _ = run(table_exe, [q(o, e, v), q(o, e, v + 1)], 1 << 16)
    assert truth == ["1", "0"]
    # at the leaf's root: "value >= v + 1" stored as TRUE
    out, counts = run(table_exe, [f"S {o:x} {e:x} {v + 1} 1 -1", q(o, e, v + 1), "P"], 1 << 16)
    assert out == ["1"] and counts[0]["steps"] == 0 and counts[0]["cutoffs"] == 1
    # below it: a child where the opponent replies, stored as worth at most -(v + 1) to the opponent, so the move reaches v + 1
    for a in range(64):
        if ob.find_correct_moves(o, e) >> a & 1:
            fl = ob.calc_flip(a, o, e)
            o2, e2 = (o ^ fl) | (1 << a), e ^ fl
            if ob.find_correct_moves(e2, o2):
                break
    else:
        pytest.fail("no child with a reply")
    out, counts = run(table_exe, [f"S {e2:x} {o2:x} {-v} 0 -1", q(o, e, v + 1), "P"], 1 << 16)
    assert out == ["1"] and counts[0]["cutoffs"] >= 1
