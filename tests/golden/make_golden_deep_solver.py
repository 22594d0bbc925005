"""Generates tests/golden/deep_solver.json: seeded endgame positions with 13..20 empty squares and their exact answers
(move, score) from the host oracle tests/support/endgame_oracle.cu (plain negamax alpha-beta, first best square), for
the deep solver's GPU tests.  Every entry also lists the exact value of each root move, so the tags below can be checked.

Tags the set must cover: `tie` (two or more root moves reach the value), `zero` (value 0), `single` (one legal move),
`pass_child` (a root move leaves the opponent without a reply), `pass_deep` (a forced pass within the first three plies,
where the split works), `wipeout` (a line within the first three plies ends the game with empty squares left).

    python tests/golden/make_golden_deep_solver.py [out.json]
"""
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import bitboard as ob  # noqa: E402

REQUIRED = ("tie", "zero", "single", "pass_child", "pass_deep", "wipeout")


def build_oracle(out_dir):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    exe = os.path.join(out_dir, "endgame_oracle")
    subprocess.run([nvcc, "-O2", "-std=c++17", "--expt-relaxed-constexpr", "-Wno-deprecated-gpu-targets", "-I",
                    os.path.join(ROOT, "reversi-alpha-zero_b200", "csrc"), os.path.join(ROOT, "tests", "support", "endgame_oracle.cu"),
                    "-o", exe], check=True)
    return exe


def oracle_solve(exe, positions):
    """[(own, enemy)] -> [(move, score)]"""
    text = "".join(f"{o:x} {e:x}\n" for o, e in positions)
    r = subprocess.run([exe], input=text, capture_output=True, text=True, check=True)
    return [tuple(int(v) for v in line.split()) for line in r.stdout.strip().split("\n")] if positions else []


def children(own, enemy):
    """root moves ascending -> (square, own', enemy', negate): the child in the frame of whoever moves next, or
    (square, None, diff, None) when the game is over after the move"""
    out = []
    legal = ob.find_correct_moves(own, enemy)
    for a in range(64):
        if not legal >> a & 1:
            continue
        fl = ob.calc_flip(a, own, enemy)
        o2, e2 = (own ^ fl) | (1 << a), enemy ^ fl
        if ob.find_correct_moves(e2, o2):
            out.append((a, e2, o2, True))
        elif ob.find_correct_moves(o2, e2):
            out.append((a, o2, e2, False))
        else:
            out.append((a, None, ob.bit_count(o2) - ob.bit_count(e2), None))
    return out


def tags_of(own, enemy, move_values, value):
    tags = []
    if sum(1 for v in move_values.values() if v == value) > 1:
        tags.append("tie")
    if value == 0:
        tags.append("zero")
    if len(move_values) == 1:
        tags.append("single")
    kids = children(own, enemy)
    if any(neg is False for _, _, _, neg in kids):
        tags.append("pass_child")
    # forced passes and early game ends within three plies
    frontier, passes, wipe = [(own, enemy)], False, False
    for _ in range(3):
        nxt = []
        for o, e in frontier:
            for _, o2, e2, neg in children(o, e):
                if neg is None:
                    wipe |= 64 - ob.bit_count(o | e) - 1 > 0
                    continue
                passes |= neg is False
                nxt.append((o2, e2))
        frontier = nxt
    if passes:
        tags.append("pass_deep")
    if wipe:
        tags.append("wipeout")
    return tags


def random_position(rng, empties, greedy):
    """a seeded game down to `empties`; with `greedy` one side plays the move flipping most (lopsided boards)"""
    e = ob.Env().reset()
    while not e.done and 60 - e.turn > empties:
        o, en = e.own_enemy()
        legal = ob.find_correct_moves(o, en)
        ms = [i for i in range(64) if legal >> i & 1]
        if greedy and e.turn % 2 == 0:
            e.step(max(ms, key=lambda a: ob.bit_count(ob.calc_flip(a, o, en))))
        else:
            e.step(ms[rng.integers(len(ms))])
    if e.done:
        return None
    o, en = e.own_enemy()
    return (o, en) if ob.find_correct_moves(o, en) else None


def entry(exe, own, enemy):
    (move, score), = oracle_solve(exe, [(own, enemy)])
    kids = children(own, enemy)
    need = [(o2, e2) for _, o2, e2, neg in kids if neg is not None]
    vals = iter(oracle_solve(exe, need))
    move_values = {}
    for a, o2, e2, neg in kids:
        if neg is None:
            move_values[a] = e2
        else:
            _, s = next(vals)
            move_values[a] = -s if neg else s
    value = max(move_values.values())
    assert value == score and move == min(a for a, v in move_values.items() if v == value), (hex(own), hex(enemy))
    return dict(own=own, enemy=enemy, empties=64 - ob.bit_count(own | enemy), move=move, score=score,
                move_values={str(a): v for a, v in sorted(move_values.items())}, tags=tags_of(own, enemy, move_values, value))


def candidates(rng, empties, n):
    out, tries = [], 0
    while len(out) < n:
        tries += 1
        pos = random_position(rng, empties, greedy=tries % 3 == 0)
        if pos is not None and pos not in out:
            out.append(pos)
    return out


def main(out):
    from multiprocessing import Pool
    tmp = tempfile.mkdtemp()
    exe = build_oracle(tmp)
    rng = np.random.default_rng(2026)
    # 7 positions per empty count, then positions at 13..16 empties while a required tag is still missing
    base = [(exe, *p) for k in range(13, 21) for p in candidates(rng, k, 7)]
    extra = [(exe, *p) for k in range(13, 17) for p in candidates(rng, k, 40)]
    with Pool(os.cpu_count()) as pool:
        entries = pool.starmap(entry, base)
        covered = {t for e in entries for t in e["tags"]}
        seen = {(e["own"], e["enemy"]) for e in entries}
        for ent in pool.starmap(entry, [c for c in extra if (c[1], c[2]) not in seen]):
            if (set(ent["tags"]) - covered) & set(REQUIRED):
                entries.append(ent)
                covered |= set(ent["tags"])
    for ent in entries:
        print(f"empties {ent['empties']} move {ent['move']:2d} score {ent['score']:3d} {ent['tags']}")
    missing = set(REQUIRED) - covered
    assert not missing, missing
    with open(out, "w") as f:
        json.dump(dict(generator="tests/golden/make_golden_deep_solver.py", oracle="tests/support/endgame_oracle.cu",
                       positions=entries), f, indent=1)
    shutil.rmtree(tmp)


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(os.path.abspath(__file__)), "deep_solver.json"))
