"""CPU suite of the growing opening book: the children step compiled for the host (tests/support/book_children_check.cu)
against a Python restatement over lib/bitboard.py; best-first growth and game learning with the host twins and a stand-in
searcher (a deterministic function of the canonical key); the book file with `levels`; the YAML keys; NBoard's `learn`
with a stand-in book and searcher; the C ABI.  No GPU needed."""
import ctypes as C
import json
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from reversi_zero_b200 import _cabi
from reversi_zero_b200.config import create_config, load_yaml
from reversi_zero_b200.lib import bitboard as bb, book as BK, openings as OP
from reversi_zero_b200.lib.ggf import convert_action_to_move, make_ggf_string
from test_book_host import graph_exe, run_graph, py_levels, child_of, negamax, stand_in_engine, session, START  # noqa: F401
from test_openings_host import forcing_pass_sequence

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "reversi-alpha-zero_b200", "csrc")
MASK = (1 << 64) - 1


@pytest.fixture(scope="module")
def children_exe(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("book_children_check") / "book_children_check")
    subprocess.run([nvcc, "-O2", "-std=c++17", "--expt-relaxed-constexpr", "-Wno-deprecated-gpu-targets", "-I", CSRC,
                    os.path.join(ROOT, "tests", "support", "book_children_check.cu"), "-o", exe], check=True)
    return exe


def twin(exe):
    """BK.book_children's signature over the host twin"""
    def children(own, enemy, next_hi, next_lo):
        text = f"{len(own)} {len(next_hi)}\n" + "".join(f"{int(o)} {int(e)}\n" for o, e in zip(own, enemy)) + \
               "".join(f"{int(h)} {int(l)}\n" for h, l in zip(next_hi, next_lo))
        out = subprocess.run([exe], input=text, capture_output=True, text=True, check=True).stdout
        offset, rows = [0], []
        for line in filter(None, out.split("\n")):
            v = [int(x) for x in line.split()]
            offset.append(offset[-1] + v[0])
            rows += [v[1 + 7 * j:8 + 7 * j] for j in range(v[0])]
        r = np.array(rows, dtype=object).reshape(-1, 7)
        return BK.Children(np.array(offset, np.uint64), r[:, 0].astype(np.uint8), r[:, 1].astype(np.int32),
                           r[:, 3].astype(np.uint64), r[:, 4].astype(np.uint64), r[:, 5].astype(np.uint64),
                           r[:, 6].astype(np.uint64), r[:, 2].astype(np.uint8))
    return children


def py_children(own, enemy, keys):
    """the children step restated: [(square, index in `keys` or -1, kind, child own, child enemy, key hi, key lo)]"""
    index = {k: j for j, k in enumerate(keys)}
    row = []
    for sq in range(64):
        if (bb.find_correct_moves(own, enemy) >> sq) & 1:
            co, ce = child_of(own, enemy, sq)
            kind = BK.KEPT if bb.find_correct_moves(co, ce) else BK.PASS if bb.find_correct_moves(ce, co) else BK.OVER
            k = OP.canonical_key(co, ce)
            row.append((sq, index.get(k, -1) if kind == BK.KEPT else -1, kind, co, ce) + k)
    return row


def rows_of(ch):
    off = ch.edge_offset.astype(np.int64)
    cols = (ch.edge_square, ch.edge_child, ch.child_kind, ch.child_own, ch.child_enemy, ch.child_hi, ch.child_lo)
    return [list(zip(*(c[off[i]:off[i + 1]].tolist() for c in cols))) for i in range(len(off) - 1)]


def check_children(children, own, enemy, keys):
    keys = sorted(keys)
    hi = np.array([k[0] for k in keys], np.uint64)
    lo = np.array([k[1] for k in keys], np.uint64)
    got = rows_of(children(np.array(own, np.uint64), np.array(enemy, np.uint64), hi, lo))
    assert got == [py_children(o, e, keys) for o, e in zip(own, enemy)]
    return got


def test_children_twin_on_levels_0_to_6(children_exe):
    children = twin(children_exe)
    levels = py_levels(6)
    for lv in range(6):
        nxt = [OP.canonical_key(o, e) for o, e in levels[lv + 1]]
        got = check_children(children, [p[0] for p in levels[lv]], [p[1] for p in levels[lv]], nxt)
        assert all(c >= 0 for row in got for _, c, kind, *_ in row if kind == BK.KEPT)   # a full level: every kept child found
    last = levels[6]
    check_children(children, [p[0] for p in last], [p[1] for p in last], [])   # no level: every index -1


def random_positions(seed, count):
    """positions of seeded random games at 10..40 discs, mover's frame, with a legal move"""
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < count:
        own, enemy = START
        target = int(rng.integers(10, 41))
        while bb.bit_count(own | enemy) < target:
            legal = [s for s in range(64) if (bb.find_correct_moves(own, enemy) >> s) & 1]
            if not legal:
                own, enemy = enemy, own
                if not bb.find_correct_moves(own, enemy):
                    break
                continue
            own, enemy = child_of(own, enemy, int(rng.choice(legal)))
        if bb.find_correct_moves(own, enemy):
            out.append((own, enemy))
    return out


def test_children_twin_on_random_positions_and_partial_levels(children_exe):
    children = twin(children_exe)
    pos = random_positions(3, 120)
    rng = np.random.default_rng(4)
    kids = sorted({r[5:] for o, e in pos for r in py_children(o, e, []) if r[2] == BK.KEPT})
    part = [k for k in kids if rng.random() < 0.5] + [(1, 2), (MASK, MASK)]   # some children, and keys of no child
    got = check_children(children, [p[0] for p in pos], [p[1] for p in pos], part)
    found = [c for row in got for _, c, kind, *_ in row if kind == BK.KEPT]
    assert min(found) == -1 and max(found) >= 0


def test_children_twin_marks_pass_and_game_over(children_exe):
    children = twin(children_exe)
    seq, passes = forcing_pass_sequence()
    own, enemy = START
    for a in seq[:-1]:
        own, enemy = child_of(own, enemy, a)
    # a move into a lone enemy disc ends the game: the new mover has no disc, and the other side no move
    over = (1 << 0, 1 << 1)
    got = check_children(children, [own, over[0]], [enemy, over[1]], [OP.canonical_key(*child_of(own, enemy, seq[-1]))])
    assert dict((r[0], (r[1], r[2])) for r in got[0])[seq[-1]] == (-1, BK.PASS if passes else BK.OVER)
    assert got[1] == [(2, -1, BK.OVER, 0, 7, 0, 7)]
    # no nodes: an empty CSR
    assert len(children(np.zeros(0, np.uint64), np.zeros(0, np.uint64), np.zeros(0, np.uint64), np.zeros(0, np.uint64)).edge_offset) == 1


def key_value(hi, lo):
    """the stand-in searcher's value of a canonical key, in (-1, 1)"""
    x = ((hi * 0x9E3779B97F4A7C15) ^ (lo * 0xC2B2AE3D27D4EB4F)) & MASK
    x ^= x >> 29
    return ((x * 0xBF58476D1CE4E5B9 & MASK) >> 11) / 2.0 ** 52 - 1.0


class KeySearch:
    """a searcher whose value is key_value of the canonical key (quantised to halves with ties=True); records its calls"""

    def __init__(self, ties=False):
        self.ties = ties
        self.calls = []

    def value(self, hi, lo):
        v = key_value(hi, lo)
        return float(np.round(v * 2) / 2) if self.ties else v

    def __call__(self, own, enemy):
        self.calls.append((np.array(own), np.array(enemy)))
        return np.array([self.value(*OP.canonical_key(int(o), int(e))) for o, e in zip(own, enemy)])

    def close(self):
        pass


def meta(plies):
    return dict(plies=plies, simulation_num_per_move=40, seed=1, model_sha256="ab" * 32, model={}, format_version=BK.FORMAT_VERSION)


def full_book(graph_exe, plies, search):
    g = run_graph(graph_exe, plies)
    flags = BK.node_flags(g)
    searched = np.array([search.value(int(h), int(l)) for h, l in zip(g.key_hi, g.key_lo)])
    return g, BK.Book(g.key_hi, g.key_lo, BK.backup(g, flags, searched), flags, g.level_counts, meta(plies))


def test_links_of_a_full_width_book_are_its_graph(graph_exe, children_exe):
    g, book = full_book(graph_exe, 5, KeySearch())
    links = BK.book_links(book, twin(children_exe))
    for name in BK.Graph._fields:
        assert np.array_equal(getattr(links, name), getattr(g, name)), name


def test_growth_by_whole_frontiers_is_the_full_width_book(graph_exe, children_exe):
    search = KeySearch()
    g6, want = full_book(graph_exe, 6, search)
    first = BK.level_starts(g6.level_counts)
    assert (want.flags[:first[6]] == BK.INTERIOR).all()   # no incomplete node in this range
    _, book = full_book(graph_exe, 3, search)
    children = twin(children_exe)
    grown = BK.grow(book, 10 ** 6, 10 ** 6, 6, 0.0, children, search)
    for k in ("keys_hi", "keys_lo", "flags", "values", "level_counts"):
        assert np.array_equal(getattr(grown, k), getattr(want, k)), k
    assert grown.plies == 3 and grown.levels == 7 and grown.meta["levels"] == 7
    # three rounds, each the next level, each searched in the enumerator's orientation
    assert [c[0].size for c in search.calls] == [int(x) for x in g6.level_counts[4:]]
    for lv, (own, enemy) in zip((4, 5, 6), search.calls):
        assert np.array_equal(own, g6.own[first[lv]:first[lv + 1]]) and np.array_equal(enemy, g6.enemy[first[lv]:first[lv + 1]])


def py_select(book, positions, count, max_level, cost):
    """the priority restated: d over INTERIOR parents by recursion over bitboard moves, then sorted tuples"""
    first = BK.level_starts(book.level_counts)
    d = {0: 0.0}
    for node in range(int(first[-1])):
        if node not in d or book.flags[node] != BK.INTERIOR:
            continue
        own, enemy = positions[node]
        for sq in range(64):
            if (bb.find_correct_moves(own, enemy) >> sq) & 1:
                c = book.find(*child_of(own, enemy, sq))
                d[c] = min(d.get(c, np.inf), d[node] + book.values[node] + book.values[c])
    level = lambda i: int(np.searchsorted(first, i, "right")) - 1
    cand = [i for i in d if book.flags[i] == BK.LEAF and level(i) < max_level]
    cand.sort(key=lambda i: (d[i] + cost * (level(i) - book.plies), level(i), int(book.keys_hi[i]), int(book.keys_lo[i])))
    return cand[:count]


def test_rounds_pick_the_priority_with_ties(graph_exe, children_exe):
    search = KeySearch(ties=True)
    _, book = full_book(graph_exe, 2, search)
    children = twin(children_exe)
    rounds = 0
    for cost in (0.0, 0.5):
        b = book
        for _ in range(5):
            graph = BK.book_links(b, children)
            d = BK.deviation(graph, b.flags, b.values)
            pick = BK.select_leaves(b, d, 4, 5, cost)
            assert pick.tolist() == py_select(b, list(zip(graph.own.tolist(), graph.enemy.tolist())), 4, 5, cost)
            if not pick.size:
                break
            b, _ = BK.grow_round(b, graph.own[pick], graph.enemy[pick], b.keys_hi[pick], b.keys_lo[pick], children, search)
            rounds += 1
        assert b.levels > 3
    assert rounds == 10


def test_backup_of_a_grown_book_is_negamax(graph_exe, children_exe):
    search = KeySearch()
    _, book = full_book(graph_exe, 3, search)
    children = twin(children_exe)
    grown = BK.grow(book, 60, 7, 9, 0.3, children, search)
    assert grown.levels > 5 and (grown.flags != BK.LEAF).sum() == (book.flags != BK.LEAF).sum() + 60
    graph = BK.book_links(grown, children)
    searched = grown.values.copy()
    searched[grown.flags == BK.INTERIOR] = np.nan
    assert np.array_equal(grown.values, np.array(negamax(graph, grown.flags, searched)))
    # a leaf's value is its search
    leaves = np.nonzero(grown.flags == BK.LEAF)[0]
    assert np.array_equal(grown.values[leaves], [search.value(int(grown.keys_hi[i]), int(grown.keys_lo[i])) for i in leaves])


def random_game(seed, plies=60):
    """a seeded random game from the initial position: its moves, with None for a pass, until the game ends"""
    rng = np.random.default_rng(seed)
    own, enemy = START
    moves = []
    while len(moves) < plies:
        legal = [s for s in range(64) if (bb.find_correct_moves(own, enemy) >> s) & 1]
        if not legal:
            if not bb.find_correct_moves(enemy, own):
                break
            moves.append(None)
            own, enemy = enemy, own
            continue
        a = int(rng.choice(legal))
        moves.append(a)
        own, enemy = child_of(own, enemy, a)
    return moves


def game_positions(moves):
    own, enemy = START
    out = [(own, enemy)]
    for a in moves:
        if a is None:
            break
        own, enemy = child_of(own, enemy, a)
        if not bb.find_correct_moves(own, enemy):
            break
        out.append((own, enemy))
    return out


def test_learn_game(graph_exe, children_exe):
    search = KeySearch()
    _, book = full_book(graph_exe, 3, search)
    children = twin(children_exe)
    for seed in range(40):   # a game without a pass before its 20th move
        moves = random_game(seed)
        if None not in moves[:20]:
            break
    learned, k = BK.learn_game(book, moves, 12, children, search)
    assert k == 9 and learned.levels == 13 and learned.meta["levels"] == 13 and learned.plies == 3
    for level, (o, e) in enumerate(game_positions(moves)[:13]):
        i = learned.find(o, e)
        assert i is not None
        if level < 12:
            assert learned.flags[i] != BK.LEAF
            assert learned.moves(o, e) is not None or learned.flags[i] == BK.INCOMPLETE
    # untouched nodes keep their values; only expanded nodes and their ancestors (through the backup) change
    for i in range(book.values.size):
        j = learned.key_index(int(np.searchsorted(book.first, i, "right")) - 1, int(book.keys_hi[i]), int(book.keys_lo[i]))
        if learned.flags[j] == BK.LEAF:
            assert learned.values[j] == book.values[i]
        elif book.flags[i] == BK.LEAF:
            assert level_of(learned, j) == 3
    # learning the same game again changes nothing and searches nothing
    n_calls = len(search.calls)
    again, k2 = BK.learn_game(learned, moves, 12, children, search)
    assert k2 == 0 and again is learned and len(search.calls) == n_calls
    # a game from another start is skipped
    same, k3 = BK.learn_game(book, moves, 12, children, search, start=(START[0], START[1], 2))
    assert same is book and k3 == 0
    assert BK.learn_game(book, moves, 12, children, search, start=(START[0], START[1], 1))[1] == 9


def level_of(book, i):
    return int(np.searchsorted(book.first, i, "right")) - 1


def test_learn_stops_at_a_pass(graph_exe, children_exe):
    search = KeySearch()
    _, book = full_book(graph_exe, 3, search)
    seq, _ = forcing_pass_sequence()
    learned, k = BK.learn_game(book, seq + [None] * 3, 30, twin(children_exe), search)
    path = game_positions(seq)
    assert len(path) == len(seq) and k == len(seq) - 3
    assert learned.flags[learned.find(*path[-1])] == BK.INCOMPLETE
    assert learned.find(*child_of(*path[-1], seq[-1])) is None and learned.levels == len(seq) + 1


def test_file_round_trip_with_levels_and_refusals(graph_exe, children_exe, tmp_path):
    search = KeySearch()
    _, book = full_book(graph_exe, 3, search)
    grown = BK.grow(book, 30, 10, 7, 0.0, twin(children_exe), search)
    p = str(tmp_path / "g.npz")
    BK.save_book(p, grown)
    back = BK.load_book(p)
    for k in ("keys_hi", "keys_lo", "values", "flags", "level_counts"):
        assert np.array_equal(getattr(back, k), getattr(grown, k))
    assert back.meta == grown.meta and back.levels == grown.levels == grown.meta["levels"] and back.plies == 3
    deep = [p for p in game_positions(random_game(1)) if bb.bit_count(p[0] | p[1]) - 4 > 3]
    assert all(back.moves(*q) == grown.moves(*q) for q in deep)

    def write(name, **changes):
        m = dict(grown.meta)
        m.update(changes.pop("meta", {}))
        arrays = dict(keys_hi=grown.keys_hi, keys_lo=grown.keys_lo, values=grown.values, flags=grown.flags,
                      level_counts=grown.level_counts)
        arrays.update(changes)
        q = str(tmp_path / name)
        with open(q, "wb") as f:
            np.savez(f, meta=np.array(json.dumps({k: v for k, v in m.items() if v is not None})), **arrays)
        return q
    n = int(grown.level_counts[-1])
    cases = {write("l42.npz", meta=dict(levels=42)): "42 levels for a book of 3 plies",
             write("l2.npz", meta=dict(levels=2)): "2 levels for a book of 3 plies",
             write("lx.npz", meta=dict(levels=grown.levels + 1)): "inconsistent array lengths",
             write("none.npz", meta=dict(levels=None)): "inconsistent array lengths",
             write("short.npz", level_counts=grown.level_counts[:-1], keys_hi=grown.keys_hi[:-n], keys_lo=grown.keys_lo[:-n],
                   values=grown.values[:-n], flags=grown.flags[:-n]): "inconsistent array lengths"}
    for q, why in cases.items():
        with pytest.raises(ValueError, match=re.escape(q) + ".*" + why):
            BK.load_book(q)
    # a full-width book is written as before: no levels entry, and it loads and answers as it did
    q = str(tmp_path / "full.npz")
    BK.save_book(q, book)
    with np.load(q) as z:
        assert sorted(z.files) == ["flags", "keys_hi", "keys_lo", "level_counts", "meta", "values"]
        assert "levels" not in json.loads(str(z["meta"]))
    old = BK.load_book(q)
    assert old.levels == 4 and old.plies == 3 and old.moves(*START) == book.moves(*START)
    # a grown 3-ply book still scores only 3-ply openings
    with pytest.raises(ValueError, match="a book of 3 plies cannot score openings of 4 plies"):
        OP.book_suite(back, 4, 10, 0.2, 1)


def test_yaml_keys_reach_consumers(tmp_path):
    import yaml
    p = tmp_path / "c.yml"
    p.write_text(yaml.safe_dump(dict(book=dict(extend=True, grow_nodes=500, grow_batch=32, max_level=30, grow_depth_cost=0.25,
                                               learn=["games/*.ggf"]), b200=dict(nboard_book_learn=True))))
    cfg = load_yaml(str(p), project_dir=str(tmp_path))
    assert [BK._field(cfg, k, None) for k in ("extend", "grow_nodes", "grow_batch", "max_level", "grow_depth_cost", "learn")] == \
           [True, 500, 32, 30, 0.25, ["games/*.ggf"]]
    assert cfg.b200.nboard_book_learn is True
    d = create_config(project_dir=str(tmp_path))
    assert (d.book.extend, d.book.grow_nodes, d.book.grow_batch, d.book.max_level, d.book.grow_depth_cost, d.book.learn) == \
           (False, 0, 256, 40, 0.0, None)
    assert d.b200.nboard_book_learn is False
    # learn: every game of every matching file, several games to a file, in sorted file order
    os.makedirs(tmp_path / "games")
    g1, g2 = random_game(5), random_game(6)
    text = lambda g: make_ggf_string(moves=[convert_action_to_move(a) for a in g])
    (tmp_path / "games" / "b.ggf").write_text(text(g1) + "\n" + text(g2) + "\n")
    (tmp_path / "games" / "a.ggf").write_text(text(g2))
    games = BK.learn_files(str(tmp_path), cfg.book.learn)
    assert [(s, m) for s, m in games] == [((START[0], START[1], 1), g) for g in (g2, g1, g2)]
    assert all(BK.is_start(s) for s, _ in games)
    # extend refuses another model or simulation count, naming the file
    book = BK.Book([0], [0], [0.0], [BK.LEAF], [1], meta(0), path="x/book.npz")
    BK.check_extend(book, "ab" * 32, 40)
    with pytest.raises(ValueError, match="x/book.npz: the book was searched with model abababab"):
        BK.check_extend(book, "cd" * 32, 40)
    with pytest.raises(ValueError, match="x/book.npz: the book was searched with 40 simulations per position, not 50"):
        BK.check_extend(book, "ab" * 32, 50)


def test_nboard_learn(graph_exe, children_exe, tmp_path, monkeypatch):
    search = KeySearch()
    _, book = full_book(graph_exe, 3, search)
    path = str(tmp_path / "book.npz")
    BK.save_book(path, book)
    monkeypatch.setattr(BK, "book_children", twin(children_exe))
    moves = random_game(2)[:14]
    assert None not in moves
    played = [f"move {convert_action_to_move(a)}" for a in moves]
    for knob in (False, True):
        eng = stand_in_engine(BK.load_book(path))
        eng.config.b200.nboard_book_learn = knob
        eng.book_searcher = lambda: search
        before = open(path, "rb").read()
        assert session(eng, played + ["learn"]) == ["learned"]
        if not knob:
            assert open(path, "rb").read() == before and eng.book.levels == 4
            continue
        disk = BK.load_book(path)
        # every position of the game is expanded, the last one included: its children make level 15
        assert disk.levels == 16 and eng.book.levels == 16 and np.array_equal(disk.values, eng.book.values)
        path_nodes = [disk.find(o, e) for o, e in game_positions(moves)]
        assert len(path_nodes) == 15 and None not in path_nodes and all(disk.flags[i] != BK.LEAF for i in path_nodes)
        # learning the game again leaves the file as it is
        mtime = os.stat(path).st_mtime_ns
        assert session(eng, ["learn"]) == ["learned"] and os.stat(path).st_mtime_ns == mtime
    # a fresh engine plays the grown book along the game, beyond its full width
    eng = stand_in_engine(BK.load_book(path))
    deep = [k for k in range(4, 15) if disk.flags[path_nodes[k]] == BK.INTERIOR]
    assert deep
    for k in deep:
        own, enemy = game_positions(moves)[k]
        eng2 = stand_in_engine(disk)
        session(eng2, played[:k])
        go = session(eng2, ["go"])
        sq, v = disk.best(own, enemy)
        assert go[1].startswith(f"=== {convert_action_to_move(sq)}/{v * 10}/") and eng2.player.searches == []
    assert eng.book.levels == 16


def test_abi():
    hdr = open(os.path.join(ROOT, "include", "rz_engine.h")).read()
    assert re.search(r"int rz_openings_book_children\(const uint64_t\* own, const uint64_t\* enemy, size_t n, const uint64_t\* next_hi,\s+"
                     r"const uint64_t\* next_lo, size_t n_next, uint64_t\* edge_offset, uint8_t\* edge_square,\s+"
                     r"int32_t\* edge_child, uint64_t\* child_own, uint64_t\* child_enemy, uint64_t\* child_hi,\s+"
                     r"uint64_t\* child_lo, uint8_t\* child_kind, size_t cap_edges, size_t\* n_edges\);", hdr)
    assert "rz_openings_book_children" in _cabi.SIGNATURES and hasattr(_cabi.lib(), "rz_openings_book_children")
    assert len(_cabi.SIGNATURES["rz_openings_book_children"][1]) == 16
    lib = _cabi.lib()
    m = C.c_size_t()
    one = np.array([START[0]], np.uint64)
    assert lib.rz_openings_book_children(None, None, 0, None, None, 0, None, None, None, None, None, None, None, None, 0, None) == -1
    assert lib.rz_openings_book_children(None, None, 1, None, None, 0, None, None, None, None, None, None, None, None, 0, C.byref(m)) == -1
    assert lib.rz_openings_book_children(one.ctypes.data_as(_cabi.u64p), one.ctypes.data_as(_cabi.u64p), 1, None, None, 3,
                                         None, None, None, None, None, None, None, None, 0, C.byref(m)) == -1
