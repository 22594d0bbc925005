"""CPU suite of the opening book: the book graph's edge step compiled for the host (tests/support/book_graph_check.cu)
against a Python restatement over lib/bitboard.py; the minimax backup against a recursive negamax; Book.moves under the
8 symmetries; the book file and its refusals; the YAML keys; NBoard's go and hint with a stand-in book; the C ABI.
No GPU needed."""
import ctypes as C
import io
import os
import re
import shutil
import subprocess
import types

import numpy as np
import pytest

from reversi_zero_b200 import _cabi
from reversi_zero_b200.config import Config, create_config, load_yaml
from reversi_zero_b200.env.reversi_env import ReversiEnv, Player
from reversi_zero_b200.lib import bitboard as bb, book as BK, openings as OP
from reversi_zero_b200.lib.ggf import convert_action_to_move
from reversi_zero_b200.lib.nonblocking_stream_reader import NonBlockingStreamReader
from reversi_zero_b200.play_game import nboard as NB
from test_openings_host import forcing_pass_sequence

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "reversi-alpha-zero_b200", "csrc")
START = (0x10 << 24) | (0x08 << 32), (0x08 << 24) | (0x10 << 32)


@pytest.fixture(scope="module")
def graph_exe(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    exe = str(tmp_path_factory.mktemp("book_graph_check") / "book_graph_check")
    subprocess.run([nvcc, "-O2", "-std=c++17", "--expt-relaxed-constexpr", "-Wno-deprecated-gpu-targets", "-I", CSRC,
                    os.path.join(ROOT, "tests", "support", "book_graph_check.cu"), "-o", exe], check=True)
    return exe


def run_graph(exe, plies, root=None):
    """-> BK.Graph as the host twin prints it (keys by lib/openings.canonical_key)"""
    args = [exe, str(plies)] + ([str(root[0]), str(root[1])] if root else [])
    lines = subprocess.run(args, capture_output=True, text=True, check=True).stdout.split("\n")
    counts = [int(x) for x in lines[0].split()[1:]]
    own, enemy, offset, square, child = [], [], [0], [], []
    for line in filter(None, lines[1:]):
        v = [int(x) for x in line.split()]
        own.append(v[0])
        enemy.append(v[1])
        square += v[3::2]
        child += v[4::2]
        offset.append(offset[-1] + v[2])
    keys = np.array([OP.canonical_key(o, e) for o, e in zip(own, enemy)], np.uint64).reshape(-1, 2)
    return BK.Graph(np.array(own, np.uint64), np.array(enemy, np.uint64), keys[:, 0].copy(), keys[:, 1].copy(),
                    np.array(counts, np.uint64), np.array(offset, np.uint64), np.array(square, np.uint8), np.array(child, np.int32))


def child_of(own, enemy, sq):
    fl = bb.calc_flip(sq, own, enemy)
    return enemy ^ fl, own | fl | (1 << sq)


def py_levels(plies, root=START):
    """the enumerator restated from `root` (test_openings_host.py_enumerate): every level's representatives"""
    levels = [[root]]
    for _ in range(plies):
        best = {}
        for own, enemy in levels[-1]:
            for sq in range(64):
                if (bb.find_correct_moves(own, enemy) >> sq) & 1:
                    co, ce = child_of(own, enemy, sq)
                    if bb.find_correct_moves(co, ce):
                        best.setdefault(OP.canonical_key(co, ce), (co, ce))
        levels.append([best[k] for k in sorted(best)])
    return levels


def py_edges(levels):
    """per node below the last level: [(square, index of the child's class in the next level, or -1)]"""
    out = []
    for lv in range(len(levels) - 1):
        index = {OP.canonical_key(o, e): j for j, (o, e) in enumerate(levels[lv + 1])}
        for own, enemy in levels[lv]:
            row = []
            for sq in range(64):
                if (bb.find_correct_moves(own, enemy) >> sq) & 1:
                    co, ce = child_of(own, enemy, sq)
                    row.append((sq, index[OP.canonical_key(co, ce)] if bb.find_correct_moves(co, ce) else -1))
            out.append(row)
    return out + [[] for _ in levels[-1]]


def graph_rows(g):
    off = g.edge_offset.astype(np.int64)
    return [list(zip(g.edge_square[off[i]:off[i + 1]].tolist(), g.edge_child[off[i]:off[i + 1]].tolist()))
            for i in range(len(g.own))]


@pytest.mark.parametrize("plies", range(0, 7))
def test_graph_host_twin_matches_python(graph_exe, plies):
    g = run_graph(graph_exe, plies)
    levels = py_levels(plies)
    assert g.level_counts.tolist() == [len(lv) for lv in levels]
    assert list(zip(g.own.tolist(), g.enemy.tolist())) == [p for lv in levels for p in lv]
    assert graph_rows(g) == py_edges(levels)
    first = BK.level_starts(g.level_counts)
    for p in range(1, plies + 1):   # level p is the enumerator's output for p plies
        _, frontier = __import__("test_openings_host").py_enumerate(p)
        assert list(zip(g.own[first[p]:first[p + 1]].tolist(), g.enemy[first[p]:first[p + 1]].tolist())) == \
               [(o, e) for o, e, _ in frontier]


def pass_root():
    """the position before the last move of the shortest sequence after which the mover must pass or the game ends"""
    seq, _ = forcing_pass_sequence()
    own, enemy = START
    for a in seq[:-1]:
        own, enemy = child_of(own, enemy, a)
    return (own, enemy), seq[-1]


def test_graph_marks_pass_and_game_over_children(graph_exe):
    root, last = pass_root()
    g = run_graph(graph_exe, 2, root)
    levels = py_levels(2, root)
    assert graph_rows(g) == py_edges(levels)
    rows = graph_rows(g)
    assert dict(rows[0])[last] == -1    # the pass child
    for i, (own, enemy) in enumerate(p for lv in levels[:-1] for p in lv):
        for sq, c in rows[i]:
            assert (c == -1) == (bb.find_correct_moves(*child_of(own, enemy, sq)) == 0)
    assert BK.node_flags(g)[0] == BK.INCOMPLETE


def negamax(g, flags, searched):
    first = BK.level_starts(g.level_counts)
    off = g.edge_offset.astype(np.int64)

    def v(level, i):
        node = first[level] + i
        if flags[node] != BK.INTERIOR:
            return searched[node]
        return max(-v(level + 1, int(c)) for c in g.edge_child[off[node]:off[node + 1]])
    return [v(lv, i) for lv in range(len(first) - 1) for i in range(int(g.level_counts[lv]))]


def test_backup_matches_negamax(graph_exe):
    rng = np.random.default_rng(3)
    g = run_graph(graph_exe, 4)
    # incomplete nodes: some edges of levels 1..3 marked -1 by hand, and a graph with a real pass
    child = g.edge_child.copy()
    first = BK.level_starts(g.level_counts)
    off = g.edge_offset.astype(np.int64)
    for node in rng.choice(np.arange(first[1], first[4]), 12, replace=False):
        child[off[node] + rng.integers(0, off[node + 1] - off[node])] = -1
    for graph in (g, g._replace(edge_child=child), run_graph(graph_exe, 3, pass_root()[0])):
        flags = BK.node_flags(graph)
        n = len(graph.own)
        searched = rng.uniform(-1, 1, n)
        searched[flags == BK.INTERIOR] = np.nan   # never read
        values = BK.backup(graph, flags, searched)
        assert np.array_equal(values, np.array(negamax(graph, flags, searched)))
        assert np.isfinite(values).all()
    assert (BK.node_flags(g._replace(edge_child=child)) == BK.INCOMPLETE).sum() >= 1


def make_book(exe, plies, rng, ties=False):
    g = run_graph(exe, plies)
    flags = BK.node_flags(g)
    searched = rng.choice([-0.5, 0.0, 0.5], len(g.own)) if ties else rng.uniform(-1, 1, len(g.own))
    values = BK.backup(g, flags, searched)
    meta = dict(plies=plies, simulation_num_per_move=40, seed=1, model_sha256="ab" * 32, model={}, format_version=BK.FORMAT_VERSION)
    return g, BK.Book(g.key_hi, g.key_lo, values, flags, g.level_counts, meta)


def square_map(t):
    return [int(bb.dihedral(1 << sq, t)).bit_length() - 1 for sq in range(64)]


def test_book_moves_under_symmetries(graph_exe):
    rng = np.random.default_rng(5)
    for ties in (False, True):
        g, book = make_book(graph_exe, 5, rng, ties)
        first = BK.level_starts(g.level_counts)
        off = g.edge_offset.astype(np.int64)
        sample = list(range(int(first[3]))) + rng.choice(np.arange(first[3], first[5]), 20, replace=False).tolist()
        for node in sample:
            own, enemy = int(g.own[node]), int(g.enemy[node])
            level = int(np.searchsorted(first, node, "right") - 1)
            mv = book.moves(own, enemy)
            want = [(int(s), -float(book.values[first[level + 1] + c]))
                    for s, c in zip(g.edge_square[off[node]:off[node + 1]], g.edge_child[off[node]:off[node + 1]])]
            assert mv == want
            for t in range(8):
                m = square_map(t)
                o, e = bb.dihedral(own, t), bb.dihedral(enemy, t)
                got = book.moves(o, e)
                assert sorted(got) == sorted((m[s], v) for s, v in mv)
                best = book.best(o, e)
                assert best[1] == max(v for _, v in got) and best[0] == min(s for s, v in got if v == best[1])
        # leaves and positions outside the book
        assert book.moves(int(g.own[-1]), int(g.enemy[-1])) is None
        assert book.moves(*child_of(int(g.own[-1]), int(g.enemy[-1]), min(s for s in range(64) if (bb.find_correct_moves(int(g.own[-1]), int(g.enemy[-1])) >> s) & 1))) is None


def test_turn_zero_is_the_forced_first_move(graph_exe):
    _, book = make_book(graph_exe, 3, np.random.default_rng(1))
    mv = book.moves(*START)
    legal = [s for s in range(64) if (bb.find_correct_moves(*START) >> s) & 1]
    assert [s for s, _ in mv] == legal and len({v for _, v in mv}) == 1   # one class
    assert book.best(*START)[0] == min(legal) == 19


def test_symmetric_positions(graph_exe):
    """a position equal to some of its images answers the same, whichever image is queried"""
    _, book = make_book(graph_exe, 4, np.random.default_rng(2), ties=True)
    seen = 0
    for own, enemy in [START] + [p for p in py_levels(2)[2]]:
        for t in range(8):
            if (bb.dihedral(own, t), bb.dihedral(enemy, t)) == (own, enemy):
                seen += t > 0
                assert book.moves(bb.dihedral(own, t), bb.dihedral(enemy, t)) == book.moves(own, enemy)
    assert seen >= 3


def test_file_round_trip_and_refusals(graph_exe, tmp_path):
    _, book = make_book(graph_exe, 3, np.random.default_rng(4))
    p = str(tmp_path / "b" / "book.npz")
    BK.save_book(p, book)
    assert not os.path.exists(p + ".tmp")
    back = BK.load_book(p)
    for k in ("keys_hi", "keys_lo", "values", "flags", "level_counts"):
        assert np.array_equal(getattr(back, k), getattr(book, k))
    assert back.meta == book.meta and back.moves(*START) == book.moves(*START)

    def write(name, **changes):
        arrays = dict(keys_hi=book.keys_hi, keys_lo=book.keys_lo, values=book.values, flags=book.flags,
                      level_counts=book.level_counts)
        meta = dict(book.meta)
        meta.update(changes.pop("meta", {}))
        arrays.update(changes)
        q = str(tmp_path / name)
        with open(q, "wb") as f:
            np.savez(f, meta=np.array(__import__("json").dumps(meta)), **arrays)
        return q
    hi = book.keys_hi.copy()
    hi[[6, 7]] = hi[[7, 6]]   # two keys of level 3 swapped
    cases = {write("v.npz", meta=dict(format_version=99)): "format version 99",
             write("n.npz", values=book.values[:-1]): "inconsistent array lengths",
             write("c.npz", level_counts=book.level_counts[:-1]): "inconsistent array lengths",
             write("o.npz", keys_hi=hi): "keys out of order in level 3"}
    for q, why in cases.items():
        with pytest.raises(ValueError, match=re.escape(q) + ".*" + why):
            BK.load_book(q)


def test_yaml_keys_reach_consumers(tmp_path):
    import yaml
    from reversi_zero_b200.agent import model as M
    from reversi_zero_b200.worker.self_play import blob_path_of
    p = tmp_path / "c.yml"
    p.write_text(yaml.safe_dump(dict(book=dict(plies=6, simulation_num_per_move=50, seed=4, model="m.npy", path="bk.npz"),
                                     b200=dict(nboard_book="bk.npz"), openings=dict(book="bk.npz", plies=5))))
    cfg = load_yaml(str(p), project_dir=str(tmp_path))
    assert [BK._field(cfg, k, None) for k in ("plies", "simulation_num_per_move", "seed", "model", "path")] == [6, 50, 4, "m.npy", "bk.npz"]
    assert OP._field(cfg, "book", None) == "bk.npz" and cfg.b200.nboard_book == "bk.npz"
    d = create_config(project_dir=str(tmp_path))
    assert (d.book.plies, d.book.simulation_num_per_move, d.book.seed, d.book.model) == (8, 400, None, None)
    assert d.book.path == os.path.join("data", "book", "book.npz") and d.b200.nboard_book is None and d.openings.book is None
    pc = BK.book_search_config(d, 77)
    assert (pc.noise_eps, pc.simulation_num_per_move, pc.parallel_search_num) == (0.0, 77, d.play_with_human.parallel_search_num)
    # NBoard: the book is used only with the loaded model's digest, and refused (logged) otherwise or when missing
    mc = M.ModelConfig(16, 3, 1, 1e-4, 16)
    cfg.model.update(dict(cnn_filter_num=16, res_layer_num=1, value_fc_size=16))
    cfg.resource.create_directories()
    blob = M.weights_to_blob(mc, M.build_random_weights(mc, 3))
    np.save(blob_path_of(cfg), blob)
    levels = py_levels(2)
    keys = np.array([OP.canonical_key(o, e) for lv in levels for o, e in lv], np.uint64).reshape(-1, 2)
    flags = np.array([BK.INTERIOR] * 2 + [BK.LEAF] * 3, np.uint8)
    meta = dict(plies=2, simulation_num_per_move=8, seed=0, model_sha256=M.blob_digest(blob), model={}, format_version=1)
    eng = NB.NBoardEngine.__new__(NB.NBoardEngine)
    eng.config = cfg
    assert eng.load_book() is None   # no file yet
    BK.save_book(str(tmp_path / "bk.npz"), BK.Book(keys[:, 0], keys[:, 1], np.zeros(5), flags, [1, 1, 3], meta))
    assert eng.load_book().plies == 2
    BK.save_book(str(tmp_path / "bk.npz"), BK.Book(keys[:, 0], keys[:, 1], np.zeros(5), flags, [1, 1, 3], dict(meta, model_sha256="0" * 64)))
    assert eng.load_book() is None
    cfg.b200.nboard_book = None
    assert eng.load_book() is None
    # openings: a book of another depth is refused before anything runs on the device
    book = BK.Book(keys[:, 0], keys[:, 1], np.zeros(5), flags, [1, 1, 3], meta, path="bk.npz")
    with pytest.raises(ValueError, match="bk.npz: a book of 2 plies cannot score openings of 5 plies"):
        OP.book_suite(book, 5, 10, 0.2, 1)


def test_book_command_parses():
    from reversi_zero_b200 import run
    assert run.create_parser().parse_args(["book", "-c", "x.yml"]).cmd == "book"


class StandInPlayer:
    """ReversiPlayer's interface to NBoardEngine: every search answers the lowest legal square with q = 0.25"""

    def __init__(self):
        self.searches = []

    def action(self, own, enemy, callback_in_mtcs=None, solve=True):
        self.searches.append((own, enemy))
        self.last = min(s for s in range(64) if (bb.find_correct_moves(own, enemy) >> s) & 1)
        return self.last

    def ask_thought_about(self, own, enemy):
        values, visit = [0.0] * 64, [0] * 64
        values[self.last], visit[self.last] = 0.25, 7
        return types.SimpleNamespace(values=values, visit=visit)

    def stop_thinking(self):
        pass


def stand_in_engine(book):
    eng = NB.NBoardEngine.__new__(NB.NBoardEngine)
    eng.config = Config()
    eng.nc = eng.config.nboard
    eng.play_config = eng.config.play
    eng.stdout = io.StringIO()
    eng.reader = NonBlockingStreamReader(io.StringIO(""))
    eng.handler = NB.NBoardProtocolVersion2(eng.config, eng)
    eng.player = StandInPlayer()
    eng.env = ReversiEnv().reset()
    eng.turn_of_nboard = Player.black
    eng.game_start = None
    eng.game_actions = []
    eng.book = book
    return eng


def session(eng, lines):
    eng.stdout.seek(0)
    eng.stdout.truncate()
    for line in lines:
        eng.handler.handle_message(line)
    return eng.stdout.getvalue().splitlines()


def test_nboard_go_and_hint_with_a_book(graph_exe):
    _, book = make_book(graph_exe, 3, np.random.default_rng(6))
    eng = stand_in_engine(book)
    out = session(eng, ["go"])
    v0 = book.best(*START)[1]
    assert out == ["status thinking...", f"=== C4/{v0 * 10}/{float(out[1].split('/')[2])}", "status waiting"]
    assert convert_action_to_move(19) == "C4" and eng.player.searches == []
    # three plies of book moves, each hint the book's best moves with the best last
    for ply in range(3):
        own, enemy = eng._states()
        mv = book.moves(own, enemy)
        hint = session(eng, ["hint 2"])
        ranked = sorted(mv, key=lambda m: (-m[1], m[0]))[:2]
        assert hint == ["status thinkng hint..."] + [f"search {convert_action_to_move(s)} {v} 0 40" for s, v in reversed(ranked)] + \
               ["status waiting"]
        go = session(eng, ["go"])[1]
        sq, v = book.best(own, enemy)
        assert go.startswith(f"=== {convert_action_to_move(sq)}/{v * 10}/")
        session(eng, [f"move {convert_action_to_move(sq)}"])
    assert eng.player.searches == []
    # level 3 is the book's last: the search takes over
    out = session(eng, ["go"])
    assert len(eng.player.searches) == 1 and out[1].startswith(f"=== {convert_action_to_move(eng.player.last)}/2.5/")


def test_nboard_without_book_or_outside_it_searches(graph_exe):
    _, book = make_book(graph_exe, 3, np.random.default_rng(7))
    plain, booked = stand_in_engine(None), stand_in_engine(book)
    # the knob off: the same replies as today, every one from the search
    out = session(plain, ["go", "hint 2"])
    assert out[1].startswith("=== C4/2.5/") and out[3:6] == ["status thinkng hint...", "search C4 0.25 0 7", "status waiting"]
    assert len(plain.player.searches) == 2
    # a game from another start position, or with a pass, leaves the book
    for start in ((START[0], START[1], Player.white), (START[0] | (1 << 0), START[1], Player.black)):
        booked.game_start = start
        session(booked, ["go"])
    booked.game_start = None
    booked.game_actions = [None]
    session(booked, ["go"])
    assert len(booked.player.searches) == 3


def test_abi():
    hdr = open(os.path.join(ROOT, "include", "rz_engine.h")).read()
    assert re.search(r"int rz_openings_book_graph\(int plies, uint64_t\* own, uint64_t\* enemy, uint64_t\* key_hi, uint64_t\* key_lo, "
                     r"size_t cap_nodes,\s+size_t\* n_nodes, uint64_t\* level_counts, uint64_t\* edge_offset, uint8_t\* edge_square,\s+"
                     r"int32_t\* edge_child, size_t cap_edges, size_t\* n_edges\);", hdr)
    assert "rz_openings_book_graph" in _cabi.SIGNATURES and hasattr(_cabi.lib(), "rz_openings_book_graph")
    assert len(_cabi.SIGNATURES["rz_openings_book_graph"][1]) == 13
    n, m = C.c_size_t(), C.c_size_t()
    for plies in (0, 11):
        assert _cabi.lib().rz_openings_book_graph(plies, None, None, None, None, 0, C.byref(n), None, None, None, None, 0, C.byref(m)) == -1
