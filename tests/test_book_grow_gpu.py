"""GPU tests of the growing opening book: rz_openings_book_children against its host twin, its size query and a short
buffer; growth by whole frontiers against the full-width book with the deterministic evaluator and a small network; grown
leaves against one-slot searches, for any chunk size; the `book` command with `extend` and `grow_nodes`; and NBoard's
`learn` in a subprocess."""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest

from reversi_zero_b200 import _cabi
from reversi_zero_b200.config import Config
from reversi_zero_b200.lib import book as BK
from reversi_zero_b200.lib.ggf import convert_action_to_move
from test_book_host import graph_exe, run_graph  # noqa: F401  (the host twin fixtures)
from test_book_grow_host import children_exe, twin, random_positions, random_game, game_positions, rows_of  # noqa: F401
from test_book_gpu import small_net, write_blob, run_cmd, SMALL_MODEL

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_device_children_match_host_twin_on_the_8_ply_graph(children_exe):
    g = BK.book_graph(8)
    first = BK.level_starts(g.level_counts)
    host = twin(children_exe)
    for level in range(9):
        a, b = int(first[level]), int(first[level + 1])
        c = int(first[level + 2]) if level < 8 else b
        args = (g.own[a:b], g.enemy[a:b], g.key_hi[b:c], g.key_lo[b:c])
        d, h = BK.book_children(*args), host(*args)
        for name in BK.Children._fields:
            assert np.array_equal(getattr(d, name), getattr(h, name)), (level, name)
        if level < 8:   # the graph's own edges
            assert np.array_equal(d.edge_child, g.edge_child[int(g.edge_offset[a]):int(g.edge_offset[b])])


def test_device_children_on_seeded_positions_repeat_and_size_query(children_exe):
    pos = random_positions(8, 3000)
    own = np.array([p[0] for p in pos], np.uint64)
    enemy = np.array([p[1] for p in pos], np.uint64)
    every = BK.book_children(own, enemy, [], [])
    rng = np.random.default_rng(2)
    pick = np.sort(rng.choice(every.child_hi.size, every.child_hi.size // 3, replace=False))
    keys = sorted(set(zip(every.child_hi[pick].tolist(), every.child_lo[pick].tolist())))
    hi, lo = np.array([k[0] for k in keys], np.uint64), np.array([k[1] for k in keys], np.uint64)
    a, b, h = BK.book_children(own, enemy, hi, lo), BK.book_children(own, enemy, hi, lo), twin(children_exe)(own, enemy, hi, lo)
    for name in BK.Children._fields:
        assert np.array_equal(getattr(a, name), getattr(b, name)) and np.array_equal(getattr(a, name), getattr(h, name)), name
    assert (a.edge_child >= 0).sum() > 0 and (a.edge_child[a.child_kind == BK.KEPT] < 0).sum() > 0
    lib = _cabi.lib()
    m = C.c_size_t()
    u64 = lambda x: x.ctypes.data_as(_cabi.u64p)
    assert lib.rz_openings_book_children(u64(own), u64(enemy), own.size, u64(hi), u64(lo), hi.size, None, None, None, None, None,
                                         None, None, None, 0, C.byref(m)) == 0
    assert m.value == a.edge_square.size
    outs = [np.zeros(own.size + 1, np.uint64), np.zeros(m.value, np.uint8), np.zeros(m.value, np.int32)] + \
           [np.zeros(m.value, np.uint64) for _ in range(4)] + [np.zeros(m.value, np.uint8)]
    ptrs = [u64(outs[0]), outs[1].ctypes.data_as(_cabi.u8p), outs[2].ctypes.data_as(_cabi.i32p)] + \
           [u64(x) for x in outs[3:7]] + [outs[7].ctypes.data_as(_cabi.u8p)]
    call = lambda cap: lib.rz_openings_book_children(u64(own), u64(enemy), own.size, u64(hi), u64(lo), hi.size, *ptrs, cap, C.byref(m))
    assert call(m.value - 1) == -5
    assert call(m.value) == 0
    for x, name in zip(outs, ("edge_offset", "edge_square", "edge_child", "child_own", "child_enemy", "child_hi", "child_lo",
                              "child_kind")):
        assert np.array_equal(x, getattr(a, name)), name


@pytest.mark.parametrize("with_net", [False, True])
def test_growing_4_plies_by_whole_frontiers_is_build_book_6(with_net):
    cfg = Config()
    net = small_net() if with_net else None
    try:
        want = BK.build_book(cfg, net, 6, 16, 5, chunk=256)
        book = BK.build_book(cfg, net, 4, 16, 5, chunk=256)
        grown = BK.extend_book(cfg, net, book, (), 10 ** 6, 10 ** 6, 6, 0.0, chunk=256)
    finally:
        if net is not None:
            net.close()
    assert (want.flags[:int(want.first[6])] != BK.INCOMPLETE).all()
    for k in ("keys_hi", "keys_lo", "flags", "values", "level_counts"):
        assert np.array_equal(getattr(grown, k), getattr(want, k)), k
    assert grown.levels == 7 and grown.plies == 4


def test_grown_leaves_are_one_slot_searches_for_any_chunk():
    cfg = Config()
    net = small_net()
    try:
        base = BK.build_book(cfg, net, 3, 24, 7, chunk=64)
        runs = [BK.extend_book(cfg, net, base, (), 40, 9, 12, 0.2, chunk=chunk) for chunk in (64, 5, 64)]
        for r in runs[1:]:
            for k in ("keys_hi", "keys_lo", "flags", "values", "level_counts"):
                assert np.array_equal(getattr(r, k), getattr(runs[0], k)), k
        grown = runs[0]
        assert grown.levels > 5 and (grown.flags != BK.LEAF).sum() == (base.flags != BK.LEAF).sum() + 40
        graph = BK.book_links(grown)
        new = np.nonzero((grown.flags == BK.LEAF) & (np.arange(grown.values.size) >= int(grown.first[4])))[0]
        one = BK.search_engine(cfg, net, 24, 1, seed=7)
        try:
            for i in new[::max(1, new.size // 40)]:
                n, w = one.search_root(int(graph.own[i]), int(graph.enemy[i]), 1, 0)
                assert BK.leaf_values(n, w)[0] == grown.values[i]
        finally:
            one.close()
    finally:
        net.close()


def test_book_command_extends_and_grows(tmp_path):
    write_blob(str(tmp_path / "data" / "model" / "model_best_weight.rzblob.npy"))
    base = tmp_path / "b.yml"
    base.write_text(SMALL_MODEL + "b200: {games_per_gpu: 64}\nbook: {plies: 3, simulation_num_per_move: 16, seed: 3, path: out/book.npz}\n")
    run_cmd(tmp_path, "book", base)
    shutil.copy(tmp_path / "out" / "book.npz", tmp_path / "base.npz")
    first = BK.load_book(str(tmp_path / "base.npz"))
    grow = tmp_path / "g.yml"
    grow.write_text(SMALL_MODEL + "b200: {games_per_gpu: 64}\nbook: {simulation_num_per_move: 16, path: out/book.npz, extend: true, "
                                  "grow_nodes: 50, grow_batch: 16, max_level: 12, grow_depth_cost: 0.1}\n")
    books = []
    for _ in range(2):
        shutil.copy(tmp_path / "base.npz", tmp_path / "out" / "book.npz")
        run_cmd(tmp_path, "book", grow)
        books.append(BK.load_book(str(tmp_path / "out" / "book.npz")))
    a, b = books
    for k in ("keys_hi", "keys_lo", "values", "flags", "level_counts"):
        assert np.array_equal(getattr(a, k), getattr(b, k)), k
    assert a.meta == b.meta and a.plies == 3 and a.levels == a.meta["levels"] > 4
    assert (a.flags != BK.LEAF).sum() == (first.flags != BK.LEAF).sum() + 50
    # the full-width part's leaves keep their searched values
    for i in np.nonzero(first.flags == BK.LEAF)[0]:
        j = a.key_index(3, int(first.keys_hi[i]), int(first.keys_lo[i]))
        assert a.flags[j] != BK.LEAF or a.values[j] == first.values[i]
    # another simulation count is refused, and the file stays as it is
    bad = tmp_path / "bad.yml"
    bad.write_text(SMALL_MODEL + "book: {simulation_num_per_move: 17, path: out/book.npz, extend: true, grow_nodes: 5}\n")
    before = open(tmp_path / "out" / "book.npz", "rb").read()
    with pytest.raises(subprocess.CalledProcessError) as e:
        run_cmd(tmp_path, "book", bad)
    assert "searched with 16 simulations per position, not 17" in e.value.stderr
    assert open(tmp_path / "out" / "book.npz", "rb").read() == before


def nboard_session(tmp, yml, lines, until):
    from test_nboard_gpu import Session
    env = dict(os.environ, PROJECT_DIR=str(tmp), PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "reversi-alpha-zero_b200"), ROOT]))
    env.pop("DATA_DIR", None)
    env.pop("MODEL_DIR", None)
    s = Session([sys.executable, "-m", "reversi_zero_b200.run", "nboard", "-c", str(yml)], str(tmp), env)
    out = []
    try:
        s.send("nboard 2")
        s.until(lambda l: l.startswith("status"))
        for line, pred in zip(lines, until):   # pred None: a line without a reply
            s.send(line)
            if pred is not None:
                out.append(s.until(pred, timeout=300)[-1])
        s.p.stdin.close()
        s.p.wait(timeout=120)
        assert s.p.returncode == 0, "".join(s.err)[-3000:]
    finally:
        if s.p.poll() is None:
            s.p.kill()
        s.p.wait(timeout=30)
    return out


def test_nboard_learns_the_game_into_the_book(tmp_path):
    from test_nboard_gpu import _ggf
    write_blob(str(tmp_path / "data" / "model" / "model_best_weight.rzblob.npy"))
    yml = tmp_path / "b.yml"
    yml.write_text(SMALL_MODEL + "b200: {games_per_gpu: 64}\nbook: {plies: 3, simulation_num_per_move: 16, seed: 3, path: out/book.npz}\n")
    run_cmd(tmp_path, "book", yml)
    path = tmp_path / "out" / "book.npz"
    before = open(path, "rb").read()
    moves = random_game(2)[:16]
    assert None not in moves
    game = _ggf([convert_action_to_move(a) for a in moves])
    is_learned = lambda l: l == "learned"
    # the knob off: `learned` and the file as it was
    off = tmp_path / "off.yml"
    off.write_text(SMALL_MODEL + "b200: {nboard_book: out/book.npz}\nplay: {simulation_num_per_move: 16}\n")
    assert nboard_session(tmp_path, off, [f"set game {game}", "learn"], [None, is_learned]) == ["learned"]
    assert open(path, "rb").read() == before
    # the knob on: the game is in the book beyond its 3 plies
    on = tmp_path / "on.yml"
    on.write_text(SMALL_MODEL + "b200: {nboard_book: out/book.npz, nboard_book_learn: true}\nplay: {simulation_num_per_move: 16}\n"
                                "book: {max_level: 14}\n")
    assert nboard_session(tmp_path, on, [f"set game {game}", "learn"], [None, is_learned]) == ["learned"]
    book = BK.load_book(str(path))
    assert book.levels == 15 and book.meta["levels"] == 15 and book.plies == 3
    nodes = [book.find(o, e) for o, e in game_positions(moves)[:15]]
    assert None not in nodes and all(book.flags[i] != BK.LEAF for i in nodes[:14])
    # a fresh session plays the learned book moves
    deep = [k for k in range(4, 14) if book.flags[nodes[k]] == BK.INTERIOR][:3]
    assert deep
    lines, preds = [], []
    for k in deep:
        lines += [f"set game {_ggf([convert_action_to_move(a) for a in moves[:k]])}", "go"]
        preds += [None, lambda l: l.startswith("=== ")]
    out = nboard_session(tmp_path, off, lines, preds)
    for k, line in zip(deep, out):
        sq, v = book.best(*game_positions(moves)[k])
        assert line.startswith(f"=== {convert_action_to_move(sq)}/{v * 10}/"), (k, line)
