"""GPU tests of the opening book: the device graph against its host twin, the size query and a short buffer; chunked
leaf searches against one-slot searches; the `book` command end to end; NBoard in a subprocess with a book; and an
`openings` suite scored by a book."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np
import pytest

from reversi_zero_b200 import _cabi
from reversi_zero_b200.lib import book as BK, openings as OP
from reversi_zero_b200.lib.ggf import convert_action_to_move, convert_move_to_action
from test_book_host import graph_exe, run_graph  # noqa: F401  (the host twin fixture)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMALL_MODEL = "model: {cnn_filter_num: 16, res_layer_num: 1, value_fc_size: 16}\n"


@pytest.mark.parametrize("plies", range(1, 9))
def test_device_graph_matches_host_twin(graph_exe, plies):  # noqa: F811
    d, h = BK.book_graph(plies), run_graph(graph_exe, plies)
    for name in BK.Graph._fields:
        assert np.array_equal(getattr(d, name), getattr(h, name)), name
    first = BK.level_starts(d.level_counts)
    ops = OP.enumerate_openings(plies)
    assert np.array_equal(d.own[first[plies]:], ops.own) and np.array_equal(d.enemy[first[plies]:], ops.enemy)


def test_graph_repeats_size_query_and_short_buffer():
    a, b = BK.book_graph(8), BK.book_graph(8)
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    lib = _cabi.lib()
    n, m = C.c_size_t(), C.c_size_t()
    assert lib.rz_openings_book_graph(8, None, None, None, None, 0, C.byref(n), None, None, None, None, 0, C.byref(m)) == 0
    assert (n.value, m.value) == (a.own.size, a.edge_square.size) and int(a.level_counts[-1]) == 67239
    own, enemy = np.zeros(n.value, np.uint64), np.zeros(n.value, np.uint64)
    off = np.zeros(n.value + 1, np.uint64)
    sq, ch = np.zeros(m.value, np.uint8), np.zeros(m.value, np.int32)
    args = lambda cap_n, cap_m: (8, own.ctypes.data_as(_cabi.u64p), enemy.ctypes.data_as(_cabi.u64p), None, None, cap_n, C.byref(n),
                                 None, off.ctypes.data_as(_cabi.u64p), sq.ctypes.data_as(_cabi.u8p), ch.ctypes.data_as(_cabi.i32p),
                                 cap_m, C.byref(m))
    assert lib.rz_openings_book_graph(*args(n.value - 1, m.value)) == -5
    assert lib.rz_openings_book_graph(*args(n.value, m.value - 1)) == -5
    assert lib.rz_openings_book_graph(*args(n.value, m.value)) == 0
    assert np.array_equal(own, a.own) and np.array_equal(ch, a.edge_child)
    # -1 edges appear by 10 plies, and the flags follow them
    g = BK.book_graph(10)
    flags = BK.node_flags(g)
    assert (g.edge_child == -1).sum() > 0 and (flags == BK.INCOMPLETE).sum() > 0


def small_net(seed=11):
    from reversi_zero_b200 import net as N
    from reversi_zero_b200.agent import model as M
    mc = M.ModelConfig(16, 3, 1, 1e-4, 16)
    net = N.Net(mc)
    net.load_weights(M.build_random_weights(mc, seed))
    return net


def test_chunked_leaf_values_equal_one_slot_searches():
    from reversi_zero_b200.config import Config
    cfg = Config()
    net = small_net()
    ops = OP.enumerate_openings(6)
    pick = np.arange(0, ops.own.size, 37)[:48]
    own, enemy = ops.own[pick], ops.enemy[pick]
    runs = []
    for chunk in (16, 48):
        eng = BK.search_engine(cfg, net, 32, chunk, seed=9)
        n_all, w_all = [], []
        for s in range(0, own.size, chunk):
            n, w = eng.search_roots(own[s:s + chunk], enemy[s:s + chunk], 1)
            n_all.append(n)
            w_all.append(w)
        runs.append((np.concatenate(n_all), np.concatenate(w_all), BK.search_positions(eng, own, enemy, chunk)))
        eng.close()
    assert np.array_equal(runs[0][0], runs[1][0]) and np.array_equal(runs[0][1], runs[1][1])
    assert np.array_equal(runs[0][2], runs[1][2]) and np.array_equal(runs[0][2], BK.leaf_values(runs[0][0], runs[0][1]))
    one = BK.search_engine(cfg, net, 32, 1, seed=9)
    for i in range(0, own.size, 5):
        n, w = one.search_root(int(own[i]), int(enemy[i]), 1, 0)
        assert np.array_equal(n, runs[0][0][i]) and np.array_equal(w.view(np.uint32), runs[0][1][i].view(np.uint32))
    one.close()
    net.close()


def write_blob(path, seed=10):
    from reversi_zero_b200.agent import model as M
    mc = M.ModelConfig(16, 3, 1, 1e-4, 16)
    os.makedirs(os.path.dirname(path), exist_ok=True)
    blob = M.weights_to_blob(mc, M.build_random_weights(mc, seed))
    np.save(path, blob)
    return blob


def run_cmd(tmp_path, cmd, yml):
    env = dict(os.environ, PROJECT_DIR=str(tmp_path), PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "reversi-alpha-zero_b200"), ROOT]))
    env.pop("DATA_DIR", None)
    env.pop("MODEL_DIR", None)
    subprocess.run([sys.executable, "-m", "reversi_zero_b200.run", cmd, "-c", str(yml)], env=env, cwd=str(tmp_path),
                   check=True, timeout=900, capture_output=True, text=True)


@pytest.fixture(scope="module")
def built_book(tmp_path_factory):
    """the `book` command at 4 plies with the best model's blob, run twice"""
    from reversi_zero_b200.agent import model as M
    tmp = tmp_path_factory.mktemp("book")
    blob = write_blob(str(tmp / "data" / "model" / "model_best_weight.rzblob.npy"))
    yml = tmp / "b.yml"
    yml.write_text(SMALL_MODEL + "b200: {games_per_gpu: 64}\nbook: {plies: 4, simulation_num_per_move: 24, seed: 3, path: out/book.npz}\n")
    books = []
    for _ in range(2):
        run_cmd(tmp, "book", yml)
        books.append(BK.load_book(str(tmp / "out" / "book.npz")))
    return tmp, books, M.blob_digest(blob)


def test_book_command_end_to_end(built_book):
    tmp, (a, b), digest = built_book
    for k in ("keys_hi", "keys_lo", "values", "flags", "level_counts"):
        assert np.array_equal(getattr(a, k), getattr(b, k)), k
    assert a.meta == b.meta and a.meta["model_sha256"] == digest and a.meta["plies"] == 4
    assert a.meta["simulation_num_per_move"] == 24 and a.meta["seed"] == 3 and a.meta["model"]["cnn_filter_num"] == 16
    assert a.level_counts.tolist() == [1, 1, 3, 14, 60] and (a.flags[:19] == BK.INTERIOR).all()
    log = open(tmp / "logs" / "main.log").read()
    assert re.search(r"book: level 4: 60 nodes", log) and "positions searched in" in log
    # the leaves are the searches of an engine of another slot count
    from reversi_zero_b200 import net as N
    from reversi_zero_b200.config import load_yaml
    cfg = load_yaml(str(tmp / "b.yml"), project_dir=str(tmp))
    net = N.Net(cfg.model)
    net.load_blob(np.load(tmp / "data" / "model" / "model_best_weight.rzblob.npy"))
    g = BK.book_graph(4)
    eng = BK.search_engine(cfg, net, 24, 7, seed=3)
    leaves = BK.search_positions(eng, g.own[19:], g.enemy[19:], 7)
    eng.close()
    net.close()
    assert np.array_equal(leaves, a.values[19:])
    assert np.array_equal(BK.backup(g, a.flags, np.concatenate([np.zeros(19), leaves])), a.values)


def test_openings_scored_by_the_book(built_book):
    tmp, (book, _), _ = built_book
    yml = tmp / "o.yml"
    yml.write_text(SMALL_MODEL + "openings: {plies: 4, count: 30, max_abs_value: 1.0, seed: 9, book: out/book.npz, path: out/suite.txt}\n")
    run_cmd(tmp, "openings", yml)
    suite = OP.load_suite(str(tmp / "out" / "suite.txt"))
    text = open(tmp / "out" / "suite.txt").read()
    assert "book out/book.npz" in text and len(suite) == 30
    for line, moves in zip([l for l in text.splitlines() if l and not l.startswith("#")], suite):
        v = float(line.split("v=")[1])
        assert abs(v - float(book.level_values(4)[book.find(*OP.replay(moves)) - int(book.first[4])])) < 1e-4
    # the same selection as a value-head suite would make from these values
    want = OP.select_balanced(OP.enumerate_openings(4), book.level_values(4), 30, 1.0, 9)
    assert [e.moves for e in want] == suite
    bad = tmp / "bad.yml"
    bad.write_text(SMALL_MODEL + "openings: {plies: 5, book: out/book.npz, path: out/s5.txt}\n")
    with pytest.raises(subprocess.CalledProcessError) as e:
        run_cmd(tmp, "openings", bad)
    assert "a book of 4 plies cannot score openings of 5 plies" in e.value.stderr
    assert not os.path.exists(tmp / "out" / "s5.txt")


def test_nboard_plays_the_book_then_searches(built_book):
    from test_nboard_gpu import Session, _ggf
    tmp, (book, _), _ = built_book
    yml = tmp / "n.yml"
    yml.write_text(SMALL_MODEL + "b200: {nboard_book: out/book.npz}\nplay: {simulation_num_per_move: 16}\n")
    env = dict(os.environ, PROJECT_DIR=str(tmp), PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "reversi-alpha-zero_b200"), ROOT]))
    env.pop("DATA_DIR", None)
    env.pop("MODEL_DIR", None)
    s = Session([sys.executable, "-m", "reversi_zero_b200.run", "nboard", "-c", str(yml)], str(tmp), env)
    from reversi_zero_b200.env.reversi_env import ReversiEnv
    try:
        s.send("nboard 2")
        s.until(lambda l: l.startswith("status"))
        s.send("set depth 1")
        moves = []
        env_ = ReversiEnv().reset()
        for ply in range(6):
            s.send(f"set game {_ggf(moves)}")
            s.send("go")
            line = s.until(lambda l: l.startswith("=== "))[-1]
            move, ev = line[4:].split("/")[:2]
            own, enemy = env_.get_own_and_enemy()
            if ply < 4:   # inside the book: its move and value
                sq, v = book.best(own, enemy)
                assert (move, float(ev)) == (convert_action_to_move(sq), v * 10), (ply, line)
            moves.append(move)
            env_.step(convert_move_to_action(move))
        s.p.stdin.close()
        s.p.wait(timeout=120)
        assert s.p.returncode == 0, "".join(s.err)[-3000:]
    finally:
        if s.p.poll() is None:
            s.p.kill()
        s.p.wait(timeout=30)
    log = open(tmp / "logs" / "main.log").read()
    assert "nboard: book" in log and len(re.findall(r"book move ", log)) == 4
