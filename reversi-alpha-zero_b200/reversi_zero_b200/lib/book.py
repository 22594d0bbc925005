"""Opening book: a minimax book over every distinct opening of up to P plies, searched on the device.

``book_graph(P)`` lists the openings of 0 .. P plies and the moves between consecutive levels (``rz_openings_book_graph``:
transpositions and the 8 board symmetries merged, no passes).  Every node is one of

* a leaf: a node of level P;
* interior: a node below level P all of whose moves lead to an opening of the next level;
* incomplete: a node below level P with a move after which the opponent must pass or the game ends.

Leaves and incomplete nodes are searched, all on one engine, one root per slot (``Engine.search_roots``) with the
player's search configuration, no root noise and ``book.simulation_num_per_move`` simulations.  Their value is the Q of
the most visited root move (first index on ties), ``w_sum[a] / n_visit[a]``, from the mover's view: 1/10 of the
evaluation ``go`` reports.  Interior nodes are backed up level by level: v(node) = max over its moves of -v(child).

``Book.moves`` answers in the queried orientation, for interior nodes only; the book move is the move of largest value,
the lowest square on ties.  ``save_book`` / ``load_book`` keep a book in one ``.npz`` file.  ``start`` is the ``book``
command; settings in the YAML ``book:`` section: ``plies`` (8), ``simulation_num_per_move`` (400), ``seed`` (default
``b200.seed``), ``model`` (a blob path relative to the project directory, with the ``model`` section's shape; default the
best model's blob) and ``path`` (``data/book/book.npz``, relative to the project directory).
"""
import ctypes as C
import json
import os
import time
from collections import namedtuple
from logging import getLogger

import numpy as np

from .. import _cabi
from . import bitboard as bb
from .openings import canonical_key

logger = getLogger(__name__)

FORMAT_VERSION = 1
LEAF, INTERIOR, INCOMPLETE = 0, 1, 2
MAX_BOOK_PLIES = 10

Graph = namedtuple("Graph", "own enemy key_hi key_lo level_counts edge_offset edge_square edge_child")


def book_graph(plies):
    """-> Graph(own, enemy, key_hi, key_lo: uint64 [n], level_counts: uint64 [plies + 1], edge_offset: uint64 [n + 1],
    edge_square: uint8 [m], edge_child: int32 [m]) as rz_openings_book_graph gives it; edge_child indexes the next level"""
    lib = _cabi.lib()
    n, m = C.c_size_t(), C.c_size_t()
    _cabi.check(lib.rz_openings_book_graph(int(plies), None, None, None, None, 0, C.byref(n), None, None, None, None, 0,
                                           C.byref(m)), "rz_openings_book_graph")
    own, enemy, hi, lo = (np.zeros(n.value, np.uint64) for _ in range(4))
    counts = np.zeros(int(plies) + 1, np.uint64)
    offset = np.zeros(n.value + 1, np.uint64)
    square, child = np.zeros(m.value, np.uint8), np.zeros(m.value, np.int32)
    _cabi.check(lib.rz_openings_book_graph(int(plies), own.ctypes.data_as(_cabi.u64p), enemy.ctypes.data_as(_cabi.u64p),
                                           hi.ctypes.data_as(_cabi.u64p), lo.ctypes.data_as(_cabi.u64p), n.value, C.byref(n),
                                           counts.ctypes.data_as(_cabi.u64p), offset.ctypes.data_as(_cabi.u64p),
                                           square.ctypes.data_as(_cabi.u8p), child.ctypes.data_as(_cabi.i32p), m.value, C.byref(m)),
                "rz_openings_book_graph")
    return Graph(own, enemy, hi, lo, counts, offset, square, child)


def level_starts(level_counts):
    """first node index of every level, and the total: [0, c_0, c_0 + c_1, ...]"""
    return np.concatenate([[0], np.cumsum(np.asarray(level_counts, np.int64))]).astype(np.int64)


def node_flags(graph):
    """LEAF for the last level; below it INCOMPLETE where a move has edge_child -1, else INTERIOR -> uint8 [n]"""
    first = level_starts(graph.level_counts)
    n_inner = int(first[-2])
    flags = np.full(int(first[-1]), LEAF, np.uint8)
    off = graph.edge_offset.astype(np.int64)
    if n_inner:
        bad = np.add.reduceat((graph.edge_child < 0).astype(np.int64), off[:n_inner])
        flags[:n_inner] = np.where(bad > 0, INCOMPLETE, INTERIOR)
    return flags


def backup(graph, flags, searched):
    """the book's values: `searched` (float64 [n], read at LEAF and INCOMPLETE nodes) as they are, and bottom-up for every
    INTERIOR node the largest -v(child) over its moves: a segmented max over the level's CSR edges"""
    first = level_starts(graph.level_counts)
    values = np.asarray(searched, np.float64).copy()
    off = graph.edge_offset.astype(np.int64)
    for level in range(len(first) - 3, -1, -1):
        a, b = int(first[level]), int(first[level + 1])
        e0, e1 = int(off[a]), int(off[b])
        child = graph.edge_child[e0:e1].astype(np.int64)
        cv = np.where(child >= 0, -values[first[level + 1] + np.maximum(child, 0)], -np.inf)
        best = np.maximum.reduceat(cv, off[a:b] - e0)   # every opening has a legal move: no empty segment
        inner = flags[a:b] == INTERIOR
        values[a:b][inner] = best[inner]
    return values


def leaf_values(n_visit, w_sum):
    """Q of the most visited root move (first index on ties), w_sum[a] / n_visit[a] in float64, per row"""
    n = np.asarray(n_visit).reshape(-1, 64)
    w = np.asarray(w_sum).reshape(-1, 64)
    a = np.argmax(n, axis=1)
    rows = np.arange(n.shape[0])
    return w[rows, a].astype(np.float64) / n[rows, a].astype(np.float64)


def book_search_config(config, simulation_num_per_move):
    """ReversiPlayer's search configuration (agent/player.search_play_config over the play section as NBoard sets it up),
    with root noise off and `simulation_num_per_move` simulations"""
    from ..agent.player import search_play_config
    pc = search_play_config(config, config.play)
    human = getattr(config, "play_with_human", None)
    if human is not None:
        human.update_play_config(pc)
    pc.noise_eps = 0.0
    pc.simulation_num_per_move = int(simulation_num_per_move)
    return pc


def search_engine(config, net, simulation_num_per_move, slots, seed, device=0):
    """an engine of `slots` slots for one search per slot with book_search_config (net None: the deterministic evaluator)"""
    from ..engine import Engine, engine_cfg_from_play_config, EVAL_NET, EVAL_FAKE
    ecfg = engine_cfg_from_play_config(book_search_config(config, simulation_num_per_move), games=int(slots), seed=int(seed),
                                       eval_mode=EVAL_NET if net is not None else EVAL_FAKE, max_searches_per_game=1)
    return Engine(ecfg, net, device)


def search_positions(engine, own, enemy, chunk):
    """leaf_values of every (own[i], enemy[i]), searched `chunk` roots per rz_engine_search_roots call"""
    out = np.empty(len(own), np.float64)
    for s in range(0, len(own), chunk):
        n, w = engine.search_roots(own[s:s + chunk], enemy[s:s + chunk], 1)
        out[s:s + chunk] = leaf_values(n, w)
    return out


def best_move(moves):
    """the book move of a Book.moves list: the largest value, the lowest square among equal values -> (square, value)"""
    return max(moves, key=lambda m: (m[1], -m[0]))


class Book:
    """keys_hi / keys_lo (canonical keys, ascending within each level), values (mover's view), flags and level_counts as
    build_book makes them; meta: plies, simulation_num_per_move, model_sha256, model, seed, format_version"""

    def __init__(self, keys_hi, keys_lo, values, flags, level_counts, meta, path=None):
        self.keys_hi = np.asarray(keys_hi, np.uint64)
        self.keys_lo = np.asarray(keys_lo, np.uint64)
        self.values = np.asarray(values, np.float64)
        self.flags = np.asarray(flags, np.uint8)
        self.level_counts = np.asarray(level_counts, np.uint64)
        self.meta = dict(meta)
        self.path = path
        self.first = level_starts(self.level_counts)

    @property
    def plies(self):
        return len(self.level_counts) - 1

    def level_values(self, level):
        return self.values[self.first[level]:self.first[level + 1]]

    def find(self, own, enemy):
        """-> the node index of (own, enemy) (mover's frame, any orientation), or None when it is not in the book"""
        level = bb.bit_count(own | enemy) - 4
        if not 0 <= level <= self.plies:
            return None
        hi, lo = canonical_key(int(own), int(enemy))
        a, b = int(self.first[level]), int(self.first[level + 1])
        lo_i = a + int(np.searchsorted(self.keys_hi[a:b], np.uint64(hi), "left"))
        hi_i = a + int(np.searchsorted(self.keys_hi[a:b], np.uint64(hi), "right"))
        j = lo_i + int(np.searchsorted(self.keys_lo[lo_i:hi_i], np.uint64(lo), "left"))
        return j if j < hi_i and int(self.keys_lo[j]) == lo else None

    def moves(self, own, enemy):
        """[(square, value)] for every legal move of an interior node, in ascending square order of the queried frame,
        value = -v(child) from this mover's view; None for a position not in the book, a leaf or an incomplete node"""
        i = self.find(own, enemy)
        if i is None or self.flags[i] != INTERIOR:
            return None
        out = []
        legal = bb.find_correct_moves(own, enemy)
        for sq in range(64):
            if (legal >> sq) & 1:
                fl = bb.calc_flip(sq, own, enemy)
                j = self.find(enemy ^ fl, own | fl | (1 << sq))
                if j is None:
                    return None
                out.append((sq, -float(self.values[j])))
        return out

    def best(self, own, enemy):
        """the book move (square, value): the largest value, the lowest square among equal values; None outside the book"""
        mv = self.moves(own, enemy)
        return best_move(mv) if mv else None


def build_book(config, net, plies, simulation_num_per_move, seed, chunk=None, device=0, meta=None):
    """the book of `plies` plies (1..10) searched with `net` (a reversi_zero_b200.net.Net; None: the deterministic
    evaluator) on one engine of `chunk` slots (default b200.games_per_gpu) -> Book"""
    plies = int(plies)
    if not 1 <= plies <= MAX_BOOK_PLIES:
        raise ValueError(f"book: plies = {plies} outside 1..{MAX_BOOK_PLIES}")
    chunk = int(chunk or getattr(getattr(config, "b200", None), "games_per_gpu", 4096))
    t0 = time.perf_counter()
    g = book_graph(plies)
    flags = node_flags(g)
    first = level_starts(g.level_counts)
    for level in range(plies + 1):
        f = flags[first[level]:first[level + 1]]
        logger.info(f"book: level {level}: {f.size} nodes ({int((f == INTERIOR).sum())} interior, "
                    f"{int((f == INCOMPLETE).sum())} incomplete, {int((f == LEAF).sum())} leaves)")
    todo = np.nonzero(flags != INTERIOR)[0]
    searched = np.zeros(flags.size, np.float64)
    t1 = time.perf_counter()
    engine = search_engine(config, net, simulation_num_per_move, min(chunk, todo.size), seed, device)
    try:
        searched[todo] = search_positions(engine, g.own[todo], g.enemy[todo], chunk)
    finally:
        engine.close()
    t2 = time.perf_counter()
    values = backup(g, flags, searched)
    logger.info(f"book: graph {t1 - t0:.2f} s, {todo.size} positions searched in {t2 - t1:.2f} s "
                f"({todo.size / max(t2 - t1, 1e-9):.0f}/s), backup {time.perf_counter() - t2:.3f} s")
    meta = dict(meta or {}, plies=plies, simulation_num_per_move=int(simulation_num_per_move), seed=int(seed),
                format_version=FORMAT_VERSION)
    return Book(g.key_hi, g.key_lo, values, flags, g.level_counts, meta)


def save_book(path, book):
    """one .npz: keys_hi, keys_lo, values, flags, level_counts and meta (a JSON string).  Written to path + ".tmp" and
    renamed."""
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path + ".tmp", "wb") as f:
        np.savez(f, keys_hi=book.keys_hi, keys_lo=book.keys_lo, values=book.values, flags=book.flags,
                 level_counts=book.level_counts, meta=np.array(json.dumps(book.meta, sort_keys=True)))
    os.replace(path + ".tmp", path)


def load_book(path):
    """-> Book.  Refuses, naming the file: a missing array, a format version other than FORMAT_VERSION, array lengths
    that disagree with the level counts, and keys out of ascending order within a level."""
    with np.load(path, allow_pickle=False) as z:
        missing = [k for k in ("keys_hi", "keys_lo", "values", "flags", "level_counts", "meta") if k not in z.files]
        if missing:
            raise ValueError(f"{path}: not a book (no {', '.join(missing)})")
        meta = json.loads(str(z["meta"]))
        arrays = {k: z[k] for k in ("keys_hi", "keys_lo", "values", "flags", "level_counts")}
    if meta.get("format_version") != FORMAT_VERSION:
        raise ValueError(f"{path}: book format version {meta.get('format_version')}, this build reads {FORMAT_VERSION}")
    counts = arrays["level_counts"].astype(np.int64)
    n = int(counts.sum())
    lengths = {k: len(v) for k, v in arrays.items() if k != "level_counts"}
    if len(counts) != int(meta.get("plies", -1)) + 1 or any(v != n for v in lengths.values()):
        raise ValueError(f"{path}: inconsistent array lengths {lengths} for level counts {counts.tolist()} "
                         f"and plies {meta.get('plies')}")
    first = level_starts(counts)
    hi, lo = arrays["keys_hi"], arrays["keys_lo"]
    for level in range(len(counts)):
        a, b = int(first[level]), int(first[level + 1])
        h, l = hi[a:b], lo[a:b]
        ok = (h[1:] > h[:-1]) | ((h[1:] == h[:-1]) & (l[1:] > l[:-1]))
        if not ok.all():
            raise ValueError(f"{path}: keys out of order in level {level} at node {a + 1 + int(np.argmin(ok))}")
    return Book(hi, lo, arrays["values"], arrays["flags"], counts.astype(np.uint64), meta, path=path)


def _field(config, name, default):
    sec = getattr(config, "book", None)
    if isinstance(sec, dict):
        return sec.get(name, default)
    return getattr(sec, name, default) if sec is not None else default


def model_meta(config):
    m = config.model
    return {k: getattr(m, k) for k in ("cnn_filter_num", "cnn_filter_size", "res_layer_num", "value_fc_size")}


def start(config, device=0):
    """the ``book`` command: builds and writes a book as the YAML ``book:`` section says -> its path"""
    from ..agent.model import blob_digest
    from ..net import Net
    from ..worker.self_play import blob_path_of
    rc = config.resource
    plies = int(_field(config, "plies", 8))
    sims = int(_field(config, "simulation_num_per_move", 400))
    seed = _field(config, "seed", None)
    seed = int(getattr(getattr(config, "b200", None), "seed", 0) if seed is None else seed)
    model = _field(config, "model", None)
    blob_path = os.path.join(rc.project_dir, model) if model else blob_path_of(config)
    path = os.path.join(rc.project_dir, _field(config, "path", os.path.join("data", "book", "book.npz")))
    blob = np.load(blob_path)
    net = Net(config.model, device)
    try:
        net.load_blob(blob)
        book = build_book(config, net, plies, sims, seed, device=device,
                          meta=dict(model_sha256=blob_digest(blob), model=model_meta(config)))
    finally:
        net.close()
    save_book(path, book)
    logger.info(f"book: {book.values.size} positions of 0..{plies} plies written to {path}")
    return path
