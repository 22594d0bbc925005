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
the lowest square on ties.  ``save_book`` / ``load_book`` keep a book in one ``.npz`` file.

A book grows beyond its full width one batch of leaves at a time (``grow``, best first, and ``learn_game``, along a played
game).  Level L always holds positions with L + 4 discs; levels above P are sparse, up to ``MAX_LEVEL``.  An expanded leaf
becomes interior, or incomplete when one of its moves leads to a pass or the end of the game; all its kept children become
leaves (``rz_openings_book_children``).  New leaves are searched as above, with the book's simulation count and seed, and
the book is backed up again.  A leaf that becomes incomplete keeps the value of its search.

``start`` is the ``book`` command; settings in the YAML ``book:`` section: ``plies`` (8), ``simulation_num_per_move``
(400), ``seed`` (default ``b200.seed``), ``model`` (a blob path relative to the project directory, with the ``model``
section's shape; default the best model's blob), ``path`` (``data/book/book.npz``, relative to the project directory), and
for growth ``extend`` (grow the book at ``path`` instead of building one), ``grow_nodes`` (expansions, 0), ``grow_batch``
(expansions per round, 256), ``max_level`` (40), ``grow_depth_cost`` (0.0) and ``learn`` (GGF file globs relative to the
project directory whose games are learned).
"""
import ctypes as C
import glob
import json
import os
import re
import time
from collections import namedtuple
from logging import getLogger

import numpy as np

from .. import _cabi
from . import bitboard as bb
from .ggf import parse_ggf, convert_to_bitboard_and_actions
from .openings import canonical_key

logger = getLogger(__name__)

FORMAT_VERSION = 1
LEAF, INTERIOR, INCOMPLETE = 0, 1, 2
MAX_BOOK_PLIES = 10
MAX_LEVEL = 40                  # the deepest level growth may add: 44 discs, 20 empties, the deep endgame solver's range
KEPT, PASS, OVER = 0, 1, 2      # a child's kind (rz_openings_book_children): an opening, its mover must pass, game over
START = (0x10 << 24) | (0x08 << 32), (0x08 << 24) | (0x10 << 32)   # the initial position, black to move

Graph = namedtuple("Graph", "own enemy key_hi key_lo level_counts edge_offset edge_square edge_child")
Children = namedtuple("Children", "edge_offset edge_square edge_child child_own child_enemy child_hi child_lo child_kind")


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


def book_children(own, enemy, next_hi, next_lo):
    """-> Children(edge_offset: uint64 [n + 1], edge_square: uint8 [m], edge_child: int32 [m], child_own, child_enemy,
    child_hi, child_lo: uint64 [m], child_kind: uint8 [m]) of the n nodes (own[i], enemy[i]) against the ascending keys
    (next_hi, next_lo) of a sorted level, as rz_openings_book_children gives them"""
    lib = _cabi.lib()
    own, enemy, next_hi, next_lo = (np.ascontiguousarray(a, np.uint64) for a in (own, enemy, next_hi, next_lo))
    ptr = lambda a: a.ctypes.data_as(_cabi.u64p) if a.size else None
    m = C.c_size_t()
    _cabi.check(lib.rz_openings_book_children(ptr(own), ptr(enemy), own.size, ptr(next_hi), ptr(next_lo), next_hi.size, None, None,
                                              None, None, None, None, None, None, 0, C.byref(m)), "rz_openings_book_children")
    offset = np.zeros(own.size + 1, np.uint64)
    square, kind, child = np.zeros(m.value, np.uint8), np.zeros(m.value, np.uint8), np.zeros(m.value, np.int32)
    c_own, c_enemy, c_hi, c_lo = (np.zeros(m.value, np.uint64) for _ in range(4))
    _cabi.check(lib.rz_openings_book_children(ptr(own), ptr(enemy), own.size, ptr(next_hi), ptr(next_lo), next_hi.size,
                                              offset.ctypes.data_as(_cabi.u64p), square.ctypes.data_as(_cabi.u8p),
                                              child.ctypes.data_as(_cabi.i32p), c_own.ctypes.data_as(_cabi.u64p),
                                              c_enemy.ctypes.data_as(_cabi.u64p), c_hi.ctypes.data_as(_cabi.u64p),
                                              c_lo.ctypes.data_as(_cabi.u64p), kind.ctypes.data_as(_cabi.u8p), m.value, C.byref(m)),
                "rz_openings_book_children")
    return Children(offset, square, child, c_own, c_enemy, c_hi, c_lo, kind)


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


def _edges_of(offset, nodes):
    """the CSR edges of `nodes` (ascending node indices): (the node of every edge, the edge's index, the start of every
    node's run in that list)"""
    start = offset[nodes]
    lens = offset[nodes + 1] - start
    base = np.cumsum(lens) - lens
    edge = np.arange(int(lens.sum()), dtype=np.int64) - np.repeat(base, lens) + np.repeat(start, lens)
    return np.repeat(nodes, lens), edge, base


def backup(graph, flags, searched):
    """the book's values: `searched` (float64 [n], read at LEAF and INCOMPLETE nodes) as they are, and bottom-up for every
    INTERIOR node the largest -v(child) over its moves: a segmented max over the level's CSR edges"""
    first = level_starts(graph.level_counts)
    values = np.asarray(searched, np.float64).copy()
    off = graph.edge_offset.astype(np.int64)
    for level in range(len(first) - 3, -1, -1):
        inner = int(first[level]) + np.nonzero(flags[first[level]:first[level + 1]] == INTERIOR)[0]
        if not inner.size:
            continue
        _, edge, base = _edges_of(off, inner)
        child = graph.edge_child[edge].astype(np.int64)
        cv = np.where(child >= 0, -values[first[level + 1] + np.maximum(child, 0)], -np.inf)
        values[inner] = np.maximum.reduceat(cv, base)   # an interior node has a legal move: no empty segment
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
    build_book, grow and learn_game make them; meta: plies, simulation_num_per_move, model_sha256, model, seed,
    format_version, and levels once the book holds more than plies + 1 levels"""

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
        """the full-width depth: every opening of 0 .. plies plies is a node"""
        return int(self.meta.get("plies", len(self.level_counts) - 1))

    @property
    def levels(self):
        """the number of stored levels: plies + 1, more once the book has grown"""
        return len(self.level_counts)

    def level_values(self, level):
        return self.values[self.first[level]:self.first[level + 1]]

    def find(self, own, enemy):
        """-> the node index of (own, enemy) (mover's frame, any orientation), or None when it is not in the book"""
        level = bb.bit_count(own | enemy) - 4
        if not 0 <= level < self.levels:
            return None
        return self.key_index(level, *canonical_key(int(own), int(enemy)))

    def key_index(self, level, hi, lo):
        """-> the node index of canonical key (hi, lo) in `level`, or None"""
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


def book_links(book, children=None):
    """-> Graph of a book of any depth from rz_openings_book_children (`children`, default book_children), level by
    level: level 0 is the initial position; a node of level L + 1 is held in the orientation of its first parent by
    (index, square) among the expanded (INTERIOR or INCOMPLETE) nodes of level L, as the enumerator picks its
    representatives; expanded nodes have one edge per legal move, leaves none.  For a full-width book this is
    book_graph(plies).  Raises ValueError for a node without an expanded parent or an expanded node missing a child."""
    children = children or book_children
    first = level_starts(book.level_counts)
    where = book.path or "the book"
    n = int(first[-1])
    own, enemy = np.zeros(n, np.uint64), np.zeros(n, np.uint64)
    own[0], enemy[0] = START
    counts = np.zeros(n, np.int64)
    squares, childs = [np.zeros(0, np.uint8)], [np.zeros(0, np.int32)]
    for level in range(book.levels - 1):
        a, b, c = (int(first[level + k]) for k in range(3))
        exp = a + np.nonzero(book.flags[a:b] != LEAF)[0]
        ch = children(own[exp], enemy[exp], book.keys_hi[b:c], book.keys_lo[b:c])
        kept = ch.child_kind == KEPT
        if (kept & (ch.edge_child < 0)).any():
            raise ValueError(f"{where}: an expanded node of level {level} has a child that is not in level {level + 1}")
        idx, at = np.unique(ch.edge_child[kept], return_index=True)   # the first edge into every child
        if idx.size != c - b:
            raise ValueError(f"{where}: {c - b - idx.size} nodes of level {level + 1} have no expanded parent")
        own[b:c], enemy[b:c] = ch.child_own[kept][at], ch.child_enemy[kept][at]
        counts[exp] = np.diff(ch.edge_offset.astype(np.int64))
        squares.append(ch.edge_square)
        childs.append(ch.edge_child)
    offset = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint64)
    return Graph(own, enemy, book.keys_hi.copy(), book.keys_lo.copy(), book.level_counts.copy(), offset,
                 np.concatenate(squares).astype(np.uint8), np.concatenate(childs).astype(np.int32))


def deviation(graph, flags, values):
    """d of every node reachable from the root through INTERIOR nodes, inf elsewhere: d(root) = 0 and d(c) = the least
    d(u) + v(u) - (-v(c)) over INTERIOR parents u, the value given up by playing into c summed along the cheapest path"""
    first = level_starts(graph.level_counts)
    d = np.full(int(first[-1]), np.inf)
    d[0] = 0.0
    off = graph.edge_offset.astype(np.int64)
    for level in range(len(first) - 2):
        a, b = int(first[level]), int(first[level + 1])
        inner = a + np.nonzero((flags[a:b] == INTERIOR) & np.isfinite(d[a:b]))[0]
        if not inner.size:
            continue
        u, edge, _ = _edges_of(off, inner)
        c = b + graph.edge_child[edge].astype(np.int64)
        np.minimum.at(d, c, d[u] + values[u] + values[c])
    return d


def select_leaves(book, d, count, max_level, depth_cost):
    """the next round's expansions: up to `count` LEAF nodes below `max_level` with a finite deviation d, least by
    (d + depth_cost x (level - plies), level, key) -> node indices in that order"""
    level = np.repeat(np.arange(book.levels), book.level_counts.astype(np.int64))
    cand = np.nonzero((book.flags == LEAF) & np.isfinite(d) & (level < int(max_level)))[0]
    priority = d[cand] + float(depth_cost) * (level[cand] - book.plies)
    order = np.lexsort((book.keys_lo[cand], book.keys_hi[cand], level[cand], priority))
    return cand[order[:int(count)]]


def _sorted_unique(hi, lo):
    """the distinct keys (hi[i], lo[i]) in ascending order"""
    order = np.lexsort((lo, hi))
    hi, lo = hi[order], lo[order]
    keep = np.ones(hi.size, bool)
    keep[1:] = (hi[1:] != hi[:-1]) | (lo[1:] != lo[:-1])
    return hi[keep], lo[keep]


def expand(book, own, enemy, key_hi, key_lo, children=None):
    """the book with the positions (own[i], enemy[i]) of canonical keys (key_hi[i], key_lo[i]) expanded in one batch: each
    is a LEAF of the book or a kept child of another position of the batch.  Each becomes INTERIOR, or INCOMPLETE when a
    move leads to a pass or the end of the game; its kept children not yet in the next level are added there as LEAF
    nodes with value NaN (to be searched).  -> Book (meta gains `levels` when levels > plies + 1)"""
    children = children or book_children
    own, enemy = np.asarray(own, np.uint64), np.asarray(enemy, np.uint64)
    level = np.array([bb.bit_count(int(o) | int(e)) - 4 for o, e in zip(own, enemy)], np.int64)
    first = level_starts(book.level_counts)
    if level.size and (level.min() < 0 or level.max() >= MAX_LEVEL):
        raise ValueError(f"book: a position of level {int(level.min())} .. {int(level.max())} cannot be expanded "
                         f"(levels 0 .. {MAX_LEVEL - 1})")
    levels = max(book.levels, int(level.max()) + 2 if level.size else 0)
    add_hi, add_lo = [[] for _ in range(levels)], [[] for _ in range(levels)]
    flag_of = {}
    for lv in np.unique(level):
        at = np.nonzero(level == lv)[0]
        b, c = (int(first[lv + 1]), int(first[lv + 2])) if lv + 1 < book.levels else (0, 0)
        ch = children(own[at], enemy[at], book.keys_hi[b:c], book.keys_lo[b:c])
        off = ch.edge_offset.astype(np.int64)
        bad = np.add.reduceat((ch.child_kind != KEPT).astype(np.int64), off[:-1])   # a kept position has a legal move
        for i, nbad in zip(at, bad):
            flag_of[(int(lv), int(key_hi[i]), int(key_lo[i]))] = INCOMPLETE if nbad else INTERIOR
        new = (ch.child_kind == KEPT) & (ch.edge_child < 0)
        add_hi[lv + 1].append(ch.child_hi[new])
        add_lo[lv + 1].append(ch.child_lo[new])
    his, los, vals, flags, counts = [], [], [], [], []
    for lv in range(levels):
        a, b = (int(first[lv]), int(first[lv + 1])) if lv < book.levels else (0, 0)
        nh, nl = _sorted_unique(np.concatenate([np.zeros(0, np.uint64)] + add_hi[lv]),
                                np.concatenate([np.zeros(0, np.uint64)] + add_lo[lv]))
        hi = np.concatenate([book.keys_hi[a:b], nh])
        lo = np.concatenate([book.keys_lo[a:b], nl])
        order = np.lexsort((lo, hi))
        his.append(hi[order])
        los.append(lo[order])
        vals.append(np.concatenate([book.values[a:b], np.full(nh.size, np.nan)])[order])
        flags.append(np.concatenate([book.flags[a:b], np.full(nh.size, LEAF, np.uint8)])[order])
        counts.append(hi.size)
    meta = dict(book.meta)
    if levels > book.plies + 1:
        meta["levels"] = levels
    out = Book(np.concatenate(his), np.concatenate(los), np.concatenate(vals), np.concatenate(flags), counts, meta,
               path=book.path)
    for (lv, hi, lo), flag in flag_of.items():
        i = out.key_index(lv, hi, lo)
        if i is None or out.flags[i] != LEAF:
            raise ValueError(f"book: an expanded position of level {lv} is {'not linked' if i is None else 'not a leaf'}")
        out.flags[i] = flag
    return out


def grow_round(book, own, enemy, key_hi, key_lo, children=None, search=None):
    """expand (one batch), then search every new leaf in the orientation book_links gives it with `search(own, enemy)
    -> values`, and back up -> (Book, its Graph)"""
    book = expand(book, own, enemy, key_hi, key_lo, children)
    graph = book_links(book, children)
    values = book.values.copy()
    todo = np.nonzero(np.isnan(values))[0]
    if todo.size:
        values[todo] = search(graph.own[todo], graph.enemy[todo])
    book.values = backup(graph, book.flags, values)
    return book, graph


def grow(book, nodes, batch, max_level, depth_cost, children=None, search=None):
    """best-first growth: rounds of up to `batch` expansions picked by select_leaves over the deviations of the current
    book, until `nodes` expansions in all or no candidate is left -> Book"""
    if not 0 < int(max_level) <= MAX_LEVEL:
        raise ValueError(f"book: max_level = {max_level} outside 1..{MAX_LEVEL}")
    if int(batch) < 1:
        raise ValueError(f"book: grow_batch = {batch} below 1")
    graph = book_links(book, children)
    done = 0
    while done < int(nodes):
        pick = select_leaves(book, deviation(graph, book.flags, book.values), min(int(batch), int(nodes) - done), max_level,
                             depth_cost)
        if not pick.size:
            break
        book, graph = grow_round(book, graph.own[pick], graph.enemy[pick], book.keys_hi[pick], book.keys_lo[pick],
                                 children, search)
        done += pick.size
        logger.info(f"book: grown by {done} of {int(nodes)} nodes, {book.values.size} positions in {book.levels} levels")
    return book


def is_start(start):
    """True for a game start (black, white, player) that is the initial position with black to move; None counts as it"""
    if start is None:
        return True
    black, white, player = start
    return (int(black), int(white), int(getattr(player, "value", player))) == (START[0], START[1], 1)


def learn_game(book, moves, max_level, children=None, search=None, start=None):
    """learns one game: its moves (squares, None for a pass) from `start` ((black, white, player); None: the initial
    position) are replayed until the first pass, the end of the game or `max_level`, and every position that is a LEAF
    or not yet in the book is expanded in one batch, so that each position's successor becomes its child; the new leaves
    are searched and the book backed up.  A game from another start is skipped.  -> (Book, positions expanded)"""
    if not is_start(start):
        logger.info("book: a game from another start position is not learned")
        return book, 0
    if not 0 < int(max_level) <= MAX_LEVEL:
        raise ValueError(f"book: max_level = {max_level} outside 1..{MAX_LEVEL}")
    own, enemy = START
    path = [(own, enemy)]
    for j, a in enumerate(moves):
        if a is None or len(path) > int(max_level):
            break
        if not (bb.find_correct_moves(own, enemy) >> int(a)) & 1:
            raise ValueError(f"book: move {j + 1} of the game is illegal")
        fl = bb.calc_flip(int(a), own, enemy)
        own, enemy = enemy ^ fl, own | fl | (1 << int(a))
        if not bb.find_correct_moves(own, enemy):
            break
        path.append((own, enemy))
    todo = []
    for level, (o, e) in enumerate(path[:int(max_level)]):
        i = book.find(o, e)
        if i is None or book.flags[i] == LEAF:
            todo.append((o, e) + canonical_key(o, e))
    if not todo:
        return book, 0
    o, e, hi, lo = (np.array(x, np.uint64) for x in zip(*todo))
    book, _ = grow_round(book, o, e, hi, lo, children, search)
    return book, len(todo)


def ggf_games(text):
    """the games of a GGF file (one or several "(;...;)" records) -> [((black, white, player), actions)]"""
    out = []
    for record in re.findall(r"\(;.*?;\)", text, re.S):
        ggf = parse_ggf(record)
        if ggf.BO is None:
            continue
        black, white, actions = convert_to_bitboard_and_actions(ggf)
        out.append(((black, white, 1 if ggf.BO.color == "*" else 2), actions))
    return out


class Searcher:
    """search(own, enemy) -> leaf values with a book's simulation count and seed (search_positions), on one engine made at
    the first call with min(chunk, that call's positions) slots; close() frees it"""

    def __init__(self, config, net, book, chunk=None, device=0):
        self.config, self.net, self.device = config, net, device
        self.sims = int(book.meta["simulation_num_per_move"])
        self.seed = int(book.meta["seed"])
        self.chunk = int(chunk or getattr(getattr(config, "b200", None), "games_per_gpu", 4096))
        self.engine = None
        self.slots = 0

    def __call__(self, own, enemy):
        if self.engine is None:
            self.slots = max(1, min(self.chunk, len(own)))
            self.engine = search_engine(self.config, self.net, self.sims, self.slots, self.seed, self.device)
        return search_positions(self.engine, own, enemy, self.slots)

    def close(self):
        if self.engine is not None:
            self.engine.close()
            self.engine = None


def extend_book(config, net, book, games=(), grow_nodes=0, grow_batch=256, max_level=MAX_LEVEL, depth_cost=0.0, chunk=None,
                device=0):
    """learns `games` ([(start, actions)], learn_game) one by one, then grows the book by `grow_nodes` expansions (grow),
    searching with `net` (None: the deterministic evaluator) -> Book"""
    search = Searcher(config, net, book, chunk, device)
    try:
        for start, actions in games:
            book, k = learn_game(book, actions, max_level, search=search, start=start)
            logger.info(f"book: learned a game of {len(actions)} moves, {k} positions expanded")
        if int(grow_nodes) > 0:
            book = grow(book, grow_nodes, grow_batch, max_level, depth_cost, search=search)
    finally:
        search.close()
    return book


def save_book(path, book):
    """one .npz: keys_hi, keys_lo, values, flags, level_counts and meta (a JSON string).  Written to path + ".tmp" and
    renamed."""
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path + ".tmp", "wb") as f:
        np.savez(f, keys_hi=book.keys_hi, keys_lo=book.keys_lo, values=book.values, flags=book.flags,
                 level_counts=book.level_counts, meta=np.array(json.dumps(book.meta, sort_keys=True)))
    os.replace(path + ".tmp", path)


def load_book(path):
    """-> Book.  Refuses, naming the file: a missing array, a format version other than FORMAT_VERSION, a `levels` entry
    outside plies + 1 .. MAX_LEVEL + 1, array lengths that disagree with the level counts (plies + 1 of them, or `levels`),
    and keys out of ascending order within a level."""
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
    levels = meta.get("levels")
    if levels is not None and not int(meta.get("plies", -1)) + 1 <= int(levels) <= MAX_LEVEL + 1:
        raise ValueError(f"{path}: {levels} levels for a book of {meta.get('plies')} plies, a book holds plies + 1 .. "
                         f"{MAX_LEVEL + 1} levels")
    if len(counts) != (int(meta.get("plies", -1)) + 1 if levels is None else int(levels)) or \
            any(v != n for v in lengths.values()):
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


def learn_files(project_dir, patterns):
    """the games of the GGF files matching `patterns` (globs relative to the project directory, sorted) -> [(start, actions)]"""
    games = []
    for pattern in [patterns] if isinstance(patterns, str) else list(patterns or []):
        for path in sorted(glob.glob(os.path.join(project_dir, pattern))):
            with open(path) as f:
                found = ggf_games(f.read())
            logger.info(f"book: {len(found)} games in {path}")
            games += found
    return games


def check_extend(book, digest, simulation_num_per_move):
    """refuses (ValueError, naming the file) to extend a book searched with another model or simulation count"""
    if book.meta.get("model_sha256") != digest:
        raise ValueError(f"{book.path}: the book was searched with model {str(book.meta.get('model_sha256'))[:16]}, "
                         f"this one is {digest[:16]}")
    if int(book.meta.get("simulation_num_per_move", -1)) != int(simulation_num_per_move):
        raise ValueError(f"{book.path}: the book was searched with {book.meta.get('simulation_num_per_move')} simulations "
                         f"per position, not {simulation_num_per_move}")


def start(config, device=0):
    """the ``book`` command: builds a book (or, with ``extend``, loads the one at ``path``), learns the games of ``learn``
    and grows it by ``grow_nodes`` expansions, and writes it as the YAML ``book:`` section says -> its path"""
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
    grow_nodes = int(_field(config, "grow_nodes", 0))
    games = learn_files(rc.project_dir, _field(config, "learn", None))
    blob = np.load(blob_path)
    digest = blob_digest(blob)
    net = Net(config.model, device)
    try:
        net.load_blob(blob)
        if _field(config, "extend", False):
            book = load_book(path)
            check_extend(book, digest, sims)
        else:
            book = build_book(config, net, plies, sims, seed, device=device,
                              meta=dict(model_sha256=digest, model=model_meta(config)))
        if grow_nodes > 0 or games:
            book = extend_book(config, net, book, games, grow_nodes, int(_field(config, "grow_batch", 256)),
                               int(_field(config, "max_level", MAX_LEVEL)), float(_field(config, "grow_depth_cost", 0.0)),
                               device=device)
    finally:
        net.close()
    save_book(path, book)
    logger.info(f"book: {book.values.size} positions of 0..{book.levels - 1} plies written to {path}")
    return path
