"""Opening suites: balanced positions to start the games of a match or a league from.

``enumerate_openings(p)`` lists every distinct opening of p plies on the device (``rz_openings_enumerate``: transpositions
and the 8 board symmetries merged, no passes).  ``balanced_suite`` keeps the openings whose value, by a network's value
head from the mover's view, lies within ``max_abs_value`` of 0, and draws ``count`` of them in an order fixed by a seed.
``save_suite`` / ``load_suite`` keep a suite in a text file: one opening per line, its moves in the GGF notation of
``lib/ggf.py`` ("F5 D6 C3 ..."), ``#`` starting a comment.  ``start`` is the ``openings`` command.

Settings (YAML ``openings:`` section): ``plies`` (8), ``count`` (500), ``max_abs_value`` (0.2), ``seed`` (default
``b200.seed``), ``model`` (a blob path relative to the project directory, with the ``model`` section's shape; default
the best model's blob), ``path`` (``data/openings/openings.txt``, relative to the project directory) and ``book`` (an
opening book of ``plies`` plies, lib/book.py, whose searched values score the openings instead of the value head; default
none).
"""
import ctypes as C
import hashlib
import os
import re
from collections import namedtuple
from logging import getLogger

import numpy as np

from .. import _cabi
from . import bitboard as bb
from .ggf import convert_action_to_move, convert_move_to_action

logger = getLogger(__name__)

MAX_OPENING_PLIES = 20  # RZ_MAX_OPENING_PLIES
_START_BLACK, _START_WHITE = (0x10 << 24) | (0x08 << 32), (0x08 << 24) | (0x10 << 32)
_SQUARE = re.compile(r"^[A-Ha-h][1-8]$")

Openings = namedtuple("Openings", "own enemy moves level_counts")
SuiteEntry = namedtuple("SuiteEntry", "moves value")


def enumerate_openings(plies):
    """-> Openings(own, enemy: uint64 [n], moves: uint8 [n, plies], level_counts: uint64 [plies + 1]) in ascending
    canonical-key order; own / enemy is the position reached, in the mover's frame"""
    lib = _cabi.lib()
    n = C.c_size_t()
    _cabi.check(lib.rz_openings_enumerate(int(plies), None, None, None, 0, C.byref(n), None), "rz_openings_enumerate")
    own, enemy = np.zeros(n.value, np.uint64), np.zeros(n.value, np.uint64)
    moves = np.zeros((n.value, int(plies)), np.uint8)
    counts = np.zeros(int(plies) + 1, np.uint64)
    _cabi.check(lib.rz_openings_enumerate(int(plies), own.ctypes.data_as(_cabi.u64p), enemy.ctypes.data_as(_cabi.u64p),
                                          moves.ctypes.data_as(_cabi.u8p), n.value, C.byref(n), counts.ctypes.data_as(_cabi.u64p)),
                "rz_openings_enumerate")
    return Openings(own, enemy, moves, counts)


def canonical_key(own, enemy):
    """the least (own, enemy) pair over the 8 dihedral images (lib/bitboard.dihedral), own compared first"""
    return min((bb.dihedral(own, t), bb.dihedral(enemy, t)) for t in range(8))


def replay(moves):
    """plays the squares `moves` from the initial position -> (own, enemy) in the mover's frame.  Raises ValueError for an
    illegal move, a move after which the other side must pass, and a move that ends the game."""
    own, enemy = _START_BLACK, _START_WHITE
    for j, a in enumerate(moves):
        if a is None or not (bb.find_correct_moves(own, enemy) >> int(a)) & 1:
            raise ValueError(f"move {j + 1} ({convert_action_to_move(a)}) is illegal")
        fl = bb.calc_flip(int(a), own, enemy)
        own, enemy = enemy ^ fl, own | fl | (1 << int(a))
        if not bb.find_correct_moves(own, enemy):
            if bb.find_correct_moves(enemy, own):
                raise ValueError(f"after move {j + 1} ({convert_action_to_move(a)}) the other side must pass")
            raise ValueError(f"move {j + 1} ({convert_action_to_move(a)}) ends the game")
    return own, enemy


def _order_digest(seed, own, enemy):
    hi, lo = canonical_key(int(own), int(enemy))
    return hashlib.sha256(f"{int(seed)}:{hi:016x}{lo:016x}".encode()).digest()


def balanced_suite(net, plies, count, max_abs_value, seed, batch=65536):
    """Every distinct opening of `plies` plies whose value by `net` (a reversi_zero_b200.net.Net, value head, mover's view,
    board as it is) satisfies |v| <= max_abs_value, ordered by a hash of (seed, canonical key); the first `count` of them.
    -> [SuiteEntry(moves: list of squares, value: float)].  Fewer than `count` when fewer qualify (logged)."""
    import torch
    ops = enumerate_openings(plies)
    n = ops.own.size
    dev = torch.device("cuda", net.device)
    values = np.empty(n, np.float32)
    with torch.cuda.device(dev):
        for s in range(0, n, batch):
            e = min(n, s + batch)
            own_t = torch.from_numpy(ops.own[s:e].view(np.int64)).to(dev)
            enemy_t = torch.from_numpy(ops.enemy[s:e].view(np.int64)).to(dev)
            policy_t = torch.empty((e - s, 64), dtype=torch.float32, device=dev)
            value_t = torch.empty((e - s,), dtype=torch.float32, device=dev)
            net.predict_dev(own_t, enemy_t, policy_t, value_t, e - s)
            torch.cuda.synchronize(dev)
            values[s:e] = value_t.cpu().numpy()
    return select_balanced(ops, values, count, max_abs_value, seed)


def book_suite(book, plies, count, max_abs_value, seed):
    """balanced_suite with each opening's value taken from `book` (a lib.book.Book of `plies` plies: its searched leaf
    values) instead of a value head.  Refuses a book of another depth."""
    if book.plies != int(plies):
        raise ValueError(f"{book.path or 'the book'}: a book of {book.plies} plies cannot score openings of {plies} plies")
    ops = enumerate_openings(plies)
    a, b = int(book.first[plies]), int(book.first[plies + 1])
    if b - a != ops.own.size or any(canonical_key(int(ops.own[i]), int(ops.enemy[i])) !=
                                    (int(book.keys_hi[a + i]), int(book.keys_lo[a + i])) for i in (0, ops.own.size - 1)):
        raise ValueError(f"{book.path or 'the book'}: its level {plies} is not the openings of {plies} plies")
    return select_balanced(ops, book.level_values(plies), count, max_abs_value, seed)


def select_balanced(ops, values, count, max_abs_value, seed):
    """the openings of `ops` (enumerate_openings) whose value satisfies |v| <= max_abs_value, ordered by a hash of
    (seed, canonical key); the first `count` of them -> [SuiteEntry]"""
    n, plies = ops.own.size, ops.moves.shape[1]
    kept = np.nonzero(np.abs(values) <= max_abs_value)[0]
    kept = sorted(kept, key=lambda i: _order_digest(seed, ops.own[i], ops.enemy[i]))[:count]
    if len(kept) < count:
        logger.info(f"openings: {len(kept)} of the {n} openings of {plies} plies have |value| <= {max_abs_value}, "
                    f"fewer than the {count} asked for")
    return [SuiteEntry([int(a) for a in ops.moves[i]], float(values[i])) for i in kept]


def save_suite(path, suite, header=None):
    """writes one opening per line ("F5 D6 C3 ..."); SuiteEntry values go into a trailing comment.  `header`: comment
    lines put first.  Written to path + ".tmp" and renamed."""
    os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    with open(path + ".tmp", "wt") as f:
        for line in (header or []):
            f.write(f"# {line}\n")
        for entry in suite:
            moves, value = (entry.moves, entry.value) if isinstance(entry, SuiteEntry) else (entry, None)
            text = " ".join(convert_action_to_move(int(a)) for a in moves)
            f.write(text + (f"  # v={value:+.4f}" if value is not None else "") + "\n")
    os.replace(path + ".tmp", path)


def load_suite(path):
    """-> list of openings (lists of squares 0..63).  Refuses, naming the line: an unknown square, an illegal move, a pass
    ("PA") or a move that forces one, a move that ends the game, more than MAX_OPENING_PLIES moves, and a file without
    an opening."""
    suite = []
    with open(path, "rt") as f:
        for no, line in enumerate(f, 1):
            tokens = line.split("#", 1)[0].split()
            if not tokens:
                continue
            where = f"{path}:{no}"
            moves = []
            for tok in tokens:
                if tok[:2].lower() == "pa":
                    raise ValueError(f"{where}: a pass ({tok}) in an opening")
                if not _SQUARE.match(tok):
                    raise ValueError(f"{where}: {tok!r} is not a square")
                moves.append(convert_move_to_action(tok))
            if len(moves) > MAX_OPENING_PLIES:
                raise ValueError(f"{where}: {len(moves)} moves, at most {MAX_OPENING_PLIES}")
            try:
                replay(moves)
            except ValueError as e:
                raise ValueError(f"{where}: {e}") from None
            suite.append(moves)
    if not suite:
        raise ValueError(f"{path}: no opening")
    return suite


def suite_digest(path):
    with open(path, "rb") as f:
        return hashlib.sha256(f.read()).hexdigest()


def _field(config, name, default):
    sec = getattr(config, "openings", None)
    if isinstance(sec, dict):
        return sec.get(name, default)
    return getattr(sec, name, default) if sec is not None else default


def start(config, device=0):
    """the ``openings`` command: writes a balanced suite as the YAML ``openings:`` section says -> its path"""
    from ..net import Net
    from ..worker.self_play import blob_path_of
    rc = config.resource
    plies = int(_field(config, "plies", 8))
    count = int(_field(config, "count", 500))
    max_abs_value = float(_field(config, "max_abs_value", 0.2))
    seed = _field(config, "seed", None)
    seed = int(getattr(getattr(config, "b200", None), "seed", 0) if seed is None else seed)
    model = _field(config, "model", None)
    blob = os.path.join(rc.project_dir, model) if model else blob_path_of(config)
    path = os.path.join(rc.project_dir, _field(config, "path", os.path.join("data", "openings", "openings.txt")))
    book_path = _field(config, "book", None)
    if book_path:
        from .book import load_book
        book = load_book(os.path.join(rc.project_dir, book_path))
        suite = book_suite(book, plies, count, max_abs_value, seed)
        source = f"book {book_path} ({book.meta.get('simulation_num_per_move')} simulations per position)"
    else:
        net = Net(config.model, device)
        try:
            net.load_blob(np.load(blob))
            suite = balanced_suite(net, plies, count, max_abs_value, seed)
        finally:
            net.close()
        source = f"model {os.path.relpath(blob, rc.project_dir)}"
    save_suite(path, suite, header=[f"{len(suite)} openings of {plies} plies, |value| <= {max_abs_value}, seed {seed}", source])
    logger.info(f"openings: {len(suite)} openings of {plies} plies written to {path}")
    return path
