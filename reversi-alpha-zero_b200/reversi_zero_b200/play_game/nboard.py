"""NBoard protocol 2 engine (reference play_game/nboard.py:23-333): ``python -m reversi_zero_b200.run nboard -c <yml>``
(or the ``nboard_engine`` launcher) lets the NBoard GUI, NTest matches or reversi-arena play and analyse with a model
of this project.

Commands arrive on stdin, one per line; stdout carries protocol replies only (logging goes to the log file that
``run.py`` sets up).  ``go`` and ``hint`` search with the one-slot ``ReversiPlayer`` mirror, whose simulations run on
the device; the tree is kept across the moves of a game and dropped when NBoard sends the opening position.  A
``ping`` interrupts a running search from the reader thread, so NBoard gets its ``pong`` as soon as the current chunk
of ``hint_callback_per_sim`` simulations ends.  With ``b200.nboard_analyze`` on, ``analyze`` answers with a retrograde
analysis of the game (play_game/analysis.py), which a ``ping`` interrupts as well.  With ``b200.nboard_exact_hint`` on,
``hint n`` in a position the player would solve reports the exact value of the best n moves (``100%`` lines, after
``100%W`` lines for moves whose sign is proven first); a ``ping`` interrupts it within one slice of the deep solver.
With ``b200.nboard_book`` set to an opening book (lib/book.py) of the loaded model, ``go`` plays the book move and ``hint
n`` reports the best n book moves, without a search, in every interior node of the book reached from the initial
position without a pass; everywhere else they search as without a book.  With ``b200.nboard_book_learn`` on as well,
``learn`` adds the game since ``set game`` to the book (lib/book.learn_game, up to ``book.max_level``), writes it back to
its file and plays from the grown book, before it replies ``learned``; a ``ping`` does not interrupt it.
"""
import ctypes as C
import os
import re
import sys
from collections import namedtuple
from logging import getLogger, StreamHandler, FileHandler
from time import time

import numpy as np

from ..agent.model import blob_digest
from ..agent.player import ReversiPlayer, CallbackInMCTS, solver_max_empties, solves_exactly
from ..env.reversi_env import ReversiEnv, Player
from ..lib import book as book_lib
from ..lib.book import best_move, load_book
from ..lib.ggf import parse_ggf, convert_to_bitboard_and_actions, convert_move_to_action, convert_action_to_move
from ..lib.nonblocking_stream_reader import NonBlockingStreamReader
from .common import load_model, model_source_path

logger = getLogger(__name__)

GameState = namedtuple("GameState", "black white actions player")
GoResponse = namedtuple("GoResponse", "action eval time")
HintResponse = namedtuple("HintResponse", "action value visit")
ExactHint = namedtuple("ExactHint", "action value depth")   # depth: "100%" exact, "100%W" win/loss proven
HINT_TIMEOUT = 30   # the reference solver's timeout (ReversiSolver.solve)
START_BLACK, START_WHITE = (0x10 << 24) | (0x08 << 32), (0x08 << 24) | (0x10 << 32)


def start(config):
    config.play_with_human.update_play_config(config.play)
    root_logger = getLogger()
    for h in list(root_logger.handlers):
        if isinstance(h, StreamHandler) and not isinstance(h, FileHandler):
            root_logger.removeHandler(h)
    logger.info(f"config type={config.type}")
    NBoardEngine(config).start()
    logger.info("finish nboard")


class NBoardEngine:
    # play_game.analysis.GameAnalyser, created at the first analysis.  A class attribute, so that the reader thread's
    # push_callback finds it on every engine, also one whose analysis has never run.
    analyser = None
    # the exact hint's solver and its stop flag (a ctypes.c_int32), created at the first exact hint; class attributes for
    # the same reason
    hint_solver = None
    hint_stop = None
    book = None   # lib.book.Book of b200.nboard_book, None without a usable one

    def __init__(self, config, stdin=None, stdout=None):
        self.config = config
        self.stdout = stdout or sys.stdout
        self.reader = NonBlockingStreamReader(stdin or sys.stdin)
        self.handler = NBoardProtocolVersion2(config, self)
        self.running = False
        self.nc = self.config.nboard
        self.env = ReversiEnv().reset()
        self.model = load_model(self.config)
        self.play_config = self.config.play
        self.player = self.create_player()
        self.book = self.load_book()
        self.turn_of_nboard = None
        self.game_start = None      # (black, white, player) of `set game`, and the actions since: the game `analyze` analyses
        self.game_actions = []

    def load_book(self):
        """the book of b200.nboard_book (relative to the project directory); None, logged, when none is set, the file is
        missing or refused, or the book was searched with another model than the one loaded"""
        path = getattr(getattr(self.config, "b200", None), "nboard_book", None)
        if not path:
            return None
        full = os.path.join(self.config.resource.project_dir, path)
        try:
            book = load_book(full)
        except (OSError, ValueError) as e:
            logger.warning(f"nboard: book not used: {e}")
            return None
        digest = blob_digest(np.load(model_source_path(self.config)))
        if book.meta.get("model_sha256") != digest:
            logger.warning(f"nboard: book not used: {full} was searched with model {str(book.meta.get('model_sha256'))[:16]}, "
                           f"the loaded model is {digest[:16]}")
            return None
        logger.info(f"nboard: book {full}: {book.plies} plies, {book.values.size} positions")
        return book

    def book_moves(self, own, enemy):
        """Book.moves of the position, in a game from the initial position without a pass; else None"""
        if self.book is None or None in self.game_actions:
            return None
        if self.game_start is not None:
            black, white, player = self.game_start
            if (black, white, int(getattr(player, "value", player))) != (START_BLACK, START_WHITE, 1):
                return None
        return self.book.moves(own, enemy)

    def book_searcher(self):
        """the searcher of learned positions: the loaded model with the book's simulation count and seed"""
        return book_lib.Searcher(self.config, self.model, self.book)

    def learn(self):
        """`learn` with b200.nboard_book_learn on and a book loaded: the game since `set game` is learned into the book,
        which is written back to its file and used from then on.  A game the book cannot learn is logged."""
        if self.book is None:
            return
        start_time = time()
        search = self.book_searcher()
        try:
            max_level = int(book_lib._field(self.config, "max_level", book_lib.MAX_LEVEL))
            book, k = book_lib.learn_game(self.book, self.game_actions, max_level, search=search, start=self.game_start)
        except ValueError as e:
            logger.warning(f"nboard: game not learned: {e}")
            return
        finally:
            search.close()
        if k:
            book_lib.save_book(self.book.path, book)
            self.book = book
        logger.info(f"nboard: learned the game: {k} positions expanded, {self.book.values.size} positions in the book "
                    f"({time() - start_time:.2f} s)")

    def create_player(self):
        logger.debug("create new ReversiPlayer()")
        return ReversiPlayer(self.config, self.model, self.play_config, enable_resign=False)

    def start(self):
        """Handles lines until the stream ends.  Lines that arrived before the end are still handled (the reference
        leaves as soon as its reader sees the end, dropping them)."""
        self.running = True
        self.reader.start(push_callback=self.push_callback)
        while self.running:
            closed = self.reader.closed   # read before polling: every line is queued before the stream is marked closed
            message = self.reader.readline(self.nc.read_stdin_timeout)
            if message is None:
                if closed:
                    break
                continue
            message = message.strip()
            logger.debug(f"> {message}")
            self.handler.handle_message(message)

    def push_callback(self, message):
        # called on the reader thread: a ping ends the running search
        if message.startswith("ping"):
            self.stop_thinking()
            if self.analyser is not None:
                self.analyser.stop()
            if self.hint_stop is not None:
                self.hint_stop.value = 1

    def stop(self):
        self.running = False

    def reply(self, message):
        logger.debug(f"< {message}")
        self.stdout.write(message + "\n")
        self.stdout.flush()

    def stop_thinking(self):
        self.player.stop_thinking()

    def set_depth(self, n):
        """nboard.py:79-91: depth n asks for n * simulation_num_per_depth_about visits on the chosen move, with up to
        min(30, 5 x that / simulation_num_per_move) thinking loops."""
        try:
            n = int(n)
            self.play_config.required_visit_to_decide_action = n * self.nc.simulation_num_per_depth_about
            self.play_config.thinking_loop = min(
                30, int(self.play_config.required_visit_to_decide_action * 5 / self.play_config.simulation_num_per_move))
            logger.info(f"set required_visit_to_decide_action to {self.play_config.required_visit_to_decide_action}")
        except ValueError:
            pass

    def reset_state(self):
        self.player.engine.close()
        self.player = self.create_player()

    def set_game(self, game_state):
        self.env.reset()
        self.env.update(game_state.black, game_state.white, game_state.player)
        self.turn_of_nboard = game_state.player
        self.game_start = (game_state.black, game_state.white, game_state.player)
        self.game_actions = list(game_state.actions)
        for action in game_state.actions:
            self._change_turn()
            if action is not None:
                self.env.step(action)

    def _change_turn(self):
        if self.turn_of_nboard:
            self.turn_of_nboard = Player.black if self.turn_of_nboard == Player.white else Player.white

    def move(self, action):
        self.game_actions.append(action)
        self._change_turn()
        if action is not None:
            self.env.step(action)

    def _states(self):
        board = self.env.board
        return (board.black, board.white) if self.env.next_player == Player.black else (board.white, board.black)

    def go(self):
        if self.env.next_player != self.turn_of_nboard:   # NBoard's side to move has no legal move: pass
            return GoResponse(None, 0, 0)
        states = self._states()
        start_time = time()
        book = self.book_moves(*states)
        if book:
            action, value = best_move(book)
            logger.debug(f"book move {convert_action_to_move(action)} ({value:+.4f})")
            return GoResponse(action, value, time() - start_time)
        action = self.player.action(*states)
        item = self.player.ask_thought_about(*states)
        return GoResponse(action, item.values[action], time() - start_time)

    def hint(self, n_hint):
        states = self._states()
        book = self.book_moves(*states)
        if book:
            self.handler.report_hint(book_hints(book, n_hint, self.book.meta.get("simulation_num_per_move", 0)))
            return
        exact = getattr(getattr(self.config, "b200", None), "nboard_exact_hint", False) and \
            solves_exactly(self.play_config, *states, solver_max_empties(self.config))
        if exact and self.exact_hint(*states, n_hint):
            return

        def hint_report_callback(values, visits):
            hint_list = []
            for action, visit in list(sorted(enumerate(visits), key=lambda x: -x[1]))[:n_hint]:
                if visit > 0:
                    hint_list.append(HintResponse(action, values[action], visit))
            self.handler.report_hint(hint_list)

        # after an exact solve that proved nothing (a timeout), the search answers without solving again
        self.player.action(*states, callback_in_mtcs=CallbackInMCTS(self.nc.hint_callback_per_sim, hint_report_callback),
                           solve=not exact)
        item = self.player.ask_thought_about(*states)
        hint_report_callback(item.values, item.visit)

    def exact_hint(self, own, enemy, n_hint):
        """`hint n` with b200.nboard_exact_hint on, in solver range: the value of every move from the exact solvers
        (ReversiSolver.solve_moves, n_best = n, the solver's 30 s timeout), reported as it is proven: after each deep round
        a `100%W` line for every move whose sign is proven before its value, then the best n proven moves.  A ping stops
        the solve and nothing more is sent.  False when nothing was proven, not even a sign: then the search answers."""
        if self.hint_solver is None:
            from ..lib.reversi_solver import ReversiSolver
            self.hint_solver = ReversiSolver(solver_max_empties(self.config))
            self.hint_stop = C.c_int32(0)
        self.hint_stop.value = 0

        def on_bounds(bounds):
            if not self.hint_stop.value:
                self.handler.report_exact_hint(wld_hints(bounds))

        bounds = self.hint_solver.solve_moves(own, enemy, 1, n_hint, HINT_TIMEOUT, self.hint_stop, on_bounds)
        if self.hint_stop.value:
            return True
        hints = exact_hints(bounds or {}, n_hint)
        if not hints:
            return False
        self.handler.report_exact_hint(hints)
        return True


    def begin_analysis(self):
        """before `status analyzing...`: the analyser exists and no earlier ping stops the analysis about to start"""
        if self.analyser is None:
            from .analysis import GameAnalyser
            self.analyser = GameAnalyser(self.config, self.model, self.play_config)
        self.analyser.reset_stop()

    def analyze(self, report):
        """report(moves_made, value, exact) for every position of the game since `set game`, until a ping stops it"""
        if self.game_start is None:
            return
        black, white, player = self.game_start
        self.analyser.analyse(black, white, player, self.game_actions, report)


def book_hints(moves, n_hint, visits):
    """the best `n_hint` book moves, best first as the search hint's list is (report_hint puts the best last), each with
    the book's simulation count in the search hint's visit field"""
    ranked = sorted(moves, key=lambda m: (-m[1], m[0]))[:n_hint]
    return [HintResponse(sq, value, visits) for sq, value in ranked]


def _best_last(hints):
    """ascending value, and among equal values the lowest square last: NBoard takes the last line as the best, and it
    is then go's move"""
    return sorted(hints, key=lambda h: (h.value, -h.action))


def wld_hints(bounds):
    """The `100%W` hints of a deep round's bounds {square: (lo, hi)}: every move whose sign is proven and whose value
    is not, with lo for a proven win and hi for a proven loss"""
    out = [ExactHint(s, lo if lo >= 1 else hi, "100%W") for s, (lo, hi) in bounds.items()
           if lo < hi and (lo >= 1 or hi <= -1)]
    return _best_last(out)


def exact_hints(bounds, n_hint):
    """The final hint list of a solve: the best `n_hint` (0: all) of the moves with an exact value (`100%`) or a proven
    sign (`100%W`, as in wld_hints; only after a timeout), best last"""
    out = [ExactHint(s, lo, "100%") for s, (lo, hi) in bounds.items() if lo == hi] + wld_hints(bounds)
    out.sort(key=lambda h: (-h.value, h.action))
    return _best_last(out[:n_hint] if n_hint > 0 else out)


def analysis_line(moves_made, value, exact):
    """NBoard's `analysis {movesMade} {eval}` line.  `value` is from the viewpoint of the side to move in that position,
    like the `===` and `search` lines (INTEGRATION §5); exact values (final disc differences) print as integers, searched
    ones (10 * q) in `go`'s float format."""
    return f"analysis {moves_made} {int(value) if exact else float(value)}"


class NBoardProtocolVersion2:
    """nboard.py:154-333; the protocol is described at https://github.com/weltyc/ntest/blob/master/instructions/Protocol.htm"""

    def __init__(self, config, engine):
        self.config = config
        self.engine = engine
        self.handlers = [
            (re.compile(r'nboard ([0-9]+)'), self.nboard),
            (re.compile(r'set depth ([0-9]+)'), self.set_depth),
            (re.compile(r'set game (.+)'), self.set_game),
            (re.compile(r'move ([^/]+)(/[^/]*)?(/[^/]*)?'), self.move),
            (re.compile(r'hint ([0-9]+)'), self.hint),
            (re.compile(r'go'), self.go),
            (re.compile(r'ping ([0-9]+)'), self.ping),
            (re.compile(r'learn'), self.learn),
            (re.compile(r'analyze'), self.analyze),
        ]

    def handle_message(self, message):
        for regexp, func in self.handlers:
            match = regexp.match(message)
            if match:
                func(*match.groups())
                return
        logger.debug(f"ignore message: {message}")

    def nboard(self, version):
        if version != "2":
            logger.warning(f"UNKNOWN NBoard Version {version}!!!")
        self.engine.reply(f"set myname {self.config.nboard.my_name}({self.config.type})")
        self.tell_status("waiting")

    def set_depth(self, depth):
        self.engine.set_depth(depth)

    def set_game(self, ggf_str):
        """The position at the end of the GGF game ``ggf_str``; a game of at most one move starts a new game, which
        drops the search tree."""
        ggf = parse_ggf(ggf_str)
        black, white, actions = convert_to_bitboard_and_actions(ggf)
        player = Player.black if ggf.BO.color == "*" else Player.white
        self.engine.set_game(GameState(black, white, actions, player))
        if len(actions) <= 1:
            self.engine.reset_state()

    def move(self, move, evaluation, time_sec):
        self.engine.move(convert_move_to_action(move))

    def hint(self, n):
        self.tell_status("thinkng hint...")
        self.engine.hint(int(n))
        self.tell_status("waiting")

    def report_hint(self, hint_list):
        for hint in reversed(hint_list):  # NBoard takes the last line as the best
            move = convert_action_to_move(hint.action)
            self.engine.reply(f"search {move} {hint.value} 0 {int(hint.visit)}")

    def report_exact_hint(self, hints):
        """ExactHint lines, already in NBoard's order (best last): `search {move} {disc difference} 0 100%` for an
        exact value, `... 100%W` for a proven win (lower bound) or loss (upper bound)"""
        for hint in hints:
            self.engine.reply(f"search {convert_action_to_move(hint.action)} {int(hint.value)} 0 {hint.depth}")

    def go(self):
        """Replies "=== {move}/{eval}/{time}"; the engine's board is not changed (NBoard sends a "move" next)."""
        self.tell_status("thinking...")
        gr = self.engine.go()
        move = convert_action_to_move(gr.action)
        self.engine.reply(f"=== {move}/{gr.eval * 10}/{gr.time}")
        self.tell_status("waiting")

    def ping(self, n):
        # the search has already been stopped by NBoardEngine.push_callback on the reader thread
        self.engine.reply(f"pong {n}")

    def learn(self):
        """With b200.nboard_book_learn on, the engine learns the game into its book first (NBoardEngine.learn)."""
        if getattr(getattr(self.config, "b200", None), "nboard_book_learn", False):
            self.engine.learn()
        self.engine.reply("learned")

    def analyze(self):
        """Retrograde analysis is optional in the protocol and the reference leaves it out; with b200.nboard_analyze on,
        one `analysis` line per position between `status analyzing...` and `status waiting`."""
        if not getattr(getattr(self.config, "b200", None), "nboard_analyze", False):
            return
        self.engine.begin_analysis()
        self.tell_status("analyzing...")
        self.engine.analyze(self.report_analysis)
        self.tell_status("waiting")

    def report_analysis(self, moves_made, value, exact):
        self.engine.reply(analysis_line(moves_made, value, exact))

    def tell_status(self, status):
        self.engine.reply(f"status {status}")
