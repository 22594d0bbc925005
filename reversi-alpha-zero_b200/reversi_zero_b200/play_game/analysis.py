"""Retrograde analysis of a whole game, NBoard's "Analyze game" (``analyze`` in protocol 2): one value per position of the
game, from the viewpoint of the side the record puts to move there.

* A finished game is worth its final disc difference (empties not awarded, the solver convention).
* A position whose mover has to pass is worth the negated value of the position after the pass.
* A position ``ReversiPlayer.action_with_evaluation`` would solve exactly (``use_solver_turn`` set, ``turn >=
  use_solver_turn`` and at most ``b200.solver_max_empties`` empties) is solved: up to 12 empties all in one lane-solver
  batch, 13 or more one at a time on the whole device in ascending order of empties, so that the deep solver's table
  carries each proof into the next, larger position.  A deep solve that times out or is stopped falls back to the search.
* Every other position is searched, all of them at once, one per slot of a 64-slot engine
  (``Engine.search_roots``), in chunks of ``nboard.hint_callback_per_sim`` simulations up to
  ``simulation_num_per_move``; the value is ``10 * q`` of the most visited move (first index), as ``go`` reports it.

Values are reported as they become known: the exact ones from the end of the game backwards, then the searched ones
from the end backwards.  ``stop()`` (from another thread) ends an analysis: nothing more is reported, a running deep
solve returns within one slice and a partial search is dropped.
"""
import ctypes as C
import threading
from collections import namedtuple
from logging import getLogger

import numpy as np

from ..agent.player import search_play_config, solver_max_empties, solves_exactly
from ..engine import Engine, engine_cfg_from_play_config, EVAL_NET, EVAL_FAKE
from ..lib.bitboard import find_correct_moves, calc_flip, bit_count

logger = getLogger(__name__)

ANALYSIS_SLOTS = 64          # no game from the standard start has more than 60 positions with a legal move
ANALYSIS_CACHE_MB = 64       # evaluation cache of the analysis engine (see DESIGN §5)
LANE_MAX_EMPTIES = 12
DEEP_TIMEOUT = 30            # ReversiSolver.solve's default, which ReversiPlayer uses

# one position of a game: the record's side to move there (1 black, 2 white), its discs and the opponent's
Position = namedtuple("Position", "moves_made player own enemy")


def enumerate_positions(black, white, player, actions):
    """Positions 0..len(actions) of a game that starts from (black, white) with `player` (1 black, 2 white) to move and
    goes on with `actions` (square 0..63, None for a pass, as NBoard's ``set game`` and ``move`` give them).  A move the
    record's mover cannot play but the other side can is the other side's after an unrecorded pass, as ReversiEnv plays
    it.  -> list of Position."""
    p = int(getattr(player, "value", player))
    own, enemy = (black, white) if p == 1 else (white, black)
    out = [Position(0, p, own, enemy)]
    for k, a in enumerate(actions):
        if a is not None:
            if not (find_correct_moves(own, enemy) >> a) & 1:
                if not (find_correct_moves(enemy, own) >> a) & 1:
                    raise ValueError(f"move {k + 1} (square {a}) is illegal")
                own, enemy, p = enemy, own, 3 - p
            flip = calc_flip(a, own, enemy)
            own, enemy = own | flip | (1 << a), enemy ^ flip
        own, enemy, p = enemy, own, 3 - p
        out.append(Position(k + 1, p, own, enemy))
    return out


def classify(positions):
    """-> list of (kind, sign, own, enemy) per position: kind "over" (value = sign * disc difference of own / enemy),
    else the value is sign * the value of (own, enemy) with its mover to move, which has a legal move ("pass" positions
    refer to the position after the pass, sign -1)."""
    out = []
    for pos in positions:
        own, enemy = pos.own, pos.enemy
        if find_correct_moves(own, enemy):
            out.append(("move", 1, own, enemy))
        elif find_correct_moves(enemy, own):
            out.append(("pass", -1, enemy, own))
        else:
            out.append(("over", 1, own, enemy))
    return out


def analyse(positions, play_config, max_empties, report, stopped, solve_lane, solve_deep, search):
    """The analysis of `positions` (enumerate_positions) with the given exact solvers and search; `report(moves_made,
    value, exact)` receives the values in report order, and nothing once `stopped()` is true.
      solve_lane(own list, enemy list) -> exact scores (mover's frame), positions with at most 12 empties;
      solve_deep(own, enemy) -> exact score, or None when it timed out or was stopped;
      search(own list, enemy list) -> list of values (10 * q), or None when stopped.
    Returns False when stopped, else True."""
    kinds = classify(positions)
    value = {}   # (own, enemy) -> (value for its mover, exact)

    def solvable(own, enemy):
        return solves_exactly(play_config, own, enemy, max_empties)

    targets = []   # (own, enemy) to evaluate, without repeats, in game order
    for kind, _, own, enemy in kinds:
        if kind != "over" and (own, enemy) not in targets:
            targets.append((own, enemy))
    reported = set()

    def report_known(exact):
        """report, from the end backwards, every position not yet reported whose value is known (exact ones only when
        `exact`); False when stopped"""
        for i in range(len(positions) - 1, -1, -1):
            if i in reported:
                continue
            kind, sign, own, enemy = kinds[i]
            if kind == "over":
                v, ex = sign * (bit_count(own) - bit_count(enemy)), True
            elif (own, enemy) in value:
                v, ex = value[(own, enemy)]
                v = sign * v
            else:
                continue
            if ex != exact:
                continue
            if stopped():
                return False
            reported.add(i)
            report(positions[i].moves_made, v, ex)
        return True

    lane = [t for t in targets if solvable(*t) and 64 - bit_count(t[0] | t[1]) <= LANE_MAX_EMPTIES]
    deep = sorted((t for t in targets if solvable(*t) and 64 - bit_count(t[0] | t[1]) > LANE_MAX_EMPTIES),
                  key=lambda t: (64 - bit_count(t[0] | t[1]), -targets.index(t)))
    if lane:
        for t, sc in zip(lane, solve_lane([t[0] for t in lane], [t[1] for t in lane])):
            value[t] = (int(sc), True)
    if not report_known(True):
        return False
    for t in deep:
        if stopped():
            return False
        sc = solve_deep(*t)
        if sc is not None:
            value[t] = (int(sc), True)
            if not report_known(True):
                return False
    rest = [t for t in targets if t not in value]
    if rest:
        if stopped():
            return False
        vals = search([t[0] for t in rest], [t[1] for t in rest])
        if vals is None or stopped():
            return False
        for t, v in zip(rest, vals):
            value[t] = (float(v), False)
    return report_known(False)


def search_value(n, w):
    """go's evaluation of a searched position from its root statistics: 10 * q of the most visited move (first index),
    q = w / (n + 1e-5) in float64"""
    n, w = np.asarray(n, np.float64), np.asarray(w, np.float64)
    a = int(np.argmax(n))
    return float(w[a] / (n[a] + 1e-5)) * 10


def chunk_steps(total, per_sim):
    """the simulation counts of the chunks of a `total`-simulation search reported every `per_sim` simulations, as
    ReversiPlayer._search runs them: a remainder first (25 in chunks of 10 -> 5, 10, 10)"""
    chunk = int(per_sim) if per_sim and per_sim > 0 else int(total)
    steps, done = [], 0
    while done < total:
        step = (total - done) % chunk or chunk
        steps.append(step)
        done += step
    return steps


class GameAnalyser:
    """The device side of an analysis: a 64-slot engine with ReversiPlayer's search configuration (created at the first
    analysis and kept; it never touches the player's engine), the lane solver and the deep solver with a stop flag."""

    def __init__(self, config, model, play_config, device=0, seed=0):
        self.config = config
        self.play_config = play_config
        self.per_sim = int(config.nboard.hint_callback_per_sim)
        self.max_empties = solver_max_empties(config)
        self._stop_event = threading.Event()
        self._stop_flag = C.c_int32(0)
        pc = search_play_config(config, play_config)
        self._sims = int(pc.simulation_num_per_move)
        # one search per slot per analysis, from a fresh tree: arenas for simulation_num_per_move simulations
        ecfg = engine_cfg_from_play_config(pc, games=ANALYSIS_SLOTS, seed=seed, eval_mode=EVAL_NET if model is not None else EVAL_FAKE,
                                           max_searches_per_game=1, eval_cache_mb=ANALYSIS_CACHE_MB)
        self.engine = Engine(ecfg, model, device)
        self._engine_sims = self._sims
        self.deep_stats = []   # (empties, stats dict) of every deep solve, for tests and measurements

    def stop(self):
        """end a running analysis (any thread)"""
        self._stop_event.set()
        self._stop_flag.value = 1

    def reset_stop(self):
        self._stop_event.clear()
        self._stop_flag.value = 0

    def stopped(self):
        return self._stop_event.is_set()

    def analyse(self, black, white, player, actions, report):
        """report(moves_made, value, exact) for every position of the game; False when stopped"""
        return analyse(enumerate_positions(black, white, player, actions), self.play_config, self.max_empties, report,
                       self.stopped, self.solve_lane, self.solve_deep, self.search)

    def solve_lane(self, own, enemy):
        from ..lib.reversi_solver import solve_batch
        _, score = solve_batch(np.array(own, np.uint64), np.array(enemy, np.uint64), True)
        return [int(s) for s in score]

    def solve_deep(self, own, enemy):
        from ..lib.reversi_solver import solve_deep_batch
        mv, sc, st = solve_deep_batch([own], [enemy], DEEP_TIMEOUT, stats=True, stop=self._stop_flag)
        self.deep_stats.append((64 - bit_count(own | enemy), st[0]))
        return None if mv[0] < 0 else int(sc[0])

    def search(self, own, enemy):
        out = []
        for i in range(0, len(own), ANALYSIS_SLOTS):
            o, e = own[i:i + ANALYSIS_SLOTS], enemy[i:i + ANALYSIS_SLOTS]
            n = w = None
            for k, step in enumerate(chunk_steps(self._sims, self.per_sim)):
                if self.stopped():
                    return None
                if step != self._engine_sims:
                    self.engine.set_simulation_num(step)
                    self._engine_sims = step
                n, w = self.engine.search_roots(o, e, 1, keep_tree=k > 0)
            out += [search_value(n[j], w[j]) for j in range(len(o))]
        return out

    def close(self):
        self.engine.close()
