"""Mirror of the reference's ``ReversiPlayer`` (agent/player.py:28-436) for its single-game callers
(worker/evaluate.py:66-96, play_game/game_model.py, play_game/nboard.py): same constructor, ``action``,
``action_with_evaluation``, ``moves``, ``finish_game``, ``resigned``, ``stop_thinking``,
``ask_thought_about`` and the namedtuples.  The search itself runs on the device: a one-slot engine keeps
the transposition table across the moves of the game (the reference's MCTSInfo) and
``rz_engine_search_root`` performs ``simulation_num_per_move`` simulations per call.  Move choice,
resignation and the 8-symmetry training records follow agent/player.py:105-134,166-179 on the host.

Self-play does NOT go through this class -- thousands of games are played concurrently inside
``worker.self_play.SelfPlayWorker`` -- it exists so that the reference's other callers keep working.
"""
from collections import namedtuple
from logging import getLogger
from types import SimpleNamespace

import numpy as np

from ..engine import Engine, engine_cfg_from_play_config, EVAL_NET, EVAL_FAKE
from ..lib.bitboard import find_correct_moves, bit_to_array, flip_vertical, rotate90, bit_count

CounterKey = namedtuple("CounterKey", "black white next_player")
HistoryItem = namedtuple("HistoryItem", "action policy values visit enemy_values enemy_visit")
CallbackInMCTS = namedtuple("CallbackInMCTS", "per_sim callback")
MCTSInfo = namedtuple("MCTSInfo", "var_n var_w var_p")
ActionWithEvaluation = namedtuple("ActionWithEvaluation", "action n q")

logger = getLogger(__name__)


def solver_max_empties(config):
    """b200.solver_max_empties of a config; 12 (the lane solver alone) for a reference ``Config`` without ``b200``"""
    return int(getattr(getattr(config, "b200", None), "solver_max_empties", 12))


def solves_exactly(play_config, own, enemy, max_empties=64):
    """True where ReversiPlayer asks its exact root solver: ``use_solver_turn`` set and the turn (discs - 4) at least
    that.  With `max_empties`, also at most that many empty squares: the positions the solver answers rather than
    refuses, which the game analysis and NBoard's exact hints solve."""
    use_solver_turn = getattr(play_config, "use_solver_turn", None)
    discs = bit_count(own) + bit_count(enemy)
    return bool(use_solver_turn) and discs - 4 >= use_solver_turn and 64 - discs <= max_empties


def search_play_config(config, play_config):
    """The search parameters ReversiPlayer's engine runs with: `play_config`, except that the reference reads three of
    them from config.play even when a separate play_config is given (evaluate.py / play_game callers):
    allowed_resign_turn (agent/player.py:127, handled in action_with_evaluation), use_solver_turn_in_simulation
    (:237-238) and virtual_loss (:264).  thinking_loop is at least 1 (the loop runs on the host, see there)."""
    search_pc = SimpleNamespace(**vars(play_config))
    for k in ("use_solver_turn_in_simulation", "virtual_loss"):
        if hasattr(config.play, k):
            setattr(search_pc, k, getattr(config.play, k))
    search_pc.thinking_loop = max(1, int(search_pc.thinking_loop))
    return search_pc


class ReversiPlayer:
    def __init__(self, config, model, play_config=None, enable_resign=True, mtcs_info=None, api=None, seed=0, device=0):
        """model: a ``reversi_zero_b200.net.Net`` (None selects the deterministic test evaluator).
        mtcs_info / api are accepted for signature compatibility; statistics live on the device."""
        self.config = config
        self.model = model
        self.play_config = play_config or self.config.play
        self.enable_resign = enable_resign
        self.api = api
        ecfg = engine_cfg_from_play_config(search_play_config(self.config, self.play_config), games=1, seed=seed,
                                           eval_mode=EVAL_NET if model is not None else EVAL_FAKE)
        self.engine = Engine(ecfg, model, device)
        self._fresh = True
        self._engine_sims = int(self.play_config.simulation_num_per_move)
        self.solver = None
        self.moves = []
        self.thinking_history = {}
        self.resigned = False
        self.requested_stop_thinking = False
        self.callback_in_mtcs = None

    @staticmethod
    def create_mtcs_info():
        from collections import defaultdict
        return MCTSInfo(defaultdict(lambda: np.zeros((64,))), defaultdict(lambda: np.zeros((64,))),
                        defaultdict(lambda: np.zeros((64,))))

    def action(self, own, enemy, callback_in_mtcs=None, solve=True):
        return self.action_with_evaluation(own, enemy, callback_in_mtcs=callback_in_mtcs, solve=solve).action

    def _search(self, own, enemy):
        """simulation_num_per_move simulations from (own, enemy); with a CallbackInMCTS the search runs in chunks of
        `per_sim` simulations (the tree is kept between chunks) and reports (q, n) after each, like
        agent/player.py:212-214; stop_thinking() ends it early (:206-208).  The reference reports whenever the number of
        simulations still to finish is a multiple of `per_sim`, so a remainder comes first: 25 in chunks of 10 -> 5, 10, 10."""
        total = int(self.play_config.simulation_num_per_move)
        cb = self.callback_in_mtcs
        chunk = int(cb.per_sim) if cb and cb.per_sim > 0 else total
        done, n, w = 0, None, None
        while done < total and not (self.requested_stop_thinking and done > 0):
            step = (total - done) % chunk or chunk
            if step != self._engine_sims:
                self.engine.set_simulation_num(step)
                self._engine_sims = step
            n, w = self.engine.search_root(int(own), int(enemy), 1, 0, keep_tree=not self._fresh)
            self._fresh = False
            done += step
            if cb and cb.per_sim > 0:
                cb.callback(list(w / (n + 1e-5)), list(n))
        return n.astype(np.float64), w.astype(np.float64)

    def action_with_evaluation(self, own, enemy, callback_in_mtcs=None, solve=True):
        """agent/player.py:82-134; the exact root solver (:100-103,150-161) runs through lib/reversi_solver (rz_solve), the
        WLD solver inside simulations (:237-251) inside the engine.  solve=False searches even where the root solver would
        answer (NBoard's hint, after an exact solve that proved nothing)."""
        pc = self.play_config
        turn = bit_count(own) + bit_count(enemy) - 4
        self.callback_in_mtcs = callback_in_mtcs
        self.requested_stop_thinking = False
        if solve and solves_exactly(pc, own, enemy):  # action_by_searching, agent/player.py:100-103,150-161
            if self.solver is None:
                from ..lib import reversi_solver
                self.solver = reversi_solver.ReversiSolver(solver_max_empties(self.config))
            mv, score = self.solver.solve(own, enemy, 1, exactly=True)
            if mv is not None:
                policy = np.zeros(64)
                policy[mv] = 1
                # :157-160: N = 999 and W = sign(score) * 999 on the solved move
                n, w = np.zeros(64), np.zeros(64)
                n[mv], w[mv] = 999, np.sign(score) * 999
                self.thinking_history[(own, enemy)] = HistoryItem(mv, policy, list(w / (n + 1e-5)), list(n), None, None)
                return ActionWithEvaluation(action=mv, n=999, q=float(np.sign(score)))  # not saved as play data
        n = w = None
        # at least one search: NBoard's `set depth` can make thinking_loop 0 (e.g. depth 1 at 200 simulations per move),
        # where the reference fails with an unbound `action`
        for tl in range(max(1, pc.thinking_loop)):
            if turn > 0:
                n, w = self._search(own, enemy)
            else:  # bypass_first_move, agent/player.py:143-148
                legal = bit_to_array(find_correct_moves(own, enemy), 64)
                n, w = np.zeros(64), np.zeros(64)
                n[int(np.argmax(legal))] = 1
            q = w / (n + 1e-5)
            policy = self.calc_policy_from(n, turn)
            action = int(np.random.choice(range(64), p=policy))
            action_by_value = int(np.argmax(q + (n > 0) * 100))
            value_diff = q[action] - q[action_by_value]
            if turn <= pc.start_rethinking_turn or self.requested_stop_thinking or \
                    (value_diff > -0.01 and n[action] >= pc.required_visit_to_decide_action):
                break
        self.thinking_history[(own, enemy)] = HistoryItem(action, policy, list(q), list(n), None, None)
        if pc.resign_threshold is not None and np.max(q - (n == 0) * 10) <= pc.resign_threshold:
            self.resigned = True
            if self.enable_resign and turn >= self.config.play.allowed_resign_turn:
                return ActionWithEvaluation(None, 0, 0)
        saved_policy = n / np.sum(n) if self.config.play_data.save_policy_of_tau_1 else policy
        self.add_data_to_move_buffer_with_8_symmetries(own, enemy, saved_policy)
        return ActionWithEvaluation(action=action, n=n[action], q=q[action])

    def calc_policy_from(self, n, turn):
        """agent/player.py:366-385"""
        if turn < self.play_config.change_tau_turn:
            return n / np.sum(n)
        ret = np.zeros(64)
        ret[int(np.argmax(n))] = 1
        return ret

    def add_data_to_move_buffer_with_8_symmetries(self, own, enemy, policy):
        """agent/player.py:166-179"""
        for flip in (False, True):
            for rot_right in range(4):
                o, e, p = own, enemy, np.asarray(policy).reshape((8, 8))
                if flip:
                    o, e, p = flip_vertical(o), flip_vertical(e), np.flipud(p)
                for _ in range(rot_right):
                    o, e = rotate90(o), rotate90(e)
                if rot_right:
                    p = np.rot90(p, k=-rot_right)
                self.moves.append([(o, e), list(p.reshape((64,)))])

    def stop_thinking(self):
        self.requested_stop_thinking = True

    def ask_thought_about(self, own, enemy):
        return self.thinking_history.get((own, enemy))

    def finish_game(self, z):
        """agent/player.py:357-364"""
        for move in self.moves:
            move += [z]
