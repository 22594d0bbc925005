"""Python handle of the on-device self-play engine (rz_engine_* in include/rz_engine.h)."""
import ctypes as C
import math

import numpy as np

from . import _cabi

EVAL_NET, EVAL_FAKE = 0, 1
MAX_OPENING_PLIES = 20  # RZ_MAX_OPENING_PLIES


def engine_cfg_from_play_config(pc, pdc=None, games=1024, seed=0, eval_mode=EVAL_NET, net_impl=0, first_game_id=0,
                                game_id_stride=1, max_games=0, warm_start=False, overlap_groups=0,
                                max_searches_per_game=0, use_solver=True, arena_simulation_num=0, eval_cache_mb=0):
    """Build an rz_engine_cfg from objects with the reference's PlayConfig / PlayDataConfig fields
    (config.py:116-166).  eval_cache_mb: size of the evaluation cache (0 = default, < 0 = off; include/rz_engine.h)."""
    cfg = _cabi.EngineCfg()
    cfg.games = games
    cfg.simulation_num_per_move = int(pc.simulation_num_per_move)
    cfg.parallel_search_num = int(pc.parallel_search_num)
    cfg.virtual_loss = int(pc.virtual_loss)
    cfg.change_tau_turn = int(pc.change_tau_turn)
    cfg.thinking_loop = int(pc.thinking_loop)
    cfg.required_visit_to_decide_action = int(pc.required_visit_to_decide_action)
    cfg.start_rethinking_turn = int(pc.start_rethinking_turn)
    cfg.allowed_resign_turn = int(pc.allowed_resign_turn)
    cfg.use_resign_threshold = 0 if pc.resign_threshold is None else 1
    cfg.share_mtcs_info = 1 if pc.share_mtcs_info_in_self_play else 0
    cfg.eval_mode = eval_mode
    cfg.net_impl = net_impl
    cfg.max_plies = 64
    cfg.warm_start = 1 if warm_start else 0
    cfg.overlap_groups = overlap_groups
    cfg.max_searches_per_game = max_searches_per_game
    cfg.arena_simulation_num = int(arena_simulation_num or 0)
    cfg.eval_cache_mb = int(eval_cache_mb)
    cfg.max_sims_per_wave = int(getattr(pc, "max_sims_per_wave", 0) or 0)
    cfg.reset_mtcs_info_per_game = int(getattr(pc, "reset_mtcs_info_per_game", 1) or 1) if cfg.share_mtcs_info else 1
    cfg.use_solver_turn = int(getattr(pc, "use_solver_turn", 0) or 0) if use_solver else 0
    cfg.use_solver_turn_in_simulation = int(getattr(pc, "use_solver_turn_in_simulation", 0) or 0) if use_solver else 0
    cfg.c_puct = float(pc.c_puct)
    cfg.noise_eps = float(pc.noise_eps)
    cfg.dirichlet_alpha = float(pc.dirichlet_alpha)
    cfg.resign_threshold = 0.0 if pc.resign_threshold is None else float(pc.resign_threshold)
    cfg.disable_resignation_rate = float(pc.disable_resignation_rate)
    cfg.seed = seed
    cfg.first_game_id = first_game_id
    cfg.game_id_stride = game_id_stride
    cfg.max_games = max_games
    return cfg


class Engine:
    def __init__(self, cfg, net=None, device=0):
        self.cfg = cfg
        self.net = net  # keep alive
        self._h = C.c_void_p()
        _cabi.check(_cabi.lib().rz_engine_create(C.byref(cfg), net.handle if net is not None else None, device, C.byref(self._h)),
                    "rz_engine_create")
        self._games = (_cabi.Game * 256)()
        self._plies = (_cabi.Ply * (256 * 64))()

    def run(self, finished_target=0, max_waves=0):
        _cabi.check(_cabi.lib().rz_engine_run(self._h, finished_target, max_waves), "rz_engine_run")

    def poll_raw(self):
        """-> (games ctypes array slice, plies ctypes array slice) for up to 256 games."""
        ng, npl = C.c_size_t(), C.c_size_t()
        _cabi.check(_cabi.lib().rz_engine_poll(self._h, self._games, 256, C.byref(ng), self._plies, 256 * 64, C.byref(npl)),
                    "rz_engine_poll")
        return self._games, ng.value, self._plies, npl.value

    def poll(self):
        """-> list of dicts (one per finished game) with python ints and numpy visit counts."""
        out = []
        while True:
            games, ng, plies, _ = self.poll_raw()
            if ng == 0:
                break
            for i in range(ng):
                g = games[i]
                pl = []
                for j in range(g.first_ply, g.first_ply + g.n_plies):
                    p = plies[j]
                    pl.append(dict(own=int(p.own), enemy=int(p.enemy), N=np.array(p.n_visit[:], dtype=np.int64), action=int(p.action),
                                   pid=int(p.player), loops=int(p.loops), recorded=bool(p.recorded), n=float(p.n), q=float(p.q),
                                   waves=int(p.waves)))
                out.append(dict(game_id=int(g.game_id), black=int(g.black), white=int(g.white), winner=int(g.winner),
                                black_z=int(g.black_z), expansions=int(g.expansions), simulations=int(g.simulations),
                                resign_enabled=bool(g.resign_enabled), resigned_mask=int(g.resigned_mask), turn=int(g.turn),
                                black_net=int(g.black_net), white_net=int(g.white_net), opening_plies=int(g.opening_plies),
                                table_nodes=int(g.table_nodes), plies=pl))
        return out

    def stats(self):
        s = _cabi.Stats()
        _cabi.check(_cabi.lib().rz_engine_stats(self._h, C.byref(s)), "rz_engine_stats")
        return {n: (float if t is C.c_double else int)(getattr(s, n)) for n, t in _cabi.Stats._fields_}

    def cache_turn_stats(self):
        """-> (lookups, hits): numpy uint64 [61]; entry t < 60 counts searches at turn t, entry 60 the warm-started first
        games of the slots (rz_engine_cache_turn_stats)."""
        lookups, hits = np.zeros(61, np.uint64), np.zeros(61, np.uint64)
        _cabi.check(_cabi.lib().rz_engine_cache_turn_stats(self._h, lookups.ctypes.data_as(_cabi.u64p), hits.ctypes.data_as(_cabi.u64p), 61),
                    "rz_engine_cache_turn_stats")
        return lookups, hits

    def set_simulation_num(self, sims):
        _cabi.check(_cabi.lib().rz_engine_set_simulation_num(self._h, int(sims)), "rz_engine_set_simulation_num")

    def set_max_games(self, n):
        """no slot starts a game whose local index is >= n (0 = unlimited); 1 drains the engine"""
        _cabi.check(_cabi.lib().rz_engine_set_max_games(self._h, int(n)), "rz_engine_set_max_games")

    def set_warm_start_profile(self, weights):
        w = np.ascontiguousarray(weights, dtype=np.float32)
        _cabi.check(_cabi.lib().rz_engine_set_warm_start_profile(self._h, w.ctypes.data_as(_cabi.f32p), int(w.size)),
                    "rz_engine_set_warm_start_profile")

    def set_second_net(self, net_b=None, enable=True):
        """evaluation matches: even local game indices -> first network plays black, odd -> second network."""
        self.net_b = net_b  # keep alive
        _cabi.check(_cabi.lib().rz_engine_set_second_net(self._h, net_b.handle if net_b is not None else None, int(bool(enable))),
                    "rz_engine_set_second_net")

    def set_nets(self, nets, black, white, fake_scales=None):
        """leagues (rz_engine_set_nets): the game with local index i is played by nets[black[i]] as black and
        nets[white[i]] as white.  ``nets`` may hold None with the deterministic evaluator, whose network k then has its
        value multiplied by fake_scales[k] (None: all 1).  Call before the first run, with max_games in 1..len(black)."""
        black = np.ascontiguousarray(black, dtype=np.uint8).reshape(-1)
        white = np.ascontiguousarray(white, dtype=np.uint8).reshape(-1)
        if black.shape != white.shape:
            raise ValueError("black and white differ in length")
        handles = (C.c_void_p * max(len(nets), 1))(*[n.handle if n is not None else None for n in nets])
        scales = None
        if fake_scales is not None:
            sc = np.ascontiguousarray(fake_scales, dtype=np.float32)
            if sc.size != len(nets):
                raise ValueError("one fake scale per network")
            scales = sc.ctypes.data_as(_cabi.f32p)
        _cabi.check(_cabi.lib().rz_engine_set_nets(self._h, handles, scales, len(nets), black.ctypes.data_as(_cabi.u8p),
                                                    white.ctypes.data_as(_cabi.u8p), int(black.size)), "rz_engine_set_nets")
        self.nets = list(nets)  # keep alive

    def set_openings(self, openings):
        """games from openings (rz_engine_set_openings): the game with local index i starts after the squares openings[i]
        (a sequence of 0..RZ_MAX_OPENING_PLIES moves, 0..63), played without a search and not recorded.  Call before the
        first run, with max_games in 1..len(openings)."""
        n = len(openings)
        moves = np.zeros((max(n, 1), MAX_OPENING_PLIES), np.uint8)
        n_moves = np.zeros(max(n, 1), np.uint8)
        for i, seq in enumerate(openings):
            seq = [int(a) for a in seq]
            if len(seq) > MAX_OPENING_PLIES or any(not 0 <= a < 64 for a in seq):
                raise ValueError(f"opening {i}: {seq} is not a sequence of at most {MAX_OPENING_PLIES} squares 0..63")
            moves[i, :len(seq)] = seq
            n_moves[i] = len(seq)
        _cabi.check(_cabi.lib().rz_engine_set_openings(self._h, moves.ctypes.data_as(_cabi.u8p), n_moves.ctypes.data_as(_cabi.u8p), n),
                    "rz_engine_set_openings")

    def set_resign_threshold(self, threshold):
        _cabi.check(_cabi.lib().rz_engine_set_resign_threshold(self._h, 0 if threshold is None else 1,
                                                               0.0 if threshold is None else float(threshold)),
                    "rz_engine_set_resign_threshold")

    def search_root(self, own, enemy, player, slot=0, keep_tree=False):
        n = np.zeros(64, np.int32)
        w = np.zeros(64, np.float32)
        _cabi.check(_cabi.lib().rz_engine_search_root(self._h, own, enemy, player, slot, int(keep_tree), n.ctypes.data_as(_cabi.i32p),
                                                       w.ctypes.data_as(_cabi.f32p)), "rz_engine_search_root")
        return n, w

    def search_roots(self, own, enemy, player, keep_tree=False):
        """One root per slot (rz_engine_search_roots): slot i searches (own[i], enemy[i]) in the mover's frame with
        player[i] (1 or 2, or one value for all) to move.  -> (n int32 [len(own), 64], w float32 [len(own), 64])."""
        own = np.ascontiguousarray(own, dtype=np.uint64).reshape(-1)
        enemy = np.ascontiguousarray(enemy, dtype=np.uint64).reshape(-1)
        pl = np.ascontiguousarray(np.broadcast_to(np.asarray(player, dtype=np.uint8), own.shape))
        if enemy.shape != own.shape:
            raise ValueError("own and enemy differ in length")
        n = np.zeros((own.size, 64), np.int32)
        w = np.zeros((own.size, 64), np.float32)
        _cabi.check(_cabi.lib().rz_engine_search_roots(self._h, own.ctypes.data_as(_cabi.u64p), enemy.ctypes.data_as(_cabi.u64p),
                                                        pl.ctypes.data_as(_cabi.u8p), int(own.size), int(keep_tree),
                                                        n.ctypes.data_as(_cabi.i32p), w.ctypes.data_as(_cabi.f32p)),
                    "rz_engine_search_roots")
        return n, w

    def close(self):
        if self._h:
            _cabi.lib().rz_engine_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def write_play_data(path, games, n_games, plies, save_policy_of_tau_1=True, change_tau_turn=4):
    """games / plies: ctypes arrays as returned by Engine.poll_raw()."""
    n = C.c_size_t()
    _cabi.check(_cabi.lib().rz_write_play_data(path.encode(), games, n_games, plies, int(bool(save_policy_of_tau_1)),
                                                int(change_tau_turn), C.byref(n)), "rz_write_play_data")
    return n.value
