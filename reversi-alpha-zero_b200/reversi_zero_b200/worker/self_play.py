"""Mirror of the reference's self-play worker (worker/self_play.py) on the H100 engine.

``start(config)`` / ``SelfPlayWorker(config, env, api, shared_var, worker_index).start()`` keep the
reference's entry points (manager.py:51-53, worker/self_play.py:28-41,64-93) and output contract:
``play_%Y%m%d-%H%M%S.%f.json`` files of ``[[own, enemy], [64 floats], z]`` records (self_play.py:180-194),
``self_play-*.ggf`` game records (:196-207), pruning to ``max_file_num`` files (:209-217), the
``.self-play-game-idx`` counter (:35,136-137), the simulation-count schedule / ``.force-sim`` override
(:262-272), draw dropping (:182) and the resignation-threshold auto-tuner (:219-260).

What differs by design: the reference forks ``multi_process_num`` Python workers that play one game
each and talk to a Keras server through pipes; here ONE process per GPU drives ``b200.games_per_gpu``
concurrent games that live entirely on the device (csrc/rz_engine.cu); finished games are harvested and
written by a second host thread (``rz_engine_poll`` is the consumer end of a single-producer / single-consumer
queue) while the first keeps the waves going, so the GPU never waits for the Python bookkeeping or the files
(the reference overlaps the same work through its worker processes, worker/self_play.py:36-41).  Across GPUs the game-id space is strided by rank and every rank writes its own files
(SURVEY 8(e)); the only collective is the weight broadcast.
"""
import os
import threading
import time
from datetime import datetime
from logging import getLogger

import numpy as np

from .. import _cabi
from ..agent import model as M
from ..engine import Engine, engine_cfg_from_play_config, write_play_data, EVAL_NET
from ..lib.ggf import convert_action_to_move, make_ggf_string
from ..net import Net

logger = getLogger(__name__)


def start(config):
    return SelfPlayWorker(config).start()


def read_as_int(filename):
    """lib/file_util.py:4-13"""
    if os.path.exists(filename):
        try:
            with open(filename, "rt") as f:
                ret = int(str(f.read()).strip())
                if ret:
                    return ret
        except ValueError:
            pass


def _b200(config):
    from ..config import B200Config
    return getattr(config, "b200", None) or B200Config()


NEXT_GENERATION_BLOB = "model_weight.rzblob.npy"  # next to model_weight.h5 in next_generation/model_*/ (tools/export_keras_weights.py)


def load_or_build_weights(config, net):
    """agent/api.py:102-115 load_model: with ``play.use_newest_next_generation_model`` (the default, config.py:166) the
    newest next-generation weights, else -- or if there are none -- the best weights; nothing there (or ``--new``):
    build() + save_as_best.  The engine-side hand-off files are float32 .npy blobs (SURVEY 8(f).1) written next to the
    trainer's h5 files by tools/export_keras_weights.py; a model directory that holds ONLY h5 files is refused loudly
    (reading HDF5 without libhdf5 cannot be pinned in this image, and start-up and hot reload must see the same files)."""
    new = getattr(config.opts, "new", False)
    path = None if new else weight_source_path(config)
    if path is not None:
        blob = np.load(path)
        logger.debug(f"loading weights from {path}")
    else:
        h5_path = None if new else keras_h5_source_path(config)
        if h5_path is not None:
            raise RuntimeError(f"{h5_path} exists but its engine-side twin (*.rzblob.npy) does not: run "
                               f"`python tools/export_keras_weights.py <model_config.json> {h5_path}` on the trainer side "
                               f"(INTEGRATION.md section 4), or start with opts.new to random-initialise")
        path = blob_path_of(config)
        blob = M.weights_to_blob(config.model, M.build_random_weights(config.model, _b200(config).weight_seed))
        os.makedirs(os.path.dirname(path), exist_ok=True)
        np.save(path, blob)
        logger.debug(f"built random-init weights, saved to {path}")
    net.load_blob(blob)
    return blob


def blob_path_of(config):
    rc = config.resource
    return getattr(rc, "model_best_blob_path", os.path.join(rc.model_dir, "model_best_weight.rzblob.npy"))


def newest_next_generation_blob(config):
    """lib/model_helpler.py:50-63 + lib/data_helper.py:17-20: the weight blob in the last (sorted) next_generation/model_* directory"""
    from glob import glob
    rc = config.resource
    base = getattr(rc, "next_generation_model_dir", os.path.join(rc.model_dir, "next_generation"))
    tmpl = getattr(rc, "next_generation_model_dirname_tmpl", "model_%s")
    for d in reversed(sorted(glob(os.path.join(base, tmpl % "*")))):
        path = os.path.join(d, NEXT_GENERATION_BLOB)
        return path if os.path.exists(path) else None   # only the newest directory counts, like the reference
    return None


def keras_h5_source_path(config):
    """The reference's own weight files (config.py:30-40), same newest-first / best-first rule as weight_source_path."""
    from glob import glob
    rc = config.resource
    best = getattr(rc, "model_best_weight_path", os.path.join(rc.model_dir, "model_best_weight.h5"))
    best = best if os.path.exists(best) else None
    base = getattr(rc, "next_generation_model_dir", os.path.join(rc.model_dir, "next_generation"))
    tmpl = getattr(rc, "next_generation_model_dirname_tmpl", "model_%s")
    newest = None
    for d in reversed(sorted(glob(os.path.join(base, tmpl % "*")))):
        cand = os.path.join(d, getattr(rc, "next_generation_model_weight_filename", "model_weight.h5"))
        newest = cand if os.path.exists(cand) else None
        break
    if getattr(config.play, "use_newest_next_generation_model", True):
        return newest or best
    return best or newest


def weight_source_path(config):
    """The file self-play takes its weights from right now (agent/api.py:107-110,120-123), or None."""
    best = blob_path_of(config)
    best = best if os.path.exists(best) else None
    newest = newest_next_generation_blob(config)
    if getattr(config.play, "use_newest_next_generation_model", True):
        return newest or best
    return best or newest


class SelfPlayWorker:
    MODEL_CHECK_INTERVAL_SEC = 60  # agent/api.py:80-82
    WAVES_PER_RUN = 32             # waves between two control points of the driving thread (commands of the writer thread,
                                   # weight-reload check, stop rules); rz_engine_run itself looks at the device every 8 waves

    def __init__(self, config, env=None, api=None, shared_var=None, worker_index=0, net=None, device=0, rank=0,
                 world_size=1):
        """env / api / shared_var are accepted for signature compatibility with the reference
        (worker/self_play.py:65-86); games run on the device and ``net`` (a ``reversi_zero_b200.net.Net``)
        takes the place of the API client."""
        self.config = config
        self.env = env
        self.api = api
        self.shared_var = shared_var
        self.worker_index = worker_index
        self.net = net
        self.device = device
        self.rank, self.world_size = rank, world_size
        self.buffer_games = []        # (Game header copy, [Ply copies]) kept for the next play_data file
        self.ggf_lines = []
        self.false_positive_count_of_resign = 0
        self.resign_test_game_count = 0
        self.engine = None
        self.local_idx = 0
        self.game_idx = 0
        self.files_written = []
        self.bytes_written = 0
        self.last_model_check_time = time.time()
        self.tensor_board = None
        # the writer thread: harvests finished games (rz_engine_poll), keeps the reference's per-game bookkeeping and writes
        # the files while the driving thread is inside rz_engine_run.  Engine calls it wants made (new simulation count,
        # new resignation threshold) are queued and made by the driving thread between two runs: handles are not thread-safe.
        self._writer = None
        self._writer_stop = threading.Event()
        self._writer_error = None
        self._cmds = []
        self._cmd_lock = threading.Lock()

    # -- reference helpers ---------------------------------------------------------------------------------
    def decide_simulation_num_per_move(self, idx):
        """worker/self_play.py:262-272"""
        ret = read_as_int(self.config.resource.force_simulation_num_file)
        if ret:
            return ret
        for min_idx, num in self.config.play.schedule_of_simulation_num_per_move:
            if idx >= min_idx:
                ret = num
        return ret

    def largest_simulation_num(self):
        """The largest count decide_simulation_num_per_move can return during this run as far as it is known now: every
        entry of the schedule and the current ``.force-sim`` value.  The engine's arenas are sized for it
        (rz_engine_cfg.arena_simulation_num); a later, larger ``.force-sim`` makes the worker drain and re-create the
        engine (_rebuild_engine)."""
        nums = [int(num) for _, num in self.config.play.schedule_of_simulation_num_per_move]
        nums.append(read_as_int(self.config.resource.force_simulation_num_file) or 0)
        return max(nums + [1])

    @property
    def false_positive_rate(self):
        if self.resign_test_game_count == 0:
            return 0
        return self.false_positive_count_of_resign / self.resign_test_game_count

    def check_and_update_resignation_threshold(self):
        """worker/self_play.py:250-260"""
        pc = self.config.play
        if self.resign_test_game_count < 100 or pc.resign_threshold is None:
            return
        old = pc.resign_threshold
        if self.false_positive_rate >= pc.false_positive_threshold:
            pc.resign_threshold -= pc.resign_threshold_delta
        else:
            pc.resign_threshold += pc.resign_threshold_delta
        logger.debug(f"update resign_threshold: {old} -> {pc.resign_threshold}")
        self.false_positive_count_of_resign = 0
        self.resign_test_game_count = 0
        self._engine_cmd("set_resign_threshold", pc.resign_threshold)

    def try_reload_model(self, force_check=False, check_now=None):
        """agent/api.py:117-125 + lib/model_helpler.py digest logic: every 60 s look at the weight hand-off file
        and, if its sha256 differs from the loaded weights, load it between two waves.  With several ranks every rank
        must call this at the same control point (start() sees to that: the decision to check is part of the control
        all-reduce); rank 0 reads the file and broadcasts flag + blob, so all GPUs switch at the same point."""
        if check_now is None:
            check_now = force_check or time.time() - self.last_model_check_time >= self.MODEL_CHECK_INTERVAL_SEC
        if not check_now:
            return False
        self.last_model_check_time = time.time()
        # agent/api.py:117-125: the newest next-generation model if configured (and present), else the best model (the
        # reference checks ONLY the newest model when configured; also looking at the best file when there is no
        # next-generation model is a harmless superset: after a promotion both hold the same weights)
        newest = newest_next_generation_blob(self.config) if getattr(self.config.play, "use_newest_next_generation_model", True) else None
        path = newest or blob_path_of(self.config)
        blob = None
        changed = False
        if self.rank == 0 and os.path.exists(path):
            try:
                blob = np.load(path)
                changed = blob.size == self.net.blob_floats and M.blob_digest(blob) != self.net.digest
            except Exception as e:  # partially written file: try again at the next check
                logger.error(e)
        if self.world_size > 1:
            import torch
            import torch.distributed as dist
            from ..parallel import broadcast_blob, control_device
            dev = control_device(self.device)
            flag = torch.tensor([1 if changed else 0], dtype=torch.int32, device=dev)
            dist.broadcast(flag, src=0)
            if not int(flag.item()):
                return False
            t = broadcast_blob(self.config.model, blob, f"cuda:{self.device}" if dev != "cpu" else "cpu")
            if dev != "cpu":
                torch.cuda.synchronize()
                self.net.load_blob_dev(t)
                self.net.digest = M.blob_digest(t.cpu().numpy())
            else:
                self.net.load_blob(t.numpy())
            return True
        if changed:
            self.net.load_blob(blob)
            logger.debug(f"reloaded weights, digest = {self.net.digest}")
        return changed

    # -- engine plumbing ------------------------------------------------------------------------------------
    def _make_engine(self):
        cfg, b = self.config, _b200(self.config)
        rc = cfg.resource
        rc.create_directories() if hasattr(rc, "create_directories") else None
        if self.net is None:
            self.net = Net(cfg.model, self.device)
            load_or_build_weights(cfg, self.net)
        self.game_idx = read_as_int(rc.self_play_game_idx_file) or 0
        sims = self.decide_simulation_num_per_move(self.game_idx)
        cfg.play.simulation_num_per_move = sims
        ecfg = engine_cfg_from_play_config(cfg.play, games=b.games_per_gpu, seed=b.seed, eval_mode=EVAL_NET, net_impl=b.net_impl,
                                           first_game_id=self.game_idx + self.rank, game_id_stride=self.world_size,
                                           arena_simulation_num=max(sims, self.largest_simulation_num()),
                                           warm_start=getattr(b, "warm_start", False))
        self.engine = Engine(ecfg, self.net, self.device)
        profile = getattr(b, "warm_start_profile", None)
        if profile is not None and getattr(b, "warm_start", False):
            self.engine.set_warm_start_profile(profile)

    def _engine_cmd(self, name, *args):
        """An engine call asked for by the per-game bookkeeping: made at once on the driving thread, queued for it when the
        bookkeeping runs on the writer thread."""
        if self._writer is not None and threading.current_thread() is self._writer:
            with self._cmd_lock:
                self._cmds.append((name, args))
        else:
            self._apply_cmd(name, args)

    def _apply_cmd(self, name, args):
        if name == "set_simulation_num":
            if getattr(self, "_rebuilding", False):
                return   # the engine being created takes its count from decide_simulation_num_per_move
            try:
                self.engine.set_simulation_num(*args)
            except _cabi.RzError as ex:   # the arenas were sized for fewer simulations (a new, larger .force-sim)
                logger.info(f"{ex}: draining the resident games and re-creating the engine")
                self._rebuild_engine()
        else:
            getattr(self.engine, name)(*args)

    def _apply_pending_cmds(self):
        with self._cmd_lock:
            cmds, self._cmds = self._cmds, []
        for name, args in cmds:
            self._apply_cmd(name, args)

    def _rebuild_engine(self):
        """The simulation count asked for does not fit the arenas: let the resident games finish (no slot starts another
        one), harvest them, and create a new engine sized for the new count; game ids go on where the old engine stopped."""
        threaded = self._writer is not None
        self._rebuilding = True
        try:
            self.engine.set_max_games(1)
            self.engine.run()                  # returns when every slot is idle
            self._stop_writer()
            self._finished_before = getattr(self, "_finished_before", 0) + self.engine.stats()["games_finished"]
            self.engine.close()
            self.engine = None
            self._make_engine()
        finally:
            self._rebuilding = False
        if threaded:
            self._start_writer()

    def _start_writer(self):
        self._writer_stop.clear()
        self._writer = threading.Thread(target=self._writer_loop, name=f"rz-writer-{self.rank}", daemon=True)
        self._writer.start()

    def _stop_writer(self):
        """join the writer thread and take what is left in the engine's queue"""
        if self._writer is not None:
            self._writer_stop.set()
            self._writer.join()
            self._writer = None
        if self._writer_error is not None:
            err, self._writer_error = self._writer_error, None
            raise err
        self._harvest()

    def _writer_loop(self):
        try:
            while not self._writer_stop.is_set():
                if self._harvest() == 0:
                    self._writer_stop.wait(0.02)
        except BaseException as ex:  # reported by the driving thread at its next control point
            self._writer_error = ex

    def _control(self, want_check, time_up, games_done):
        """One control point per run of WAVES_PER_RUN waves.  With several ranks the three decisions are all-reduced, so
        that every rank checks for new weights (a collective) and leaves the loop at the same iteration: the check is
        rank 0's decision, time is up when it is up anywhere, the game target is reached when it is reached everywhere."""
        if self.world_size == 1:
            return want_check, time_up or games_done
        import torch
        import torch.distributed as dist
        from ..parallel import control_device
        t = torch.tensor([int(want_check and self.rank == 0), int(time_up), int(not games_done)], dtype=torch.int32,
                         device=control_device(self.device))
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        check, up, not_done = (int(x) for x in t.tolist())
        return bool(check), bool(up) or not not_done

    def start(self, max_games=None, max_seconds=None, max_waves=None, threaded=True):
        """Runs until max_games finished / max_seconds elapsed / max_waves executed (all None: forever, like the
        reference).  Returns the number of games harvested by this call.  Engine requests the bookkeeping queued after the last
        control point (e.g. a simulation count that needs new arenas) stay queued and are applied by the next call.  ``threaded=False`` harvests on the driving
        thread between two runs (the round-1 behaviour, kept for A/B measurements)."""
        if self.engine is None:
            self._make_engine()
        t0 = time.time()
        local0 = self.local_idx
        self._finished_before = -self.engine.stats()["games_finished"]   # games finished before this call do not count
        waves0 = self.engine.stats()["waves"]
        waves_done = 0
        if threaded:
            self._start_writer()
        try:
            while True:
                chunk = self.WAVES_PER_RUN if max_waves is None else min(self.WAVES_PER_RUN, max_waves - waves_done)
                target = 0
                if max_games is not None:
                    # rz_engine_run's target is cumulative per engine
                    target = max(1, max_games - self._finished_before)
                eng = self.engine
                eng.run(finished_target=target, max_waves=max(1, chunk))
                if not threaded:
                    self._harvest()
                if self._writer_error is not None:
                    raise self._writer_error
                st = eng.stats()
                waves_done = st["waves"] - waves0
                finished = self._finished_before + st["games_finished"]
                self._apply_pending_cmds()       # may re-create the engine
                if self.engine is not eng:
                    waves0 = -waves_done
                want_check = time.time() - self.last_model_check_time >= self.MODEL_CHECK_INTERVAL_SEC
                check, stop = self._control(want_check, max_seconds is not None and time.time() - t0 >= max_seconds,
                                            (max_games is not None and finished >= max_games) or
                                            (max_waves is not None and waves_done >= max_waves))
                if check:
                    # agent/api.py:80-83: at every model check the reference's prediction server logs its mean batch size
                    last = getattr(self, "_batch_stats", (0, 0))
                    cur = (st.get("expansions", 0), st.get("nn_launches", 0))
                    if self.engine is eng and cur[1] > last[1]:
                        logger.debug(f"average_prediction_size={(cur[0] - last[0]) / (cur[1] - last[1]):.1f}")
                    self._batch_stats = cur if self.engine is eng else (0, 0)
                    self.try_reload_model(check_now=True)
                if stop:
                    break
        finally:
            if threaded:
                self._stop_writer()
        self._flush_files(force=True)
        return self.local_idx - local0

    def _log_scalars(self, g, n_plies, seconds_per_game):
        """worker/self_play.py:125-129: self/time, self/turn, self/mcts_buffer_size (+ engine counters) under
        logs/tensorboard/self_play/workerNNN"""
        if self.tensor_board is None:
            try:
                from torch.utils.tensorboard import SummaryWriter
                self.tensor_board = SummaryWriter(os.path.join(self.config.resource.self_play_log_dir, f"worker{self.rank:03d}"))
            except Exception:  # tensorboard not installed: scalars are optional
                self.tensor_board = False
        if self.tensor_board:
            self.tensor_board.add_scalar("self/time", seconds_per_game, self.game_idx)
            self.tensor_board.add_scalar("self/turn", int(g.turn), self.game_idx)
            # len(mtcs_info.var_p): the reference stores every prior under the key and its colour-swapped mirror (player.py:323)
            self.tensor_board.add_scalar("self/mcts_buffer_size", 2 * int(g.table_nodes), self.game_idx)
            self.tensor_board.add_scalar("self/expansions", int(g.expansions), self.game_idx)

    def _harvest(self):
        n_total = 0
        pdc, pc = self.config.play_data, self.config.play
        now = time.time()
        elapsed, self._last_harvest_time = now - getattr(self, "_last_harvest_time", now), now
        while True:
            games, ng, plies, _ = self.engine.poll_raw()
            if ng == 0:
                break
            for i in range(ng):
                g = games[i]
                n_total += 1
                self.local_idx += 1
                self.game_idx += self.world_size
                gp = [plies[j] for j in range(g.first_ply, g.first_ply + g.n_plies)]
                self._finish_game(g)
                if getattr(self.config.b200 if hasattr(self.config, "b200") else None, "tensorboard", False):
                    self._log_scalars(g, len(gp), elapsed / max(1, ng))
                # drop draw games with probability drop_draw_game_rate (self_play.py:182)
                if g.black_z != 0 or pdc.drop_draw_game_rate <= np.random.random():
                    self.buffer_games.append((_copy(g), [_copy(p) for p in gp]))
                if pdc.enable_ggf_data:
                    self.ggf_lines.append(self._ggf_of(g, gp))
                    if self.local_idx % pdc.nb_game_in_ggf_file == 0 or self.local_idx <= 5:   # worker/self_play.py:169-172
                        self._flush_ggf()
                if self.local_idx % pdc.nb_game_in_file == 0:
                    self._flush_files(ggf=False)
            with open(self.config.resource.self_play_game_idx_file, "wt") as f:
                f.write(str(self.game_idx))
            new_sims = self.decide_simulation_num_per_move(self.game_idx)
            if new_sims and new_sims != pc.simulation_num_per_move:
                pc.simulation_num_per_move = new_sims
                self._engine_cmd("set_simulation_num", new_sims)
        return n_total

    def _finish_game(self, g):
        """worker/self_play.py:219-238 (resign false-positive statistics)"""
        if g.winner == 1:
            fp = bool(g.resigned_mask & 1)
        elif g.winner == 2:
            fp = bool(g.resigned_mask & 2)
        else:
            fp = bool(g.resigned_mask)
        if not g.resign_enabled:
            self.resign_test_game_count += 1
            if fp:
                self.false_positive_count_of_resign += 1
            self.check_and_update_resignation_threshold()

    def _ggf_of(self, g, gp):
        """MoveHistory, worker/self_play.py:275-299"""
        moves = []
        for p in gp:
            if p.action < 0:
                continue
            if (len(moves) % 2 == 0) == (p.player == 2):
                moves.append(convert_action_to_move(None))
            moves.append(f"{convert_action_to_move(int(p.action))}/{p.q * 10}/{p.n}")
        return make_ggf_string("RAZ", "RAZ", moves=moves)

    def _flush_ggf(self):
        """worker/self_play.py:196-207"""
        if not self.ggf_lines:
            return
        rc = self.config.resource
        game_id = datetime.now().strftime("%Y%m%d-%H%M%S.%f")
        if self.world_size > 1:   # ranks share the directory: same suffix rule as the play_data files
            game_id += f"_r{self.rank}"
        path = os.path.join(rc.self_play_ggf_data_dir, rc.ggf_filename_tmpl % game_id)
        with open(path, "wt") as f:
            for line in self.ggf_lines:
                f.write(line + "\n")
        self.ggf_lines = []

    def _flush_files(self, force=False, ggf=True):
        rc, pdc = self.config.resource, self.config.play_data
        if self.buffer_games:
            n_plies = sum(len(pl) for _, pl in self.buffer_games)
            G = (_cabi.Game * len(self.buffer_games))()
            P = (_cabi.Ply * max(1, n_plies))()
            at = 0
            for i, (g, pl) in enumerate(self.buffer_games):
                G[i] = g
                G[i].first_ply = at
                for p in pl:
                    P[at] = p
                    at += 1
            game_id = datetime.now().strftime("%Y%m%d-%H%M%S.%f")
            if self.world_size > 1:
                game_id += f"_r{self.rank}"
            path = os.path.join(rc.play_data_dir, rc.play_data_filename_tmpl % game_id)
            write_play_data(path, G, len(self.buffer_games), P, pdc.save_policy_of_tau_1, self.config.play.change_tau_turn)
            if getattr(getattr(self.config, "b200", None), "write_play_rows", False):  # compact twin for worker/ingest.py
                from .ingest import rows_path_of, write_play_rows
                write_play_rows(rows_path_of(path), G, len(self.buffer_games), P, pdc.save_policy_of_tau_1, self.config.play.change_tau_turn)
            logger.info(f"save play data to {path}")
            self.files_written.append(path)
            self.bytes_written += os.path.getsize(path)
            self.buffer_games = []
            self.remove_play_data()
        if ggf and force:
            self._flush_ggf()

    def remove_play_data(self):
        """worker/self_play.py:209-217"""
        rc = self.config.resource
        from glob import glob
        files = sorted(glob(os.path.join(rc.play_data_dir, rc.play_data_filename_tmpl % "*")))
        if len(files) < self.config.play_data.max_file_num:
            return
        for i in range(len(files) - self.config.play_data.max_file_num):
            for victim in (files[i], os.path.splitext(files[i])[0] + ".rzrows"):  # the JSON file and its compact twin, if any
                try:
                    os.remove(victim)
                except OSError:
                    pass


def _copy(struct):
    c = type(struct)()
    import ctypes
    ctypes.memmove(ctypes.byref(c), ctypes.byref(struct), ctypes.sizeof(struct))
    return c
