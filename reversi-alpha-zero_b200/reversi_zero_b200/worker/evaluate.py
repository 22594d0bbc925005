"""Mirror of the reference's evaluator (worker/evaluate.py:17-124) on the H100 engine: the challenger
("next generation") network plays ``eval.game_num`` games against the best network and replaces it when its
winning rate over the decided games reaches ``eval.replace_rate``.

The reference plays the games one after the other with two in-process ``ReversiPlayer`` objects; here ALL games of
a match run concurrently on the device (``rz_engine_set_second_net``): each search is evaluated by the mover's own
network, colours alternate by game index (the reference draws them at random, :70), each player keeps its own
statistics (``share_mtcs_info = 0``, as ``ReversiPlayer(config, model, play_config=...)`` does in :69-70).  The
verdict follows the reference's sequential bookkeeping (:44-64) over the games in game-index order, including its
early-stop rules -- games after the point where the reference would have stopped do not count.  Weights are exchanged as float32 blobs (``*.rzblob.npy``, DESIGN.md section 9).

With ``eval.openings: <path>`` (a suite written by the ``openings`` command, relative to the project directory) game i
starts from opening (i div 2) mod n of the suite, so every opening is played once with each colour."""
import hashlib
import os
import shutil
from datetime import datetime
from glob import glob
from logging import getLogger
from time import sleep
from types import SimpleNamespace

import numpy as np

from ..engine import Engine, engine_cfg_from_play_config, EVAL_NET
from ..net import Net
from .self_play import blob_path_of

logger = getLogger(__name__)

NEXT_GENERATION_BLOB = "model_weight.rzblob.npy"
PROMOTED_DIR = "promoted"  # under the model directory: every promoted blob, when b200.keep_promoted_models is on


def start(config):
    return EvaluateWorker(config).start()


def eval_play_config(config):
    """The play configuration an evaluation game really runs with in the reference:

    * ``EvaluateConfig.play_config`` is a FRESH ``PlayConfig()`` -- the defaults, not a copy of the self-play section --
      with five overrides (config.py:103-113), overlaid with the ``eval.play_config`` mapping of a YAML file (mini.yml and
      alpha_go_zero.yml merge their ``play`` section into it with a YAML anchor; ch5.yml has no eval section, so e.g.
      ``c_puct`` is the default 1 there and the exact root solver is on from turn 50);
    * three fields are read from the SELF-PLAY section even in evaluation games, because ``ReversiPlayer`` uses
      ``self.config.play`` for them: ``allowed_resign_turn`` (agent/player.py:127), ``use_solver_turn_in_simulation``
      (:237-238) and ``virtual_loss`` (:264);
    * the two players never share statistics (``ReversiPlayer(config, model, play_config=...)``, worker/evaluate.py:69-70).
    """
    from ..config import PlayConfig
    ev = getattr(config, "eval", None)
    user = (ev.get("play_config") if isinstance(ev, dict) else getattr(ev, "play_config", None)) or {}
    if not isinstance(user, dict) and all(hasattr(user, k) for k in ("simulation_num_per_move", "c_puct", "thinking_loop")):
        pc = SimpleNamespace(**vars(user))       # a complete PlayConfig object (the reference's own Config): use it as it is
    else:
        pc = SimpleNamespace(**vars(PlayConfig()))
        over = dict(simulation_num_per_move=400, thinking_loop=1, change_tau_turn=0, noise_eps=0, disable_resignation_rate=0)
        over.update(user if isinstance(user, dict) else vars(user))
        for k, v in over.items():
            setattr(pc, k, v)
    for k in ("allowed_resign_turn", "use_solver_turn_in_simulation", "virtual_loss"):
        setattr(pc, k, getattr(config.play, k))
    pc.share_mtcs_info_in_self_play = False
    return pc


def _eval_field(config, name, default):
    ev = getattr(config, "eval", None)
    if isinstance(ev, dict):
        return ev.get(name, default)
    return getattr(ev, name, default) if ev is not None else default


def match_openings(game_num, suite):
    """the opening of each game of a match: game i plays suite[(i div 2) mod n], and colours alternate with i"""
    return [suite[(i // 2) % len(suite)] for i in range(game_num)]


def play_match(config, best_net, ng_net, game_num, device=0, seed=0, first_game_id=0, suite=None):
    """-> (results, games): results[i] = 1 challenger won, 0 lost, None draw (worker/evaluate.py:84-96).
    ``seed`` / ``first_game_id`` select the Philox streams (dihedral choices, move sampling) of the match: callers give
    every match its own, so that the randomness of consecutive matches is independent like the reference's.
    ``suite``: openings (lists of squares) the games start from, as ``match_openings`` assigns them; None: none."""
    pc = eval_play_config(config)
    slots = min(game_num, getattr(getattr(config, "b200", None), "games_per_gpu", 4096))
    cfg = engine_cfg_from_play_config(pc, games=slots, seed=seed, eval_mode=EVAL_NET, max_games=game_num, first_game_id=first_game_id)
    eng = Engine(cfg, best_net, device)
    eng.set_second_net(ng_net)
    if suite:
        eng.set_openings(match_openings(game_num, suite))
    eng.run(finished_target=game_num)
    games = sorted(eng.poll(), key=lambda g: g["game_id"])   # game-id order == local game index order (colours alternate with it)
    eng.close()
    results = []
    for g in games:
        best_is_black = g["black_net"] == 0
        if g["winner"] == 1:
            results.append(0 if best_is_black else 1)
        elif g["winner"] == 2:
            results.append(1 if best_is_black else 0)
        else:
            results.append(None)
    return results, games


def match_verdict(results, game_num, replace_rate):
    """worker/evaluate.py:44-64 replayed over ``results`` (game-index order; 1 challenger won, 0 lost, None draw):
    returns (replace: bool, winning_rate, games_counted).  The reference stops as soon as the losses reach
    game_num * (1 - replace_rate) or the wins reach game_num * replace_rate, and then decides on the winning rate so far."""
    decided = []
    counted = 0
    for r in results[:game_num]:
        counted += 1
        if r is not None:
            decided.append(r)
        if decided.count(0) >= game_num * (1 - replace_rate):
            break
        if decided.count(1) >= game_num * replace_rate:
            break
    winning_rate = sum(decided) / len(decided) if decided else 0.0   # the reference divides by zero when every game is a draw
    return winning_rate >= replace_rate, winning_rate, counted


class EvaluateWorker:
    def __init__(self, config, device=0):
        self.config = config
        self.device = device
        self.best_net = None
        self.match_count = 0   # matches played by this worker: every match gets its own game-id range (= its own random streams)

    def start(self, max_models=None):
        self.best_net = self._load(blob_path_of(self.config))
        if self._keep_promoted():
            self.archive_best_model()
        done = 0
        while max_models is None or done < max_models:
            model_dir = self.next_generation_dir()
            ng_net = self._load(os.path.join(model_dir, NEXT_GENERATION_BLOB))
            logger.debug(f"start evaluate model {model_dir}")
            if self.evaluate_model(ng_net, model_dir):
                logger.debug(f"New Model become best model: {model_dir}")
                self.save_as_best_model(model_dir)
                self.best_net = ng_net
            self.remove_model(model_dir)
            done += 1
        return done

    def save_as_best_model(self, model_dir):
        """lib/model_helpler.py:22-28 save_as_best_model: the challenger becomes the best model for EVERY consumer -- the
        engine-side blob, and the Keras-side model_best_config.json / model_best_weight.h5 the reference trainer
        (worker/optimize.py load_model) and load_best_model_weight read -- when the trainer put them into the directory."""
        rc = self.config.resource
        shutil.copyfile(os.path.join(model_dir, NEXT_GENERATION_BLOB), blob_path_of(self.config))
        if self._keep_promoted():
            self._archive(os.path.join(model_dir, NEXT_GENERATION_BLOB), os.path.basename(os.path.normpath(model_dir)))
        for name, dst in ((rc.next_generation_model_config_filename, rc.model_best_config_path),
                          (rc.next_generation_model_weight_filename, rc.model_best_weight_path)):
            src = os.path.join(model_dir, name)
            if os.path.exists(src):
                shutil.copyfile(src, dst + ".tmp")
                os.replace(dst + ".tmp", dst)

    def _keep_promoted(self):
        return bool(getattr(getattr(self.config, "b200", None), "keep_promoted_models", False))

    def _archive(self, src, name):
        """copies the blob `src` to <model_dir>/promoted/<name>.rzblob.npy (a temporary file, then an atomic rename), so
        that a league (worker/league.py) can rate every generation"""
        d = os.path.join(self.config.resource.model_dir, PROMOTED_DIR)
        os.makedirs(d, exist_ok=True)
        dst = os.path.join(d, name + ".rzblob.npy")
        shutil.copyfile(src, dst + ".tmp")
        os.replace(dst + ".tmp", dst)
        return dst

    def archive_best_model(self):
        """archives the current best blob as promoted/model_<its mtime>.rzblob.npy, unless a promoted blob with the same
        content is there already: the first generation is then rated too"""
        src = blob_path_of(self.config)

        def digest(path):
            with open(path, "rb") as f:
                return hashlib.sha256(f.read()).hexdigest()
        mine = digest(src)
        for p in sorted(glob(os.path.join(self.config.resource.model_dir, PROMOTED_DIR, "*.rzblob.npy"))):
            if digest(p) == mine:
                return None
        stamp = datetime.fromtimestamp(os.path.getmtime(src)).strftime("%Y%m%d-%H%M%S.%f")
        return self._archive(src, self.config.resource.next_generation_model_dirname_tmpl % stamp)

    def remove_model(self, model_dir):
        """worker/evaluate.py:115-121: the reference removes its two files and then the directory (os.rmdir fails, loudly,
        on anything else in there); the mirror removes those two and the blob it added, nothing more."""
        rc = self.config.resource
        for name in (rc.next_generation_model_config_filename, rc.next_generation_model_weight_filename, NEXT_GENERATION_BLOB):
            try:
                os.remove(os.path.join(model_dir, name))
            except FileNotFoundError:
                pass
        os.rmdir(model_dir)

    def evaluate_model(self, ng_net, model_dir=""):
        """worker/evaluate.py:44-64"""
        game_num = int(_eval_field(self.config, "game_num", 200))
        replace_rate = float(_eval_field(self.config, "replace_rate", 0.55))
        # a fresh game-id range per match and a seed tied to the challenger's directory: consecutive matches (and
        # restarts of the worker) do not replay the same dihedral / move-sampling streams
        import zlib
        seed = int(getattr(getattr(self.config, "b200", None), "seed", 0)) ^ zlib.crc32(os.path.basename(model_dir).encode())
        suite = self.load_openings()
        results, _ = play_match(self.config, self.best_net, ng_net, game_num, self.device, seed=seed,
                                first_game_id=self.match_count * 2 * game_num, suite=suite)
        self.match_count += 1
        replace, winning_rate, counted = match_verdict(results, game_num, replace_rate)
        logger.debug(f"winning rate {winning_rate * 100:.1f}% after {counted} games")
        return replace

    def load_openings(self):
        """the suite of ``eval.openings`` (None without one)"""
        path = _eval_field(self.config, "openings", None)
        if not path:
            return None
        from ..lib.openings import load_suite, suite_digest
        full = os.path.join(self.config.resource.project_dir, path)
        suite = load_suite(full)
        logger.info(f"eval: {len(suite)} openings from {path} (sha256 {suite_digest(full)[:16]})")
        return suite

    def next_generation_dir(self):
        rc = self.config.resource
        while True:
            dirs = sorted(glob(os.path.join(rc.next_generation_model_dir, rc.next_generation_model_dirname_tmpl % "*")))
            dirs = [d for d in dirs if os.path.exists(os.path.join(d, NEXT_GENERATION_BLOB))]
            if dirs:
                return dirs[-1] if _eval_field(self.config, "evaluate_latest_first", True) else dirs[0]
            logger.info("There is no next generation model to evaluate")
            sleep(60)

    def _load(self, path):
        net = Net(self.config.model, self.device)
        net.load_blob(np.load(path))
        return net
