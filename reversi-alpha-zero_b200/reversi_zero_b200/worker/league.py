"""League: a round-robin between saved models on one GPU, rated with Elo.

Every pair of the 2 .. 16 models plays ``league.game_num_per_pair`` games, and all games of all pairs run concurrently in
one engine (``rz_engine_set_nets``): each search is evaluated by the mover's own network, so models of different widths
and depths can meet.  The games follow the rules of ``eval`` (``eval_play_config``), overlaid with ``league.play_config``.
The results are fitted by a Bradley-Terry model on the Elo scale, with one model (``league.anchor``, an index into the
model list) fixed at 0.

Settings (YAML ``league:`` section):

* ``models``: a list of blob paths or globs relative to the project directory, or mappings
  ``{path: ..., model: {cnn_filter_num: 128, ...}}`` whose ``model`` overrides ``config.model`` for that entry.  Default:
  ``<model_dir>/promoted/*.rzblob.npy`` sorted by name (``b200.keep_promoted_models`` fills that directory);
* ``game_num_per_pair`` (default 100), ``play_config`` (a mapping), ``anchor`` (default 0);
* ``openings``: a suite written by the ``openings`` command (path relative to the project directory).  Game k, in round
  r = k div P (P pairs), starts from opening (r div 2) mod n: each pair plays every opening once with each colour, and
  with an odd ``game_num_per_pair`` the last opening once.  Default: every game starts from the initial position.

The result goes to ``logs/league_<timestamp>.json`` and a rating table to the log.
"""
import copy
import glob
import hashlib
import json
import math
import os
from datetime import datetime
from logging import getLogger

import numpy as np

from ..engine import Engine, engine_cfg_from_play_config, EVAL_NET
from .evaluate import eval_play_config

logger = getLogger(__name__)

MAX_MODELS = 16  # RZ_MAX_NETS
_ELO = 400.0 / math.log(10.0)  # Elo points per natural-log unit of the odds


def start(config):
    return LeagueWorker(config).start()


def _field(config, name, default):
    lg = getattr(config, "league", None)
    if isinstance(lg, dict):
        return lg.get(name, default)
    return getattr(lg, name, default) if lg is not None else default


def league_play_config(config):
    """``eval_play_config(config)`` overlaid with the ``league.play_config`` mapping"""
    pc = eval_play_config(config)
    for k, v in (_field(config, "play_config", None) or {}).items():
        setattr(pc, k, v)
    return pc


def schedule(n_models, games_per_pair):
    """-> (black, white) uint8 arrays of P x games_per_pair model indices, P = the unordered pairs i < j in lexicographic
    order.  Game k belongs to pair k mod P; in round k div P the lower index plays black when the round is even, so the
    pairs progress evenly through the run and every pair's colours are balanced to within one game."""
    if not 2 <= n_models <= MAX_MODELS:
        raise ValueError(f"a league needs 2..{MAX_MODELS} models, got {n_models}")
    if games_per_pair < 1:
        raise ValueError(f"games per pair must be >= 1, got {games_per_pair}")
    pairs = np.array([(i, j) for i in range(n_models) for j in range(i + 1, n_models)], dtype=np.uint8)
    k = np.arange(len(pairs) * games_per_pair)
    pk, lower_black = pairs[k % len(pairs)], (k // len(pairs)) % 2 == 0
    black = np.where(lower_black, pk[:, 0], pk[:, 1]).astype(np.uint8)
    white = np.where(lower_black, pk[:, 1], pk[:, 0]).astype(np.uint8)
    return black, white


def league_openings(n_models, games_per_pair, suite):
    """the opening of each game of ``schedule(n_models, games_per_pair)``: game k, in round r = k div P, plays
    suite[(r div 2) mod n]; colours swap between rounds 2q and 2q + 1"""
    n_pairs = n_models * (n_models - 1) // 2
    return [suite[(k // n_pairs // 2) % len(suite)] for k in range(n_pairs * games_per_pair)]


def play_league(config, nets, games_per_pair, device=0, seed=0, first_game_id=0, suite=None):
    """Plays the whole round-robin in one engine, from the openings of ``suite`` (``league_openings``) when given.  -> one record per game, in game-id order: game_id, black and white
    (model indices), winner (1 black, 2 white, 3 draw) and disc_diff (black's discs minus white's at the end)."""
    pc = league_play_config(config)
    black, white = schedule(len(nets), games_per_pair)
    total = int(black.size)
    slots = min(total, getattr(getattr(config, "b200", None), "games_per_gpu", 4096))
    # the evaluation cache stays off while several networks are set: none is allocated
    cfg = engine_cfg_from_play_config(pc, games=slots, seed=seed, eval_mode=EVAL_NET, max_games=total, first_game_id=first_game_id,
                                      eval_cache_mb=-1)
    eng = Engine(cfg, nets[0], device)
    try:
        eng.set_nets(nets, black, white)
        if suite:
            eng.set_openings(league_openings(len(nets), games_per_pair, suite))
        eng.run(finished_target=total)
        games = sorted(eng.poll(), key=lambda g: g["game_id"])
    finally:
        eng.close()
    if len(games) != total:
        raise RuntimeError(f"league: {len(games)} of {total} games finished")
    records = []
    for g in games:
        local = g["game_id"] - first_game_id
        assert (g["black_net"], g["white_net"]) == (black[local], white[local]), g["game_id"]
        records.append(dict(game_id=g["game_id"], black=g["black_net"], white=g["white_net"], winner=g["winner"],
                            disc_diff=bin(g["black"]).count("1") - bin(g["white"]).count("1")))
    return records


def _scores(records, n_models):
    """-> (s, n): s[i, j] = points of i against j (a win 1, a draw 1/2), n[i, j] = games between i and j"""
    s, n = np.zeros((n_models, n_models)), np.zeros((n_models, n_models))
    for r in records:
        b, w = int(r["black"]), int(r["white"])
        n[b, w] += 1
        n[w, b] += 1
        pb = 1.0 if r["winner"] == 1 else (0.0 if r["winner"] == 2 else 0.5)
        s[b, w] += pb
        s[w, b] += 1.0 - pb
    return s, n


def fit_elo(records, n_models, anchor=0, prior_draws=1):
    """Bradley-Terry maximum-likelihood ratings on the Elo scale: P(i beats j) = 1 / (1 + 10^((r_j - r_i) / 400)).
    A draw counts as half a win for each side, and ``prior_draws`` virtual draws are added to every pair that played, so
    that a clean sweep still has a finite maximum.  Newton's method to 1e-9 Elo, with model ``anchor`` fixed at 0.
    -> (ratings, ci95): numpy arrays, ci95 = 1.96 standard errors from the inverse observed information with the anchor
    removed (0 for the anchor)."""
    if not 0 <= anchor < n_models:
        raise ValueError(f"anchor {anchor} is not a model index (0..{n_models - 1})")
    s, n = _scores(records, n_models)
    played = n > 0
    s = s + 0.5 * prior_draws * played
    n = n + prior_draws * played
    free = np.array([i for i in range(n_models) if i != anchor])
    theta = np.zeros(n_models)

    def loglik(t):
        d = t[:, None] - t[None, :]
        return float(np.sum(s * -np.logaddexp(0.0, -d)))

    def info(t):
        p = 1.0 / (1.0 + np.exp(-(t[:, None] - t[None, :])))
        grad = np.sum(s - n * p, axis=1)
        w = n * p * (1.0 - p)
        h = np.diag(w.sum(axis=1)) - w  # observed information (negative Hessian of the log-likelihood)
        return grad[free], h[np.ix_(free, free)]

    for _ in range(200):
        g, h = info(theta)
        try:
            step = np.linalg.solve(h, g)
        except np.linalg.LinAlgError:
            raise ValueError("fit_elo: the results do not connect every model") from None
        ll, t = loglik(theta), 1.0
        while True:  # Newton's step, halved while it would lower the likelihood (the log-likelihood is concave)
            cand = theta.copy()
            cand[free] += t * step
            if loglik(cand) >= ll - 1e-12 * abs(ll) or t < 1e-6:
                break
            t *= 0.5
        theta = cand
        if np.max(np.abs(t * step)) * _ELO < 1e-9:
            break
    else:
        raise ValueError("fit_elo: no finite maximum (a clean sweep without prior draws?)")
    _, h = info(theta)
    ci = np.zeros(n_models)
    ci[free] = 1.96 * np.sqrt(np.diag(np.linalg.inv(h))) * _ELO
    return theta * _ELO, ci


def pair_table(records):
    """-> {(i, j): {"W", "D", "L", "as_black": [W, D, L], "as_white": [W, D, L]}} from model i's side, for every ordered
    pair that played"""
    out = {}
    for r in records:
        b, w, win = int(r["black"]), int(r["white"]), int(r["winner"])
        for me, opp, colour, res in ((b, w, "as_black", {1: 0, 3: 1, 2: 2}[win]), (w, b, "as_white", {2: 0, 3: 1, 1: 2}[win])):
            e = out.setdefault((me, opp), {"W": 0, "D": 0, "L": 0, "as_black": [0, 0, 0], "as_white": [0, 0, 0]})
            e["WDL"[res]] += 1
            e[colour][res] += 1
    return out


class LeagueWorker:
    def __init__(self, config, device=0):
        self.config = config
        self.device = device

    def model_entries(self):
        """-> [(absolute blob path, model config)] from ``league.models`` (default: the promoted blobs); refuses fewer than 2
        models, more than 16, a missing file and a blob whose size does not match its model configuration"""
        from ..agent import model as M
        rc = self.config.resource
        listed = _field(self.config, "models", None)
        entries = []
        if listed is None:
            for p in sorted(glob.glob(os.path.join(rc.model_dir, "promoted", "*.rzblob.npy"))):
                entries.append((p, self.config.model))
        else:
            if isinstance(listed, (str, dict)):
                listed = [listed]
            for item in listed:
                path, over = (item.get("path"), item.get("model")) if isinstance(item, dict) else (item, None)
                if not isinstance(path, str):
                    raise ValueError(f"league.models: entry {item!r} has no path")
                mc = self.config.model
                if over:
                    mc = copy.copy(mc)
                    for k, v in over.items():
                        setattr(mc, k, v)
                full = os.path.join(rc.project_dir, path)
                if glob.has_magic(path):
                    found = sorted(glob.glob(full))
                    if not found:
                        raise ValueError(f"league.models: {path} matches no file")
                    entries += [(p, mc) for p in found]
                else:
                    entries.append((full, mc))
        names = ", ".join(p for p, _ in entries) or "none"
        if len(entries) < 2:
            raise ValueError(f"a league needs at least 2 models, found {len(entries)}: {names}")
        if len(entries) > MAX_MODELS:
            raise ValueError(f"a league takes at most {MAX_MODELS} models, found {len(entries)}: {names}")
        missing = [p for p, _ in entries if not os.path.isfile(p)]
        if missing:
            raise ValueError(f"league.models: missing file(s): {', '.join(missing)}")
        for p, mc in entries:
            size, want = np.load(p, mmap_mode="r").size, M.blob_size(mc)
            if size != want:
                raise ValueError(f"league.models: {p} holds {size} floats, but its model configuration "
                                 f"({mc.cnn_filter_num} filters, {mc.res_layer_num} blocks, value_fc {mc.value_fc_size}) needs {want}")
        return entries

    def start(self):
        from ..net import Net
        rc = self.config.resource
        entries = self.model_entries()
        games_per_pair = int(_field(self.config, "game_num_per_pair", 100))
        anchor = int(_field(self.config, "anchor", 0))
        if not 0 <= anchor < len(entries):
            raise ValueError(f"league.anchor = {anchor} is not an index into the {len(entries)} models")
        seed = int(getattr(getattr(self.config, "b200", None), "seed", 0))
        suite, openings = None, None
        suite_path = _field(self.config, "openings", None)
        if suite_path:
            from ..lib.openings import load_suite, suite_digest
            full = os.path.join(rc.project_dir, suite_path)
            suite = load_suite(full)
            openings = dict(path=os.path.relpath(full, rc.project_dir), sha256=suite_digest(full), count=len(suite))
            logger.info(f"league: {len(suite)} openings from {openings['path']} (sha256 {openings['sha256'][:16]})")
        nets = []
        try:
            for p, mc in entries:
                net = Net(mc, self.device)
                net.load_blob(np.load(p))
                nets.append(net)
            records = play_league(self.config, nets, games_per_pair, self.device, seed=seed, suite=suite)
        finally:
            for net in nets:
                net.close()
        n = len(entries)
        ratings, ci = fit_elo(records, n, anchor=anchor)
        s, played = _scores(records, n)
        pairs = pair_table(records)
        models = []
        for i, (p, mc) in enumerate(entries):
            with open(p, "rb") as f:
                digest = hashlib.sha256(f.read()).hexdigest()
            models.append(dict(index=i, path=os.path.relpath(p, rc.project_dir), sha256=digest,
                               model={k: getattr(mc, k) for k in ("cnn_filter_num", "cnn_filter_size", "res_layer_num", "value_fc_size")},
                               games=int(played[i].sum()), score=float(s[i].sum()), elo=float(ratings[i]), ci95=float(ci[i])))
        pc = league_play_config(self.config)
        out = dict(timestamp=datetime.now().strftime("%Y%m%d-%H%M%S.%f"), seed=seed, games_per_pair=games_per_pair,
                   games=len(records), anchor=anchor, openings=openings, play_config={k: v for k, v in sorted(vars(pc).items())}, models=models,
                   pairs=[dict(model=i, opponent=j, **pairs[(i, j)]) for (i, j) in sorted(pairs)])
        os.makedirs(rc.log_dir, exist_ok=True)
        path = os.path.join(rc.log_dir, f"league_{out['timestamp']}.json")
        with open(path + ".tmp", "wt") as f:
            json.dump(out, f, indent=1, default=list)
        os.replace(path + ".tmp", path)
        lines = [f"league: {n} models, {games_per_pair} games per pair, {len(records)} games, anchor {anchor}",
                 f"{'#':>3} {'elo':>8} {'+-95%':>7} {'score':>8} {'games':>6}  model"]
        for m in sorted(models, key=lambda m: -m["elo"]):
            lines.append(f"{m['index']:>3} {m['elo']:8.1f} {m['ci95']:7.1f} {m['score']:8.1f} {m['games']:>6}  {m['path']}")
        logger.info("\n".join(lines))
        logger.info(f"league result: {path}")
        return path
