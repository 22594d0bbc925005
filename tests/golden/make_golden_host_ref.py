"""Writes what the UNMODIFIED reference (imported through oracle/ref_shims) produces for the host-logic comparisons of
tests/test_host_logic.py and tests/test_playdata_writer.py, so that those tests run without its checkout:

  * host_ref.json    GGF move names and record strings (lib/ggf.py, worker/self_play.py MoveHistory), the resignation tuner's
                     trajectory and the simulation schedule of worker/self_play.py over the tests' seeded sequences, the
                     effective model / play / play_data / eval.play_config values of the reference's Config for its
                     defaults and each config/*.yml
  * ref_config/*.yml the reference's own config files (inputs of the mirror's YAML loader in the tests)
  * trainer_ref.npz  OptimizeWorker.convert_to_training_data(read_game_data_from_file(f)) for the tests' fixed two-game file

Run once where the reference checkout exists:

    python tests/golden/make_golden_host_ref.py
"""
import json
import os
import shutil
import sys
import tempfile
import types
from datetime import datetime

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "reversi-alpha-zero_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

import oracle.ref_shims.install as shims  # noqa: E402

REF_CONFIG_DIR = "/root/reference/config"
GGF_DT = datetime(2026, 9, 22, 13, 5, 9)
GGF_MOVES = ["C4/2.5/10.0", "C3/-5.0/7.0", "PA", "C2/0.0/3.0"]
GGF_KW = (dict(), dict(result="+12.0", think_time_sec=125))
GGF_PLIES = ((19, 1, 0.25, 10.0), (18, 2, -0.5, 7.0), (17, 2, 0.0, 3.0), (-1, 1, 0.0, 0.0))
SCHEDULE = [(0, 8), (300, 50), (2000, 200)]
SCHEDULE_IDX = (0, 1, 299, 300, 301, 1999, 2000, 123456)
FORCE_TEXTS = ("77\n", "0", "abc", "")


def plain(v):
    return [plain(x) for x in v] if isinstance(v, (list, tuple)) else v


def resign_sequence():
    """the seeded (winner, resigned mask, resign enabled) sequence of test_resign_tuner_and_schedule_match_reference_worker"""
    rng = np.random.default_rng(9)
    out = []
    for _ in range(1500):
        winner = int(rng.integers(1, 4))
        mask = int(rng.integers(0, 4)) if rng.random() < 0.2 else 0
        enabled = bool(rng.random() < 0.4)
        out.append((winner, mask, enabled))
    return out


def ggf_golden():
    from reversi_zero.lib import ggf as ref
    from reversi_zero.worker.self_play import MoveHistory
    from reversi_zero.agent.player import ActionWithEvaluation
    from reversi_zero.env.reversi_env import Player
    moves = {str(a): ref.convert_action_to_move(a) for a in list(range(64)) + [None]}
    actions = {mv: ref.convert_move_to_action(mv) for mv in moves.values()}
    records = [ref.make_ggf_string("RAZ", "RAZ", dt=GGF_DT, moves=GGF_MOVES, **kw) for kw in GGF_KW]
    mh = MoveHistory()
    for action, player, q, n in GGF_PLIES:
        env = types.SimpleNamespace(next_player=Player.black if player == 1 else Player.white)
        mh.move(env, ActionWithEvaluation(None if action < 0 else action, n, q))
    return dict(moves=moves, actions=actions, f5=ref.convert_move_to_action("f5"), records=records,
                record_dt_only=ref.make_ggf_string(dt=GGF_DT), record_now_prefix=ref.make_ggf_string()[: len("(;GM[Othello]PC[RAZSelf]DT[")],
                move_history_after_bo=mh.make_ggf_string("RAZ", "RAZ").split("BO[")[1])


def resign_golden(tmp):
    from reversi_zero.worker.self_play import SelfPlayWorker as Ref
    from reversi_zero.env.reversi_env import Winner

    class RefSelf:
        pass
    r = RefSelf()
    r.config = types.SimpleNamespace(play=types.SimpleNamespace(resign_threshold=-0.8, false_positive_threshold=0.05, resign_threshold_delta=0.01,
                                                                 schedule_of_simulation_num_per_move=SCHEDULE),
                                     resource=types.SimpleNamespace(force_simulation_num_file=os.path.join(tmp, "force_sim")))
    r.resign_test_game_count = r.false_positive_count_of_resign = 0
    r.check_and_update_resignation_threshold = lambda: Ref.check_and_update_resignation_threshold(r)
    r.reset_false_positive_count = lambda: Ref.reset_false_positive_count(r)
    type(r).false_positive_rate = Ref.false_positive_rate
    winners = {1: Winner.black, 2: Winner.white, 3: Winner.draw}
    trajectory = []
    for winner, mask, enabled in resign_sequence():
        player = lambda bit: types.SimpleNamespace(resigned=bool(mask & bit), finish_game=lambda z: None)   # noqa: E731
        r.env = types.SimpleNamespace(winner=winners[winner])
        r.black, r.white = player(1), player(2)
        Ref.finish_game(r, resign_enabled=enabled)
        trajectory.append([r.config.play.resign_threshold, r.resign_test_game_count, r.false_positive_count_of_resign])
    schedule = {str(i): Ref.decide_simulation_num_per_move(r, i) for i in SCHEDULE_IDX}
    force = {}
    for text in FORCE_TEXTS:
        with open(r.config.resource.force_simulation_num_file, "wt") as f:
            f.write(text)
        force[text] = {str(i): Ref.decide_simulation_num_per_move(r, i) for i in (0, 5000)}
    return dict(trajectory=trajectory, schedule=schedule, force=force)


def config_golden():
    import yaml
    from moke_config import create_config as ref_create
    from reversi_zero.config import Config as RefConfig

    def sections(cfg, names):
        out = {}
        for sec in names:
            d = {}
            for k, v in vars(getattr(cfg, sec)).items():
                if sec == "resource":
                    if not isinstance(v, str):
                        continue
                    d[k] = dict(relpath=os.path.relpath(v, cfg.resource.project_dir)) if os.sep in v else v
                else:
                    d[k] = plain(v)
            out[sec] = d
        return out

    cases = {"defaults": RefConfig()}
    names = sorted(n for n in os.listdir(REF_CONFIG_DIR) if n.endswith(".yml"))
    for name in names:
        with open(os.path.join(REF_CONFIG_DIR, name), "rt") as f:
            cases[name] = ref_create(RefConfig, yaml.safe_load(f))
    out = {}
    for name, cfg in cases.items():
        d = sections(cfg, ("resource", "model", "play", "play_data") if name == "defaults" else ("model", "play", "play_data"))
        d["eval_play_config"] = {k: plain(v) for k, v in vars(cfg.eval.play_config).items()}
        d["play_all"] = {k: plain(v) for k, v in vars(cfg.play).items()}
        out[name] = d
    os.makedirs(os.path.join(HERE, "ref_config"), exist_ok=True)
    for name in names:
        shutil.copy(os.path.join(REF_CONFIG_DIR, name), os.path.join(HERE, "ref_config", name))
    return out


def trainer_golden(tmp):
    from reversi_zero.lib.data_helper import read_game_data_from_file
    from reversi_zero.worker.optimize import OptimizeWorker
    import test_playdata_writer as T
    from reversi_zero_b200 import engine as E
    games = T.fixed_games()
    G, P = T.to_ctypes(games)
    path = os.path.join(tmp, "play_20260922-000000.000000.json")
    E.write_play_data(path, G, len(games), P, True, 4)
    states, policies, zs = OptimizeWorker.convert_to_training_data(read_game_data_from_file(path))
    np.savez_compressed(os.path.join(HERE, "trainer_ref.npz"), states=states, policies=policies, zs=zs)


def main():
    assert shims.available(), "reference sources not present"
    shims.install()
    with tempfile.TemporaryDirectory() as tmp:
        golden = dict(ggf=ggf_golden(), resign=resign_golden(tmp), config=config_golden())
        trainer_golden(tmp)
    with open(os.path.join(HERE, "host_ref.json"), "w") as f:
        json.dump(golden, f, separators=(",", ":"))


if __name__ == "__main__":
    main()
