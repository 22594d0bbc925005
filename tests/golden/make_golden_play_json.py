"""Writes tests/golden/play_json_ref.npz for tests/test_ingest_json*.py: play_*.json text written by the UNMODIFIED
reference (lib/data_helper.py:23-25 write_game_data_to_file, imported through oracle/ref_shims) from whole reference
self-play games, and what its trainer builds from that file (read_game_data_from_file + OptimizeWorker.
convert_to_training_data, worker/optimize.py:215-231).  Run once where the reference checkout exists:

    python tests/golden/make_golden_play_json.py

Per case <name>: <name>_text (uint8, the file's bytes), <name>_states_packed (the [N,2,8,8] states, packbits little),
<name>_policy (float64 [N,64]) and <name>_z (int64 [N]).  The cases cover tau-1 policies, the tau rule and one-hot
(tau-0) policies from the first move, with records of both z signs.
"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import make_golden as G  # noqa: E402  (installs the reference shims)

CASES = (("tau1", True, 4, 20), ("tau_rule", False, 6, 16), ("one_hot", False, 0, 10))


def gen():
    from reversi_zero.lib.data_helper import write_game_data_to_file, read_game_data_from_file
    from reversi_zero.worker.optimize import OptimizeWorker
    out = {}
    for name, tau1, ctt, sims in CASES:
        cfg = G.ref_config(sims=sims, k=1, noise_eps=0, change_tau_turn=ctt)
        cfg.play_data.save_policy_of_tau_1 = tau1
        _, recs, z = G.ref_selfplay_game(cfg, G.FakeNet())
        assert z != 0, "a drawn game has no records of both z signs"
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "play_x.json")
            write_game_data_to_file(path, recs)
            with open(path, "rb") as f:
                text = f.read()
            states, policies, zs = OptimizeWorker.convert_to_training_data(read_game_data_from_file(path))
        out[name + "_text"] = np.frombuffer(text, np.uint8)
        out[name + "_states_packed"] = np.packbits(states.reshape(len(states), -1), axis=1, bitorder="little")
        out[name + "_policy"] = np.asarray(policies, np.float64)
        out[name + "_z"] = np.asarray(zs, np.int64)
    return out


if __name__ == "__main__":
    np.savez_compressed(os.path.join(HERE, "play_json_ref.npz"), **gen())
    print("play JSON golden vectors written")
