"""GPU suite for the NBoard engine: the reference's recorded protocol sessions (tests/golden/nboard_ref.json) replayed
through the engine with the deterministic evaluator, and the engine as NBoard runs it -- a subprocess speaking the
protocol over stdin / stdout with a ch5 network."""
import io
import json
import os
import queue
import re
import subprocess
import sys
import threading
import time

import numpy as np
import pytest

from reversi_zero_b200.agent import model as M
from reversi_zero_b200.config import create_config, load_yaml
from reversi_zero_b200.lib.bitboard import find_correct_moves
from reversi_zero_b200.lib.ggf import convert_move_to_action, convert_to_bitboard_and_actions, parse_ggf
from reversi_zero_b200.play_game import nboard as NB

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def golden(golden_dir):
    with open(os.path.join(golden_dir, "nboard_ref.json")) as f:
        return json.load(f)


def _same_reply(mine, ref):
    """equal token by token, except the evaluations (the engine accumulates W in fp32) and the time"""
    a, b = mine.split(" "), ref.split(" ")
    assert len(a) == len(b), (mine, ref)
    if a[0] == "===":
        (ma, ea, ta), (mb, eb, _) = a[1].split("/"), b[1].split("/")
        assert ma == mb, (mine, ref)
        assert abs(float(ea) - float(eb)) <= 1e-5 * 10, (mine, ref)
        assert float(ta) >= 0.0
    elif a[0] == "search":
        assert a[1] == b[1] and a[3:] == b[3:], (mine, ref)
        assert abs(float(a[2]) - float(b[2])) <= 1e-5, (mine, ref)
    else:
        assert mine == ref


@pytest.mark.parametrize("name", ["opening", "midgame", "endgame_solver", "endgame_search", "pass"])
def test_sessions_match_reference(golden, name, monkeypatch):
    s = golden["sessions"][name]
    cfg = create_config(golden["config"])
    cfg.play.use_solver_turn = cfg.play.use_solver_turn_in_simulation = 50 if s["solver"] else 0
    cfg.play_with_human.update_play_config(cfg.play)
    monkeypatch.setattr(NB, "load_model", lambda config: None)   # None: the deterministic evaluator (RZ_EVAL_FAKE)
    out = io.StringIO()
    eng = NB.NBoardEngine(cfg, stdin=io.StringIO(), stdout=out)
    try:
        for step in s["transcript"]:
            line = step["line"]
            if line.startswith("ping"):
                eng.push_callback(line)
            n0 = len(out.getvalue().splitlines())
            eng.handler.handle_message(line.strip())
            replies = out.getvalue().splitlines()[n0:]
            assert len(replies) == len(step["replies"]), (line, replies, step["replies"])
            for mine, ref in zip(replies, step["replies"]):
                _same_reply(mine, ref)
    finally:
        eng.player.engine.close()


PROTOCOL = re.compile(r"^(set myname \S+|status .*|=== \S+|search \S+ \S+ 0 \d+|pong \d+|learned)$")


class Session:
    """the engine as NBoard starts it; every stdout line is collected by a thread, so reads can time out"""

    def __init__(self, args, cwd, env):
        self.p = subprocess.Popen(args, cwd=cwd, env=env, stdin=subprocess.PIPE, stdout=subprocess.PIPE,
                                  stderr=subprocess.PIPE, text=True, bufsize=1)
        self.lines = queue.Queue()
        self.all = []
        self.err = []
        threading.Thread(target=self._pump, daemon=True).start()
        threading.Thread(target=lambda: self.err.extend(self.p.stderr), daemon=True).start()

    def _pump(self):
        for line in self.p.stdout:
            self.lines.put(line.rstrip("\n"))

    def send(self, line):
        self.p.stdin.write(line + "\n")
        self.p.stdin.flush()

    def until(self, pred, timeout=120.0):
        got = []
        end = time.time() + timeout
        while True:
            left = end - time.time()
            if left <= 0:
                raise AssertionError(f"no matching line within {timeout} s: {got}; exit code {self.p.poll()}, "
                                     f"stderr: {''.join(self.err)[-3000:]}")
            try:
                line = self.lines.get(timeout=left)
            except queue.Empty:
                continue
            got.append(line)
            self.all.append(line)
            if pred(line):
                return got


def _ggf(moves):
    body = "".join(f"{'B' if i % 2 == 0 else 'W'}[{m}]" for i, m in enumerate(moves))
    return f"(;GM[Othello]PC[NBoard]BO[8 ---------------------------O*------*O--------------------------- *]{body};)"


def _legal(ggf_text, move):
    b, w, actions = convert_to_bitboard_and_actions(parse_ggf(ggf_text))
    from reversi_zero_b200.env.reversi_env import ReversiEnv, Player
    env = ReversiEnv().update(b, w, Player.black)
    for a in actions:
        env.step(a)
    own, enemy = env.get_own_and_enemy()
    return (find_correct_moves(own, enemy) >> convert_move_to_action(move)) & 1 == 1


def test_engine_subprocess_plays_over_stdin_stdout(golden, tmp_path):
    yml = os.path.join(ROOT, "tests", "golden", "ref_config", "ch5.yml")
    cfg = load_yaml(yml, project_dir=str(tmp_path))
    cfg.resource.create_directories()
    np.save(cfg.resource.model_best_blob_path, M.weights_to_blob(cfg.model, M.build_random_weights(cfg.model, 5)))
    env = dict(os.environ, PROJECT_DIR=str(tmp_path), PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "reversi-alpha-zero_b200"), ROOT]))
    env.pop("DATA_DIR", None)
    env.pop("MODEL_DIR", None)
    s = Session([sys.executable, "-m", "reversi_zero_b200.run", "nboard", "-c", yml], str(tmp_path), env)
    try:
        s.send("nboard 2")
        assert s.until(lambda l: l.startswith("status"))[0] == "set myname RAZ(ch5)"
        # the opening: a legal move
        s.send("set depth 1")
        s.send(f"set game {_ggf([])}")
        s.send("go")
        move = s.until(lambda l: l.startswith("=== "))[-1][4:].split("/")[0]
        assert _legal(_ggf([]), move), move
        # a long analysis, interrupted: the pong comes after the search has stopped and is answered promptly
        moves = [step["line"][5:] for step in golden["sessions"]["opening"]["transcript"] if step["line"].startswith("move ")][:12]
        game = _ggf(moves)
        s.send("set depth 60")
        s.send(f"set game {game}")
        s.send("hint 3")
        s.until(lambda l: l.startswith("search "))
        t0 = time.time()
        s.send("ping 9")
        got = s.until(lambda l: l.startswith("pong"), timeout=120.0)
        assert got[-1] == "pong 9" and got[-2] == "status waiting", got
        assert time.time() - t0 < 60.0
        s.send("go")
        move = s.until(lambda l: l.startswith("=== "))[-1][4:].split("/")[0]
        assert _legal(game, move), move
        # past use_solver_turn (50): the exact solver's move, which does not depend on the network
        end = next(step for step in golden["sessions"]["endgame_solver"]["transcript"] if step["line"].startswith("set game "))
        solved = next(r for step in golden["sessions"]["endgame_solver"]["transcript"] for r in step["replies"] if r.startswith("=== "))
        s.send(end["line"])
        s.send("go")
        assert s.until(lambda l: l.startswith("=== "))[-1].split("/")[0] == solved.split("/")[0]
        s.send("learn")
        s.until(lambda l: l == "learned")
        # end of input: the engine leaves on its own
        s.p.stdin.close()
        s.p.wait(timeout=60)
        assert s.p.returncode == 0, "".join(s.err)[-3000:]
        time.sleep(0.2)
        while not s.lines.empty():
            s.all.append(s.lines.get())
        bad = [l for l in s.all if not PROTOCOL.match(l)]
        assert not bad, bad
        assert os.path.getsize(os.path.join(str(tmp_path), "logs", "main.log")) > 0
    finally:
        if s.p.poll() is None:
            s.p.kill()
        s.p.wait(timeout=30)
