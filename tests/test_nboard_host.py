"""CPU suite for the NBoard engine (reversi_zero_b200/play_game/nboard.py) and the command line (run.py): GGF parsing, the
protocol handler in front of a stand-in engine, the stdin reader, the config sections and the argument parsing against
what the unmodified reference does (tests/golden/nboard_ref.json, tests/golden/make_golden_nboard.py), and the model
lookup of play_game/common.py."""
import io
import json
import os
import types

import numpy as np
import pytest

from reversi_zero_b200 import run
from reversi_zero_b200.config import Config, PlayConfig, PlayWithHumanConfig, NBoardConfig, create_config
from reversi_zero_b200.env.reversi_env import Player
from reversi_zero_b200.lib import ggf as G
from reversi_zero_b200.lib.nonblocking_stream_reader import NonBlockingStreamReader
from reversi_zero_b200.play_game import common, nboard as NB


@pytest.fixture(scope="module")
def golden(golden_dir):
    with open(os.path.join(golden_dir, "nboard_ref.json")) as f:
        return json.load(f)


def test_ggf_parsing_matches_reference(golden):
    for case in golden["ggf"]:
        p = G.parse_ggf(case["text"])
        assert list(p.BO) == case["bo"]
        assert [list(m) for m in p.MOVES] == case["moves"]
        black, white, actions = G.convert_to_bitboard_and_actions(p)
        assert (black, white, actions) == (case["black"], case["white"], case["actions"])


class StandInEngine:
    """NBoardEngine's interface to the protocol handler, recording calls; go / hint answer with canned results"""

    def __init__(self, handler_config):
        self.calls, self.out = [], []
        self.handler = NB.NBoardProtocolVersion2(handler_config, self)

    def reply(self, message):
        self.out.append(message)

    def __getattr__(self, name):
        if name in ("set_depth", "set_game", "reset_state", "move", "stop_thinking"):
            return lambda *a: self.calls.append((name,) + a)
        raise AttributeError(name)

    def go(self):
        self.calls.append(("go",))
        return NB.GoResponse(37, 0.25, 1.5)

    def hint(self, n):
        self.calls.append(("hint", n))
        self.handler.report_hint([NB.HintResponse(19, 0.5, 30.0), NB.HintResponse(26, -0.125, 12.0)])


def test_protocol_dispatch_and_replies():
    cfg = Config()
    cfg.type = "ch5"
    e = StandInEngine(cfg)
    h = e.handler
    opening = "(;GM[Othello]BO[8 ---------------------------O*------*O--------------------------- *];)"
    for line in ("nboard 2", "set depth 7", f"set game {opening}", "move f5/1.25/3.0", "move PA", "go", "hint 2", "ping 4",
                 "learn", "analyze", "who are you", "nboard 3"):
        h.handle_message(line)
    black, white = 1 << 28 | 1 << 35, 1 << 27 | 1 << 36
    assert e.calls == [("set_depth", "7"), ("set_game", NB.GameState(black, white, [], Player.black)), ("reset_state",),
                       ("move", 44), ("move", None), ("go",), ("hint", 2)]
    assert e.out == ["set myname RAZ(ch5)", "status waiting",
                     "status thinking...", "=== E6/2.5/1.5", "status waiting",
                     "status thinkng hint...", "search D3 -0.125 0 12", "search C4 0.5 0 30", "status waiting",
                     "pong 4", "learned",
                     "set myname RAZ(ch5)", "status waiting"]


def test_set_game_resets_the_search_only_for_a_new_game():
    e = StandInEngine(Config())
    bo = "BO[8 ---------------------------O*------*O--------------------------- *]"
    for moves, resets in (("", True), ("B[F5]", True), ("B[F5]W[F6]", False), ("B[F5]W[F6]B[E6]W[F4]", False)):
        e.calls.clear()
        e.handler.handle_message(f"set game (;GM[Othello]{bo}{moves};)")
        assert (("reset_state",) in e.calls) == resets
    e.calls.clear()
    e.handler.handle_message("set game (;GM[Othello]BO[8 ---------------------------O*------*O--------------------------- O];)")
    assert e.calls[0][1].player == Player.white


def test_protocol_lines_without_a_search_match_reference(golden):
    """every reply of the recorded sessions that does not depend on a search: greeting, pong, learned, silence"""
    cfg = create_config(golden["config"])
    for s in golden["sessions"].values():
        for step in s["transcript"]:
            line = step["line"]
            if line.split(" ")[0] in ("go", "hint"):
                continue
            e = StandInEngine(cfg)
            e.handler.handle_message(line)
            assert e.out == step["replies"], line


def test_set_depth_matches_reference(golden):
    for case in golden["set_depth"]:
        pc = PlayConfig()
        pc.simulation_num_per_move = case["sims"]
        fake = types.SimpleNamespace(play_config=pc, nc=NBoardConfig())
        NB.NBoardEngine.set_depth(fake, case["depth"])
        assert (pc.required_visit_to_decide_action, pc.thinking_loop) == (case["required_visit_to_decide_action"],
                                                                         case["thinking_loop"]), case


def test_config_defaults_match_reference(golden):
    d = golden["defaults"]
    assert vars(PlayWithHumanConfig()) == d["play_with_human"]
    assert vars(NBoardConfig()) == d["nboard"]
    pc = PlayConfig()
    PlayWithHumanConfig().update_play_config(pc)
    mine = {k: (v if not isinstance(v, list) else [list(x) for x in v]) for k, v in vars(pc).items()}
    assert mine == d["updated_play"]
    cfg = Config()
    assert isinstance(cfg.nboard, NBoardConfig) and isinstance(cfg.play_with_human, PlayWithHumanConfig)
    # a YAML section overlays the defaults (alpha_go_zero.yml sets one field of play_with_human)
    cfg = create_config({"play_with_human": {"use_newest_next_generation_model": False}, "nboard": {"my_name": "X"}})
    assert cfg.play_with_human.use_newest_next_generation_model is False and cfg.play_with_human.parallel_search_num == 8
    assert cfg.nboard.my_name == "X" and cfg.nboard.hint_callback_per_sim == 10


def test_reader_delivers_lines_then_reports_end():
    seen = []
    r = NonBlockingStreamReader(io.StringIO("ping 1\nnboard 2\n"))
    r.start(push_callback=seen.append)
    got = [r.readline(5.0), r.readline(5.0)]
    r._thread.join(5.0)
    assert got == ["ping 1\n", "nboard 2\n"] and seen == got
    assert r.closed and r.readline(0.01) is None


def _engine_without_device(lines):
    """an NBoardEngine whose player is a stand-in: the main loop, the reader thread and the handler are the real ones"""
    eng = NB.NBoardEngine.__new__(NB.NBoardEngine)
    eng.config = Config()
    eng.nc = eng.config.nboard
    eng.stdout = io.StringIO()
    eng.reader = NonBlockingStreamReader(io.StringIO("".join(l + "\n" for l in lines)))
    eng.handler = NB.NBoardProtocolVersion2(eng.config, eng)
    eng.player = types.SimpleNamespace(stopped=0)
    eng.player.stop_thinking = lambda: setattr(eng.player, "stopped", eng.player.stopped + 1)
    return eng


def test_main_loop_handles_every_line_and_ends_at_eof():
    eng = _engine_without_device(["nboard 2", "ping 1", "learn", "ping 2"])
    eng.start()   # returns: the stream has ended
    assert eng.stdout.getvalue().splitlines() == ["set myname RAZ(default)", "status waiting", "pong 1", "learned", "pong 2"]
    assert eng.player.stopped == 2   # each ping stopped the search from the reader thread


def _model_tree(tmp_path, best=False, newest=False, older=False, h5_best=False, h5_newest=False):
    cfg = Config(project_dir=str(tmp_path))
    rc = cfg.resource
    rc.create_directories()
    if best:
        np.save(rc.model_best_blob_path, np.zeros(3, np.float32))
    if h5_best:
        open(rc.model_best_weight_path, "wb").close()
    for stamp, want, h5 in (("20260101-000000.000000", older, False), ("20260102-000000.000000", newest, h5_newest)):
        if want or h5:
            d = os.path.join(rc.next_generation_model_dir, rc.next_generation_model_dirname_tmpl % stamp)
            os.makedirs(d)
            if want:
                np.save(os.path.join(d, "model_weight.rzblob.npy"), np.zeros(3, np.float32))
            if h5:
                open(os.path.join(d, rc.next_generation_model_weight_filename), "wb").close()
    return cfg


def test_model_lookup_order(tmp_path):
    cfg = _model_tree(tmp_path / "a", best=True, newest=True, older=True)
    newest = os.path.join(cfg.resource.next_generation_model_dir, "model_20260102-000000.000000", "model_weight.rzblob.npy")
    assert common.model_source_path(cfg) == newest
    cfg.play.use_newest_next_generation_model = False
    assert common.model_source_path(cfg) == cfg.resource.model_best_blob_path
    cfg = _model_tree(tmp_path / "b", best=True)
    assert common.model_source_path(cfg) == cfg.resource.model_best_blob_path
    cfg = _model_tree(tmp_path / "c", newest=True)
    cfg.play.use_newest_next_generation_model = False
    assert common.model_source_path(cfg).endswith(os.path.join("model_20260102-000000.000000", "model_weight.rzblob.npy"))


def test_model_lookup_refuses_without_weights(tmp_path):
    with pytest.raises(RuntimeError, match="^No models found!$"):
        common.model_source_path(_model_tree(tmp_path / "none"))
    with pytest.raises(RuntimeError, match="export_keras_weights"):
        common.model_source_path(_model_tree(tmp_path / "h5", h5_best=True))
    with pytest.raises(RuntimeError, match="export_keras_weights"):
        common.model_source_path(_model_tree(tmp_path / "h5n", h5_newest=True))
    assert not os.listdir(os.path.join(tmp_path / "none", "data", "model", "next_generation"))   # nothing was created


def test_argument_parsing_matches_reference(golden, capsys):
    for case in golden["parser"]:
        if "exit" in case:
            with pytest.raises(SystemExit) as ex:
                run.create_parser().parse_args(case["argv"])
            assert ex.value.code == case["exit"]
        else:
            assert vars(run.create_parser().parse_args(case["argv"])) == case["args"]
    with pytest.raises(SystemExit):
        run.create_parser().parse_args(["play_gui"])   # needs wxPython: not offered


def test_start_dispatches_and_sets_up_like_the_reference(tmp_path, monkeypatch, capsys):
    assert run.start(["self", "--type", "mini"]) == 1
    assert "--type option was deprecated" in capsys.readouterr().out
    monkeypatch.setenv("PROJECT_DIR", str(tmp_path))
    monkeypatch.setattr(run, "setup_logger", lambda path: seen.append(("log", path)))
    seen = []
    from reversi_zero_b200.worker import optimize
    from reversi_zero_b200.play_game import nboard
    monkeypatch.setattr(optimize, "start", lambda config: seen.append(("opt", config)) or "opt done")
    monkeypatch.setattr(nboard, "start", lambda config: seen.append(("nboard", config)) or "nboard done")
    assert run.start(["opt", "--new", "--total-step", "77"]) == "opt done"
    cfg = seen[1][1]
    assert seen[0] == ("log", os.path.join(str(tmp_path), "logs", "main.log"))
    assert cfg.opts.new is True and optimize.trainer_field(cfg, "start_total_steps") == 77
    assert os.path.isdir(cfg.resource.next_generation_model_dir) and os.path.isdir(cfg.resource.play_data_dir)
    yml = tmp_path / "c.yml"
    yml.write_text("type: mine\ntrainer:\n  batch_size: 16\nnboard:\n  my_name: Z\n")
    seen.clear()
    assert run.start(["nboard", "-c", str(yml), "--total-step", "5"]) == "nboard done"
    cfg = seen[1][1]
    assert cfg.type == "mine" and cfg.nboard.my_name == "Z" and cfg.opts.new is False
    assert optimize.trainer_field(cfg, "start_total_steps") == 5 and optimize.trainer_field(cfg, "batch_size") == 16


def test_launcher_runs_the_nboard_command():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    path = os.path.join(root, "nboard_engine")
    assert os.access(path, os.X_OK)
    with open(path) as f:
        text = f.read()
    assert "-m reversi_zero_b200.run nboard \"$@\"" in text
