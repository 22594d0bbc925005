"""Writes what the UNMODIFIED reference NBoard engine (play_game/nboard.py, imported through oracle/ref_shims) replies,
for tests/test_nboard_host.py and tests/test_nboard_gpu.py:

  * scripted protocol sessions, each on a fresh engine: every input line and every reply line.  The engine's model is
    the deterministic FakeNet evaluator (policy 1/64, value (#own - #enemy)/64, the engine's RZ_EVAL_FAKE) and
    play_with_human.parallel_search_num = 1, so the reference's search is deterministic; the time field of "===" replies
    is recorded as "<time>";
  * parse_ggf / convert_to_bitboard_and_actions on GGF strings as NBoard sends them;
  * NBoardEngine.set_depth over depths x simulation counts;
  * the defaults of the play_with_human and nboard config sections, and what update_play_config changes;
  * manager.py's argument parsing.

-> nboard_ref.json.  Run once where the reference checkout exists:

    python tests/golden/make_golden_nboard.py
"""
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import oracle.ref_shims.install as shims  # noqa: E402

shims.install()

from make_golden import FakeNet  # noqa: E402  (same deterministic evaluator as mcts.json)
from reversi_zero.config import Config, PlayConfig, PlayWithHumanConfig, NBoardConfig  # noqa: E402
from reversi_zero.env.reversi_env import ReversiEnv  # noqa: E402
from reversi_zero.lib import bitboard as rb  # noqa: E402
from reversi_zero.lib.ggf import parse_ggf, convert_to_bitboard_and_actions, convert_action_to_move  # noqa: E402
import reversi_zero.agent.player as ref_player  # noqa: E402
import reversi_zero.play_game.nboard as ref_nboard  # noqa: E402

SEED = 20261015
START_BO = "8 ---------------------------O*------*O--------------------------- *"
# config overrides of every session (the mirror test applies the same ones)
CONFIG = dict(type="golden", play=dict(simulation_num_per_move=20, c_puct=5), play_with_human=dict(parallel_search_num=1))


def scripted_game(seed, want_pass=False):
    """moves ("F5" / "PA") of a random game from the opening; with want_pass, one that contains a pass"""
    rng = np.random.default_rng(seed)
    while True:
        env = ReversiEnv().reset()
        moves = []
        while not env.done:
            o, e = env.get_own_and_enemy()
            legal = rb.find_correct_moves(o, e)
            ms = [i for i in range(64) if legal >> i & 1]
            before = env.next_player
            a = int(ms[rng.integers(len(ms))])
            env.step(a)
            moves.append(convert_action_to_move(a))
            if not env.done and env.next_player == before:   # the other side had to pass
                moves.append("PA")
        if not want_pass or "PA" in moves:
            return moves


def ggf(moves, decorate=False):
    """a GGF game as NBoard sends it with ``set game``; decorate adds NBoard's /eval/time fields to some moves"""
    body = []
    for i, m in enumerate(moves):
        tag = "B" if i % 2 == 0 else "W"
        if decorate and i % 3 == 1:
            m = f"{m}/{(i % 7) - 3}.25/{i * 0.5}"
        body.append(f"{tag}[{m}]")
    return (f"(;GM[Othello]PC[NBoard]DT[2026-10-15 12:00:00 GMT]PB[RAZ]PW[human]RE[?]TI[5:00]TY[8]BO[{START_BO}]"
            + "".join(body) + ";)")


def configure(solver):
    cfg = Config()
    cfg.type = CONFIG["type"]
    for section in ("play", "play_with_human"):
        for k, v in CONFIG[section].items():
            setattr(getattr(cfg, section), k, v)
    cfg.play.use_solver_turn = cfg.play.use_solver_turn_in_simulation = 50 if solver else 0
    cfg.play_with_human.update_play_config(cfg.play)
    return cfg


def run_session(lines, solver):
    cfg = configure(solver)
    np.random.seed(0)
    ref_nboard.load_model = lambda config: None
    ref_nboard.ReversiPlayer = lambda config, model, play_config=None, enable_resign=True: ref_player.ReversiPlayer(
        config, model, play_config, enable_resign, api=FakeNet())
    eng = ref_nboard.NBoardEngine(cfg)
    out = []
    eng.reply = lambda message: out.append(message)
    transcript = []
    for line in lines:
        if line.startswith("ping"):
            eng.push_callback(line)   # what the reader thread does before the line is handled
        n0 = len(out)
        eng.handler.handle_message(line.strip())
        replies = []
        for r in out[n0:]:
            if r.startswith("=== "):
                head, ev, _ = r.split("/")
                r = f"{head}/{ev}/<time>"
            replies.append(r)
        transcript.append(dict(line=line, replies=replies))
    return dict(solver=solver, transcript=transcript)


def sessions():
    g = scripted_game(SEED)
    gp = scripted_game(SEED + 1, want_pass=True)
    ip = gp.index("PA")
    out = {}
    # opening: the first moves, rethinking turns (> start_rethinking_turn = 8), hint, ping, learn and unknown lines
    lines = ["nboard 2", "set depth 1", f"set game {ggf([])}", "go", "hint 3"]
    for k in range(12):
        lines.append(f"move {g[k]}")
        if k in (0, 5, 9, 11):
            lines += ["go", "hint 2"]
    lines += ["ping 7", "learn", "analyze", "hello engine", "set depth 2", "go", "set game " + ggf(g[:1]), "go"]
    out["opening"] = run_session(lines, True)
    # midgame, solver off, decorated moves, deeper search
    lines = ["nboard 2", "set depth 3", f"set game {ggf(g[:30], decorate=True)}", "go", "hint 4", f"move {g[30]}/1.5/2.0",
             f"move {g[31]}", "go"]
    out["midgame"] = run_session(lines, False)
    # endgame from turn 50 with the exact root solver, and the same positions without it.  The searches reuse the tree
    # for the same side only: the reference marks a node expanded for the side that evaluated it (agent/player.py:325), so
    # the first simulation at a root last seen from the other side re-evaluates it and adds no visit, which the engine's
    # shared statistics do not reproduce
    for name, solver in (("endgame_solver", True), ("endgame_search", False)):
        lines = ["nboard 2", "set depth 1", f"set game {ggf(g[:50])}", "go", "hint 3", f"move {g[50]}", f"move {g[51]}", "go",
                 "hint 2", f"move {g[52]}", f"move {g[53]}", "go"]
        out[name] = run_session(lines, solver)
    # a pass: NBoard's side to move has no legal move -> "=== PA"; then NBoard sends "move PA"
    lines = ["nboard 2", "set depth 1", f"set game {ggf(gp[:ip])}", "go", f"move {gp[ip]}", "go", "hint 1"]
    out["pass"] = run_session(lines, True)
    return out


def ggf_golden():
    g = scripted_game(SEED)
    gp = scripted_game(SEED + 1, want_pass=True)
    texts = [ggf([]), ggf(g[:7]), ggf(g[:30], decorate=True), ggf(gp),
             f"(;GM[Othello]PC[NBoard]BO[{START_BO}]b[f5]w[f6//0.1];)",
             "(;GM[Othello]PC[NBoard]BO[8 -------------------------O-O**----*O--------------------------- O]W[c4]B[PA];)"]
    out = []
    for t in texts:
        p = parse_ggf(t)
        black, white, actions = convert_to_bitboard_and_actions(p)
        out.append(dict(text=t, bo=list(p.BO), moves=[list(m) for m in p.MOVES], black=black, white=white, actions=actions))
    return out


def set_depth_golden():
    out = []
    for sims in (20, 200, 800):
        for depth in ("0", "1", "2", "5", "20", "60", "x"):
            pc = PlayConfig()
            pc.simulation_num_per_move = sims
            fake = types.SimpleNamespace(play_config=pc, nc=NBoardConfig())
            ref_nboard.NBoardEngine.set_depth(fake, depth)
            out.append(dict(sims=sims, depth=depth, required_visit_to_decide_action=pc.required_visit_to_decide_action,
                            thinking_loop=pc.thinking_loop))
    return out


def config_golden():
    pc = PlayConfig()
    PlayWithHumanConfig().update_play_config(pc)
    return dict(play_with_human=vars(PlayWithHumanConfig()), nboard=vars(NBoardConfig()), updated_play=vars(pc))


def parser_golden():
    from reversi_zero.manager import create_parser
    argvs = [["self"], ["opt", "-c", "config/ch5.yml"], ["eval", "--new"], ["nboard", "-c", "x.yml", "--new"],
             ["opt", "--total-step", "123"], ["self", "--type", "mini"], ["nboard"], ["bogus"], [], ["opt", "--total-step", "x"]]
    out = []
    for argv in argvs:
        try:
            out.append(dict(argv=argv, args=vars(create_parser().parse_args(argv))))
        except SystemExit as e:
            out.append(dict(argv=argv, exit=e.code))
    return out


def main():
    import contextlib
    import io
    with contextlib.redirect_stderr(io.StringIO()):
        parser = parser_golden()
    golden = dict(config=CONFIG, sessions=sessions(), ggf=ggf_golden(), set_depth=set_depth_golden(), defaults=config_golden(),
                  parser=parser)
    with open(os.path.join(HERE, "nboard_ref.json"), "w") as f:
        json.dump(golden, f, indent=1)


if __name__ == "__main__":
    main()
