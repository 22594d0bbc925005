"""GGF game records (reference lib/ggf.py): parsing for the NBoard engine, move text and record formatting for the
self-play worker."""
import re
from collections import namedtuple
from datetime import datetime, timezone

GGF = namedtuple("GGF", "BO MOVES")
BO = namedtuple("BO", "board_type, square_cont, color")  # color: {O, *}  (O is white, * is black)
MOVE = namedtuple("MOVE", "color pos")  # color={B, W} pos: like 'F5'

_TAG = re.compile(r'([a-zA-Z]+)\[([^\]]+)\]')


def parse_ggf(ggf):
    """lib/ggf.py:13-32: the board (BO) and the moves (B / W) of a GGF game; every other tag is ignored."""
    moves = []
    bo = None
    for token in re.split(r'([a-zA-Z]+\[[^\]]+\])', ggf):
        match = _TAG.search(token)
        if not match:
            continue
        key, value = match.groups()
        key = key.upper()
        if key == "BO":
            bo = BO(*value.split(" "))
        elif key in ("B", "W"):
            moves.append(MOVE(key, value))
    return GGF(bo, moves)


def parse_ggf_board_to_bitboard(string):
    """lib/util.py:22-29: '*' = black, 'O' = white, square i = bit i."""
    white = black = 0
    for i, ch in enumerate(string):
        if ch == "*":
            black |= 1 << i
        elif ch == "O":
            white |= 1 << i
    return black, white


def convert_to_bitboard_and_actions(ggf):
    """lib/ggf.py:62-67 -> (black, white, [action or None for a pass])"""
    black, white = parse_ggf_board_to_bitboard(ggf.BO.square_cont)
    return black, white, [convert_move_to_action(move.pos) for move in ggf.MOVES]


def convert_action_to_move(action):
    """lib/ggf.py: 0 -> 'A1' ... 63 -> 'H8' (letter = row, digit = column+1); None -> 'PA'."""
    if action is None:
        return "PA"
    y, x = action // 8, action % 8
    return chr(ord("A") + y) + str(x + 1)


def convert_move_to_action(move_str):
    if move_str[:2].lower() == "pa":
        return None
    return (ord(move_str[0].upper()) - ord("A")) * 8 + int(move_str[1]) - 1


def make_ggf_string(black_name=None, white_name=None, dt=None, moves=None, result=None, think_time_sec=60):
    dt = dt or datetime.now(timezone.utc).replace(tzinfo=None)  # the reference's naive datetime.utcnow(): "%Z" prints nothing
    body = "".join(f"{'B' if i % 2 == 0 else 'W'}[{m}]" for i, m in enumerate(moves or []))
    return ("(;GM[Othello]PC[RAZSelf]DT[%s]PB[%s]PW[%s]RE[%s]TI[%d:%d]TY[8]"
            "BO[8 ---------------------------O*------*O--------------------------- *]%s;)") % (
        dt.strftime("%Y.%m.%d_%H:%M:%S.%Z"), black_name or "black", white_name or "white", result or "?",
        think_time_sec // 60, think_time_sec % 60, body)
