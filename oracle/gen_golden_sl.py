"""What the REAL supervised workers load from human game records -> tests/golden/sl_games.json.gz.

Needs the reference tree (oracle/ref_import.py) and pandas; Keras / TensorFlow imports are satisfied by the empty stand-in
modules of oracle/ref_worker_harness.py.  No human dataset is committed: the games are seeded random playouts on the
reference's light board, written as WXF (verified move by move against the reference's own parse_WXF_move) and as
onegreen digit strings, plus crafted records for the parser's corners (tandem pieces, a digit file holding the piece
twice, '.' and '=', unequal turn counts, an absent piece, an illegal but applicable move, a move without a label,
missing and duplicated CSV rows, onegreen endgames from a non-standard init with '99' squares, every result string).

For every game the fixture stores the records, then what `SupervisedWorker.load_game` of worker/sl.py and of
worker/sl_onegreen.py appends to `self.buffer`: the observation's state string, the one-hot index and the float32 value
of each entry, or that the reference raised / dropped the game.

    python -m oracle.gen_golden_sl
"""
import copy
import gzip
import json
import os
import random

import numpy as np

from . import ref_import
from .ref_worker_harness import install_shims

GOLD = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")
OUT = os.path.join(GOLD, "sl_games.json.gz")
LETTER = {'k': 'K', 'a': 'A', 'b': 'E', 'n': 'H', 'r': 'R', 'c': 'C', 'p': 'P'}
PIECES = 'rnbakabnrccpppppRNBAKABNRCCPPPPP'


def modules():
    ref_import.setup()
    install_shims()
    import cchess_alphazero.worker.sl as sl
    import cchess_alphazero.worker.sl_onegreen as slo
    from cchess_alphazero.environment.light_env.chessboard import L_Chessboard
    from cchess_alphazero.config import Config
    return sl, slo, L_Chessboard, Config


def wxf_candidates(board, action):
    """WXF spellings of a light-board move (red = lower case inside the board = upper case WXF)."""
    x0, y0, x1, y1 = (int(c) for c in action)
    ch = board.board[y0][x0]
    red = ch.islower()
    letter = LETTER[ch.lower()]
    letter = letter if red else letter.lower()
    fcol = (lambda x: str(x + 1)) if red else (lambda x: str(9 - x))
    if y1 == y0:
        tails = ['.' + fcol(x1), '=' + fcol(x1)]
    else:
        up = y1 > y0
        mov = ('+' if up else '-') if red else ('-' if up else '+')
        tails = [mov + (fcol(x1) if letter.upper() in 'HEA' else str(abs(y1 - y0)))]
    out = []
    for t in tails:
        out += [letter + '+' + t, letter + '-' + t, letter + fcol(x0) + t]
    return out


def playout(L, rng, plies, board=None):
    """Random moves on the reference's light board; returns the board and [(action, wxf or None)]."""
    b = board or L()
    start = copy.deepcopy(b)
    out = []
    for _ in range(plies):
        if b.is_end():
            break
        moves = b.legal_moves()
        b._legal_moves = None
        if not moves:
            break
        a = moves[rng.randrange(len(moves))]
        spell = [w for w in wxf_candidates(b, a) if copy.deepcopy(b).parse_WXF_move(w) == a]
        # prefer the tandem spelling where it resolves, then '=' now and then
        tand = [w for w in spell if w[1] in '+-']
        w = (tand[0] if tand and rng.random() < 0.7 else (spell[-1] if spell else None))
        if w and w[2] == '.' and rng.random() < 0.3:
            w = w[:2] + '=' + w[3]
        out.append((a, w))
        b.move_action_str(a)
    return start, out


def wxf_rows(gid, moves):
    rows = []
    for k, (_, w) in enumerate(moves):
        rows.append({"gameID": gid, "turn": k // 2 + 1, "side": "red" if k % 2 == 0 else "black", "move": w})
    return rows


def ref_sl(sl, Config, pd, rows, winner):
    """worker/sl.py load_game on this game's rows -> {"raised": bool, "records": [[state, label, value], ...]}."""
    cfg = Config("mini")
    w = sl.SupervisedWorker(cfg)
    df = pd.DataFrame(rows, columns=["gameID", "turn", "side", "move"])
    red, black = df[df.side == 'red'], df[df.side == 'black']
    try:
        w.load_game(red, black, winner, 0)
    except Exception as e:                                           # the reference aborts its run here
        return {"raised": type(e).__name__, "records": []}
    return {"raised": None, "records": [[fen.split(' ')[0], int(np.argmax(p)), float(np.float32(v))] for fen, p, v in w.buffer]}


def ref_onegreen(slo, Config, game):
    from cchess_alphazero.environment.lookup_tables import Winner
    cfg = Config("mini")
    cfg.opts.light = True
    w = slo.SupervisedWorker(cfg)
    if game['result'] == '红胜' or '胜' in game['title']:
        winner = Winner.red
    elif game['result'] == '黑胜' or '负' in game['title']:
        winner = Winner.black
    else:
        winner = Winner.draw
    try:
        v = w.load_game(game['init'], game['move_list'], winner, 0, game['title'], game['url'])
    except Exception as e:
        return {"raised": type(e).__name__, "dropped": False, "records": []}
    return {"raised": None, "dropped": v is None,
            "records": [[fen.split(' ')[0], int(np.argmax(p)), float(np.float32(v_))] for fen, p, v_ in w.buffer]}


def onegreen_init(board):
    """The light board as a onegreen init string (pieces in PIECES order, '99' = captured)."""
    squares = {}
    for y in range(10):
        for x in range(9):
            ch = board.board[y][x]
            if ch != '.':
                squares.setdefault(ch, []).append(f"{x}{9 - y}")
    out = []
    for p in PIECES:
        lst = squares.get(p, [])
        out.append(lst.pop(0) if lst else '99')
    return ''.join(out)


def onegreen_move(a):
    x0, y0, x1, y1 = (int(c) for c in a)
    return f"{x0}{9 - y0}{x1}{9 - y1}"


def main(n_random=40, seed=11):
    import pandas as pd
    sl, slo, L, Config = modules()
    rng = random.Random(seed)
    wxf_games = []

    def add(rows, winner, tag):
        gid = len(wxf_games) + 1
        rows = [dict(r) for r in rows]
        for r in rows:
            r["gameID"] = gid
        wxf_games.append({"id": gid, "tag": tag, "winner": winner, "rows": rows, "ref": ref_sl(sl, Config, pd, rows, winner)})

    winners = ['red', 'black', 'peace']
    for i in range(n_random):
        _, mv = playout(L, rng, rng.randrange(6, 120))
        if any(w is None for _, w in mv):
            mv = mv[:next(k for k, (_, w) in enumerate(mv) if w is None)]
        add(wxf_rows(0, mv), winners[i % 3], "random")
    # crafted
    _, mv = playout(L, random.Random(5), 40)
    mv = [m for m in mv if m[1]]
    rows = wxf_rows(0, mv)
    add([r for r in rows if not (r["side"] == "black" and r["turn"] > 10)], "red", "unequal_turns_red_longer")
    add([r for r in rows if not (r["side"] == "red" and r["turn"] > 12)], "black", "unequal_turns_black_longer")
    add([r for r in rows if not (r["side"] == "red" and r["turn"] == 4)], "red", "missing_turn_row")
    add(rows + [dict(rows[6])], "red", "duplicate_turn_row")
    add([{"turn": 1, "side": "red", "move": "R1+5"}, {"turn": 1, "side": "black", "move": "h2+3"},
         {"turn": 2, "side": "red", "move": "C2.5"}, {"turn": 2, "side": "black", "move": "c8.5"},
         {"turn": 3, "side": "red", "move": "P5+1"}, {"turn": 3, "side": "black", "move": "p5+1"}], "red", "illegal_but_applicable")
    add([{"turn": 1, "side": "red", "move": "C2.5"}, {"turn": 1, "side": "black", "move": "h8+7"},
         {"turn": 2, "side": "red", "move": "R1.1"}, {"turn": 2, "side": "black", "move": "r9.8"},
         {"turn": 3, "side": "red", "move": "H2+3"}, {"turn": 3, "side": "black", "move": "c2.5"},
         {"turn": 4, "side": "red", "move": "R9+1"}, {"turn": 4, "side": "black", "move": "e3+5"}], "black", "no_label_move")
    add([{"turn": 1, "side": "red", "move": "C2.5"}, {"turn": 1, "side": "black", "move": "h8+7"},
         {"turn": 2, "side": "red", "move": "H5+3"}, {"turn": 2, "side": "black", "move": "c2.5"},
         {"turn": 3, "side": "red", "move": "P1+1"}], "red", "absent_piece")
    add([{"turn": 1, "side": "red", "move": "C2.5"}, {"turn": 1, "side": "black", "move": "c8.5"},
         {"turn": 2, "side": "red", "move": "C8=5"}, {"turn": 2, "side": "black", "move": "c2=5"},
         {"turn": 3, "side": "red", "move": "C+.4"}, {"turn": 3, "side": "black", "move": "c-+2"},
         {"turn": 4, "side": "red", "move": "R1+1"}, {"turn": 4, "side": "black", "move": "r9+1"},
         {"turn": 5, "side": "red", "move": "R1.4"}, {"turn": 5, "side": "black", "move": "r9.6"},
         {"turn": 6, "side": "red", "move": "R9+1"}, {"turn": 6, "side": "black", "move": "r1+1"},
         {"turn": 7, "side": "red", "move": "R9.6"}, {"turn": 7, "side": "black", "move": "r1.4"},
         {"turn": 8, "side": "red", "move": "R-+2"}, {"turn": 8, "side": "black", "move": "r++2"},
         {"turn": 9, "side": "red", "move": "P5+1"}, {"turn": 9, "side": "black", "move": "p5+1"},
         {"turn": 10, "side": "red", "move": "P5+1"}, {"turn": 10, "side": "black", "move": "x"}], "peace", "tandem_and_separators")
    add([{"turn": 1, "side": "red", "move": "P3+1"}, {"turn": 1, "side": "black", "move": "p7+1"},
         {"turn": 2, "side": "red", "move": "P3+1"}, {"turn": 2, "side": "black", "move": "p7+1"},
         {"turn": 3, "side": "red", "move": "P3.4"}, {"turn": 3, "side": "black", "move": "p7.6"},
         {"turn": 4, "side": "red", "move": "P5+1"}, {"turn": 4, "side": "black", "move": "p5+1"},
         {"turn": 5, "side": "red", "move": "P4+1"}, {"turn": 5, "side": "black", "move": "p6+1"},
         {"turn": 6, "side": "red", "move": "P4+1"}, {"turn": 6, "side": "black", "move": "k5.4"},
         {"turn": 7, "side": "red", "move": "A4+5"}, {"turn": 7, "side": "black", "move": "a6+5"},
         {"turn": 8, "side": "red", "move": "E3+5"}, {"turn": 8, "side": "black", "move": "e7+5"}], "red", "digit_file_twice")
    add([{"turn": 1, "side": "red", "move": "C2.5"}, {"turn": 1, "side": "black", "move": "?2.5"},
         {"turn": 2, "side": "red", "move": "R1+1"}], "black", "unparseable_move")
    add([{"turn": 1, "side": "red", "move": "C2.5"}, {"turn": 1, "side": "black", "move": "h8+7"},
         {"turn": 2, "side": "red", "move": "H2+3"}], "red", "short_game")

    # onegreen: openings from the start, endgames from a non-standard init
    results = [("红胜", "甲 先胜 乙"), ("黑胜", "甲 先负 乙"), ("和棋", "甲 先和 乙"), ("", "甲 胜 乙"), ("", "甲 负 乙"),
               ("和棋", "残局")]
    og = []
    for i in range(n_random):
        r = random.Random(1000 + i)
        if i % 2 == 0:
            start, mv = playout(L, r, r.randrange(4, 80))
            init = ""
        else:
            pre, mv0 = playout(L, r, r.randrange(30, 90))
            for a, _ in mv0:
                pre.move_action_str(a)
            # an endgame: keep kings and a few pieces, side to move red (parse_init's board starts with red to move)
            b = L()
            b.board = [['.'] * 9 for _ in range(10)]
            for y in range(10):
                for x in range(9):
                    ch = pre.board[y][x]
                    if ch != '.' and (ch in 'kK' or r.random() < 0.4):
                        b.board[y][x] = ch
            init = onegreen_init(b)
            b2 = L(init)
            start, mv = playout(L, r, r.randrange(2, 50), board=b2)
        res, title = results[i % len(results)]
        og.append({"init": init, "move_list": ''.join(onegreen_move(a) for a, _ in mv), "result": res, "title": title,
                   "url": f"synthetic/{i}", "tag": "random"})
    og.append({"init": "", "move_list": "77470919" + "0000" + "1927", "result": "红胜", "title": "", "url": "", "tag": "no_label"})
    og.append({"init": "", "move_list": "7747091x", "result": "黑胜", "title": "", "url": "", "tag": "non_digit"})
    og.append({"init": "", "move_list": "774709191", "result": "和棋", "title": "", "url": "", "tag": "short_tail"})
    og.append({"init": "", "move_list": "", "result": "和棋", "title": "", "url": "", "tag": "empty"})
    for g in og:
        g["ref"] = ref_onegreen(slo, Config, g)

    os.makedirs(GOLD, exist_ok=True)
    with gzip.open(OUT, "wt", encoding="utf-8") as f:
        json.dump({"wxf": wxf_games, "onegreen": og}, f, ensure_ascii=False)
    n_rec = sum(len(g["ref"]["records"]) for g in wxf_games) + sum(len(g["ref"]["records"]) for g in og)
    print(f"{OUT}: {len(wxf_games)} WXF games, {len(og)} onegreen games, {n_rec} records, {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
