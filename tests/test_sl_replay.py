"""Replay of human game records (cz_sl_replay) against what the REAL worker/sl.py and worker/sl_onegreen.py load_game
append (tests/golden/sl_games.json.gz, oracle/gen_golden_sl.py), on the emulator build of the same kernel source; the
host packing of CSV / JSON records; the float64 Adam restatement on a hand-evaluated example."""
import gzip
import json
import os

import numpy as np
import pytest

from cczero_b200 import sl_data as sd
from cczero_b200.env import board_to_state
from cczero_b200.lib import CzLib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "sl_games.json.gz")


def fixture():
    with gzip.open(GOLD, "rt", encoding="utf-8") as f:
        return json.load(f)


@pytest.fixture(scope="module")
def emul():
    return CzLib(os.path.join(ROOT, "tests", "simt_emul", "libcz_emul.so"))


def wxf_sides(rows):
    red = [(int(r["turn"]), r["move"]) for r in rows if r["side"] == "red"]
    black = [(int(r["turn"]), r["move"]) for r in rows if r["side"] == "black"]
    return red, black


def check_replay(lib, device, data):
    """Every fixture game: records (state, label, float32 value bits) and failures equal the reference's."""
    games = [(*wxf_sides(g["rows"]), g["winner"]) for g in data["wxf"]]
    rep, wins, keep, skipped = sd.replay_wxf_games(lib, device, games)
    got = {}
    ds = sd.build_dataset(rep, wins)
    # per-game slices of the dataset, in game order
    labels = rep.labels.cpu().numpy()
    sides = rep.sides.cpu().numpy()
    pos = 0
    boards, labs, vals = ds.boards.cpu().numpy(), ds.labels.cpu().numpy(), ds.values.cpu().numpy()
    for j, k in enumerate(keep):
        if rep.game[j, 1] != sd.OK:
            got[k] = None
            continue
        m = len(sd.record_order(labels, sides, int(rep.offsets[j]), int(rep.offsets[j + 1])))
        got[k] = [[board_to_state(boards[i]), int(labs[i]), vals[i]] for i in range(pos, pos + m)]
        pos += m
    assert pos == len(ds)
    n_fail = 0
    for k, g in enumerate(data["wxf"]):
        ref = g["ref"]
        if ref["raised"]:
            assert got.get(k) is None, (g["tag"], "the reference raised")
            n_fail += 1
            continue
        recs = got[k]
        assert len(recs) == len(ref["records"]), (g["tag"], len(recs), len(ref["records"]))
        for (s, lab, v), (rs, rl, rv) in zip(recs, ref["records"]):
            assert s == rs and lab == rl, g["tag"]
            assert np.float32(v).tobytes() == np.float32(rv).tobytes(), g["tag"]
    assert n_fail >= 3 and skipped >= 2                      # missing and duplicated rows are skipped on the host

    og = data["onegreen"]
    rep, wins, keep, skipped = sd.replay_onegreen_games(lib, device, og)
    assert keep == list(range(len(og)))
    labels, sides = rep.labels.cpu().numpy(), rep.sides.cpu().numpy()
    ds = sd.build_dataset(rep, wins)
    boards, labs, vals = ds.boards.cpu().numpy(), ds.labels.cpu().numpy(), ds.values.cpu().numpy()
    pos = 0
    draws = 0
    for j, g in enumerate(og):
        ref = g["ref"]
        if ref["raised"] or ref["dropped"]:
            assert rep.game[j, 1] == sd.FAILED, g["tag"]
            continue
        assert rep.game[j, 1] == sd.OK, g["tag"]
        m = len(sd.record_order(labels, sides, int(rep.offsets[j]), int(rep.offsets[j + 1])))
        assert m == len(ref["records"]), g["tag"]
        for i, (rs, rl, rv) in zip(range(pos, pos + m), ref["records"]):
            assert board_to_state(boards[i]) == rs and int(labs[i]) == rl, g["tag"]
            assert vals[i].tobytes() == np.float32(rv).tobytes(), (g["tag"], vals[i], rv)
        draws += sd.onegreen_winner(g) == 0 and m > 0 and abs(float(ref["records"][0][2])) not in (0.0, 1.0)
        pos += m
    assert pos == len(ds)
    assert draws >= 3                                        # draws valued by evaluate, not 0 / 1
    return rep


def test_replay_matches_reference_emul(emul):
    check_replay(emul, "cpu", fixture())


def test_illegal_ply_is_flagged_exactly(emul):
    """The legality index flags the crafted illegal ply (a rook through its own pawn) and nothing in legal playouts."""
    data = fixture()
    sel = [g for g in data["wxf"] if g["tag"] in ("illegal_but_applicable", "random")]
    games = [(*wxf_sides(g["rows"]), g["winner"]) for g in sel]
    rep, _, keep, _ = sd.replay_wxf_games(emul, "cpu", games)
    fi = {sel[k]["tag"] + str(k): int(rep.first_illegal[j]) for j, k in enumerate(keep)}
    ill = [v for t, v in fi.items() if t.startswith("illegal")]
    assert ill == [0]                                         # R1+5 is the first ply
    assert all(v == -1 for t, v in fi.items() if t.startswith("random"))


def test_wxf_packing_drops_last_turn_and_skips_bad_rows():
    red = [(1, "C2.5"), (2, "H2+3"), (3, "R1.2")]
    black = [(1, "h8+7"), (2, "c8.5")]
    plies, sides = sd.pack_wxf_game(red, black)
    # turns < max: red 1, 2 and black 1 only; red then black per turn
    assert [p.rstrip(b"\0").decode() for p in plies] == ["C2.5", "h8+7", "H2+3"] and sides == [1, -1, 1]
    with pytest.raises(sd.RecordError):
        sd.pack_wxf_game([(1, "C2.5"), (3, "R1.2")], black)                # no row for red turn 2
    with pytest.raises(sd.RecordError):
        sd.pack_wxf_game(red + [(2, "R1.1")], black)                       # two rows for red turn 2
    assert sd.pack_wxf_game([], []) == ([], [])
    assert sd.ply_bytes("C2") == b"C2\0\0" and sd.ply_bytes("C2.5x") == b"C2.5"


def test_record_interleave_stops_at_red_list():
    labels = np.array([5, 6, 7, -1, 8, 9, 10])
    sides = np.array([1, -1, 1, -1, -1, 1, -1])
    # red: 0, 2, 5; black (labelled): 1, 4, 6 -> r0 b1 r2 b4 r5 b6
    assert sd.record_order(labels, sides, 0, 7) == [0, 1, 2, 4, 5, 6]
    assert sd.record_order(labels, np.array([1, -1, -1, -1, -1, -1, -1]), 0, 7) == [0, 1]


def test_csv_and_json_readers(tmp_path):
    data = fixture()
    info, moves = tmp_path / "gameinfo.csv", tmp_path / "moves.csv"
    info.write_text("gameID,winner\n" + "".join(f"{g['id']},{g['winner']}\n" for g in data["wxf"]))
    moves.write_text("gameID,turn,side,move\n" + "".join(f"{r['gameID']},{r['turn']},{r['side']},{r['move']}\n"
                                                         for g in data["wxf"] for r in g["rows"]))
    gi = sd.read_gameinfo(str(info))
    mv = sd.read_moves(str(moves))
    assert [int(r["gameID"]) for r in gi] == [g["id"] for g in data["wxf"]]
    for g in data["wxf"]:
        red, black = wxf_sides(g["rows"])
        got = mv.get(g["id"], {"red": [], "black": []})          # a game without move rows has no entry
        assert sorted(got["red"]) == sorted(red) and sorted(got["black"]) == sorted(black)
    assert [sd.onegreen_winner(g) for g in data["onegreen"][:6]] == [1, -1, 0, 1, -1, 0]


def test_onegreen_init_board():
    b = sd.onegreen_board("")
    assert (b == sd.start_board()).all()
    # the standard position written as an init string is the standard board
    std = "0919293949596979891777062646668600102030405060708012720323436383"
    assert (sd.onegreen_board(std) == sd.start_board()).all()
    b = sd.onegreen_board("99" * 4 + "49" + "99" * 11 + "99" * 4 + "40" + "99" * 11)
    assert int((b != 0).sum()) == 2 and b[4] == 7 and b[9 * 9 + 4] == 15
    with pytest.raises(sd.RecordError):
        sd.onegreen_board("90" + "99" * 31)                                 # x = 9: board[y][9] raises


def test_adam_oracle_two_steps_by_hand():
    from tests import adam_oracle as ao
    w = np.array([1.0, -2.0]); g1 = np.array([0.5, 0.0]); g2 = np.array([-1.0, 2.0])
    st = ao.AdamState.zeros_like({"k": w})
    ws = {"k": w.copy()}
    ao.adam_update(ws, {"k": g1}, st, lr=0.1)
    # t=1: m = 0.1 g, v = 0.001 g^2, lr_t = 0.1 sqrt(0.001) / 0.1; step = lr_t m / (sqrt(v) + eps) = 0.1 sign(g) (g != 0)
    assert abs(ws["k"][0] - (1.0 - 0.1 * 0.05 / (np.sqrt(0.001 * 0.25) + 1e-8) * np.sqrt(0.001) / 0.1 * 1.0)) < 1e-12
    assert ws["k"][1] == -2.0
    ao.adam_update(ws, {"k": g2}, st, lr=0.1)
    m = 0.9 * 0.05 + 0.1 * -1.0
    v = 0.999 * 0.00025 + 0.001 * 1.0
    lr_t = 0.1 * np.sqrt(1 - 0.999 ** 2) / (1 - 0.9 ** 2)
    w0 = 1.0 - 0.1 * np.sqrt(0.001) / 0.1 * 0.05 / (np.sqrt(0.00025) + 1e-8)
    assert abs(ws["k"][0] - (w0 - lr_t * m / (np.sqrt(v) + 1e-8))) < 1e-12
    assert abs(ws["k"][1] - (-2.0 - lr_t * 0.2 / (np.sqrt(0.004) + 1e-8))) < 1e-12
    assert st.iterations == 2
