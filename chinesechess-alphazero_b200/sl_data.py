"""Human game records as a device-resident training set (worker/sl.py, worker/sl_onegreen.py).

The host reads the records and packs every game as a start board plus its plies (4 bytes each, the WXF characters or the
four onegreen digits, with the side list the ply belongs to).  `replay()` walks all games at once on the rules kernels
(`cz_sl_replay`, csrc/cz_replay.cu: one warp per game) and leaves the observation before every ply and its label in device
tensors.  `build_dataset()` keeps the records `load_game` appends, in its order, and computes their values with numpy.
A position then costs 96 + 2 + 4 bytes on the device instead of the 14x10x9 float32 planes and 2086-wide float32 policy
row (13 388 bytes) of the reference's host arrays; `SlDataset.batch()` expands a batch on the device.  The same dataset
holds OptimizeWorker's self-play records (records.replay_play_games) with a fourth column, the ply in the game.
"""
import ctypes as C
import csv

import numpy as np
import torch

from .env import INIT_STATE, state_to_board
from .lib import BOARD_STRIDE, N_LABELS

WXF, ONEGREEN = 0, 1                   # cz_sl_replay modes
OK, FAILED = 0, 1                      # per-game status
GAME_FIELDS = 6                        # plies applied, status, first illegal ply, ans, tot, red to move
ONEGREEN_PIECES = 'rnbakabnrccpppppRNBAKABNRCCPPPPP'
_LIGHT_CODE = {'p': 1, 'c': 2, 'r': 3, 'n': 4, 'b': 5, 'a': 6, 'k': 7}


class RecordError(ValueError):
    """The reference raises on this record (it would abort the whole run); the game is skipped."""


def _ptr(t):
    return C.c_void_p(t.data_ptr())


def start_board():
    """The standard start in the replay's frame (the light board's rows, red = codes 1..7): the engine's INIT_STATE."""
    return state_to_board(INIT_STATE)


def onegreen_board(init):
    """L_Chessboard.parse_init (light_env/chessboard.py:47-53): 32 two-digit squares in ONEGREEN_PIECES order, '99' =
    captured, y counted from black's side.  Raises RecordError where the reference raises."""
    if init is None or init == '':
        return start_board()
    b = np.zeros(BOARD_STRIDE, np.uint8)
    for pos, piece in zip([init[i:i + 2] for i in range(0, len(init), 2)], ONEGREEN_PIECES):
        if pos == '99':
            continue
        if len(pos) != 2 or not (pos[0].isdigit() and pos[1].isdigit() and pos.isascii()):
            raise RecordError(f"init square {pos!r}")
        x, y = int(pos[0]), 9 - int(pos[1])
        if x > 8:
            raise RecordError(f"init square {pos!r} is off the board")
        b[y * 9 + x] = _LIGHT_CODE[piece.lower()] | (8 if piece.isupper() else 0)
    return b


def ply_bytes(move):
    """The first four characters of a move as bytes; missing characters are 0, characters outside ASCII 0x7f (no
    character the replay interprets)."""
    out = bytearray(4)
    if isinstance(move, str):
        for i, ch in enumerate(move[:4]):
            out[i] = ord(ch) if ord(ch) < 128 else 0x7F
    return bytes(out)


# ------------------------------------------------------------------------------------------------ readers
def _key(v):
    v = str(v).strip()
    try:
        return int(v)
    except ValueError:
        return v


def read_gameinfo(path):
    """gameinfo.csv rows (dicts), in file order."""
    with open(path, newline='', encoding='utf-8') as f:
        return list(csv.DictReader(f))


def read_moves(path):
    """moves.csv grouped by gameID in one pass: gameID -> {"red": [(turn, move)], "black": [...]}."""
    games = {}
    with open(path, newline='', encoding='utf-8') as f:
        for row in csv.DictReader(f):
            g = games.setdefault(_key(row['gameID']), {'red': [], 'black': []})
            side = row.get('side')
            if side in g:
                g[side].append((int(float(row['turn'])), row.get('move')))
    return games


def pack_wxf_game(red, black):
    """sl.py load_game :124-155 on the CSV rows: turns 1 .. max - 1 of each side (`turns < max_turn`), red then black
    per turn, each turn exactly one row (`.item()`).  Returns (plies, sides); RecordError where `.item()` raises."""
    rmax = max((t for t, _ in red), default=None)
    bmax = max((t for t, _ in black), default=None)
    plies, sides = [], []
    turns = 1

    def one(rows, t, side):
        hit = [m for tt, m in rows if tt == t]
        if len(hit) != 1:
            raise RecordError(f"{side} turn {t}: {len(hit)} rows")
        return hit[0]

    while (rmax is not None and turns < rmax) or (bmax is not None and turns < bmax):
        if rmax is not None and turns < rmax:
            plies.append(ply_bytes(one(red, turns, 'red')))
            sides.append(1)
        if bmax is not None and turns < bmax:
            plies.append(ply_bytes(one(black, turns, 'black')))
            sides.append(-1)
        turns += 1
    return plies, sides


def wxf_red_win(winner):
    return 1 if winner == 'red' else (-1 if winner == 'black' else 0)


def pack_onegreen_game(move_list):
    """sl_onegreen.py load_game :139-147: 4-character moves, even plies red."""
    moves = [move_list[i:i + 4] for i in range(0, len(move_list), 4)]
    return [ply_bytes(m) for m in moves], [1 if k % 2 == 0 else -1 for k in range(len(moves))]


def onegreen_winner(game):
    """sl_onegreen.py:119-125: 1 red, -1 black, 0 draw."""
    if game['result'] == '红胜' or '胜' in game['title']:
        return 1
    if game['result'] == '黑胜' or '负' in game['title']:
        return -1
    return 0


# ------------------------------------------------------------------------------------------------ replay
class Replay:
    """Device outputs of one cz_sl_replay call plus the host copies the dataset builder needs."""

    def __init__(self, boards, labels, sides, game, offsets):
        self.boards, self.labels, self.sides = boards, labels, sides          # [P][96] u8, [P] i16, [P] i8 (device)
        self.game = game                                                      # np.int32 [n][GAME_FIELDS]
        self.offsets = offsets                                                # np.int64 [n + 1]

    @property
    def status(self):
        return self.game[:, 1]

    @property
    def first_illegal(self):
        return self.game[:, 2]


def replay(lib, device, boards0, plies, sides, mode, lut=None, stream=None):
    """Replays n games: boards0 u8 [n][96] start boards, plies / sides one list per game (ply_bytes / +-1)."""
    device = torch.device(device)
    n = len(plies)
    counts = np.array([len(p) for p in plies], np.int64)
    offsets = np.zeros(n + 1, np.int64)
    np.cumsum(counts, out=offsets[1:])
    total = int(offsets[-1])
    flat = np.frombuffer(b''.join(b''.join(p) for p in plies), np.uint8).reshape(total, 4).copy() if total else np.zeros((0, 4), np.uint8)
    side_arr = np.concatenate([np.asarray(s, np.int8) for s in sides]) if total else np.zeros(0, np.int8)
    if lut is None:
        lut = np.empty(8100, np.int16)
        lib.call("cz_action_labels", C.c_void_p(0), C.c_void_p(lut.ctypes.data))

    def dev(a):
        return torch.from_numpy(np.ascontiguousarray(a)).to(device)

    t_init = dev(np.asarray(boards0, np.uint8).reshape(n, BOARD_STRIDE))
    t_off, t_plies, t_sides, t_lut = dev(offsets.astype(np.int32)), dev(flat), dev(side_arr), dev(lut)
    boards = torch.zeros((max(total, 1), BOARD_STRIDE), dtype=torch.uint8, device=device)
    labels = torch.full((max(total, 1),), -1, dtype=torch.int16, device=device)
    game = torch.zeros((max(n, 1), GAME_FIELDS), dtype=torch.int32, device=device)
    if stream is None:
        stream = C.c_void_p(torch.cuda.current_stream(device).cuda_stream) if lib.is_cuda else C.c_void_p(0)
    lib.call("cz_sl_replay", _ptr(t_init), _ptr(t_off), _ptr(t_plies), _ptr(t_sides), n, mode, _ptr(t_lut), _ptr(boards),
             _ptr(labels), _ptr(game), stream)
    return Replay(boards[:total], labels[:total], t_sides, game[:n].cpu().numpy(), offsets)


def onegreen_draw_value(ans, tot, red_to_move):
    """static_env.evaluate :100-115 (np.tanh(ans / tot * 3) in float64) and the sign flip of sl_onegreen.py:160-162."""
    v = np.tanh(float(ans) / int(tot) * 3)
    return v if red_to_move else -v


def record_order(labels, sides, o0, o1):
    """load_game :164-174: the red and black lists (plies with a label), interleaved up to len(red_moves)."""
    red = [o for o in range(o0, o1) if sides[o] > 0 and labels[o] >= 0]
    black = [o for o in range(o0, o1) if sides[o] < 0 and labels[o] >= 0]
    out = []
    for i in range(len(red)):
        out.append(red[i])
        if i < len(black):
            out.append(black[i])
    return out


class SlDataset:
    """boards u8 [N][96], labels i16 [N], values f32 [N] on one device, and optionally ply i16 [N]: the position's ply in
    its game (saturating at 32767), for datasets whose games are stored in consecutive rows (self-play records,
    records.replay_play_games); it lets `batch` build the 28 history planes.  104 bytes per position with it.
    visits: optional CSR columns (offsets i64 [N+1], labels [pairs] int16 holding the u16 labels, counts [pairs] int32
    holding the u32 counts) of records with root visit counts: `batch` then builds the visit-count targets
    (cz_visit_targets).  8 bytes per position plus 6 per pair."""

    def __init__(self, boards, labels, values, ply=None, visits=None):
        self.boards, self.labels, self.values, self.ply, self.visits = boards, labels, values, ply, visits

    def __len__(self):
        return int(self.boards.shape[0])

    @staticmethod
    def empty(device, with_ply=False):
        return SlDataset(torch.zeros((0, BOARD_STRIDE), dtype=torch.uint8, device=device),
                         torch.zeros(0, dtype=torch.int16, device=device), torch.zeros(0, dtype=torch.float32, device=device),
                         torch.zeros(0, dtype=torch.int16, device=device) if with_ply else None)

    def extend(self, other):
        if other is None or not len(other):
            return self
        if (self.ply is None) != (other.ply is None):
            raise ValueError("cannot join a dataset with a ply column and one without")
        if (self.visits is None) != (other.visits is None):
            raise ValueError("cannot join a dataset with visit columns and one without")
        visits = None
        if self.visits is not None:
            (o0, l0, n0), (o1, l1, n1) = self.visits, other.visits
            visits = (torch.cat([o0, o1[1:] + o0[-1]]), torch.cat([l0, l1]), torch.cat([n0, n1]))
        return SlDataset(torch.cat([self.boards, other.boards]), torch.cat([self.labels, other.labels]),
                         torch.cat([self.values, other.values]),
                         None if self.ply is None else torch.cat([self.ply, other.ply]), visits)

    def batch(self, env, idx, history=False, mirror=None):
        """Training tensors of samples idx (host int array): boards gathered on the device, planes by
        cz_env_encode_planes, the one-hot policy scattered into a zeroed [B][2086] tensor.  history=True: 28 planes,
        planes 14-27 of a sample those of row idx - 2 (the same game's position two plies earlier) where its ply is >= 2,
        zero otherwise (an empty board encodes to zero planes) — records.expanding_data(..., use_history=True).
        mirror: optional host array of per-sample flags; a flagged sample is reflected across the central file (its
        board and history board by cz_env_mirror, its policy target's columns permuted by env.mirror_labels), its value
        kept."""
        ids = torch.from_numpy(np.ascontiguousarray(idx, np.int64)).to(self.boards.device)
        flags = None if mirror is None else torch.from_numpy(np.ascontiguousarray(mirror, np.uint8)).to(self.boards.device)
        boards = self.boards.index_select(0, ids)
        if history:
            if self.ply is None:
                raise ValueError("28-plane batches need the dataset's ply column")
            earlier = self.boards.index_select(0, (ids - 2).clamp_min(0))
            earlier = torch.where((self.ply.index_select(0, ids) >= 2).unsqueeze(1), earlier, torch.zeros_like(earlier))
            both = torch.cat([boards, earlier])
            if flags is not None:
                both = env.mirror(both, torch.cat([flags, flags]))
            both = env.planes_batch(both)
            planes = torch.cat([both[:len(ids)], both[len(ids):]], dim=1)
        else:
            planes = env.planes_batch(boards.contiguous() if flags is None else env.mirror(boards, flags))
        if self.visits is not None:
            policy = self.visit_targets(env.lib, ids)
        else:
            policy = torch.zeros((len(ids), N_LABELS), dtype=torch.float32, device=self.boards.device)
            policy.scatter_(1, self.labels.index_select(0, ids).long().unsqueeze(1), 1.0)
        if flags is not None:
            policy = env.mirror_policy(policy, flags)
        return planes, policy, self.values.index_select(0, ids)

    def visit_targets(self, lib, ids):
        """cz_visit_targets for the rows ids (int64 device tensor): [B][2086] f32, one-hot where a row has no pairs."""
        off, lab, n = self.visits
        out = torch.empty((len(ids), N_LABELS), dtype=torch.float32, device=self.boards.device)
        stream = C.c_void_p(torch.cuda.current_stream(out.device).cuda_stream) if lib.is_cuda else C.c_void_p(0)
        lib.call("cz_visit_targets", _ptr(off), _ptr(lab), _ptr(n), _ptr(self.labels), _ptr(ids.contiguous()), len(ids),
                 _ptr(out), stream)
        return out


def build_dataset(rep, red_wins):
    """The records load_game appends, in order, with value red_win x side as float32 (np.asarray(value_list, float32)).
    red_wins: one float64 (or int) per game; games whose status is FAILED contribute nothing."""
    labels = rep.labels.cpu().numpy()
    sides = rep.sides.cpu().numpy()
    idx, vals = [], []
    for g in range(len(rep.game)):
        if rep.game[g, 1] != OK:
            continue
        order = record_order(labels, sides, int(rep.offsets[g]), int(rep.offsets[g + 1]))
        idx += order
        vals += [red_wins[g] * int(sides[o]) for o in order]
    dev = rep.boards.device
    ids = torch.as_tensor(np.asarray(idx, np.int64), device=dev)
    return SlDataset(rep.boards.index_select(0, ids).contiguous(), rep.labels.index_select(0, ids).contiguous(),
                     torch.as_tensor(np.asarray(vals, np.float64).astype(np.float32), device=dev))


def replay_wxf_games(lib, device, games):
    """games: list of (red rows, black rows, winner) -> (Replay or None, red_win per game, list of packed indices, skipped).
    A game whose rows make the reference raise before any move is replayed is skipped (counted)."""
    packed, wins, keep, skipped = [], [], [], 0
    for k, (red, black, winner) in enumerate(games):
        try:
            packed.append(pack_wxf_game(red, black))
        except RecordError:
            skipped += 1
            continue
        wins.append(wxf_red_win(winner))
        keep.append(k)
    if not packed:
        return None, wins, keep, skipped
    b0 = np.stack([start_board()] * len(packed))
    rep = replay(lib, device, b0, [p for p, _ in packed], [s for _, s in packed], WXF)
    return rep, wins, keep, skipped


def replay_onegreen_games(lib, device, games):
    """games: onegreen.json entries -> (Replay or None, red_win per replayed game, kept indices, skipped)."""
    boards, plies, sides, keep, skipped = [], [], [], [], 0
    for k, g in enumerate(games):
        try:
            b = onegreen_board(g['init'])
        except RecordError:
            skipped += 1
            continue
        p, s = pack_onegreen_game(g['move_list'])
        boards.append(b); plies.append(p); sides.append(s); keep.append(k)
    if not plies:
        return None, [], keep, skipped
    rep = replay(lib, device, np.stack(boards), plies, sides, ONEGREEN)
    wins = []
    for j, k in enumerate(keep):
        w = onegreen_winner(games[k])
        if w == 0 and rep.game[j, 1] == OK:
            ans, tot, red = int(rep.game[j, 3]), int(rep.game[j, 4]), bool(rep.game[j, 5])
            if tot == 0:                              # evaluate divides by zero: the reference raises
                rep.game[j, 1] = FAILED
                wins.append(0.0)
                continue
            w = onegreen_draw_value(ans, tot, red)
        wins.append(w)
    return rep, wins, keep, skipped
