"""Host-side mirror of `cchess_alphazero.environment.static_env` backed by the CUDA rules kernels.

Same function names, argument meaning and return values as the reference module
(static_env.py: INIT_STATE :9, done :14, step :79, new_step :88, state_to_planes :137,
fliped_state :245, get_legal_moves :256, will_check_or_catch :390, be_catched :456,
has_attack_chessman :471), so reference callers and tests can swap `senv` for a `StaticEnv`.
Strings are only a codec here: every rule is evaluated by the kernels behind the C-ABI
(include/cczero_b200.h, cz_env_*).  The `*_batch` methods are the efficient entry points.
"""
import ctypes as C

import numpy as np
import torch

from .lib import BOARD_STRIDE, MAX_MOVES, N_LABELS, get_lib

INIT_STATE = 'rkemsmekr/9/1c5c1/p1p1p1p1p/9/9/P1P1P1P1P/1C5C1/9/RKEMSMEKR'

# state alphabet (light_env/common.py:32-64): k = knight, e = elephant, m = advisor, s = king;
# UPPER case = side to move.  Codes: 1..7 = P C R N E A K (plane order, lookup_tables.py:27-42).
_L2C = {'P': 1, 'C': 2, 'R': 3, 'K': 4, 'E': 5, 'M': 6, 'S': 7}
_L2C.update({k.lower(): v | 8 for k, v in list(_L2C.items())})
_C2L = {v: k for k, v in _L2C.items()}


def state_to_board(state):
    """Canonical state string -> uint8[BOARD_STRIDE] packed board (rows of the string run y=9..0)."""
    b = np.zeros(BOARD_STRIDE, dtype=np.uint8)
    y, x = 9, 0
    for ch in state:
        if ch == ' ':
            break
        if ch == '/':
            y -= 1
            x = 0
        elif '1' <= ch <= '9':
            x += ord(ch) - 48
        else:
            b[y * 9 + x] = _L2C[ch]
            x += 1
    return b


def board_to_state(b):
    rows = []
    for y in range(9, -1, -1):
        s, gap = [], 0
        for x in range(9):
            c = int(b[y * 9 + x])
            if c == 0:
                gap += 1
                continue
            if gap:
                s.append(str(gap))
                gap = 0
            s.append(_C2L[c])
        if gap:
            s.append(str(gap))
        rows.append(''.join(s))
    return '/'.join(rows)


def move_to_u16(m):
    return ((int(m[1]) * 9 + int(m[0])) << 8) | (int(m[3]) * 9 + int(m[2]))


def u16_to_move(v):
    f, t = int(v) >> 8, int(v) & 0xFF
    return '%d%d%d%d' % (f % 9, f // 9, t % 9, t // 9)


def flip_move(m):
    """lookup_tables.py:50-56."""
    return '%d%d%d%d' % (8 - int(m[0]), 9 - int(m[1]), 8 - int(m[2]), 9 - int(m[3]))


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


# ---- UCI / FEN notation (static_env.py:224-228,380-388)
_FEN_TO_STATE = str.maketrans("nNbBaAkK", "kKeEmMsS")      # FEN knight/bishop/advisor/king -> state letters k/e/m/s


def fen_to_state(fen):
    return fen.split(' ')[0].translate(_FEN_TO_STATE)


_STATE_TO_FEN = str.maketrans("kKeEmMsS", "nNbBaAkK")


def state_to_fen(state, turns):
    """static_env.py:215-243: FEN of the position; on black's turns (odd) the canonical state is turned back to the
    board's orientation (rows reversed, each row mirrored, colours swapped) and the side-to-move field becomes b."""
    fen = state.translate(_STATE_TO_FEN)
    if turns % 2 == 0:
        return f"{fen} w - - 0 {turns}"
    rows = ["".join(c.swapcase() for c in reversed(row)) for row in reversed(fen.split('/'))]
    return "/".join(rows) + f" b - - 0 {turns}"


def parse_ucci_move(move):
    return str(ord(move[0]) - ord('a')) + move[1] + str(ord(move[2]) - ord('a')) + move[3]


def to_uci_move(action):
    return chr(ord('a') + int(action[0])) + action[1] + chr(ord('a') + int(action[2])) + action[3]


class StaticEnv:
    """Rules engine bound to one library + device ('cuda' for the product)."""

    def __init__(self, lib=None, device=None):
        self.lib = lib or get_lib()
        if device is None:
            device = 'cuda' if self.lib.is_cuda else 'cpu'
        if self.lib.is_cuda and not str(device).startswith('cuda'):
            raise ValueError("the CUDA library needs CUDA tensors")
        self.device = torch.device(device)
        labels = C.create_string_buffer(N_LABELS * 4)
        lut = np.empty(8100, dtype=np.int16)
        self.lib.call("cz_action_labels", C.cast(labels, C.c_void_p), C.c_void_p(lut.ctypes.data))
        raw = labels.raw.decode()
        self.labels = [raw[i * 4:i * 4 + 4] for i in range(N_LABELS)]
        self.label_lut = lut
        self._mirror_labels = self._mirror_labels_dev = None
        self.INIT_STATE = INIT_STATE

    # ---- plumbing
    def _stream(self):
        if self.lib.is_cuda:
            return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        return C.c_void_p(0)

    def to_dev(self, arr):
        return torch.from_numpy(np.ascontiguousarray(arr)).to(self.device)

    def boards_from_states(self, states):
        return self.to_dev(np.stack([state_to_board(s) for s in states]))

    # ---- batch entry points (tensors in, tensors out, all on self.device)
    def movegen_batch(self, boards):
        n = boards.shape[0]
        moves = torch.empty((n, MAX_MOVES), dtype=torch.int16, device=self.device)
        counts = torch.empty((n,), dtype=torch.int32, device=self.device)
        self.lib.call("cz_env_movegen", _ptr(boards), n, _ptr(moves), _ptr(counts), self._stream())
        return moves, counts

    def done_batch(self, boards, need_check=False):
        n = boards.shape[0]
        out = torch.empty((n, 4), dtype=torch.int8, device=self.device)
        fm = torch.empty((n,), dtype=torch.int16, device=self.device)
        self.lib.call("cz_env_done", _ptr(boards), n, int(need_check), _ptr(out), _ptr(fm), self._stream())
        return out, fm

    def step_batch(self, boards, moves):
        n = boards.shape[0]
        out = torch.empty_like(boards)
        no_eat = torch.empty((n,), dtype=torch.uint8, device=self.device)
        self.lib.call("cz_env_step", _ptr(boards), _ptr(moves), n, _ptr(out), _ptr(no_eat), self._stream())
        return out, no_eat

    def planes_batch(self, boards):
        n = boards.shape[0]
        planes = torch.empty((n, 14, 10, 9), dtype=torch.float32, device=self.device)
        self.lib.call("cz_env_encode_planes", _ptr(boards), n, _ptr(planes), self._stream())
        return planes

    def check_catch_batch(self, boards, moves):
        n = boards.shape[0]
        wcc = torch.empty((n,), dtype=torch.uint8, device=self.device)
        bc = torch.empty((n,), dtype=torch.uint8, device=self.device)
        ha = torch.empty((n,), dtype=torch.uint8, device=self.device)
        self.lib.call("cz_env_check_catch", _ptr(boards), _ptr(moves), n, _ptr(wcc), _ptr(bc), _ptr(ha), self._stream())
        return wcc, bc, ha

    def keys_batch(self, boards):
        n = boards.shape[0]
        keys = torch.empty((n, 2), dtype=torch.int64, device=self.device)
        self.lib.call("cz_env_keys", _ptr(boards), n, _ptr(keys), self._stream())
        return keys

    @property
    def mirror_labels(self):
        """int16 [2086]: the label of each label's move reflected across the central file (cz_mirror_labels)."""
        if self._mirror_labels is None:
            m = np.empty(N_LABELS, dtype=np.int16)
            self.lib.call("cz_mirror_labels", C.c_void_p(m.ctypes.data))
            self._mirror_labels = m
        return self._mirror_labels

    def mirror(self, boards, flags=None):
        """Boards reflected across the central file (x -> 8 - x).  flags: optional uint8/bool [n] tensor on the device,
        rows with flag 0 come back unchanged."""
        n = boards.shape[0]
        out = torch.empty_like(boards)
        if flags is not None:
            flags = flags.to(torch.uint8).contiguous()
        self.lib.call("cz_env_mirror", _ptr(boards), _ptr(flags), n, _ptr(out), self._stream())
        return out

    def mirror_policy(self, policy, flags):
        """Policy rows [n][2086] of mirrored positions: row'[l] = row[M l] where flags (bool [n] tensor) is set."""
        if self._mirror_labels_dev is None:
            self._mirror_labels_dev = self.to_dev(self.mirror_labels.astype(np.int64))
        return torch.where(flags.bool().unsqueeze(1), policy.index_select(1, self._mirror_labels_dev), policy)

    def moves_tensor(self, moves):
        return self.to_dev(np.array([move_to_u16(m) for m in moves], dtype=np.uint16).view(np.int16))

    # ---- static_env-compatible single-position API
    def get_legal_moves(self, state, board=None):
        mv, cnt = self.movegen_batch(self.boards_from_states([state]))
        k = int(cnt[0])
        return [u16_to_move(v) for v in mv[0, :k].cpu().numpy().view(np.uint16)]

    def done(self, state, turns=-1, need_check=False):
        out, fm = self.done_batch(self.boards_from_states([state]), need_check)
        o = out[0].cpu().numpy()
        f = int(fm.cpu().numpy().view(np.uint16)[0])
        final = None if f == 0xFFFF else u16_to_move(f)
        if need_check and ('s' in state and 'S' in state):
            return (bool(o[0]), int(o[1]), final, bool(o[2]))
        return (bool(o[0]), int(o[1]), final)

    def step(self, state, action):
        b = state_to_board(state)
        if b[move_to_u16(action) >> 8] == 0:
            raise ValueError(f"No chessman in {action}, state = {state}")
        out, _ = self.step_batch(self.to_dev(b[None]), self.moves_tensor([action]))
        return board_to_state(out[0].cpu().numpy())

    def new_step(self, state, action):
        b = state_to_board(state)
        if b[move_to_u16(action) >> 8] == 0:
            raise ValueError(f"No chessman in {action}, state = {state}")
        out, ne = self.step_batch(self.to_dev(b[None]), self.moves_tensor([action]))
        return board_to_state(out[0].cpu().numpy()), bool(ne[0])

    def state_to_planes(self, state):
        return self.planes_batch(self.boards_from_states([state]))[0].cpu().numpy()

    def state_history_to_planes(self, state, history):
        """static_env.py:158-194: planes 0-13 = state, 14-27 = history[-5] when the list holds >= 5 entries, else zero."""
        states = [state] + ([history[-5]] if history and len(history) >= 5 else [])
        p = self.planes_batch(self.boards_from_states(states)).cpu().numpy()
        out = np.zeros((28, 10, 9), dtype=np.float32)
        out[:14] = p[0]
        if len(states) == 2:
            out[14:] = p[1]
        return out

    def fliped_state(self, state):
        b = state_to_board(state)[:90]
        f = np.where(b[::-1] != 0, b[::-1] ^ 8, 0).astype(np.uint8)
        return board_to_state(f)

    def will_check_or_catch(self, ori_state, action):
        wcc, _, _ = self.check_catch_batch(self.boards_from_states([ori_state]), self.moves_tensor([action]))
        return bool(wcc[0])

    def be_catched(self, state, mov):
        _, bc, _ = self.check_catch_batch(self.boards_from_states([state]), self.moves_tensor([mov]))
        return bool(bc[0])

    def has_attack_chessman(self, state):
        _, _, ha = self.check_catch_batch(self.boards_from_states([state]), self.moves_tensor(['0000']))
        return bool(ha[0])
