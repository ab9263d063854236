"""Play records and host staging.

Record format of the reference (worker/self_play.py:202-208 -> lib/data_helper.py:17-19): one JSON list per game,
`[init_state, [move, value], [move, -value], ...]` with `value` the result from red's view for the first entry and
alternating sign after it; moves are the 4-digit strings in the mover's own frame.

Engines created with record_visits also keep the search's visit counts, the policy calc_policy builds (agent/player.py:
375-406) that the reference's self_play.py:112,134 left commented out.  Such a ply is written `[move, value, [l0, n0, l1,
n1, ...]]`: a flat list of ints, the root's edges with n > 0 in ascending label order, labels indexing ActionLabelsRed in
the mover's frame (the index space of the policy vector `action()` returns).  A ply without visits (the appended final
king capture, or any ply of an older file) stays `[move, value]`.  Every reader that takes only item[0] and item[1], the
reference's expanding_data included, reads both forms.
"""
import ctypes as C
import json
import os
from datetime import datetime, timedelta, timezone

import numpy as np
import torch

from .env import INIT_STATE, state_to_board
from .lib import BOARD_STRIDE, MAX_MOVES

CZ_PLAY_OK, CZ_PLAY_FAILED = 0, 1          # cz_play_replay's per-game status


def record_to_play_data(rec, init_state=INIT_STATE):
    """cz_drain_records entry -> the list self_play.py:202-208 builds; a ply with recorded visits gets its flat
    [l0, n0, l1, n1, ...] list as a third element."""
    data = [init_state]
    value = rec["value_red"]
    visits = rec.get("visits")
    for i, m in enumerate(rec["moves"]):
        pairs = visits[i] if visits is not None else None
        data.append([m, value, [int(x) for p in pairs for x in p]] if pairs else [m, value])
        value = -value
    return data


def split_visit_pairs(per_ply, n_plies, pairs):
    """Drained visit data -> per record, per ply, the list of (label, n) tuples.  per_ply u8 [n][>= plies] pairs per ply,
    pairs u32 [P][2] concatenated in record and ply order."""
    out, at = [], 0
    flat = pairs.tolist()
    for i, t in enumerate(n_plies):
        rec = []
        for c in per_ply[i, :t].tolist():
            rec.append([tuple(x) for x in flat[at:at + c]])
            at += c
        out.append(rec)
    return out


def write_play_data(play_data_dir, data, filename_tmpl="play_%s.json"):
    """save_play_data (self_play.py:214-227): Beijing-time stamped file, json.dump of the buffer."""
    os.makedirs(play_data_dir, exist_ok=True)
    bj = datetime.now(timezone.utc).astimezone(timezone(timedelta(hours=8)))
    path = os.path.join(play_data_dir, filename_tmpl % bj.strftime("%Y%m%d-%H%M%S.%f"))
    with open(path, "wt") as f:
        json.dump(data, f)
    return path


def init_boards_pinned(n_games):
    b = torch.from_numpy(np.tile(state_to_board(INIT_STATE), (n_games, 1)))
    return b.pin_memory() if torch.cuda.is_available() else b


class RootStage:
    """Pinned host buffers for the per-step host<->device traffic of the end-to-end path."""

    def __init__(self, engine):
        g = engine.n_games
        pin = engine.lib.is_cuda and torch.cuda.is_available()

        def mk(shape, dtype):
            t = torch.zeros(shape, dtype=dtype)
            return t.pin_memory() if pin else t
        self.boards = mk((g, BOARD_STRIDE), torch.uint8)
        self.n = mk((g, MAX_MOVES), torch.int32)
        self.moves = mk((g, MAX_MOVES), torch.int16)
        self.counts = mk((g,), torch.int32)
        self.sims = mk((g,), torch.int32)
        self.d2h_bytes_acc = 0

    @property
    def h2d_bytes(self):
        return self.boards.numel()

    @property
    def d2h_bytes(self):
        return self.boards.numel() + self.n.numel() * 4 + self.moves.numel() * 2 + self.counts.numel() * 4 + self.sims.numel() * 4


def decode_ring(ring_u8, count, layout):
    """A record ring as the collective delivered it (uint8 tensor / array) -> the dicts `Engine.drain_records` returns."""
    from .env import u16_to_move
    cap, stride, moves_off, _ = layout
    raw = ring_u8.cpu().numpy() if hasattr(ring_u8, "cpu") else np.asarray(ring_u8)
    count = min(int(count), cap)
    hdr = raw[:cap * 16].view(np.int32).reshape(cap, 4)
    moves = raw[moves_off:moves_off + cap * stride * 2].view(np.uint16).reshape(cap, stride)
    out = []
    for i in range(count):
        n_plies, value_red, game_index, flags = (int(x) for x in hdr[i])
        out.append({"n_plies": n_plies, "value_red": value_red, "game_index": game_index, "flags": flags,
                    "moves": [u16_to_move(int(v)) for v in moves[i, :n_plies]]})
    return out


def decode_visits(block_u8, recs, stride, layout):
    """A visit block as the collective delivered it (cz_record_visits_layout; at least its used prefix) -> sets "visits"
    on the ring's records `recs` (decode_ring's dicts, in ring order), as Engine.drain_records returns them.  stride =
    cz_record_layout out[1]."""
    offs_off, cnt_off, heap_off, _ = layout
    raw = block_u8.cpu().numpy() if hasattr(block_u8, "cpu") else np.asarray(block_u8)
    n = len(recs)
    offs = raw[offs_off:offs_off + 8 * n].view(np.int64)
    per = raw[cnt_off:cnt_off + n * stride].reshape(n, stride) if n else np.zeros((0, stride), np.uint8)
    heap = raw[heap_off:len(raw) - (len(raw) - heap_off) % 8].view(np.uint32).reshape(-1, 2)
    for i, rec in enumerate(recs):
        t = rec["n_plies"]
        c = per[i, :t]
        o = int(offs[i])
        rec["visits"] = split_visit_pairs(c.reshape(1, -1), [t], heap[o:o + int(c.sum())])[0]
    return recs


def record_layout(engine):
    import ctypes as C
    a = np.zeros(4, dtype=np.int64)
    engine.lib.call("cz_record_layout", engine._h, C.c_void_p(a.ctypes.data))
    return tuple(int(x) for x in a)


def gather_records(engine, dist, world, decode_on=0, clear=True, warm=False):
    """all_gather (NCCL on GPUs, gloo in the CPU tests) of the finished-game record ring of every rank — SURVEY.md §8e:
    the only inter-GPU traffic of the path, the analogue of the reference uploading its play-data files
    (worker/self_play.py:228-241).  The ring lives inside the engine's workspace tensor, so the collective reads it in
    place; every rank must call this at the same point of its loop.  Returns (records, total): on rank `decode_on` the
    decoded records of ALL ranks as [(rank, record dict), ...] (None elsewhere: other ranks only forward), and the
    number of records gathered.  clear=True empties the local ring afterwards (its content now lives on rank decode_on).
    warm=True: also run the ring collective when no rank has a record yet (first call of a long run, bench warm-up)."""
    import ctypes as C
    ptr, nbytes, ready = C.c_void_p(0), C.c_uint64(0), C.c_int32(0)
    engine.lib.call("cz_record_buffer", engine._h, C.byref(ptr), C.byref(nbytes), C.byref(ready))
    off = ptr.value - engine.workspace.data_ptr()
    ring = engine.workspace[off:off + nbytes.value]
    count = torch.tensor([ready.value], device=engine.device, dtype=torch.int32)
    counts = [torch.zeros_like(count) for _ in range(world)]
    dist.all_gather(counts, count)
    counts = [int(c.item()) for c in counts]
    total = sum(counts)
    records = None
    if warm and total == 0:                     # warm-up call: run the ring collective once so that its one-off set-up (NCCL picks
        dist.all_gather([torch.empty_like(ring) for _ in range(world)], ring)   # channels per message size) is not paid later
    if total > 0:                               # same decision on every rank (they all hold the same counts)
        rings = [torch.empty_like(ring) for _ in range(world)]
        dist.all_gather(rings, ring)
        blocks = gather_visits(engine, dist, world) if engine.record_visits else None
        if dist.get_rank() == decode_on:
            layout = record_layout(engine)
            per_rank = [decode_ring(rings[r], counts[r], layout) for r in range(world)]
            if blocks is not None:
                vl = engine.visits_layout()
                for r in range(world):
                    decode_visits(blocks[r], per_rank[r], layout[1], vl)
            records = [(r, rec) for r in range(world) for rec in per_rank[r]]
    elif dist.get_rank() == decode_on:
        records = []
    if clear:
        engine.lib.call("cz_clear_records", engine._h)
    return records, total


def gather_visits(engine, dist, world):
    """all_gather of the visit blocks beside the rings (record_visits engines): the ranks first exchange the used length
    of their block, then ship max(used) bytes each, the prefix that holds every pair of their ring, never the worst-case
    heap.  Returns the gathered uint8 tensors (engine.visits_gathered_bytes = the bytes shipped per rank)."""
    import ctypes as C
    ptr, used = C.c_void_p(0), C.c_uint64(0)
    engine.lib.call("cz_record_visits_buffer", engine._h, C.byref(ptr), C.byref(used))
    off = ptr.value - engine.workspace.data_ptr()
    n = torch.tensor([used.value], device=engine.device, dtype=torch.int64)
    ns = [torch.zeros_like(n) for _ in range(world)]
    dist.all_gather(ns, n)
    m = max(int(x.item()) for x in ns)
    block = engine.workspace[off:off + m]
    blocks = [torch.empty_like(block) for _ in range(world)]
    dist.all_gather(blocks, block)
    engine.visits_gathered_bytes = m
    return blocks


# ---- trainer-side view of the records (worker/optimize.py:223-292, lib/data_helper.py:11-24) -------------------
def get_game_data_filenames(rc):
    from glob import glob
    return sorted(glob(os.path.join(rc.play_data_dir, rc.play_data_filename_tmpl % "*")))


def read_game_data_from_file(path):
    with open(path, "rt") as f:
        return json.load(f)


def split_games(data):
    """A play-data file's list -> its games: a file holds nb_game_in_file games back to back, [state, moves..., state,
    moves...], and every state string after the first item starts a new one."""
    games = [[]]
    for item in data:
        if isinstance(item, str) and games[-1]:
            games.append([])
        games[-1].append(item)
    return games


def _move_ok(m):
    return isinstance(m, str) and len(m) == 4 and all(c in "0123456789" for c in m) and m[0] != "9" and m[2] != "9"


def move_codes(moves, source=""):
    """Moves "x0y0x1y1" (mover's frame) -> uint16 (from << 8) | to with squares y*9+x, in one numpy pass.  A move that is
    not four ASCII digits or names a square off the board (x = 9) raises ValueError naming `source` and the move."""
    if not len(moves):
        return np.zeros(0, np.uint16)
    try:
        a = np.asarray(moves)
        ok = a.ndim == 1 and a.dtype == np.dtype("<U4") and bool((np.char.str_len(a) == 4).all())
        d = a.astype("S4").view(np.uint8).reshape(-1, 4).astype(np.int32) - 48 if ok else None
    except (ValueError, TypeError, UnicodeEncodeError):
        ok = False
    if ok:
        ok = bool(((d >= 0) & (d <= 9)).all() and (d[:, 0] <= 8).all() and (d[:, 2] <= 8).all())
    if not ok:
        bad = next(m for m in moves if not _move_ok(m))
        raise ValueError(f"{source}: move {bad!r} is not four digits x0y0x1y1 naming two squares of the board")
    return (((d[:, 1] * 9 + d[:, 0]) << 8) | (d[:, 3] * 9 + d[:, 2])).astype(np.uint16)


class PlayGames:
    """Games of play-data records packed for cz_play_replay: start boards u8 [n][96], plies per game, move codes u16 [P],
    values f32 [P]; optionally `visits` = (pairs per ply i64 [P], labels u16, counts u32) from pack_visits."""

    def __init__(self, boards, counts, codes, values, visits=None):
        self.boards, self.counts, self.codes, self.values, self.visits = boards, counts, codes, values, visits

    def __len__(self):
        return len(self.codes)

    @staticmethod
    def concat(parts):
        cols = (np.concatenate([getattr(p, k) for p in parts]) for k in ("boards", "counts", "codes", "values"))
        visits = None
        if all(p.visits is not None for p in parts):
            visits = tuple(np.concatenate([p.visits[i] for p in parts]) for i in range(3))
        return PlayGames(*cols, visits=visits)


def pack_visits(items, source=""):
    """The visits of plies `[move, value(, [l0, n0, ...])]` in one numpy pass -> (pairs per ply i64 [P], labels u16,
    counts u32) in file order.  A ply without a third element has no pairs.  Raises ValueError naming `source` and the
    move for a third element that is not a flat list of ints of even length, a label outside [0, 2086), n <= 0 (or
    beyond u32), or a label twice in one ply."""
    from itertools import chain
    from .lib import N_LABELS
    lists = [it[2] if len(it) > 2 else [] for it in items]

    def bad(k, why):
        raise ValueError(f"{source}: visits of move {items[k][0]!r} (ply {k} of the file) {why}")

    for k, v in enumerate(lists):
        if not isinstance(v, list) or len(v) % 2:
            bad(k, "are not a flat list of (label, n) ints of even length")
    n_pairs = np.fromiter((len(v) // 2 for v in lists), np.int64, len(lists))
    flat = list(chain.from_iterable(lists))
    if not set(map(type, flat)) <= {int}:
        k = next(k for k, v in enumerate(lists) if any(type(x) is not int for x in v))
        bad(k, "are not a flat list of (label, n) ints of even length")
    ply = np.repeat(np.arange(len(lists)), n_pairs)
    try:
        a = np.asarray(flat, np.int64).reshape(-1, 2)
    except OverflowError:
        k = next(k for k, v in enumerate(lists) if any(abs(x) >= 2 ** 63 for x in v))
        bad(k, "hold an n outside (0, 2^32)")
    lab, n = a[:, 0], a[:, 1]
    out = np.flatnonzero((lab < 0) | (lab >= N_LABELS))
    if len(out):
        bad(int(ply[out[0]]), f"name label {int(lab[out[0]])}, outside [0, {N_LABELS})")
    out = np.flatnonzero((n <= 0) | (n >= 2 ** 32))
    if len(out):
        bad(int(ply[out[0]]), f"give label {int(lab[out[0]])} n = {int(n[out[0]])}, outside (0, 2^32)")
    key = np.sort(ply * N_LABELS + lab)
    dup = np.flatnonzero(key[1:] == key[:-1])
    if len(dup):
        k = int(key[dup[0]] // N_LABELS)
        bad(k, f"name label {int(key[dup[0]] % N_LABELS)} twice")
    return n_pairs, lab.astype(np.uint16), n.astype(np.uint32)


def pack_play_games(games, source="", visits=False):
    """Games `[init_state, [move, value], ...]` with at least one move -> PlayGames: state_to_board once per game, the
    moves in one numpy pass (move_codes) and the values as np.asarray(..., float32), as expanding_data rounds them;
    visits=True also packs every ply's visits (pack_visits).  Raises ValueError, naming `source`, for a game that does
    not start with a state or a malformed move or visits list."""
    from itertools import chain
    from operator import itemgetter
    if any(not isinstance(g[0], str) for g in games):
        raise ValueError(f"{source}: a game does not start with a state string")
    boards = np.stack([state_to_board(g[0]) for g in games])
    counts = np.array([len(g) - 1 for g in games], np.int64)
    items = list(chain.from_iterable(g[1:] for g in games))
    codes = move_codes(list(map(itemgetter(0), items)), source)
    values = np.asarray(list(map(itemgetter(1), items)), dtype=np.float32)
    return PlayGames(boards, counts, codes, values, pack_visits(items, source) if visits else None)


def load_play_file(filename, visits=False):
    """optimize.load_data_from_file without the expansion: read, split, drop games without moves, pack (with every
    ply's visits when asked).  An unreadable file is deleted (optimize.py:223-232); None when the file holds no game
    with a move."""
    import logging
    try:
        data = read_game_data_from_file(filename)
    except Exception as e:
        logging.getLogger(__name__).error(f"Error when loading data {e}")
        os.remove(filename)
        return None
    if data is None:
        return None
    games = [g for g in split_games(data) if len(g) > 1]
    return pack_play_games(games, filename, visits) if games else None


def check_labels(games, lut):
    """expanding_data's label check on PlayGames, on the host: the first move without an action label raises its
    ValueError.  OptimizeWorker runs it on every file as it loads, so a bad file stops the load where the host path
    stops it."""
    from .env import u16_to_move
    codes = games.codes.astype(np.int64)
    bad = np.flatnonzero(np.asarray(lut)[(codes >> 8) * 90 + (codes & 0xFF)] < 0)
    if len(bad):
        raise ValueError(f"move {u16_to_move(int(games.codes[bad[0]]))} is not an action label")


def play_replay(lib, device, games, lut, stream=None):
    """One cz_play_replay launch over PlayGames -> (boards u8 [P][96], labels i16 [P] on `device`, status np.int32 [n],
    offsets np.int64 [n + 1])."""
    device = torch.device(device)
    n, total = len(games.counts), len(games.codes)
    offsets = np.zeros(n + 1, np.int64)
    np.cumsum(games.counts, out=offsets[1:])

    def dev(a):
        return torch.from_numpy(np.ascontiguousarray(a)).to(device)

    t_init, t_off = dev(games.boards.astype(np.uint8)), dev(offsets.astype(np.int32))
    t_moves, t_lut = dev(games.codes.view(np.int16)), dev(np.asarray(lut, np.int16))
    boards = torch.zeros((max(total, 1), BOARD_STRIDE), dtype=torch.uint8, device=device)
    labels = torch.full((max(total, 1),), -1, dtype=torch.int16, device=device)
    status = torch.zeros(max(n, 1), dtype=torch.int32, device=device)
    if stream is None:
        stream = C.c_void_p(torch.cuda.current_stream(device).cuda_stream) if lib.is_cuda else C.c_void_p(0)
    ptr = [C.c_void_p(t.data_ptr()) for t in (t_init, t_off, t_moves, t_lut, boards, labels, status)]
    lib.call("cz_play_replay", *ptr[:3], n, *ptr[3:], stream)
    return boards[:total], labels[:total], status[:n].cpu().numpy(), offsets


def replay_play_games(lib, device, games, lut, stream=None):
    """PlayGames -> sl_data.SlDataset with the ply column, in one cz_play_replay launch: per ply the mover-relative board
    before the move, its label, the record's value and the ply's index in its game.  A game with a move that has no
    label raises expanding_data's ValueError (the first such game, and its first such move)."""
    from .env import u16_to_move
    from .sl_data import SlDataset
    boards, labels, status, offsets = play_replay(lib, device, games, lut, stream)
    failed = np.flatnonzero(status != CZ_PLAY_OK)
    if len(failed):
        g = int(failed[0])
        o = int(offsets[g]) + int(np.flatnonzero(labels[offsets[g]:offsets[g + 1]].cpu().numpy() < 0)[0])
        raise ValueError(f"move {u16_to_move(int(games.codes[o]))} is not an action label")
    ply = np.arange(len(games), dtype=np.int64) - np.repeat(offsets[:-1], games.counts)
    device = boards.device
    visits = None
    if games.visits is not None:
        n_pairs, lab, n = games.visits
        voff = np.zeros(len(n_pairs) + 1, np.int64)
        np.cumsum(n_pairs, out=voff[1:])
        visits = (torch.from_numpy(voff).to(device), torch.from_numpy(lab.view(np.int16)).to(device),
                  torch.from_numpy(n.view(np.int32)).to(device))
    return SlDataset(boards, labels, torch.from_numpy(games.values).to(device),
                     torch.from_numpy(np.minimum(ply, 32767).astype(np.int16)).to(device), visits)


def expanding_data(data, env, use_history=False, policy_target="move", source=""):
    """expanding_data + convert_to_trainging_data (optimize.py:234-281): one play record
    `[init_state, [move, value], ...]` -> (planes f32 [T,14,10,9], one-hot policy f32 [T,2086], value f32 [T]).
    use_history: planes f32 [T,28,10,9], planes 14-27 of sample i = the position of sample i-2 (history[0:2i+1][-5],
    optimize.py:264-267), zero for the first two.  The positions are replayed and encoded by the rules kernels
    (`env` is a StaticEnv).  policy_target="visits": a ply with recorded visits gets target[l] = float32(n / sum n),
    the sum and division in float64 (calc_policy's `policy /= np.sum(policy)`, player.py:403); a ply without keeps the
    one-hot of its move.  Malformed visits raise pack_visits' ValueError before any kernel runs."""
    from .env import move_to_u16
    if policy_target not in ("move", "visits"):
        raise ValueError(f"policy_target must be 'move' or 'visits', not {policy_target!r}")
    visits = pack_visits(data[1:], source) if policy_target == "visits" else None
    moves = [item[0] for item in data[1:]]
    values = np.asarray([item[1] for item in data[1:]], dtype=np.float32)
    t = len(moves)
    boards = env.boards_from_states([data[0]])
    seq = [boards]
    for m in moves[:-1]:
        boards, _ = env.step_batch(boards, env.moves_tensor([m]))
        seq.append(boards)
    if t == 0:
        return (np.zeros((0, 28 if use_history else 14, 10, 9), np.float32), np.zeros((0, len(env.labels)), np.float32), values)
    planes = env.planes_batch(torch.cat(seq, dim=0)).cpu().numpy()
    if use_history:
        hist = np.zeros_like(planes)
        hist[2:] = planes[:-2]
        planes = np.concatenate([planes, hist], axis=1)
    policy = np.zeros((t, len(env.labels)), dtype=np.float32)
    lut = env.label_lut
    for i, m in enumerate(moves):
        v = move_to_u16(m)
        lab = int(lut[(v >> 8) * 90 + (v & 0xFF)])
        if lab < 0:
            raise ValueError(f"move {m} is not an action label")
        policy[i, lab] = 1
    if visits is not None:
        n_pairs, vlab, vn = visits
        off = np.concatenate([[0], np.cumsum(n_pairs)])
        for i in np.flatnonzero(n_pairs):
            n = vn[off[i]:off[i + 1]].astype(np.float64)
            policy[i] = 0
            policy[i, vlab[off[i]:off[i + 1]]] = (n / np.sum(n)).astype(np.float32)
    return planes, policy, values


def flip_policy(pol, env):
    """lookup_tables.py:134-141: re-index a 2086-vector from black's move labels to red's
    (out[i] = pol[index of flip_move(label_i)])."""
    from .env import flip_move
    if not hasattr(env, "_unflipped_index"):
        lookup = {m: i for i, m in enumerate(env.labels)}
        env._unflipped_index = np.asarray([lookup[flip_move(m)] for m in env.labels])
    return np.asarray(pol)[env._unflipped_index]


def build_policy(action, flip, env):
    """optimize.py:283-292 / self_play.py:253-262: one-hot over the action labels, optionally seen from the other side."""
    policy = np.zeros(len(env.labels))
    policy[env.labels.index(action)] = 1
    if flip:
        policy = flip_policy(policy, env)
    return list(policy)
