"""Python handle on a `cz_engine` (include/cczero_b200.h): many concurrent games, GPU-resident trees.

PyTorch is only the allocator / stream provider here: the workspace is one uint8 CUDA tensor handed to
the library, everything else happens in the kernels behind the C-ABI.
"""
import ctypes as C

import numpy as np
import torch

from .env import move_to_u16, state_to_board, u16_to_move
from .lib import (BOARD_STRIDE, MAX_MOVES, MAX_NO_ACT, N_LABELS, CzConfig, CzPvInfo, CzRecordHdr, CzRootInfo, CzRootOpts,
                  get_lib)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


class Engine:
    def __init__(self, lib=None, device=None, n_games=1, sims_per_move=800, leaves_per_round=8, virtual_loss=3,
                 max_nodes_per_game=None, max_edges_per_game=None, max_path=128, noise_mode=1, max_game_length=100,
                 nn_filters=0, nn_blocks=0, nn_value_fc=256, c_puct=1.5, noise_eps=0.15, dirichlet_alpha=0.2,
                 tau_decay_rate=0.9, resign_threshold=-0.98, enable_resign_rate=0.5, min_resign_turn=40, seed=0, rank=0, nn_fp32_skip=None, arena=False,
                 use_history=False, game_quota=0, playouts=None, nn_policy_channels=0, nn_value_channels=0,
                 record_visits=False, eval_mirror=False):
        self.lib = lib or get_lib()
        if device is None:
            device = 'cuda' if self.lib.is_cuda else 'cpu'
        self.device = torch.device(device)
        if self.lib.is_cuda and self.device.type != 'cuda':
            raise ValueError("the CUDA library needs a CUDA device")
        if self.device.type == 'cuda' and self.device.index is None:      # "cuda" = the process's current device (one rank per GPU)
            self.device = torch.device('cuda', torch.cuda.current_device())
        if max_nodes_per_game is None:
            max_nodes_per_game = max(64, 4 * sims_per_move + 64)
        if max_edges_per_game is None:
            max_edges_per_game = max_nodes_per_game * 48
        cfg = CzConfig()
        cfg.struct_bytes = C.sizeof(CzConfig)
        cfg.device = self.device.index or 0 if self.device.type == 'cuda' else 0
        cfg.n_games, cfg.sims_per_move, cfg.leaves_per_round = n_games, sims_per_move, leaves_per_round
        cfg.virtual_loss, cfg.max_nodes_per_game, cfg.max_edges_per_game = virtual_loss, max_nodes_per_game, max_edges_per_game
        cfg.max_path, cfg.noise_mode, cfg.max_plies = max_path, noise_mode, 2 * max_game_length
        cfg.nn_filters, cfg.nn_blocks, cfg.nn_value_fc = nn_filters, nn_blocks, nn_value_fc
        cfg.c_puct, cfg.noise_eps, cfg.dirichlet_alpha = c_puct, noise_eps, dirichlet_alpha
        cfg.tau_decay_rate, cfg.resign_threshold, cfg.enable_resign_rate = tau_decay_rate, resign_threshold, enable_resign_rate
        cfg.min_resign_turn, cfg.max_game_length = min_resign_turn, max_game_length
        cfg.seed, cfg.rank = seed, rank
        cfg.arena = 1 if arena else 0
        cfg.nn_fp32_skip = 0 if nn_fp32_skip is None else (1 if nn_fp32_skip else 2)   # None = auto (fp32 when blocks >= 10)
        cfg.use_history = 1 if use_history else 0
        cfg.game_quota = int(game_quota or 0)        # > 0: play exactly the games with running index < game_quota, then retire
        cfg.playouts_lo, cfg.playouts_hi = (playouts or (0, 0))   # arena: per-game randint(lo, hi) * 100 simulations per move
        # head widths of the weight file (0 = agent/model.py's 4 policy / 2 value channels; legacy configs: 2 or 32 / 4)
        cfg.nn_policy_channels, cfg.nn_value_channels = int(nn_policy_channels or 0), int(nn_value_channels or 0)
        cfg.record_visits = 1 if record_visits else 0   # every ply's root visit counts go with the records (drain_records)
        self.record_visits = bool(record_visits)
        # the built-in network evaluates every leaf and its left-right mirror and averages them (cz_config.eval_mirror)
        cfg.eval_mirror = 1 if eval_mirror else 0
        self.use_history = bool(use_history)
        self.in_planes = 28 if use_history else 14
        self.cfg = cfg
        nbytes = C.c_uint64(0)
        self.lib.call("cz_workspace_bytes", C.byref(cfg), C.byref(nbytes))
        self.workspace_bytes = nbytes.value
        self.workspace = torch.zeros(nbytes.value, dtype=torch.uint8, device=self.device)
        self._h = C.c_void_p(0)
        self.lib.call("cz_create", C.byref(cfg), _ptr(self.workspace), nbytes, self._stream(), C.byref(self._h))
        self.n_games = n_games
        self.K = leaves_per_round
        self._keep = []

    def _stream(self):
        if self.lib.is_cuda:
            return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)
        return C.c_void_p(0)

    def close(self):
        if self._h:
            self.lib.raw("cz_destroy")(self._h)
            self._h = C.c_void_p(0)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- games
    def reset(self, states=None):
        if states is None:
            self.lib.call("cz_reset_games", self._h, C.c_void_p(0))
            return
        assert len(states) == self.n_games
        b = np.ascontiguousarray(np.stack([state_to_board(s) for s in states]))
        self.lib.call("cz_reset_games", self._h, C.c_void_p(b.ctypes.data))

    def set_root(self, game, state):
        b = np.ascontiguousarray(state_to_board(state))
        self.lib.call("cz_set_root", self._h, game, C.c_void_p(b.ctypes.data))

    # ---- search
    def make_opts(self, no_act=None, increase_temp=None, active=None, noise=None, sims_override=0, hist=None, raw_tasks=False):
        """hist (use_history engines): per game the `hist` list given to action() ([.., state, move, state]) or None.
        raw_tasks: run exactly sims_override simulations (the caller did action()'s done / depth bookkeeping)."""
        o = CzRootOpts()
        o.struct_bytes = C.sizeof(CzRootOpts)
        keep = []
        if hist is not None and any(h for h in hist):
            hb = np.zeros((self.n_games, BOARD_STRIDE), dtype=np.uint8)
            given = np.zeros(self.n_games, dtype=np.uint8)
            for g, h in enumerate(hist):
                if h:
                    given[g] = 1
                    if len(h) >= 5:
                        hb[g] = state_to_board(h[-5])
            keep += [hb, given]
            o.root_hist_host = hb.ctypes.data
            o.root_hist_given_host = given.ctypes.data
        if no_act is not None:
            a = np.full((self.n_games, MAX_NO_ACT), 0xFFFF, dtype=np.uint16)
            for g, lst in enumerate(no_act):
                for k, m in enumerate(lst or []):
                    a[g, k] = move_to_u16(m)
            keep.append(a)
            o.no_act_host = a.ctypes.data
        if increase_temp is not None:
            a = np.ascontiguousarray(np.asarray(increase_temp, dtype=np.uint8))
            keep.append(a)
            o.increase_temp_host = a.ctypes.data
        if active is not None:
            a = np.ascontiguousarray(np.asarray(active, dtype=np.uint8))
            keep.append(a)
            o.active_host = a.ctypes.data
        if noise is not None:
            t = torch.as_tensor(np.ascontiguousarray(noise, dtype=np.float64)).to(self.device)
            assert t.dim() == 2 and t.shape[0] == self.n_games
            keep.append(t)
            o.noise_dev = t.data_ptr()
            o.noise_stride = t.shape[1]
        o.sims_override = sims_override
        o.raw_tasks = 1 if raw_tasks else 0
        self._keep = keep
        return o

    def search_begin(self, opts=None):
        self.lib.call("cz_search_begin", self._h, C.byref(opts) if opts is not None else None)

    def search_wave(self):
        n, busy = C.c_int32(0), C.c_int32(0)
        self.lib.call("cz_search_wave", self._h, C.byref(n), C.byref(busy))
        return n.value, bool(busy.value)

    def leaf_planes(self, n):
        planes = torch.empty((n, self.in_planes, 10, 9), dtype=torch.float32, device=self.device)
        self.lib.call("cz_leaf_planes", self._h, _ptr(planes))
        return planes

    def leaf_boards(self, n):
        b = torch.empty((n, self.in_planes // 14 * BOARD_STRIDE), dtype=torch.uint8, device=self.device)
        self.lib.call("cz_leaf_boards", self._h, _ptr(b))
        return b

    def search_apply(self, policy, value):
        assert policy.dtype == torch.float32 and value.dtype == torch.float32
        # hold the evaluation of the last few waves (the kernels read them stream-ordered; a long `go infinite` search
        # must not accumulate one tensor pair per wave)
        self._apply_keep = (getattr(self, "_apply_keep", []) + [(policy, value)])[-4:]
        self.lib.call("cz_search_apply", self._h, _ptr(policy), _ptr(value))

    def leaf_labels(self, n):
        """Action labels of the legal moves of the n leaves of the last wave (cz_leaf_labels): (int16 [n,128], int32 [n])."""
        lab = torch.full((n, MAX_MOVES), -1, dtype=torch.int16, device=self.device)
        cnt = torch.zeros((n,), dtype=torch.int32, device=self.device)
        self.lib.call("cz_leaf_labels", self._h, _ptr(lab), _ptr(cnt))
        return lab, cnt

    def search_apply_legal(self, legal_p, value):
        """cz_search_apply_legal: legal_p f32 [n,128] = policy[label] of every legal move (see leaf_labels)."""
        assert legal_p.dtype == torch.float32 and value.dtype == torch.float32 and legal_p.shape[1] == MAX_MOVES
        self._apply_keep = (getattr(self, "_apply_keep", []) + [(legal_p, value)])[-4:]
        self.lib.call("cz_search_apply_legal", self._h, _ptr(legal_p), _ptr(value))

    def search_external(self, evaluate_planes, opts=None):
        """Whole search with `evaluate_planes(np.float32[n,14,10,9]) -> (policy[n,2086] f32, value[n] f32)`
        standing in for the network (the role CChessModelAPI plays for the reference player)."""
        self.search_begin(opts)
        stats = {"waves": 0, "positions": 0}
        while True:
            n, busy = self.search_wave()
            stats["waves"] += 1
            if n > 0:
                planes = self.leaf_planes(n).cpu().numpy()
                pol, val = evaluate_planes(planes)
                self.search_apply(torch.as_tensor(np.ascontiguousarray(pol, dtype=np.float32)).to(self.device),
                                  torch.as_tensor(np.ascontiguousarray(val, dtype=np.float32)).to(self.device))
                stats["positions"] += n
            if not busy:
                break
        return stats

    def search_more(self, n_sims):
        """n_sims more simulations inside the search search_begin opened (cz_search_more); run the wave loop after it."""
        self.lib.call("cz_search_more", self._h, int(n_sims))

    def set_noise_table(self, noise):
        """Swap the Dirichlet table of the open search for a longer one (same leading draws)."""
        t = torch.as_tensor(np.ascontiguousarray(noise, dtype=np.float64)).to(self.device)
        assert t.dim() == 2 and t.shape[0] == self.n_games
        self._noise_keep = (getattr(self, "_noise_keep", []) + [t])[-2:]     # the previous table may still be read by a queued kernel
        self.lib.call("cz_set_noise_table", self._h, _ptr(t), t.shape[1])

    def run_waves(self, evaluate_planes=None, host_loop=False):
        """The wave / evaluate / apply loop until every queued simulation is done; evaluate_planes as in search_external,
        None = the built-in network: the engine's own device-driven loop (cz_search_run), or — host_loop=True — this Python
        loop around cz_nn_forward_boards (full softmax vectors; the parity tests compare the two)."""
        if evaluate_planes is None and self.lib.is_cuda and self.cfg.nn_filters > 0 and not host_loop:
            c0 = int(self.counters()[1])
            self.lib.call("cz_search_run", self._h)          # device-driven loop, no per-wave host round trip
            return int(self.counters()[1]) - c0
        n_pos = 0
        while True:
            n, busy = self.search_wave()
            if n > 0:
                if evaluate_planes is None:
                    pol, val = self.nn_forward_boards(self.leaf_boards(n))
                    self.search_apply(pol, val)
                else:
                    pol, val = evaluate_planes(self.leaf_planes(n).cpu().numpy())
                    self.search_apply(torch.as_tensor(np.ascontiguousarray(pol, dtype=np.float32)).to(self.device),
                                      torch.as_tensor(np.ascontiguousarray(val, dtype=np.float32)).to(self.device))
                n_pos += n
            if not busy:
                return n_pos

    def pv(self, game, max_len=20):
        """print_depth_info's line (player.py:408-450): (moves as canonical strings per mover, value or None)."""
        info = CzPvInfo()
        self.lib.call("cz_get_pv", self._h, game, max_len, C.byref(info))
        return [u16_to_move(info.moves[i]) for i in range(info.n_moves)], (float(info.value) if info.has_value else None)

    def search_stats(self):
        """cz_get_search_stats as a dict (totals since the engine was created)."""
        a = np.zeros(6, dtype=np.uint64)
        self.lib.call("cz_get_search_stats", self._h, C.c_void_p(a.ctypes.data))
        sims, depth, imm, created, edges, nodes = (int(x) for x in a)
        return {"sims": sims, "path_edges": depth, "no_network": imm, "nodes_created": created, "edges_stored": edges, "nodes_stored": nodes}

    def search(self, opts=None):
        """Whole search with the built-in tensor-core network."""
        self.lib.call("cz_search", self._h, C.byref(opts) if opts is not None else None)

    def root(self, game):
        info = CzRootInfo()
        self.lib.call("cz_get_root", self._h, game, C.byref(info))
        L = info.n_moves
        return {
            "moves": [u16_to_move(info.moves[i]) for i in range(L)],
            "n": [info.n[i] for i in range(L)], "w": [info.w[i] for i in range(L)], "p": [info.p[i] for i in range(L)],
            "sum_n": info.sum_n, "noise_used": info.noise_used, "sims_run": info.sims_run,
        }

    # ---- bulk host <-> device staging (pinned buffers owned by a records.RootStage)
    def upload_roots(self, boards_pinned):
        self.lib.call("cz_set_roots", self._h, C.c_void_p(boards_pinned.data_ptr()))

    def download_roots(self, stage):
        self.lib.call("cz_get_roots", self._h, C.c_void_p(stage.boards.data_ptr()))
        stage.d2h_bytes_acc += stage.boards.numel()
        return stage.boards

    def download_root_stats(self, stage):
        self.lib.call("cz_get_root_stats", self._h, C.c_void_p(stage.n.data_ptr()), C.c_void_p(stage.moves.data_ptr()),
                      C.c_void_p(stage.counts.data_ptr()), C.c_void_p(stage.sims.data_ptr()))
        return stage.n, stage.moves, stage.counts

    def sims_run(self):
        st = getattr(self, "_sims_stage", None)
        if st is None:
            from .records import RootStage
            st = self._sims_stage = RootStage(self)
        self.download_root_stats(st)
        return st.sims.numpy()

    def compact(self):
        self.lib.call("cz_compact", self._h)

    def counters(self):
        a = np.zeros(8, dtype=np.uint64)
        self.lib.call("cz_get_counters", self._h, C.c_void_p(a.ctypes.data))
        return a

    def launch_count(self):
        n = C.c_uint64(0)
        self.lib.call("cz_launch_count", self._h, C.byref(n))
        return n.value

    def nn_profile(self, enable=True):
        """(ms, launches, flops) of the residual-tower igemm launches since the last call."""
        ms, n, fl = C.c_double(0), C.c_uint64(0), C.c_double(0)
        self.lib.call("cz_nn_profile", self._h, int(enable), C.byref(ms), C.byref(n), C.byref(fl))
        return ms.value, n.value, fl.value

    # ---- on-device game loop
    def play_move(self):
        f = C.c_int32(0)
        self.lib.call("cz_play_move", self._h, C.byref(f))
        return f.value

    def selfplay(self, target_games=0, max_moves=0):
        g, s = C.c_int32(0), C.c_int64(0)
        self.lib.call("cz_selfplay", self._h, target_games, max_moves, C.byref(g), C.byref(s))
        return g.value, s.value

    def set_game_sims(self, sims):
        """Per-slot simulations per move of the games now running (0 = the engine default): the per-game
        `config.play.simulation_num_per_move` of evaluator.py:153-154."""
        a = np.ascontiguousarray(np.asarray(sims, dtype=np.int32))
        assert a.shape == (self.n_games,)
        self.lib.call("cz_set_game_sims", self._h, C.c_void_p(a.ctypes.data))

    def any_active(self):
        """False once every slot has retired (cz_config.game_quota reached)."""
        return bool(self.active_flags().any())

    def active_flags(self):
        a = np.zeros(self.n_games, dtype=np.int32)
        self.lib.call("cz_get_active", self._h, C.c_void_p(a.ctypes.data))
        return a

    def drain_records(self, cap=None):
        """Finished games: dicts n_plies, value_red, game_index, flags, moves.  A record_visits engine adds "visits": per
        ply the root's (label, n) pairs in ascending label order (labels index ActionLabelsRed, moves in the mover's
        frame), [] for an appended final king capture."""
        cap = cap or max(64, 2 * self.n_games)
        row = self.cfg.max_plies + 1
        hdr = (CzRecordHdr * cap)()
        moves = np.zeros((cap, row), dtype=np.uint16)
        n = C.c_int32(0)
        if self.record_visits:
            from .records import split_visit_pairs
            per_ply = np.zeros((cap, row), dtype=np.uint8)
            ptr, used = C.c_void_p(0), C.c_uint64(0)       # the drained pairs are at most those in the heap
            self.lib.call("cz_record_visits_buffer", self._h, C.byref(ptr), C.byref(used))
            pair_cap = (used.value - self.visits_layout()[2]) // 8
            pairs = np.zeros((pair_cap, 2), dtype=np.uint32)
            n_pairs = C.c_int64(0)
            self.lib.call("cz_drain_records_visits", self._h, C.cast(hdr, C.c_void_p), C.c_void_p(moves.ctypes.data),
                          C.c_void_p(per_ply.ctypes.data), C.c_void_p(pairs.ctypes.data), pair_cap, cap, C.byref(n),
                          C.byref(n_pairs))
            visits = split_visit_pairs(per_ply[:n.value], [hdr[i].n_plies for i in range(n.value)], pairs[:n_pairs.value])
        else:
            self.lib.call("cz_drain_records", self._h, C.cast(hdr, C.c_void_p), C.c_void_p(moves.ctypes.data), cap, C.byref(n))
        out = []
        for i in range(n.value):
            h = hdr[i]
            out.append({"n_plies": h.n_plies, "value_red": h.value_red, "game_index": h.game_index, "flags": h.flags,
                        "moves": [u16_to_move(v) for v in moves[i, :h.n_plies]]})
            if self.record_visits:
                out[-1]["visits"] = visits[i]
        return out

    def visits_layout(self):
        """cz_record_visits_layout: byte offsets of the per-record first pair, the per-ply pair counts and the pairs inside
        the visit block, and its size."""
        a = np.zeros(4, dtype=np.int64)
        self.lib.call("cz_record_visits_layout", self._h, C.c_void_p(a.ctypes.data))
        return tuple(int(x) for x in a)

    # ---- network
    def set_weights(self, named_tensors, net=0):
        """named_tensors: dict Keras-style name -> float32 tensor on self.device (Keras layouts).  net = 1 is the second
        (next-generation) network of an arena engine."""
        from .lib import CzTensorDesc
        arr = (CzTensorDesc * len(named_tensors))()
        keep = []
        for i, (k, t) in enumerate(named_tensors.items()):
            t = t.detach().to(self.device, torch.float32).contiguous()
            keep.append(t)
            arr[i].name = k.encode()
            arr[i].dev = t.data_ptr()
            arr[i].numel = t.numel()
        self._weights_keep = getattr(self, "_weights_keep", {})
        self._weights_keep[net] = keep
        self.lib.call("cz_nn_set_weights_net", self._h, net, arr, len(named_tensors))

    def nn_forward_planes(self, planes):
        n = planes.shape[0]
        pol = torch.empty((n, N_LABELS), dtype=torch.float32, device=self.device)
        val = torch.empty((n,), dtype=torch.float32, device=self.device)
        self.lib.call("cz_nn_forward", self._h, _ptr(planes), n, _ptr(pol), _ptr(val))
        return pol, val

    def nn_forward_boards(self, boards):
        n = boards.shape[0]
        pol = torch.empty((n, N_LABELS), dtype=torch.float32, device=self.device)
        val = torch.empty((n,), dtype=torch.float32, device=self.device)
        self.lib.call("cz_nn_forward_boards", self._h, _ptr(boards), n, _ptr(pol), _ptr(val))
        return pol, val
