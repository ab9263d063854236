"""`worker.self_play` drop-in (reference: cchess_alphazero/worker/self_play.py:48-232).

`start(config)` and `SelfPlayWorker(config, pipes, pid, use_history).start() / .start_game(idx, search_tree)` keep the
reference names, arguments and return values.  Where the reference runs `max_processes` OS processes with one game
each, all talking to one prediction thread, this worker holds `config.play.max_processes x games_per_process`
concurrent games in ONE engine on the GPU: the whole per-ply loop of start_game (search, move choice, adjudication,
record) runs in the kernels behind `cz_selfplay` and the host only writes the play-data files
(`data/play_data/play_<Beijing time>.json`, self_play.py:214-227) with the reference's record layout.
"""
import os
from logging import getLogger
from time import time

from .engine import Engine
from .lib import get_lib
from .model import CChessModel, engine_net_kwargs
from .records import record_to_play_data, write_play_data
from .env import INIT_STATE, StaticEnv

logger = getLogger(__name__)


def load_model(config):
    """self_play.py:29-46: load the best model or build + save a fresh one."""
    model = CChessModel(config)
    rc = config.resource
    cfg_path, w_path = rc.model_best_config_path, rc.model_best_weight_path
    if not (os.path.exists(cfg_path) and os.path.exists(w_path) and model.load(cfg_path, w_path)):
        model.build()
        os.makedirs(os.path.dirname(w_path), exist_ok=True)
        model.save(cfg_path, w_path)
    return model, model.use_history


def start(config, games_per_process=128, max_games=None, flush_plies=8, lib=None, device=None, evaluate_planes=None,
          record_visits=False, eval_mirror=False):
    """self_play.py:48-60.  The reference fans out over `max_processes` OS processes that share one prediction thread;
    here one process drives one GPU, and data parallelism is one process per GPU under `torchrun` (RANK / LOCAL_RANK /
    WORLD_SIZE in the environment): rank r plays its own `max_processes x games_per_process` concurrent games on GPU
    LOCAL_RANK with its own Philox sub-stream (engine rank r) — no data-path collective.  Every `flush_plies` plies the
    ranks all_gather their finished-game rings (NCCL over NVLink; gloo on CPU) and rank 0 decodes them and writes the
    reference's play-data files (worker/self_play.py:202-232): the other ranks never touch the disk.
    record_visits=True also writes every ply's root visit counts into the files (records.py), the target of
    optimize's policy_target="visits".  eval_mirror=True averages the network over every leaf and its left-right mirror.
    Returns the number of games stored by this launch (rank 0; the others return the same total)."""
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    model, use_history = load_model(config) if rank == 0 or world == 1 else (None, None)
    if world == 1:
        worker = SelfPlayWorker(config, pipes=None, pid=0, use_history=use_history, model=model, lib=lib, device=device,
                                concurrent_games=config.play.max_processes * games_per_process, record_visits=record_visits,
                                eval_mirror=eval_mirror)
        return worker.start(max_games=max_games)
    import torch
    import torch.distributed as dist
    on_gpu = device is None and torch.cuda.is_available()
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if on_gpu:
        torch.cuda.set_device(local)
        device = f"cuda:{local}"
    created = not dist.is_initialized()
    if created:
        dist.init_process_group("nccl" if on_gpu else "gloo", **({"device_id": torch.device(device)} if on_gpu else {}))
    try:
        if rank != 0:                                      # rank 0 built / loaded the model (and wrote it): the others read it after
            dist.barrier()
            model, use_history = load_model(config)
        else:
            dist.barrier()
        worker = SelfPlayWorker(config, pipes=None, pid=rank, use_history=use_history, model=model, lib=lib, device=device,
                                concurrent_games=config.play.max_processes * games_per_process, rank=rank,
                                external_evaluator=evaluate_planes is not None, record_visits=record_visits,
                                eval_mirror=eval_mirror)
        return worker.start_distributed(dist, world, max_games=max_games, flush_plies=flush_plies, evaluate_planes=evaluate_planes)
    finally:
        if created:
            dist.destroy_process_group()


class SelfPlayWorker:
    def __init__(self, config, pipes=None, pid=None, use_history=False, model=None, concurrent_games=None, lib=None,
                 device=None, seed=0, rank=0, external_evaluator=False, engine_kwargs=None, record_visits=False,
                 eval_mirror=False):
        self.config = config
        self.cur_pipes = pipes          # unused: evaluation happens inside the engine
        self.id = pid
        self.pid = os.getpid()
        self.buffer = []
        self.use_history = use_history
        self.lib = lib or get_lib()
        pc, mc = config.play, config.model
        self.model = model
        if self.model is None and not external_evaluator:
            self.model, _ = load_model(config)
        g = concurrent_games or max(1, pc.max_processes)
        self.engine = Engine(
            self.lib, device, n_games=g, sims_per_move=pc.simulation_num_per_move, leaves_per_round=pc.search_threads,
            virtual_loss=pc.virtual_loss, noise_mode=1, c_puct=pc.c_puct, noise_eps=pc.noise_eps,
            dirichlet_alpha=pc.dirichlet_alpha, tau_decay_rate=pc.tau_decay_rate, resign_threshold=pc.resign_threshold,
            enable_resign_rate=pc.enable_resign_rate, min_resign_turn=pc.min_resign_turn, max_game_length=pc.max_game_length,
            **dict(dict(max_nodes_per_game=max(4096, 24 * pc.simulation_num_per_move),
                        seed=seed, rank=rank, **({} if external_evaluator else engine_net_kwargs(mc)),
                        use_history=use_history,    # the game loop never passes `hist` (self_play.py:124): path history only
                        record_visits=record_visits, eval_mirror=eval_mirror),
                   **(engine_kwargs or {})))
        if not external_evaluator:      # external evaluator: the leaves go to a caller-supplied function (CPU test tier)
            self.engine.set_weights(self.model.torch_weights())
        self.engine.reset()
        self.pending = []               # finished games not yet handed out by start_game
        self.games_written = 0          # play-data files written
        self.games_stored = 0           # games handed to save_play_data (its idx, self_play.py:199)
        self.env = None

    # ---- self_play.py:72-93
    def start(self, max_games=None):
        idx = 1
        while max_games is None or idx <= max_games:
            t0 = time()
            value, turns, state, store = self.start_game(idx, None)
            logger.debug(f"Process {self.pid}-{self.id} play game {idx} time={(time() - t0):.1f} sec, "
                         f"turn={turns / 2}, winner = {value:.2f} (1 = red, -1 = black, 0 draw)")
            if store:
                idx += 1
        return idx - 1

    def start_distributed(self, dist, world, max_games=None, flush_plies=8, evaluate_planes=None):
        """One rank of the data-parallel launch: play `flush_plies` plies, gather every rank's finished-game ring, rank 0
        stores the games (running file index over all ranks).  All ranks leave the loop together: the stop test only uses
        the gathered totals.  evaluate_planes: external evaluator (CPU tests with the emulator build); None = built-in net."""
        from .records import gather_records
        stored = 0
        self.gather_ms = 0.0
        while max_games is None or stored < max_games:
            if evaluate_planes is None:
                self.engine.selfplay(target_games=0, max_moves=flush_plies)
            else:
                for _ in range(flush_plies):
                    self.engine.search_external(evaluate_planes, None)
                    self.engine.play_move()
            t0 = time()
            recs, total = gather_records(self.engine, dist, world)
            self.gather_ms += 1e3 * (time() - t0)
            n_stored = 0
            if recs is not None:                           # rank 0: decode + write (self_play.py:202-227)
                for r, rec in recs:
                    if not (rec["flags"] & 4):
                        self.games_stored += 1
                        n_stored += 1
                        self.save_play_data(self.games_stored, record_to_play_data(rec))
            # every rank needs the stored count for the common stop test: it is a function of the gathered records'
            # flags, which only rank 0 decoded -> broadcast one integer
            import torch
            t = torch.tensor([n_stored], dtype=torch.int64, device=self.engine.device)
            dist.broadcast(t, src=0)
            stored += int(t.item())
        return stored

    # ---- self_play.py:95-212: returns (v, turns, state, store) of the next finished game
    def start_game(self, idx, search_tree):
        while not self.pending:
            self.engine.selfplay(target_games=1, max_moves=0)
            self.pending.extend(self.engine.drain_records())
        rec = self.pending.pop(0)
        store = not (rec["flags"] & 4)
        if store:
            self.save_play_data(idx, record_to_play_data(rec))
        state = self._final_state(rec["moves"])
        return rec["value_red"], rec["n_plies"], state, store

    def play_games(self, n):
        """Batch entry point: run until n games finished, write their files, return the records."""
        out = list(self.pending)
        self.pending = []
        while len(out) < n:
            self.engine.selfplay(target_games=n - len(out), max_moves=0)
            out.extend(self.engine.drain_records())
        for rec in out:
            if not (rec["flags"] & 4):
                self.games_stored += 1
                self.save_play_data(self.games_stored, record_to_play_data(rec))
        return out

    def host_step(self, stage):
        """One ply of every game with the HOST holding the positions, the way a loop around `CChessPlayer.action(state, ..)`
        drives the reference (worker/self_play.py:122-147): this ply's root positions go up from pinned host memory, the
        search runs, every root's visit counts (calc_policy's input, the training target) come back, the moves are played,
        finished games are drained and stored as play-data files (self_play.py:202-227), and the new positions are read back
        for the next ply.  `stage` is a records.RootStage (pinned buffers).  Returns (simulations run, finished records)."""
        eng = self.engine
        eng.upload_roots(stage.boards)                     # H2D: the inputs of this step
        eng.search(None)
        eng.download_root_stats(stage)                     # D2H: N(s, a) of every root + simulations run
        sims = int(stage.sims.numpy()[eng.active_flags() != 0].sum())
        recs = []
        if eng.play_move():
            recs = eng.drain_records()                     # D2H: finished games
            for rec in recs:
                if not (rec["flags"] & 4):
                    self.games_stored += 1
                    self.save_play_data(self.games_stored, record_to_play_data(rec))
        eng.download_roots(stage)                          # D2H: the positions the host holds for the next ply
        return sims, recs

    # ---- self_play.py:214-227
    def save_play_data(self, idx, data):
        self.buffer += data
        if not idx % self.config.play_data.nb_game_in_file == 0:
            return
        rc = self.config.resource
        path = write_play_data(rc.play_data_dir, self.buffer, rc.play_data_filename_tmpl)
        logger.info(f"Process {self.pid} save play data to {path}")
        self.buffer = []
        self.games_written += 1

    def _final_state(self, moves):
        if self.env is None:
            self.env = StaticEnv(self.lib, self.engine.device)
        boards = self.env.boards_from_states([INIT_STATE])
        for m in moves:
            boards, _ = self.env.step_batch(boards, self.env.moves_tensor([m]))
        from .env import board_to_state
        return board_to_state(boards[0].cpu().numpy())

    def close(self):
        self.engine.close()
