"""Drive the REAL reference game loops — worker/self_play.py SelfPlayWorker.start_game and worker/evaluator.py
EvaluateWorker.start_game, unmodified — with the deterministic fake network behind real Pipes.  Build-container only.

The two worker modules import Keras / TensorFlow at module level (agent/model.py, lib/tf_util.py); neither is installed
and neither is needed by start_game, so their imports are satisfied by empty stand-in modules (`install_shims`).  With
search_threads = 1, `random.seed` and `np.random.seed` a whole game is reproducible; `ReferenceDraws` lets the
restated loops (oracle/selfplay.py, oracle/arena.py) take their random decisions from the same two generators in the
same order, so they must replay the real games move for move.
"""
import importlib.abc
import importlib.machinery
import os
import random
import sys
import types
from collections import defaultdict

import numpy as np

from . import ref_import
from .ref_player_harness import FakeNetServer, fair_queue_lock, make_config


class _Anything:
    def __init__(self, *a, **k):
        pass

    def __call__(self, *a, **k):
        return _Anything()

    def __getattr__(self, name):
        return _Anything()


class _ShimModule(types.ModuleType):
    def __getattr__(self, name):
        if name.startswith("__"):
            raise AttributeError(name)
        return _Anything


class _ShimFinder(importlib.abc.MetaPathFinder, importlib.abc.Loader):
    ROOTS = ("keras", "tensorflow")

    def find_spec(self, fullname, path, target=None):
        if fullname.split(".")[0] in self.ROOTS:
            return importlib.machinery.ModuleSpec(fullname, self, is_package=True)
        return None

    def create_module(self, spec):
        m = _ShimModule(spec.name)
        m.__path__ = []
        return m

    def exec_module(self, module):
        pass


_installed = False


def install_shims():
    global _installed
    if not _installed:
        sys.meta_path.insert(0, _ShimFinder())
        _installed = True


def worker_modules():
    ref_import.setup()
    install_shims()
    import cchess_alphazero.worker.self_play as sp
    import cchess_alphazero.worker.evaluator as ev
    return sp, ev


class ReferenceDraws:
    """The random decisions of a game taken exactly like the reference takes them: `random()` of the random module for
    the lotteries (self_play.py:102,194), `np.random.choice` over the 2086 labels for the move (player.py:195)."""

    def resign_lottery(self):
        return random.random()

    def store_lottery(self):
        return random.random()

    def playouts(self, lo, hi):
        return random.randint(lo, hi) * 100              # evaluator.py:12,153: `from random import randint`

    def choose_with_player(self, player, state, turns, no_act, increase_temp):
        player.increase_temp = increase_temp
        policy, _ = player.calc_policy(state, turns, no_act)
        if no_act is not None:
            for act in no_act:
                policy[player.move_lookup[act]] = 0
        k = int(np.random.choice(range(len(player.labels)), p=player.apply_temperature(policy, turns)))
        return player.labels[k]


def _config(sims, **play):
    cfg = make_config(sims, 1)
    for k, v in play.items():
        setattr(cfg.play, k, v)
    cfg.internet.distributed = False
    os.makedirs(cfg.resource.play_data_dir, exist_ok=True)
    return cfg


def real_selfplay_game(seed, sims, use_history=False, player_factory=None, **play):
    """One SelfPlayWorker.start_game.  Returns dict(moves, value_red, turns, store, final_state, increase_temp_used).
    player_factory: class / callable put in place of the module's `CChessPlayer` name (the import swap of
    INTEGRATION.md §3) - the reference's own loop then drives that player."""
    sp, _ = worker_modules()
    pm = ref_import.player_module()
    cfg = _config(sims, **play)
    srv = FakeNetServer()
    worker = sp.SelfPlayWorker(cfg, pipes=[srv.you], pid=0, use_history=use_history)
    saved, temps = [], []
    worker.save_play_data = lambda idx, data: saved.append(data)
    worker.remove_play_data = lambda: None
    orig_action = pm.CChessPlayer.action

    def spy(self, state, turns, no_act=None, depth=None, infinite=False, hist=None, increase_temp=False):
        fair_queue_lock(self)
        temps.append(bool(increase_temp))
        return orig_action(self, state, turns, no_act, depth, infinite, hist, increase_temp)
    pm.CChessPlayer.action = spy
    sp_player = sp.CChessPlayer
    if player_factory is not None:
        sp.CChessPlayer = player_factory
    random.seed(seed)
    np.random.seed(seed)
    try:
        v, turns, state, store = worker.start_game(1, defaultdict(pm.VisitState))
    finally:
        pm.CChessPlayer.action = orig_action
        sp.CChessPlayer = sp_player
        srv.close()
    moves = [m for m, _ in saved[0][1:]] if saved else None
    return {"moves": moves, "value_red": v, "turns": turns, "store": bool(store), "final_state": state,
            "increase_temp_used": any(temps)}


def real_arena_game(seed, idx, sims, player_factory=None, **play):
    """One EvaluateWorker.start_game (two players, separate trees; both served by the fake network).
    sims = None: the game runs exactly as written — `playouts = randint(8, 12) * 100` (evaluator.py:153-154) drawn from the
    seeded `random` module decides the simulations per move; the drawn value is returned as "playouts".
    sims = <int>: TEST-SPEED DEVICE for the long rule-coverage games only — the per-game draw still happens but the players
    are made to search `sims` simulations (800-1200 simulations x 100 plies of pure-Python search would take minutes per
    game); such games are flagged "playouts_patched" in the fixture."""
    _, ev = worker_modules()
    pm = ref_import.player_module()
    cfg = _config(sims or 0, **play)
    s1, s2 = FakeNetServer(), FakeNetServer()
    worker = ev.EvaluateWorker(cfg, pipes1=[s1.you], pipes2=[s2.you], pid=0)
    moves, temps = [], []
    orig_action = pm.CChessPlayer.action

    def spy(self, state, turns, no_act=None, depth=None, infinite=False, hist=None, increase_temp=False):
        fair_queue_lock(self)
        if sims is not None:
            self.play_config.simulation_num_per_move = sims
        temps.append(bool(increase_temp))
        a, p = orig_action(self, state, turns, no_act, depth, infinite, hist, increase_temp)
        moves.append(a)
        return a, p
    pm.CChessPlayer.action = spy
    ev_player = ev.CChessPlayer
    if player_factory is not None:
        class Recording:                                 # same bookkeeping as the spy, around the swapped-in player
            def __init__(self, *a, **k):
                if sims is not None:                     # (the real player reads it per call; a swapped-in one at creation)
                    cfg.play.simulation_num_per_move = sims
                self.p = player_factory(*a, **k)

            def action(self, state, turns, no_act=None, increase_temp=False):
                temps.append(bool(increase_temp))
                a, pol = self.p.action(state, turns, no_act=no_act, increase_temp=increase_temp)
                moves.append(a)
                return a, pol

            def close(self, wait=True):
                self.p.close()
        ev.CChessPlayer = Recording
    random.seed(seed)
    np.random.seed(seed)
    try:
        value, turns = worker.start_game(idx)
    finally:
        pm.CChessPlayer.action = orig_action
        ev.CChessPlayer = ev_player
        s1.close()
        s2.close()
    return {"moves": moves, "value_red": value, "turns": turns, "increase_temp_used": any(temps),
            "playouts": cfg.play.simulation_num_per_move if sims is None else None}
