"""Drive the REAL reference CChessPlayer (agent/player.py, unmodified) with a deterministic fake network
over a real multiprocessing.Pipe (SURVEY.md Appendix B).  Build-container only (needs /root/reference)."""
import threading
from collections import deque
from multiprocessing import Pipe

import numpy as np

from . import ref_import
from .player import fake_eval_from_planes


class FifoLock:
    """Mutual exclusion that hands the lock to the longest waiter on release."""

    def __init__(self):
        self._guard = threading.Lock()
        self._waiters = deque()
        self._held = False

    def __enter__(self):
        with self._guard:
            if not self._held:
                self._held = True
                return self
            turn = threading.Lock()
            turn.acquire()
            self._waiters.append(turn)
        turn.acquire()                     # released by the holder's __exit__: the lock is now ours
        return self

    def __exit__(self, *exc):
        with self._guard:
            if self._waiters:
                self._waiters.popleft().release()
            else:
                self._held = False


def fair_queue_lock(player):
    """Give a real player a first-come-first-served prediction-queue lock (call it while the player is idle).

    The player's sender thread holds `q_lock` through its 1 ms sleep whenever the queue is empty and takes it again
    right after releasing it (agent/player.py:113-123).  threading.Lock is not fair: on a multi-core machine the sender
    takes it back before the woken search thread that wants to queue a leaf (expand_and_evaluate) runs, so a
    60-simulation search can take tens of seconds.  With search_threads = 1 the simulations run one after another
    whatever the timing, so the search itself is unchanged; a threaded player, whose schedule does depend on timing,
    keeps its own lock."""
    if player.config.play.search_threads == 1 and not isinstance(player.q_lock, FifoLock):
        player.q_lock = FifoLock()


class FakeNetServer:
    def __init__(self):
        self.me, self.you = Pipe()
        self.stop = False
        self.positions = 0
        self.thread = threading.Thread(target=self._run, daemon=True)
        self.thread.start()

    def _run(self):
        while not self.stop:
            if self.me.poll(0.001):
                try:
                    planes = self.me.recv()
                except EOFError:
                    return
                self.positions += len(planes)
                self.me.send([fake_eval_from_planes(p) for p in planes])

    def close(self):
        self.stop = True


def make_config(sims, search_threads=1, **over):
    cfg = ref_import.config("mini")
    pc = cfg.play
    pc.simulation_num_per_move = sims
    pc.search_threads = search_threads
    for k, v in over.items():
        setattr(pc, k, v)
    return cfg


def real_player_moves(states_and_opts, sims, seed, search_threads=1, use_history=False, **over):
    """Run action() of ONE real player object over a list of (state, turns, no_act, increase_temp[, hist]);
    returns per call: (action, {move: (n, w, q, p)}, sum_n)."""
    pm = ref_import.player_module()
    cfg = make_config(sims, search_threads, **over)
    srv = FakeNetServer()
    np.random.seed(seed)
    player = pm.CChessPlayer(cfg, pipes=srv.you, enable_resign=False, use_history=use_history)
    fair_queue_lock(player)
    out = []
    try:
        for call in states_and_opts:
            state, turns, no_act, inc = call[:4]
            hist = list(call[4]) if len(call) > 4 and call[4] is not None else None
            action, policy = player.action(state, turns, no_act, increase_temp=inc, hist=hist)
            node = player.tree[state]
            edges = {m: (int(a.n), float(a.w), float(a.q), float(a.p)) for m, a in node.a.items()}
            out.append((action, edges, int(node.sum_n)))
    finally:
        player.close(wait=False)
        srv.close()
    return out
