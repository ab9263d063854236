"""`CChessPlayer` drop-in (reference: cchess_alphazero/agent/player.py:35-470) backed by the GPU engine.

Same constructor and `action()` signature and return values as the reference class.  The search
(MCTS_search / select / expand / update_tree, player.py:198-373) runs in the CUDA kernels behind
`cz_search_*`; this class only does what the reference does once per move on the host: the visit-count
policy, temperature and the `np.random.choice` draw (player.py:187-196,375-406,453-470), with numpy, so
that the global `np.random` stream is consumed exactly like the reference consumes it:

  * root Dirichlet noise: the reference draws `np.random.dirichlet(alpha*ones(L))[0]` once per legal
    move per root selection (player.py:304).  The player pre-draws that sequence from the current
    `np.random` state into a device table, lets the engine consume a prefix, then rewinds the generator
    and re-draws exactly the consumed prefix, leaving the stream where the reference would leave it.
  * evaluation: if `pipes` is given the leaves are sent through it with the reference wire protocol
    (list of float32[14,10,9] ([28,10,9] with use_history) -> list of (float32[2086], float), api.py:48-74), so the player works
    against an unmodified CChessModelAPI; otherwise the engine's built-in tensor-core network is used.
  * UCI mode (`uci=True`, uci.py:207-209): action() runs its rounds (player.py:167-184) in slices that end exactly
    where the reference prints an `info depth .. pv ..` line (`done_tasks // 100` changed), `infinite=True` searches
    until `close_and_return_action` is called from another thread (uci.py:229-243).
"""
import sys
import threading
from time import time

import numpy as np

from .engine import Engine
from .env import StaticEnv, flip_move, to_uci_move
from .lib import get_lib
from .model import engine_net_kwargs


class EdgeView:
    """ActionState as callers read it (player.py:28-33)."""
    __slots__ = ("n", "w", "q", "p")

    def __init__(self, n, w, p):
        self.n, self.w, self.p = n, w, p
        self.q = w / n if n else 0


class NodeView:
    """VisitState as callers read it (player.py:17-25): `a` maps move -> EdgeView in legal-move order."""

    def __init__(self, root):
        self.sum_n = root["sum_n"]
        self.legal_moves = list(root["moves"])
        self.a = {m: EdgeView(n, w, p) for m, n, w, p in zip(root["moves"], root["n"], root["w"], root["p"])} if root["sum_n"] > 1 else {}
        self.p = None
        self.waiting = False
        self.visit = []


class CChessPlayer:
    def __init__(self, config, search_tree=None, pipes=None, play_config=None, enable_resign=False, debugging=False,
                 uci=False, use_history=False, side=0, lib=None, device=None, weights=None, exact_noise=True,
                 infinite_capacity=200000, eval_mirror=False):
        """eval_mirror: the built-in network's evaluations average each leaf and its left-right mirror (Engine)."""
        self.use_history = use_history          # 28 input planes (static_env.py:158-194, player.py:326-334)
        self.config = config
        self.play_config = play_config or config.play
        self.lib = lib or get_lib()
        self.env = StaticEnv(self.lib, device)
        self.labels = self.env.labels
        self.labels_n = len(self.labels)
        self.move_lookup = {m: i for i, m in enumerate(self.labels)}
        self.pipe = pipes
        self.enable_resign = enable_resign
        self.debugging = debugging
        self.uci = uci
        self.side = side
        self.increase_temp = False
        self.no_act = None
        self.root_state = None
        # The tree lives in device memory.  `search_tree` is the caller's dict (uci.py:205-209 reads the node of the position
        # after the best move out of it for its ponder move): in UCI mode the root and its children are mirrored into it
        # after every action() (`_mirror_tree`); other callers only hand it back to the next player, which cz_set_root covers.
        self.tree = search_tree if search_tree is not None else {}
        self.debug = {}
        self.search_results = {}
        self.done_tasks = 0
        self.exact_noise = exact_noise
        self.info_stream = None            # where the `info depth` lines go (None = sys.stdout, like the reference's print)
        self.infinite_capacity = infinite_capacity      # simulations an `infinite` search may run (node pool size)
        self._stop = False
        self._busy = threading.Lock()      # held while a search slice runs: close_and_return_action waits for it
        pc = self.play_config
        mc = getattr(config, "model", None)
        use_nn = pipes is None
        self.engine = Engine(
            self.lib, self.env.device, n_games=1, sims_per_move=pc.simulation_num_per_move,
            leaves_per_round=config.play.search_threads, virtual_loss=config.play.virtual_loss,
            noise_mode=0 if exact_noise else 1, c_puct=pc.c_puct, noise_eps=pc.noise_eps,
            dirichlet_alpha=pc.dirichlet_alpha, tau_decay_rate=pc.tau_decay_rate,
            resign_threshold=getattr(pc, "resign_threshold", -1.0), min_resign_turn=getattr(pc, "min_resign_turn", 0),
            max_game_length=getattr(pc, "max_game_length", 100),
            max_nodes_per_game=max(4096, 8 * pc.simulation_num_per_move, (infinite_capacity + 64) if uci else 0),
            use_history=use_history, eval_mirror=eval_mirror, **(engine_net_kwargs(mc) if (use_nn and mc) else {}))
        if use_nn:
            if weights is None:
                raise ValueError("CChessPlayer without pipes needs `weights` (Keras-named tensors) for the built-in network")
            self.engine.set_weights(weights)
        self._fresh = True

    # ---- reference API
    def close(self, wait=True):
        self._stop = True
        with self._busy:
            if self.engine is not None:
                self.engine.close()
                self.engine = None

    def action(self, state, turns, no_act=None, depth=None, infinite=False, hist=None, increase_temp=False):
        pc = self.play_config
        eng = self.engine
        with self._busy:
            self._stop = False
            self.root_state = state
            self.no_act = no_act
            self.increase_temp = increase_temp
            if self._fresh:
                eng.reset([state])
                self._fresh = False
            else:
                eng.set_root(0, state)
            # task count: player.py:153-165
            done = eng.root(0)["sum_n"]
            if no_act or increase_temp or done == pc.simulation_num_per_move:
                done = 0
            self.done_tasks = done
            num_task = pc.simulation_num_per_move - done
            if depth:
                num_task = depth - done if depth > done else 0
            if infinite:
                num_task = min(100000, self.infinite_capacity)
            self._noise_begin(state, num_task)
        start_time = time()
        shown = 0
        k = self.config.play.search_threads
        left, first = num_task, True
        while left > 0 and not self._stop:
            with self._busy:
                if self._stop or self.engine is None:
                    break
                # the rounds up to the next `info depth` line (or all of them outside UCI mode)
                n = left
                if self.uci or infinite:
                    n, dt = 0, self.done_tasks
                    while n < left:
                        r = min(k, left - n)
                        n += r
                        dt += r
                        if dt // 100 != shown:
                            break
                self._noise_reserve(n, search_open=not first)
                if first:
                    opts = eng.make_opts(no_act=[list(no_act)] if no_act else None, increase_temp=[1 if increase_temp else 0],
                                         noise=self._noise_table, sims_override=n, raw_tasks=True,
                                         hist=[list(hist)] if (self.use_history and hist) else None)
                    eng.search_begin(opts)
                    first = False
                else:
                    eng.search_more(n)
                eng.run_waves(self._evaluate_through_pipe if self.pipe is not None else None)
                self.done_tasks += n
                left -= n
                if self.uci and shown != self.done_tasks // 100:      # player.py:180-184
                    shown = self.done_tasks // 100
                    self._remember_root_value(state)
                    self.print_depth_info(state, turns, start_time, self.debug[state][1], no_act)
        with self._busy:
            if self._stop or self.engine is None:                      # close_and_return_action answered already
                if self.engine is not None:
                    self._noise_end(eng.root(0)["noise_used"])
                return None, None
            if first:                                                  # nothing to search: still a valid (empty) search
                eng.search_begin(eng.make_opts(no_act=[list(no_act)] if no_act else None,
                                               increase_temp=[1 if increase_temp else 0], sims_override=0, raw_tasks=True))
            root = eng.root(0)
            self._noise_end(root["noise_used"])
            if self.debugging or self.uci:
                self._remember_root_value(state, root)
            if self.uci:
                self._mirror_tree(state, root)
            policy, resign = self.calc_policy(root, turns, no_act)
            if resign:
                return None, list(policy)
            if no_act is not None:
                for act in no_act:
                    policy[self.move_lookup[act]] = 0
            my_action = int(np.random.choice(range(self.labels_n), p=self.apply_temperature(policy, turns)))
            return self.labels[my_action], list(policy)

    # ---- root Dirichlet noise with the reference's np.random consumption (player.py:304)
    def _noise_begin(self, state, num_task):
        self._noise_table, self._rng_state, self._noise_rows, self._n_moves = None, None, 0, 0
        # the reference draws one Dirichlet sample per legal move per root selection even when noise_eps == 0 (:304)
        if self.exact_noise and num_task > 0:
            self._n_moves = max(len(self.env.get_legal_moves(state)), 1)
            self._rng_state = np.random.get_state()
            self._noise_table = np.zeros((1, 0))
            self._noise_sims = 0

    def _noise_reserve(self, n_sims, search_open):
        """Make sure the table holds the draws `n_sims` more simulations can consume (one draw per legal move per root
        selection; parked simulations select again).  `np.random.dirichlet(alpha, size=m)` draws the same stream as m calls."""
        if self._rng_state is None:
            return
        self._noise_sims += n_sims
        want = (self._noise_sims + 2 * self.engine.K + 2) * self._n_moves
        if want > self._noise_rows:
            more = max(want - self._noise_rows, 64 * self._n_moves, self._noise_rows)     # at least double: O(log) re-uploads
            alpha = self.play_config.dirichlet_alpha * np.ones(self._n_moves)
            new = np.concatenate([np.random.dirichlet(alpha, size=min(16384, more - i))[:, 0] for i in range(0, more, 16384)])
            self._noise_table = np.concatenate([self._noise_table, new[None, :]], axis=1)
            self._noise_rows += more
            if search_open:                                            # swap the table of the running search
                self.engine.set_noise_table(self._noise_table)

    def _noise_end(self, used):
        """Rewind np.random and draw exactly what the search consumed, leaving the stream where the reference leaves it."""
        if self._rng_state is not None:
            np.random.set_state(self._rng_state)
            alpha = self.play_config.dirichlet_alpha * np.ones(self._n_moves)
            while used > 0:                                            # in slices: a long search consumed millions of draws
                m = min(used, 16384)
                np.random.dirichlet(alpha, size=m)
                used -= m
            self._rng_state = None

    def _remember_root_value(self, state, root=None):
        """debug[state] = (p, v) (player.py:349-350) for the root: v = the network's value of the root position."""
        _, v = self.engine.pv(0, 0)
        self.debug[state] = ((root or self.engine.root(0))["p"], v if v is not None else 0)

    # ---- player.py:408-450
    def print_depth_info(self, state, turns, start_time, value, no_act):
        depth = self.done_tasks // 100
        end_time = time()
        moves, end_value = self.engine.pv(0, 20)
        pv = ""
        for mv in moves:
            if turns % 2 == 1:
                mv = flip_move(mv)
            pv += " " + to_uci_move(mv)
            turns += 1
        if end_value is not None:
            value = end_value
            if turns % 2 != self.side:
                value = -value
        score = int(value * 1000)
        duration = max(end_time - start_time, 1e-9)
        nps = int(depth * 100 / duration) * 1000
        output = f"info depth {depth} score {score} time {int(duration * 1000)} pv" + pv + f" nps {nps}"
        out = self.info_stream or sys.stdout
        print(output, file=out)
        out.flush()

    def close_and_return_action(self, state, turns, no_act=None):
        """player.py:88-106 (used by the UCI front end to stop an ongoing search): answer from the tree as it stands.
        A running action() finishes its current slice of rounds, then returns (None, None)."""
        self._stop = True
        with self._busy:
            root = self.engine.root(0)
            if (self.debugging or self.uci) and state not in self.debug and root["sum_n"] > 0:
                self._remember_root_value(state, root)
            if self.uci and root["sum_n"] > 0:
                self._mirror_tree(state, root)
            policy, resign = self.calc_policy(root, turns, no_act)
            if resign:
                return None
            if no_act is not None:
                for act in no_act:
                    policy[self.move_lookup[act]] = 0
            my_action = int(np.random.choice(range(self.labels_n), p=self.apply_temperature(policy, turns)))
            value = self.debug.get(state, (None, 0))[1]
            return self.labels[my_action], value, self.done_tasks // 100

    def _mirror_tree(self, state, root):
        """tree[state] and tree[child] for every expanded child of the root, as NodeView objects (call with _busy held)."""
        self.tree[state] = NodeView(root)
        for mov, n in zip(root["moves"], root["n"]):
            if n <= 0:
                continue
            child = self.env.step(state, mov)
            self.engine.set_root(0, child)
            r = self.engine.root(0)
            if r["sum_n"] > 0:
                self.tree[child] = NodeView(r)
        self.engine.set_root(0, state)

    def engine_child_stats(self, state):
        """[(move, N)] of `state`'s node, [] if it is not in the tree or was never selected through (what iterating
        `search_tree[state].a` yields in uci.py:303-311).  Moves the engine's root: only for a player that is done searching."""
        with self._busy:
            self.engine.set_root(0, state)
            r = self.engine.root(0)
            if r["sum_n"] < 2:
                return []
            return list(zip(r["moves"], r["n"]))

    # ---- host-side tail of action(): player.py:375-406
    def calc_policy(self, root, turns, no_act):
        policy = np.zeros(self.labels_n)
        max_q_value = -100
        for mov, n, w in zip(root["moves"], root["n"], root["w"]):
            policy[self.move_lookup[mov]] = n
            if no_act and mov in no_act:
                policy[self.move_lookup[mov]] = 0
                continue
            q = w / n if n != 0 else 0
            if q > max_q_value:
                max_q_value = q
        pc = self.play_config
        if max_q_value < getattr(pc, "resign_threshold", -1e9) and self.enable_resign and turns > getattr(pc, "min_resign_turn", 0):
            return policy, True
        if self.debugging:                               # player.py:397-403: the five most visited moves
            order = sorted(range(len(root["moves"])), key=lambda i: root["n"][i], reverse=True)[:5]
            for i in order:
                n, w = root["n"][i], root["w"][i]
                if not (no_act and root["moves"][i] in no_act):
                    self.search_results[root["moves"][i]] = (n, w / n if n else 0, root["p"][i])
        policy /= np.sum(policy)
        return policy, False

    # ---- player.py:453-470
    def apply_temperature(self, policy, turn):
        pc = self.play_config
        evaluate = bool(getattr(getattr(self.config, "opts", None), "evaluate", False))
        if turn < 30 and pc.tau_decay_rate != 0:
            tau = np.power(pc.tau_decay_rate, turn + 1)
        else:
            tau = 0
        if tau < 0.1 or (turn >= 4 and evaluate):
            tau = 0
        if self.increase_temp and not evaluate:
            tau = 0.5
        if tau == 0:
            ret = np.zeros(self.labels_n)
            ret[np.argmax(policy)] = 1.0
            return ret
        ret = np.power(policy, 1 / tau)
        ret /= np.sum(ret)
        return ret

    # ---- the reference wire protocol (player.py:118-120,131-140 <-> api.py:48-74)
    def _evaluate_through_pipe(self, planes):
        out_p, out_v = [], []
        for i in range(0, len(planes), 256):
            chunk = planes[i:i + 256]
            self.pipe.send([np.ascontiguousarray(p, dtype=np.float32) for p in chunk])
            rets = self.pipe.recv()
            for p, v in rets:
                out_p.append(np.asarray(p, dtype=np.float32))
                out_v.append(np.float32(v))
        return np.stack(out_p), np.asarray(out_v, dtype=np.float32)
