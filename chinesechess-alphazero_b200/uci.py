"""UCI / UCCI front end on top of the drop-in `CChessPlayer` (behaviour of the reference's cchess_alphazero/uci.py:40-331).

Wire behaviour kept from the reference:
  uci            -> id / option lines, `uciok`; loads the network                       (uci.py:71-88)
  ucinewgame     -> start position                                                       (uci.py:90-95)
  setoption name gpu|Threads value <x>                                                   (uci.py:97-110)
  isready        -> `readyok`                                                            (uci.py:112-116)
  position {fen <fen> w|b - - <half> <full> | startpos} [moves m1 m2 ...] , fen ...      (uci.py:118-174)
  go [depth d] [movetime|time ms] [wtime ms] [btime ms] [infinite]                      (uci.py:177-227)
                 -> `info depth .. score .. time .. pv .. nps ..` while thinking (printed by the player,
                    player.py:408-450), then `info depth .. score .. time .. nps ..` and
                    `bestmove <m> [ponder <m>]`                                          (uci.py:293-327)
  stop           -> answer from the tree as it stands                                    (uci.py:229-243)
  quit

What differs does not show on the wire: the search runs in one GPU engine instead of a thread pool, and by default the
leaves are evaluated by the built-in tensor-core network (`use_pipes=True` / `pipes_factory` go through a pipe like
uci.py:205).
"""
import sys
from dataclasses import dataclass
from threading import Thread, Timer
from time import time
from typing import Optional

from .env import INIT_STATE, StaticEnv, fen_to_state, flip_move, parse_ucci_move, to_uci_move
from .lib import get_lib
from .player import CChessPlayer

ID_LINES = ('id name CCZero', 'id author https://cczero.org', 'id version 2.4',
            'option name gpu spin default 0 min 0 max 7', 'option name Threads spin default 10 min 0 max 1024', 'uciok')


@dataclass
class GoLimits:
    """What a `go` line asks for (uci.py:198-221)."""
    depth: Optional[int] = None        # simulations = 100 x the UCI depth
    infinite: bool = True
    seconds: Optional[float] = None    # stop after this long

    @classmethod
    def parse(cls, words, red_to_move):
        lim = cls()
        for key, val in zip(words, words[1:] + [None]):
            if key == 'depth':
                lim.depth, lim.infinite = int(val) * 100, False
            elif key in ('movetime', 'time'):
                lim.seconds = int(val) / 1000
            elif key == 'infinite':
                lim.infinite = True
            elif (key == 'wtime' and red_to_move) or (key == 'btime' and not red_to_move):
                lim.seconds, lim.depth, lim.infinite = int(val) / 1000, 3000, False     # own clock: at most 3000 simulations
        return lim


class Position:
    """Board + game history in the reference's canonical form: `state` is seen by the side to move, `history` is
    [state, move, state, ...] with every move written from its mover's side (uci.py:118-169)."""

    def __init__(self, env):
        self.env = env
        self.reset()

    def reset(self):
        self.state, self.red_to_move, self.turns = INIT_STATE, True, 0
        self.history = [INIT_STATE]

    def set_fen(self, fen, side, fullmove):
        state = fen_to_state(fen)
        self.env.get_legal_moves(state)               # raises on garbage
        self.history = [state]
        self.red_to_move = side != 'b'
        self.turns = (int(fullmove) - 1) * 2 + (0 if self.red_to_move else 1)
        self.state = state if self.red_to_move else self.env.fliped_state(state)

    def push(self, ucci_move):
        action = parse_ucci_move(ucci_move)
        if not self.red_to_move:
            action = flip_move(action)
        self.state = self.env.step(self.state, action)
        self.history += [action, self.state]
        self.red_to_move = not self.red_to_move
        self.turns += 1

    def repeated_replies(self):
        """Moves that were played from this very position earlier in the game (None if it is new)."""
        if self.state not in self.history[:-1]:
            return None
        return [self.history[i + 1] for i in range(len(self.history) - 1) if self.history[i] == self.state]


class UCI:
    def __init__(self, config, model=None, lib=None, device=None, stdin=None, stdout=None, use_pipes=False, pipes_factory=None,
                 infinite_capacity=200000, eval_mirror=False):
        self.config = config
        self.eval_mirror = eval_mirror          # the player's network averages every leaf and its left-right mirror
        self.lib = lib or get_lib()
        self.device = device
        self.env = StaticEnv(self.lib, device)
        self.stdin, self.stdout = stdin or sys.stdin, stdout or sys.stdout
        self.model = model
        self.use_pipes = use_pipes or pipes_factory is not None
        self.pipes_factory = pipes_factory       # () -> Connection; default: model.get_pipes(need_reload=False)
        self.infinite_capacity = infinite_capacity
        self.pos = Position(self.env)
        self.args = []
        self.player = None
        self.is_ready = False
        self.use_history = False
        self.start_time = None
        self.t = None
        self.search_worker = None

    # attribute names of the reference object, for callers that read them
    state = property(lambda self: self.pos.state)
    history = property(lambda self: self.pos.history)
    turns = property(lambda self: self.pos.turns)
    is_red_turn = property(lambda self: self.pos.red_to_move)

    def _print(self, text):
        print(text, file=self.stdout)
        self.stdout.flush()

    def main(self):
        for line in self.stdin:
            words = line.split()
            if not words:
                continue
            handler = getattr(self, 'cmd_' + words[0], None)
            self.args = words[1:]
            if handler is not None and handler() == "quit":
                return

    # ---- session
    def cmd_uci(self):
        for ln in ID_LINES:
            self._print(ln)
        self.use_history = self.load_model()
        self.pos.reset()
        self.is_ready = True

    def cmd_ucinewgame(self):
        turns = self.pos.turns                   # the reference leaves its move counter alone here (uci.py:90-95);
        self.pos.reset()                         # the `position` command that follows sets it
        self.pos.turns = turns
        self.is_ready = True

    def cmd_setoption(self):
        if len(self.args) < 4:
            return
        name, value = self.args[1], self.args[3]
        if name == 'gpu' and self.lib.is_cuda:
            self.device = f"cuda:{int(value)}"
        elif name == 'Threads':
            self.config.play.search_threads = int(value)

    def cmd_isready(self):
        if self.is_ready:
            self._print('readyok')

    def cmd_quit(self):
        if self.t:
            self.t.cancel()
        return "quit"

    def load_model(self):
        """uci.py:245-263: the best model, or a fresh one; returns whether it reads 28 planes."""
        if self.model is None:
            from .model import CChessModel
            self.model = CChessModel(self.config)
            rc = self.config.resource
            if not self.model.load(rc.model_best_config_path, rc.model_best_weight_path):
                self.model.build()
        return bool(self.model.use_history)

    # ---- position
    def cmd_position(self):
        if not self.is_ready:
            return
        a = self.args
        moves_at = None
        if not a or a[0] == 'startpos':
            self.pos.reset()
            if len(a) > 1 and a[1] == 'moves':
                moves_at = 2
        elif a[0] == 'fen':
            try:
                self.pos.set_fen(a[1], a[2], a[6])
            except Exception:
                return
            if len(a) > 7 and a[7] == 'moves':
                moves_at = 8
        elif a[0] == 'moves':
            moves_at = 1
        for mv in (a[moves_at:] if moves_at is not None else []):
            self.pos.push(mv)

    def cmd_fen(self):
        self.args = ['fen'] + self.args
        self.cmd_position()

    # ---- search
    def cmd_go(self):
        if not self.is_ready:
            return
        self.start_time = time()
        limits = GoLimits.parse(self.args, self.pos.red_to_move)
        pipes = None
        if self.use_pipes:
            if self.pipes_factory is not None:
                pipes = self.pipes_factory()
            else:
                self.model.close_pipes()
                pipes = self.model.get_pipes(need_reload=False)
        # a new player (and tree) per `go`, like uci.py:205-209
        self.player = CChessPlayer(self.config, search_tree=None, pipes=pipes, enable_resign=False, debugging=True, uci=True,
                                   use_history=self.use_history, side=self.pos.turns % 2, lib=self.lib, device=self.device,
                                   weights=None if pipes is not None else self.model.torch_weights(),
                                   infinite_capacity=self.infinite_capacity, eval_mirror=self.eval_mirror)
        self.player.info_stream = self.stdout
        self.search_worker = Thread(target=self._think, args=(self.player, limits), daemon=True)
        self.search_worker.start()
        self.t = None
        if limits.seconds:
            self.t = Timer(max(limits.seconds - 0.01, 0.0), self.cmd_stop)
            self.t.start()

    def _think(self, player, limits):
        """uci.py:265-291: ban the replies that would repeat the position with a check or a chase, search, report."""
        pos = self.pos
        res = self.env.done(pos.state, need_check=True)
        in_check = res[3] if len(res) > 3 else False
        replies = None if in_check else pos.repeated_replies()
        no_act = None if replies is None else [m for m in replies if self.env.will_check_or_catch(pos.state, m)]
        action, _ = player.action(pos.state, pos.turns, no_act=no_act, depth=limits.depth, infinite=limits.infinite,
                                  hist=pos.history)
        if self.player is not player:          # `stop` answered meanwhile
            return
        self.player = None
        if self.t:
            self.t.cancel()
        if action is not None:
            self._report(player, action, player.debug[pos.state][1], player.done_tasks // 100)
        self._release(player)

    def cmd_stop(self):
        """uci.py:229-243: every earlier reply from this position is banned, the tree answers as it stands."""
        if not self.is_ready:
            return
        player, self.player = self.player, None
        if player is None:
            return
        got = player.close_and_return_action(self.pos.state, self.pos.turns, self.pos.repeated_replies())
        if got is not None:
            self._report(player, *got)
        self._release(player)

    def _release(self, player):
        player.close(wait=False)
        if self.use_pipes and self.pipes_factory is None:
            self.model.close_pipes()

    def _report(self, player, action, value, depth):
        """uci.py:293-327: summary line, best move in board coordinates, the most visited reply as ponder move."""
        red = self.pos.red_to_move
        elapsed = max(time() - self.start_time, 1e-9)
        score = int((value if red else -value) * 1000)
        self._print(f"info depth {depth} score {score} time {int(elapsed * 1000)} nps {int(depth * 100 / elapsed) * 1000}")
        ponder, best_n = None, 0
        for mov, n in player.engine_child_stats(self.env.step(self.pos.state, action)):
            if n > best_n:                      # first maximum (uci.py:305-311)
                ponder, best_n = mov, n
        out = "bestmove " + to_uci_move(action if red else flip_move(action))
        if ponder:
            out += " ponder " + to_uci_move(flip_move(ponder) if red else ponder)
        self._print(out)


def main(config):
    UCI(config).main()
