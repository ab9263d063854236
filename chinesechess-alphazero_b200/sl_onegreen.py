"""`worker.sl_onegreen` drop-in (reference: cchess_alphazero/worker/sl_onegreen.py): supervised learning from the
onegreen.json game collection (an `init` position and a digit move list per game).

Same machinery as `sl.SupervisedWorker`; what differs is the reference's: `start(config, skip)` begins at game `skip`,
Adam's lr is 0.003, games start from their `init` (with '99' for captured pieces), the winner comes from the result and
title strings, and a drawn game is valued by static_env.evaluate on its final position (np.tanh(ans / tot * 3), from
red's side).  A game the reference drops (a move without a label) or raises on (a move that is not four digits) adds
nothing and is counted.
"""
import json
from logging import getLogger
from time import time

from . import sl_data as sd
from . import sl

logger = getLogger(__name__)


def start(config, skip, augment=None):
    return SupervisedWorker(config, augment=augment).start(skip)


class SupervisedWorker(sl.SupervisedWorker):
    LR = 0.003                                     # sl_onegreen.py:82 Adam(lr=0.003)

    def __init__(self, config, trainer_factory=None, device=None, lib=None, augment=None):
        super().__init__(config, trainer_factory, device, lib, augment)
        self.games = None

    def start(self, skip=0):
        self.model = self.load_model()
        with open(self.config.resource.sl_onegreen, 'r', encoding='utf-8') as f:
            self.games = json.load(f)
        self.training(skip)

    def training(self, skip=0):
        """sl_onegreen.py:50-66."""
        self.compile_model()
        tc = self.config.trainer
        total_steps = tc.start_total_steps
        logger.info(f"Start training, game count = {len(self.games)}, step = {tc.sl_game_step} games, skip = {skip}")
        for i in range(skip, len(self.games), tc.sl_game_step):
            games = self.games[i:i + tc.sl_game_step]
            self.fill_queue(games)
            if len(self.dataset) > tc.batch_size:
                steps = self.train_epoch(tc.epoch_to_checkpoint)
                total_steps += steps
                self.save_current_model()
                self.dataset = sd.SlDataset.empty(self._device())
                logger.debug(f"total steps = {total_steps}")
        return total_steps

    def generate_game_data(self, games):
        """sl_onegreen.py:111-132: every game of the chunk, replayed in one launch."""
        self.buffer = []
        start_time = time()
        for idx, game in enumerate(games):
            self.load_game(game['init'], game['move_list'], sd.onegreen_winner(game), idx, game.get('title'), game.get('url'))
        rep, wins, _, skipped = sd.replay_onegreen_games(self._lib(), self._device(), self.buffer)
        self.skipped += skipped
        if rep is None:
            return None
        failed = int((rep.status != sd.OK).sum())
        self.failed += failed
        if skipped or failed:
            logger.warning(f"skipped {skipped + failed} of {len(games)} games the reference drops or cannot load")
        data = sd.build_dataset(rep, wins)
        logger.debug(f"Loading {len(games)} games, {len(data)} positions, time: {time() - start_time}s")
        return data

    def load_game(self, init, move_list, winner, idx, title, url):
        """Queues one game (the board walk of sl_onegreen.py:134-175 runs for the whole chunk on the device)."""
        self.buffer.append({'init': init, 'move_list': move_list, 'result': {1: '红胜', -1: '黑胜'}.get(winner, ''),
                            'title': '', 'url': url})
