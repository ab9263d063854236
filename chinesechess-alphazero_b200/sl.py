"""`worker.sl` drop-in (reference: cchess_alphazero/worker/sl.py): supervised learning from human games (gameinfo.csv,
moves.csv in WXF notation).

`start(config)` and `SupervisedWorker(config)` keep the reference's method names and control flow: take the games in
chunks of `sl_game_step`, load each chunk, train `epoch_to_checkpoint` epochs when the chunk holds more than `batch_size`
positions, save the sl_best model and clear the dataset.  The games are replayed on the GPU (`sl_data`, cz_sl_replay)
and stay there as boards, labels and values; `fit` expands each batch on the device and steps `train.Trainer` with
Keras 2.0.8 Adam.  The restated `fit` is OptimizeWorker's: the last 2 % of the samples validate, numpy's global RNG
reshuffles the training indices every epoch, the final partial batch is kept, and the validation loss runs in inference
mode.  Deviations: a game whose records make the reference raise (a missing or duplicated turn row, a move naming no
piece, an unparseable move) is skipped and counted instead of aborting the run; a 28-plane (history) network is
rejected; TensorBoard callbacks are not built.

`augment="mirror"` reflects each training sample across the central file with probability 1/2 every epoch, as
OptimizeWorker does (optimize.py); the validation samples are never reflected.
"""
from logging import getLogger
from time import time
from types import SimpleNamespace

import numpy as np

from . import sl_data as sd
from .model import CChessModel, N_LABELS
from .optimize import check_augment, make_batches, mirror_flags, validation_split

logger = getLogger(__name__)


def start(config, augment=None):
    return SupervisedWorker(config, augment=augment).start()


def load_sl_best_model_weight(model):
    rc = model.config.resource
    return model.load(rc.sl_best_config_path, rc.sl_best_weight_path)


def save_as_sl_best_model(model):
    rc = model.config.resource
    model.save(rc.sl_best_config_path, rc.sl_best_weight_path)


class SupervisedWorker:
    LR = 1e-2                                      # sl.py:81 Adam(lr=1e-2)

    def __init__(self, config, trainer_factory=None, device=None, lib=None, augment=None):
        """trainer_factory(model, batch_size, device, optimizer="adam") builds the object whose step / validation_loss /
        export train (default train.Trainer); lib: the rules library (default the CUDA product); augment: None or
        "mirror"."""
        self.config = config
        self.augment = check_augment(augment)
        self.model = None
        self.dataset = None
        self.opt = None
        self.buffer = []
        self.gameinfo = None
        self.moves = None
        self.trainer_factory = trainer_factory
        self.device = device
        self.lib = lib
        self.trainer = None
        self.env = None
        self.history = []
        self.skipped = 0
        self.failed = 0

    def _lib(self):
        if self.lib is None:
            from .lib import get_lib
            self.lib = get_lib()
        return self.lib

    def _device(self):
        import torch
        if self.device is None:
            self.device = "cuda" if self._lib().is_cuda else "cpu"
        return torch.device(self.device)

    def _env(self):
        if self.env is None:
            from .env import StaticEnv
            self.env = StaticEnv(self._lib(), self._device())
        return self.env

    def start(self):
        self.model = self.load_model()
        rc = self.config.resource
        self.gameinfo = sd.read_gameinfo(rc.sl_data_gameinfo)
        self.moves = sd.read_moves(rc.sl_data_move)
        self.training()

    def training(self):
        """sl.py:50-65."""
        self.compile_model()
        tc = self.config.trainer
        total_steps = tc.start_total_steps
        logger.info(f"Start training, game count = {len(self.gameinfo)}, step = {tc.sl_game_step} games")
        for i in range(0, len(self.gameinfo), tc.sl_game_step):
            games = self.gameinfo[i:i + tc.sl_game_step]
            self.fill_queue(games)
            if len(self.dataset) > tc.batch_size:
                steps = self.train_epoch(tc.epoch_to_checkpoint)
                total_steps += steps
                self.save_current_model()
                self.dataset = sd.SlDataset.empty(self._device())
        return total_steps

    def train_epoch(self, epochs):
        tc = self.config.trainer
        data = self.collect_all_loaded_data()
        self.fit(data, tc.batch_size, epochs)
        return (len(data) // tc.batch_size) * epochs

    def fit(self, data, batch_size, epochs, validation=0.02):
        """Model.fit(x, [policy, value], batch_size, epochs, shuffle=True, validation_split=0.02) of Keras 2.0.8, with the
        batches expanded on the device from the replayed dataset."""
        env = self._env()
        train_idx, val_idx = validation_split(len(data), validation)
        val = None
        if len(val_idx):
            p, pol, v = data.batch(env, val_idx)
            val = (p, pol.cpu().numpy(), v.cpu().numpy())
        lr = self.opt.lr
        for epoch in range(epochs):
            order = train_idx.copy()
            np.random.shuffle(order)
            flags = mirror_flags(self.augment, len(order))
            losses = []
            for a, b in make_batches(len(order), batch_size):
                planes, policy, value = data.batch(env, order[a:b], mirror=None if flags is None else flags[a:b])
                losses.append(self.trainer.step(planes, policy, value, lr))
            rec = {"epoch": epoch, "lr": lr, "loss": float(np.mean([l[0] for l in losses])) if losses else None}
            if val is not None:
                rec["val_loss"] = self.trainer.validation_loss(*val)[0]
            logger.info(f"epoch {epoch + 1}/{epochs}: {rec}")
            self.history.append(rec)

    def compile_model(self):
        """sl.py:80-83: Adam on the two losses with config.trainer.loss_weights; one optimizer (and one `iterations`)
        for the whole run."""
        if self.model.use_history:
            raise ValueError("supervised learning produces 14-plane positions (fen_to_planes); this network reads 28 "
                             "history planes — build or load a 14-plane model")
        self.opt = SimpleNamespace(lr=self.LR)
        factory = self.trainer_factory
        if factory is None:
            from .train import Trainer
            factory = Trainer
        self.trainer = factory(self.model, self.config.trainer.batch_size, self.device, optimizer="adam")
        self.dataset = sd.SlDataset.empty(self._device())

    def fill_queue(self, games):
        chunk = self.generate_game_data(games)
        if chunk is not None:
            self.dataset = self.dataset.extend(chunk)

    def collect_all_loaded_data(self):
        """The device dataset (boards, labels, values); batches are expanded by SlDataset.batch."""
        return self.dataset

    def load_model(self):
        model = CChessModel(self.config)
        if getattr(getattr(self.config, "opts", None), "new", False) or not load_sl_best_model_weight(model):
            model.build()
            save_as_sl_best_model(model)
        return model

    def save_current_model(self):
        logger.debug("Save best sl model")
        if self.trainer is not None:
            self.model.weights = self.trainer.export()
        save_as_sl_best_model(self.model)

    def generate_game_data(self, games):
        """sl.py:110-122: every game of the chunk, replayed in one launch."""
        self.buffer = []
        start_time = time()
        for game in games:
            rows = self.moves.get(sd._key(game['gameID']), {'red': [], 'black': []})
            self.load_game(rows['red'], rows['black'], game.get('winner'), len(self.buffer))
        rep, wins, _, skipped = sd.replay_wxf_games(self._lib(), self._device(), self.buffer)
        self.skipped += skipped
        if rep is None:
            return None
        failed = int((rep.status != sd.OK).sum())
        self.failed += failed
        if skipped or failed:
            logger.warning(f"skipped {skipped + failed} of {len(games)} games the reference cannot load")
        data = sd.build_dataset(rep, wins)
        logger.debug(f"Loading {len(games)} games, {len(data)} positions, time: {time() - start_time}s")
        return data

    def load_game(self, red, black, winner, idx):
        """Queues one game: its red and black (turn, move) rows and the winner column.  The board walk of sl.py:124-174
        runs for the whole chunk on the device (generate_game_data)."""
        self.buffer.append((red, black, winner))

    def build_policy(self, action, flip):
        """sl.py:176-185: the one-hot row of a light-board move string (flip: the black list's mirrored label)."""
        from .env import flip_move
        lut = self._env().label_lut
        a = flip_move(action) if flip else action
        k = int(lut[(int(a[1]) * 9 + int(a[0])) * 90 + int(a[3]) * 9 + int(a[2])]) if len(a) == 4 else -1
        if k < 0:
            raise KeyError(action)                     # not in ActionLabelsRed, like the reference's move_lookup
        policy = np.zeros(N_LABELS)
        policy[k] = 1
        return policy
