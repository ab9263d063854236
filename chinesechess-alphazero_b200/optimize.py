"""`worker.optimize` drop-in (reference: cchess_alphazero/worker/optimize.py:37-225): learn from the play-data files.

`start(config)` and `OptimizeWorker(config)` keep the reference's method names and control flow: take the play-data
files in batches of `load_step` (`load_data_steps` where the config has no `load_step`), load them, run
`epoch_to_checkpoint` epochs of Keras-`fit`-equivalent training, save the best model, move the used files to
`data/trained/`, and when the files run out save the next generation.  The reference compiles a Keras model and calls
`fit`; here `compile_model` builds a `train.Trainer` (cz_train_step: CUDA forward, backward and SGD-momentum update) and
`fit` restates Keras 2.0.8's loop: the last 2 % of the samples (before shuffling) validate, the training indices are
reshuffled every epoch with numpy's global RNG, the final partial batch is kept, lr is constant within one call, and the
validation loss is computed in inference mode.

With the built-in trainer the play data stays on the GPU: `fill_queue` packs the files' moves on the host and replays
every game it loaded in one `cz_play_replay` launch (`records.replay_play_games`) into an `sl_data.SlDataset` of
104 bytes per position (board, label, value, ply in game), and `fit` expands each batch on the device, 14 or 28 planes.
The reference's host arrays take 13 388 bytes per position (18 428 with history planes).  With an injected
`trainer_factory` the files are expanded on the host (`records.expanding_data`) and every batch is numpy.  Both paths
load the same files in the same order, stop at the same `dataset_size`, draw the same random numbers and hand the
trainer the same values.

`policy_target="visits"` trains the policy head on the search's visit distribution where the records carry it
(self-play with `record_visits`, records.py): target[l] = float32(n_l / sum n), the AlphaZero target calc_policy builds
(agent/player.py:375-406).  Plies without visits, such as the appended final king capture or older files, keep the
one-hot of their move.  The default "move" is the reference's one-hot target (optimize.py:248).

`augment="mirror"` trains on both orientations of the data: Xiangqi's rules and action labels are symmetric across the
central file, so every epoch each training sample is reflected (planes along x, policy columns by the label mirror M)
with probability 1/2, flags drawn from numpy's global RNG right after the epoch's shuffle.  The validation samples are
never reflected, and without `augment` no flags are drawn, so the default path's random numbers are unchanged.
"""
import os
import shutil
from collections import deque
from logging import getLogger
from random import shuffle
from types import SimpleNamespace

import numpy as np

from .model import CChessModel
from .records import (PlayGames, check_labels, expanding_data, get_game_data_filenames, load_play_file, pack_visits,
                      read_game_data_from_file, replay_play_games, split_games)

logger = getLogger(__name__)


def start(config, policy_target="move", augment=None):
    return OptimizeWorker(config, policy_target=policy_target, augment=augment).start()


def load_best_model_weight(model):
    rc = model.config.resource
    return model.load(rc.model_best_config_path, rc.model_best_weight_path)


def save_as_best_model(model):
    rc = model.config.resource
    model.save(rc.model_best_config_path, rc.model_best_weight_path)


def save_as_next_generation_model(model):
    rc = model.config.resource
    model.save(rc.next_generation_config_path, rc.next_generation_weight_path)


def load_data_from_file(filename, env, use_history=False, policy_target="move"):
    """optimize.py:223-232: a file that cannot be read is deleted.  Where the reference's expanding_data reads a file as ONE
    game (and rejects files of several games: the second initial state is not a move), every game of the file is expanded.
    policy_target as in records.expanding_data; malformed visits raise before any game of the file is expanded."""
    try:
        data = read_game_data_from_file(filename)
    except Exception as e:
        logger.error(f"Error when loading data {e}")
        os.remove(filename)
        return None
    if data is None:
        return None
    games = [g for g in split_games(data) if len(g) > 1]
    if policy_target == "visits":
        pack_visits([it for g in games for it in g[1:]], filename)
    out = [expanding_data(g, env, use_history, policy_target, filename) for g in games]
    if not out:
        return None
    return tuple(np.concatenate([o[i] for o in out]) for i in range(3))


def validation_split(n, split=0.02):
    """Keras 2.0.8 fit(validation_split=...): split_at = int(n * (1 - split)), the last samples validate."""
    split_at = int(n * (1.0 - split))
    return np.arange(split_at), np.arange(split_at, n)


def check_augment(augment):
    if augment not in (None, "mirror"):
        raise ValueError(f"augment must be None or 'mirror', not {augment!r}")
    return augment


def mirror_flags(augment, n):
    """Per-sample reflection flags of one epoch (drawn only when augmenting, after the epoch's shuffle)."""
    return np.random.randint(0, 2, n) if augment else None


def mirror_batch(planes, policy, flags, mirror_labels):
    """Host form of SlDataset.batch's reflection: flagged rows' planes reversed along x, policy columns permuted by M
    (an involution, so row'[l] = row[M l]).  planes and policy are the batch's own copies and are changed in place."""
    f = np.asarray(flags).astype(bool)
    planes[f] = planes[f][..., ::-1]
    policy[f] = policy[f][:, mirror_labels]
    return planes, policy


def make_batches(size, batch_size):
    """Keras _make_batches: ceil(size / batch_size) slices, the last one partial."""
    nb = int(np.ceil(size / float(batch_size)))
    return [(i * batch_size, min(size, (i + 1) * batch_size)) for i in range(nb)]


class OptimizeWorker:
    def __init__(self, config, env=None, trainer_factory=None, device=None, dataset=None, policy_target="move",
                 augment=None):
        """env: StaticEnv for replaying records (default: the CUDA rules kernels); trainer_factory(model, batch_size, device)
        builds the object whose step(planes, policy, value, lr) / validation_loss(...) / export() train (default
        train.Trainer).  dataset: "device" keeps the positions on env's device and hands `step` device tensors, "host"
        expands them into numpy arrays; the default is "device" with the built-in trainer and "host" with a
        trainer_factory.  policy_target: "move" (one-hot of the played move) or "visits" (the recorded visit
        distribution where a ply has one).  augment: None or "mirror" (each epoch, every training sample reflected
        across the central file with probability 1/2)."""
        if dataset is None:
            dataset = "device" if trainer_factory is None else "host"
        if dataset not in ("device", "host"):
            raise ValueError(f"dataset must be 'device' or 'host', not {dataset!r}")
        self.on_device = dataset == "device"
        if policy_target not in ("move", "visits"):
            raise ValueError(f"policy_target must be 'move' or 'visits', not {policy_target!r}")
        self.policy_target = policy_target
        self.augment = check_augment(augment)
        self.config = config
        self.model = None
        self.loaded_filenames = set()
        self.loaded_data = deque(maxlen=self.config.trainer.dataset_size)
        self.clear_dataset()
        self.filenames = []
        self.opt = None
        self.count = 0
        self.eva = False
        self.env = env
        self.trainer_factory = trainer_factory
        self.device = device
        self.trainer = None
        self.history = []

    def start(self):
        self.model = self.load_model()
        self.training()

    def _env(self):
        if self.env is None:
            from .env import StaticEnv
            from .lib import get_lib
            self.env = StaticEnv(get_lib(), self.device or "cuda")
        return self.env

    def training(self):
        """optimize.py:56-100."""
        self.compile_model()
        tc = self.config.trainer
        total_steps = tc.start_total_steps
        last_file = None
        load_step = getattr(tc, "load_step", None) or tc.load_data_steps
        while True:
            files = get_game_data_filenames(self.config.resource)
            offset = tc.min_games_to_begin_learn
            if (len(files) < tc.min_games_to_begin_learn
                    or ((last_file is not None and last_file in files) and files.index(last_file) + 1 + offset > len(files))):
                if last_file is not None:
                    self.save_current_model(send=True)
                break
            if last_file is not None and last_file in files:
                idx = files.index(last_file) + 1
                files = files[idx:idx + load_step] if len(files) - idx > load_step else files[idx:]
            elif len(files) > load_step:
                files = files[0:load_step]
            last_file = files[-1]
            logger.info(f"Last file = {last_file}")
            self.filenames = deque(files)
            shuffle(self.filenames)
            self.fill_queue()
            self.update_learning_rate(total_steps)
            if self.loaded_count() > tc.batch_size:
                steps = self.train_epoch(tc.epoch_to_checkpoint)
                total_steps += steps
                self.save_current_model(send=False)
                self.update_learning_rate(total_steps)
                self.count += 1
                self.clear_dataset()
                self.backup_play_data(files)
        return total_steps

    def train_epoch(self, epochs):
        """optimize.py:102-121."""
        tc = self.config.trainer
        if self.on_device:
            data = self.collect_all_loaded_data()
            self.fit_dataset(data, tc.batch_size, epochs)
            return (len(data) // tc.batch_size) * epochs
        state_ary, policy_ary, value_ary = self.collect_all_loaded_data()
        self.fit(state_ary, policy_ary, value_ary, tc.batch_size, epochs)
        return (state_ary.shape[0] // tc.batch_size) * epochs

    def fit(self, x, policy, value, batch_size, epochs, validation=0.02):
        """Model.fit(x, [policy, value], batch_size, epochs, shuffle=True, validation_split=0.02) of Keras 2.0.8."""
        train_idx, val_idx = validation_split(len(x), validation)
        lr = self.opt.lr
        for epoch in range(epochs):
            order = train_idx.copy()
            np.random.shuffle(order)
            flags = mirror_flags(self.augment, len(order))
            losses = []
            for a, b in make_batches(len(order), batch_size):
                ids = order[a:b]
                xb, pb = x[ids], policy[ids]
                if flags is not None:
                    xb, pb = mirror_batch(xb, pb, flags[a:b], self._env().mirror_labels)
                losses.append(self.trainer.step(xb, pb, value[ids], lr))
            rec = {"epoch": epoch, "lr": lr, "loss": float(np.mean([l[0] for l in losses])) if losses else None}
            if len(val_idx):
                rec["val_loss"] = self.trainer.validation_loss(x[val_idx], policy[val_idx], value[val_idx])[0]
            logger.info(f"epoch {epoch + 1}/{epochs}: {rec}")
            self.history.append(rec)

    def fit_dataset(self, data, batch_size, epochs, validation=0.02):
        """`fit` on the device dataset: the same split, shuffles and batches, each batch expanded on the device
        (SlDataset.batch); the validation batch is built once, its targets as numpy like `fit` hands them."""
        env, history = self._env(), self.use_history()
        train_idx, val_idx = validation_split(len(data), validation)
        val = None
        if len(val_idx):
            p, pol, v = data.batch(env, val_idx, history)
            val = (p, pol.cpu().numpy(), v.cpu().numpy())
        lr = self.opt.lr
        for epoch in range(epochs):
            order = train_idx.copy()
            np.random.shuffle(order)
            flags = mirror_flags(self.augment, len(order))
            losses = []
            for a, b in make_batches(len(order), batch_size):
                mirror = None if flags is None else flags[a:b]
                losses.append(self.trainer.step(*data.batch(env, order[a:b], history, mirror), lr))
            rec = {"epoch": epoch, "lr": lr, "loss": float(np.mean([l[0] for l in losses])) if losses else None}
            if val is not None:
                rec["val_loss"] = self.trainer.validation_loss(*val)[0]
            logger.info(f"epoch {epoch + 1}/{epochs}: {rec}")
            self.history.append(rec)

    def compile_model(self):
        """optimize.py:129-136: SGD(lr=0.02, momentum) on the two losses with config.trainer.loss_weights."""
        self.opt = SimpleNamespace(lr=0.02, momentum=self.config.trainer.momentum)
        if self.trainer_factory is not None:
            self.trainer = self.trainer_factory(self.model, self.config.trainer.batch_size, self.device)
        else:
            from .train import Trainer
            self.trainer = Trainer(self.model, self.config.trainer.batch_size, self.device)

    def update_learning_rate(self, total_steps):
        lr = self.decide_learning_rate(total_steps)
        if lr:
            self.opt.lr = lr
            logger.debug(f"total step={total_steps}, set learning rate to {lr}")

    def use_history(self):
        return bool(getattr(getattr(self.config, "opts", None), "has_history", False))

    def loaded_count(self):
        if self.on_device:
            return 0 if self.dataset is None else len(self.dataset)
        return len(self.dataset[0])

    def clear_dataset(self):
        self.dataset = None if self.on_device else (deque(), deque(), deque())

    def fill_queue(self):
        """optimize.py:150-170, sequential: files popped from the end of the shuffled list until dataset_size samples.
        On the device path the files are read, packed and label-checked one by one (the same stopping test, counting
        the positions they hold, and a bad file raising where the host path raises) and then replayed together in one
        launch."""
        size = self.config.trainer.dataset_size
        if self.on_device:
            env = self._env()
            parts, pending = [], self.loaded_count()
            while self.filenames and pending < size:
                games = load_play_file(self.filenames.pop(), self.policy_target == "visits")
                if games is not None:
                    check_labels(games, env.label_lut)
                    parts.append(games)
                    pending += len(games)
            if parts:
                chunk = replay_play_games(env.lib, env.device, PlayGames.concat(parts), env.label_lut)
                self.dataset = chunk if self.dataset is None else self.dataset.extend(chunk)
            return
        while self.filenames and len(self.dataset[0]) < size:
            t = load_data_from_file(self.filenames.pop(), self._env(), self.use_history(), self.policy_target)
            if t is not None:
                for x, y in zip(self.dataset, t):
                    x.extend(y)

    def collect_all_loaded_data(self):
        """Host path: (planes, policy, value) numpy arrays.  Device path: the SlDataset."""
        if self.on_device:
            return self.dataset
        state_ary, policy_ary, value_ary = self.dataset
        return (np.asarray(state_ary, dtype=np.float32), np.asarray(policy_ary, dtype=np.float32),
                np.asarray(value_ary, dtype=np.float32))

    def load_model(self):
        model = CChessModel(self.config)
        if getattr(getattr(self.config, "opts", None), "new", False) or not load_best_model_weight(model):
            model.build()
            save_as_best_model(model)
        return model

    def save_current_model(self, send=False):
        logger.info("Save as ng model")
        if self.trainer is not None:
            self.model.weights = self.trainer.export()
        if not send:
            save_as_best_model(self.model)
        else:
            save_as_next_generation_model(self.model)

    def decide_learning_rate(self, total_steps):
        ret = None
        for step, lr in self.config.trainer.lr_schedules:
            if total_steps >= step:
                ret = lr
        return ret

    def try_reload_model(self):
        digest = self.model.fetch_digest(self.config.resource.model_best_weight_path)
        if digest and digest != self.model.digest:
            load_best_model_weight(self.model)
            return True
        return False

    def backup_play_data(self, files):
        backup_folder = os.path.join(self.config.resource.data_dir, "trained")
        cnt = 0
        os.makedirs(backup_folder, exist_ok=True)
        for f in files:
            try:
                shutil.move(f, backup_folder)
            except Exception:
                cnt += 1
        logger.info(f"backup {len(files)} files, {cnt} empty files")
