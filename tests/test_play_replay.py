"""Self-play records replayed on the device (cz_play_replay, on the emulator build of the same kernel source) and the
device dataset built from them (SlDataset with its ply column) against the host expansion records.expanding_data —
itself pinned to the reference's worker/optimize.py by test_oracle_vs_reference.py — bit for bit, at 14 and 28 planes;
input validation; and OptimizeWorker on both paths with recording trainers."""
import json
import os
import random

import numpy as np
import pytest
import torch

from cczero_b200 import records as rd
from cczero_b200.env import StaticEnv
from cczero_b200.optimize import OptimizeWorker
from oracle import senv as osenv
from tests.test_train_host import _config


def playout(rng, plies, state=osenv.INIT_STATE, value=1):
    """A seeded random legal playout from `state` as a play record (the moves stop early at a finished game)."""
    s, moves = state, []
    for _ in range(plies):
        lm = osenv.get_legal_moves(s)
        if not lm:
            break
        m = lm[rng.randint(len(lm))]
        moves.append(m)
        s = osenv.step(s, m)
    return rd.record_to_play_data({"moves": moves, "value_red": value}, init_state=state)


def host_expand(data, env, use_history):
    """optimize.load_data_from_file's expansion of one file's list (the host path)."""
    out = [rd.expanding_data(g, env, use_history) for g in rd.split_games(data) if len(g) > 1]
    return tuple(np.concatenate([o[i] for o in out]) for i in range(3))


def device_expand(data, env, use_history, source="test"):
    games = rd.pack_play_games([g for g in rd.split_games(data) if len(g) > 1], source)
    ds = rd.replay_play_games(env.lib, env.device, games, env.label_lut)
    return tuple(t.cpu().numpy() for t in ds.batch(env, np.arange(len(ds)), use_history))


def assert_same(data, env):
    for hist in (False, True):
        h, d = host_expand(data, env, hist), device_expand(data, env, hist)
        for a, b in zip(h, d):
            assert a.dtype == b.dtype and a.shape == b.shape
            assert a.tobytes() == b.tobytes()
        assert h[0].shape[1] == (28 if hist else 14)


@pytest.fixture(scope="module")
def env(emul_lib):
    return StaticEnv(emul_lib, "cpu")


def test_random_playouts_in_one_file(env):
    rng = np.random.RandomState(5)
    data = sum((playout(rng, int(rng.randint(20, 70)), value=int(rng.choice([-1, 0, 1]))) for _ in range(5)), [])
    assert_same(data, env)


@pytest.mark.parametrize("plies", [1, 2, 3])
def test_short_games_at_the_history_boundary(env, plies):
    rng = np.random.RandomState(plies)
    assert_same(playout(rng, plies), env)
    assert_same(playout(rng, plies) + playout(rng, 4) + playout(rng, plies), env)


def test_non_initial_start_state_and_dropped_empty_games(env):
    rng = np.random.RandomState(11)
    start = playout(rng, 9)
    s = osenv.INIT_STATE
    for m, _ in start[1:]:
        s = osenv.step(s, m)
    data = [osenv.INIT_STATE] + playout(rng, 12, state=s, value=-1) + [s] + playout(rng, 5)
    assert len([g for g in rd.split_games(data) if len(g) > 1]) == 2        # the lone state is a game without moves
    assert_same(data, env)


def test_labelled_illegal_move_is_applied_unchecked(env):
    # 0003: the red rook on (0,0) onto its own pawn on (0,3): a label (same file), not a legal move; then a move out of an
    # empty square.  senv.step applies both as they are.
    assert env.label_lut[0 * 90 + 27] >= 0 and "0003" not in osenv.get_legal_moves(osenv.INIT_STATE)
    data = rd.record_to_play_data({"moves": ["0003", "4544", "0313", "1719"], "value_red": 0.5})
    assert_same(data, env)


def test_float_values_round_like_the_host_path(env):
    data = rd.record_to_play_data({"moves": ["0001", "0001", "0102"], "value_red": 0.1})
    data[2][1] = 1e-40
    assert_same(data, env)


class CountingLib:
    def __init__(self, lib):
        self.lib, self.is_cuda, self.calls = lib, lib.is_cuda, []

    def call(self, name, *args):
        self.calls.append(name)
        return self.lib.call(name, *args)


def write(path, data):
    with open(path, "w") as f:
        json.dump(data, f)
    return str(path)


@pytest.mark.parametrize("bad,why", [("00a1", "not a digit"), ("001", "three characters"), ("00011", "five characters"),
                                     ("9001", "x = 9"), ("0090", "x = 9 at the destination"), ("０００１", "non-ASCII digits"),
                                     (1234, "not a string")])
def test_malformed_move_raises_before_any_launch(emul_lib, tmp_path, bad, why):
    from collections import deque
    lib = CountingLib(emul_lib)
    data = playout(np.random.RandomState(2), 6)
    data[4][0] = bad
    p = write(tmp_path / "play_bad.json", playout(np.random.RandomState(3), 5) + data)
    good = write(tmp_path / "play_good.json", playout(np.random.RandomState(4), 5))
    w = OptimizeWorker(_config(tmp_path), env=StaticEnv(lib, "cpu"), trainer_factory=RecordingTrainer, dataset="device")
    w.filenames = deque([p, good])                                  # popped from the end: the good file loads first
    with pytest.raises(ValueError) as e:
        w.fill_queue()
    assert p in str(e.value) and repr(bad) in str(e.value), why
    assert "cz_play_replay" not in lib.calls and os.path.exists(p)


def test_move_without_label_raises_the_host_paths_error(env, tmp_path):
    data = playout(np.random.RandomState(4), 7)
    data[5][0] = "0011"                                               # a diagonal step out of the corner: no label
    assert env.label_lut[0 * 90 + 10] < 0
    with pytest.raises(ValueError) as host:
        host_expand(data, env, False)
    with pytest.raises(ValueError) as dev:
        rd.replay_play_games(env.lib, env.device, rd.load_play_file(write(tmp_path / "p.json", data)), env.label_lut)
    assert str(dev.value) == str(host.value) == "move 0011 is not an action label"


@pytest.mark.parametrize("path", ["host", "device"])
def test_move_without_label_stops_the_load_at_its_file(emul_lib, tmp_path, path):
    """The file with the unlabelled move raises before the next file is read: an unreadable file after it survives, and
    nothing is replayed on the device path."""
    from collections import deque
    lib = CountingLib(emul_lib)
    data = playout(np.random.RandomState(4), 7)
    data[5][0] = "0011"
    bad = write(tmp_path / "play_nolabel.json", data)
    broken = str(tmp_path / "play_broken.json")
    with open(broken, "w") as f:
        f.write('["rkemsmekr')
    w = OptimizeWorker(_config(tmp_path), env=StaticEnv(lib, "cpu"), trainer_factory=RecordingTrainer, dataset=path)
    w.filenames = deque([broken, bad])                              # popped from the end: the unlabelled move first
    with pytest.raises(ValueError, match="move 0011 is not an action label"):
        w.fill_queue()
    assert os.path.exists(broken) and "cz_play_replay" not in lib.calls


def test_dataset_is_104_bytes_per_position(env):
    data = playout(np.random.RandomState(6), 30)
    games = rd.pack_play_games(rd.split_games(data))
    ds = rd.replay_play_games(env.lib, env.device, games, env.label_lut)
    assert len(ds) == 30
    per = sum(t.element_size() * t[0].numel() for t in (ds.boards, ds.labels, ds.values, ds.ply))
    assert per == 104
    assert ds.ply.tolist() == list(range(30))


# ---------------------------------------------------------------------------------------------- OptimizeWorker, both paths
class RecordingTrainer:
    """Records every step's and validation's batch as numpy (device tensors are converted), returns fixed losses."""

    def __init__(self, model, batch_size, device):
        self.model, self.batch_size = model, batch_size
        self.steps, self.validations = [], []

    @staticmethod
    def _np(x):
        return x.cpu().numpy().copy() if isinstance(x, torch.Tensor) else np.array(x, copy=True)

    def step(self, planes, policy, value, lr):
        assert len(planes) <= self.batch_size
        self.steps.append((self._np(planes), self._np(policy), self._np(value), lr))
        return np.array([1.0, 0.5, 0.5, 0.0])

    def validation_loss(self, planes, policy, value):
        self.validations.append((self._np(planes), self._np(policy), self._np(value)))
        return 1.0, 0.5, 0.5, 0.0

    def export(self):
        return {k: v + 1 for k, v in self.model.weights.items()}


def run_worker(root, files, env, dataset, history, **tc):
    cfg = _config(root, **tc)
    cfg.opts.has_history = history
    os.makedirs(cfg.resource.play_data_dir)
    for name, data in files:
        if isinstance(data, bytes):
            with open(os.path.join(cfg.resource.play_data_dir, name), "wb") as f:
                f.write(data)
        else:
            write(os.path.join(cfg.resource.play_data_dir, name), data)
    random.seed(3)
    np.random.seed(3)
    lrs = []
    w = OptimizeWorker(cfg, env=env, trainer_factory=RecordingTrainer, dataset=dataset)
    w.model = w.load_model()
    update = w.update_learning_rate
    w.update_learning_rate = lambda steps: (update(steps), lrs.append(w.opt.lr))
    total = w.training()
    trained = os.path.join(cfg.resource.data_dir, "trained")
    return {"steps": w.trainer.steps, "validations": w.trainer.validations, "lrs": lrs, "total_steps": total,
            "trained": sorted(os.listdir(trained)) if os.path.isdir(trained) else [],
            "left": sorted(os.listdir(cfg.resource.play_data_dir)), "history": w.history}


@pytest.mark.parametrize("history", [False, True])
@pytest.mark.parametrize("dataset_size", [100000, 40])
def test_optimize_worker_same_on_both_paths(env, tmp_path, history, dataset_size):
    rng = np.random.RandomState(7)
    files = []
    for i in range(7):
        data = playout(rng, int(rng.randint(8, 40)), value=int(rng.choice([-1, 1])))
        if i % 3 == 0:
            data += playout(rng, int(rng.randint(1, 6)))                   # several games back to back
        files.append((f"play_2026010{i}-000000.000000.json", data))
    files.insert(2, ("play_20260102-100000.000000.json", b'["rkemsmekr/9/1c5c1'))   # unreadable: deleted on both paths
    runs = {}
    for path in ("host", "device"):
        runs[path] = run_worker(tmp_path / path, files, env, path, history, load_data_steps=4, dataset_size=dataset_size,
                                batch_size=12)
    h, d = runs["host"], runs["device"]
    assert len(h["steps"]) > 4 and h["validations"]
    assert len(h["steps"]) == len(d["steps"]) and len(h["validations"]) == len(d["validations"])
    for a, b in zip(h["steps"] + h["validations"], d["steps"] + d["validations"]):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            if isinstance(x, np.ndarray):
                assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes()
            else:
                assert x == y
    assert h["steps"][0][0].shape[1] == (28 if history else 14)
    for k in ("lrs", "total_steps", "trained", "left", "history"):
        assert h[k] == d[k], k


def test_unreadable_file_is_deleted_on_the_device_path(env, tmp_path):
    p = str(tmp_path / "broken.json")
    with open(p, "w") as f:
        f.write('["rkemsmekr/9/1c5c1/p1p1p1p1p/9/9/P1P1P1P1P/1C5C1/9/RKEMSMEKR", ["00')
    assert rd.load_play_file(p) is None and not os.path.exists(p)
    assert rd.load_play_file(write(tmp_path / "state_only.json", [osenv.INIT_STATE])) is None
