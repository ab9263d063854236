"""Left-right mirror symmetry on the product library: cz_env_mirror and the label mirror equal the emulator build,
SlDataset.batch's mirror flags give the emulator's batches on the device, and the training workers with
augment="mirror" train end to end (OptimizeWorker bitwise the same on its host and device data paths)."""
import os

import numpy as np
import pytest
import torch

from cczero_b200.env import StaticEnv, state_to_board
from cczero_b200.lib import CzLib
from cczero_b200.optimize import OptimizeWorker
from tests.test_mirror import _dataset
from tests.test_play_replay_gpu import engine_games, run_worker
from tests.test_sl_gpu import end_to_end
from tests.test_sl_replay import ROOT

pytestmark = pytest.mark.gpu
EMUL = os.path.join(ROOT, "tests", "simt_emul", "libcz_emul.so")


@pytest.fixture(scope="module")
def emul():
    return StaticEnv(CzLib(EMUL), "cpu")


def test_cuda_mirror_equals_emulator(cuda_env, emul, golden_env):
    assert (cuda_env.mirror_labels == emul.mirror_labels).all()
    b = np.stack([state_to_board(r["state"]) for r in golden_env["rows"]])
    b[:, 90:] = np.arange(6, dtype=np.uint8) + 1
    flags = np.random.RandomState(1).randint(0, 2, len(b)).astype(np.uint8)
    for f in (None, flags):
        got = cuda_env.mirror(cuda_env.to_dev(b), None if f is None else cuda_env.to_dev(f)).cpu().numpy()
        want = emul.mirror(emul.to_dev(b), None if f is None else emul.to_dev(f)).numpy()
        assert got.tobytes() == want.tobytes()
    big = cuda_env.to_dev(np.tile(b, (8, 1)))                                 # 17 160 rows, several thousand blocks
    assert torch.equal(cuda_env.mirror(cuda_env.mirror(big)), big)


@pytest.mark.parametrize("visits", [False, True])
@pytest.mark.parametrize("history", [False, True])
def test_cuda_batch_mirror_equals_emulator(cuda_env, emul, visits, history):
    e, c = _dataset(emul, visits), _dataset(cuda_env, visits)
    idx = np.random.RandomState(2).permutation(len(e))
    flags = np.random.RandomState(3).randint(0, 2, len(idx))
    for x, y in zip(e.batch(emul, idx, history, mirror=flags), c.batch(cuda_env, idx, history, mirror=flags)):
        assert x.numpy().tobytes() == y.cpu().numpy().tobytes()


@pytest.mark.parametrize("in_planes", [14, 28])
def test_optimize_worker_mirror_trains_same_on_both_paths(cuda_lib, tmp_path, in_planes, monkeypatch):
    records = engine_games(cuda_lib, 60, seed=3, max_game_length=80, slots=60)
    plain_hist, plain_w = run_worker(tmp_path / "plain", records, "device", in_planes)
    orig = OptimizeWorker.__init__
    monkeypatch.setattr(OptimizeWorker, "__init__", lambda self, *a, **k: orig(self, *a, **k, augment="mirror"))
    h_hist, h_w = run_worker(tmp_path / "host", records, "host", in_planes)
    d_hist, d_w = run_worker(tmp_path / "device", records, "device", in_planes)
    assert len(h_hist) >= 4 and all(np.isfinite(r["loss"]) and np.isfinite(r["val_loss"]) for r in h_hist)
    assert h_hist == d_hist
    for k in h_w:
        assert h_w[k].tobytes() == d_w[k].tobytes(), k
    assert any(not np.array_equal(plain_w[k], d_w[k]) for k in d_w)            # the mirrored samples changed training


@pytest.mark.parametrize("onegreen", [False, True])
def test_sl_workers_mirror_end_to_end(tmp_path, cuda_lib, onegreen, monkeypatch):
    from cczero_b200 import sl, sl_onegreen
    from cczero_b200.model import CChessModel
    plain = end_to_end(tmp_path / "plain", onegreen, cuda_lib)
    wxf_start, onegreen_start = sl.start, sl_onegreen.start
    monkeypatch.setattr(sl, "start", lambda cfg: wxf_start(cfg, augment="mirror"))
    monkeypatch.setattr(sl_onegreen, "start", lambda cfg, skip: onegreen_start(cfg, skip, augment="mirror"))
    a = end_to_end(tmp_path / "a", onegreen, cuda_lib)
    b = end_to_end(tmp_path / "b", onegreen, cuda_lib)
    assert all(a.weights[k].tobytes() == b.weights[k].tobytes() for k in a.weights)        # deterministic
    assert all(np.isfinite(v).all() for v in a.weights.values())
    start = CChessModel(a.config).build(seed=5).weights
    assert any(not np.array_equal(a.weights[k], start[k]) for k in start)                   # it trained
    assert any(not np.array_equal(a.weights[k], plain.weights[k]) for k in start)           # on mirrored samples
