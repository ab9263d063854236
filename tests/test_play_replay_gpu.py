"""cz_play_replay on the product library: CUDA equals the emulator on 10 000 seeded engine self-play games (with moves
without a label planted in some), the device dataset's size per position, and OptimizeWorker with the real Trainer giving
the same losses and bitwise the same weights on its host and device data paths, at 14 and 28 planes."""
import json
import os
import random
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from cczero_b200 import records as rd
from cczero_b200.lib import CzLib
from oracle import model as om
from tests.test_sl_replay import ROOT
from tests.test_train_gpu import config

pytestmark = pytest.mark.gpu
EMUL = os.path.join(ROOT, "tests", "simt_emul", "libcz_emul.so")


def engine_games(cuda_lib, n_games, seed, max_game_length=120, slots=2500):
    """Seeded engine self-play with a random 64x2 net, `slots` games at a time -> play records (game_index order)."""
    from cczero_b200.engine import Engine
    w = om.init_weights(64, 2, 256, seed=seed)
    out = []
    for r in range((n_games + slots - 1) // slots):
        k = min(slots, n_games - len(out))
        eng = Engine(cuda_lib, "cuda", n_games=k, sims_per_move=8, leaves_per_round=4, nn_filters=64, nn_blocks=2,
                     max_game_length=max_game_length, seed=seed + r, enable_resign_rate=0.0)
        eng.set_weights({kk: torch.as_tensor(v) for kk, v in w.items()})
        eng.reset()
        recs = []
        while len(recs) < k:
            eng.selfplay(target_games=k - len(recs), max_moves=0)
            recs += eng.drain_records()
        eng.close()
        out += [rd.record_to_play_data(r) for r in sorted(recs, key=lambda r: r["game_index"])[:k]]
    return out


def test_cuda_replay_equals_emulator_on_10000_selfplay_games(cuda_lib, cuda_env):
    games = rd.pack_play_games(engine_games(cuda_lib, 10000, seed=11))
    offsets = np.concatenate([[0], np.cumsum(games.counts)])
    rng = np.random.RandomState(0)
    for g in rng.choice(len(games.counts), 500, replace=False):          # a move without a label at a random ply
        games.codes[offsets[g] + rng.randint(games.counts[g])] = (0 << 8) | 10
    emul = CzLib(EMUL)
    a = rd.play_replay(cuda_lib, "cuda", games, cuda_env.label_lut)
    b = rd.play_replay(emul, "cpu", games, cuda_env.label_lut)
    assert (a[2] == b[2]).all() and (a[2] == rd.CZ_PLAY_FAILED).sum() == 500
    assert torch.equal(a[1].cpu(), b[1]) and torch.equal(a[0].cpu(), b[0])
    assert len(games) > 200000


def test_device_dataset_is_104_bytes_per_position(cuda_lib, cuda_env):
    games = rd.pack_play_games(engine_games(cuda_lib, 64, seed=2, slots=64))
    ds = rd.replay_play_games(cuda_lib, "cuda", games, cuda_env.label_lut)
    total = sum(t.numel() * t.element_size() for t in (ds.boards, ds.labels, ds.values, ds.ply))
    assert total == 104 * len(ds) and ds.boards.is_cuda and ds.ply.is_cuda


def run_worker(root, records, path, in_planes):
    from cczero_b200.model import CChessModel
    from cczero_b200.optimize import OptimizeWorker
    d = str(root)
    cfg = config(64, 2, in_planes=in_planes, batch_size=128, lr_schedules=((0, 0.02), (20, 0.005)))
    cfg.trainer.load_data_steps, cfg.trainer.epoch_to_checkpoint, cfg.trainer.dataset_size = 6, 2, 1500
    cfg.resource = SimpleNamespace(data_dir=d, play_data_dir=os.path.join(d, "play_data"), play_data_filename_tmpl="play_%s.json",
                                   model_best_config_path=os.path.join(d, "model", "best_config.json"),
                                   model_best_weight_path=os.path.join(d, "model", "best_weight.npz"),
                                   next_generation_config_path=os.path.join(d, "model", "ng", "ng_config.json"),
                                   next_generation_weight_path=os.path.join(d, "model", "ng", "ng_weight.npz"))
    cfg.opts = SimpleNamespace(new=False, has_history=in_planes == 28)
    os.makedirs(cfg.resource.play_data_dir)
    for i in range(0, len(records), 5):                                   # nb_game_in_file = 5
        with open(os.path.join(cfg.resource.play_data_dir, f"play_20260101-0000{i // 5:02d}.000000.json"), "w") as f:
            json.dump(sum(records[i:i + 5], []), f)
    CChessModel(cfg).build(seed=5).save(cfg.resource.model_best_config_path, cfg.resource.model_best_weight_path)
    random.seed(1)
    np.random.seed(1)
    w = OptimizeWorker(cfg, device="cuda", dataset=path)
    w.start()
    w.trainer.close()
    return w.history, dict(np.load(cfg.resource.next_generation_weight_path))


@pytest.mark.parametrize("in_planes", [14, 28])
def test_optimize_worker_same_on_host_and_device_paths(cuda_lib, tmp_path, in_planes):
    records = engine_games(cuda_lib, 60, seed=3, max_game_length=80, slots=60)
    h_hist, h_w = run_worker(tmp_path / "host", records, "host", in_planes)
    d_hist, d_w = run_worker(tmp_path / "device", records, "device", in_planes)
    assert len(h_hist) >= 4 and all(np.isfinite(r["loss"]) and np.isfinite(r["val_loss"]) for r in h_hist)
    assert h_hist == d_hist
    assert sorted(h_w) == sorted(d_w)
    for k in h_w:
        assert h_w[k].tobytes() == d_w[k].tobytes(), k
