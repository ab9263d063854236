"""Visit recording and visit-count targets on the product library: CUDA recording equals the restated reference loop,
recording changes no game of the built-in network, the CUDA target kernel equals the emulator on 10 000 self-play games,
and OptimizeWorker with policy_target="visits" gives the same losses and bitwise the same weights on its host and device
data paths with the real Trainer."""
import os

import numpy as np
import pytest
import torch

from cczero_b200 import records as rd
from cczero_b200.engine import Engine
from cczero_b200.lib import CzLib
from cczero_b200.optimize import OptimizeWorker
from oracle import model as om
from oracle import senv as osenv
from tests.test_play_replay_gpu import EMUL, run_worker
from tests.test_visit_records import CONFIGS, LABEL_OF, check_visits, device_games

pytestmark = pytest.mark.gpu


def test_cuda_recorded_visits_equal_restated_calc_policy(cuda_lib, monkeypatch):
    kinds = set()
    for c in CONFIGS:
        c = dict(c, n_games=2 * c["n_games"])
        want = 2 * c.pop("want")
        recs = sorted(device_games(cuda_lib, "cuda", want=want, **c), key=lambda r: r["game_index"])
        plain = sorted(device_games(cuda_lib, "cuda", want=want, record_visits=False, **c), key=lambda r: r["game_index"])
        assert [{k: v for k, v in r.items() if k != "visits"} for r in recs] == plain
        kinds |= check_visits(monkeypatch, recs, **c)
    assert {"resign", "capture"} <= kinds, kinds


def selfplay(cuda_lib, weights, record_visits, n_games=64, sims=200, want=64, **kw):
    eng = Engine(cuda_lib, "cuda", n_games=n_games, sims_per_move=sims, leaves_per_round=8, nn_filters=128, nn_blocks=7,
                 max_game_length=60, seed=9, record_visits=record_visits, max_nodes_per_game=24 * sims, **kw)
    eng.set_weights({k: torch.as_tensor(v) for k, v in weights.items()})
    eng.reset()
    recs = []
    while len(recs) < want:
        eng.selfplay(target_games=want - len(recs), max_moves=0)
        recs += eng.drain_records()
    eng.close()
    return sorted(recs, key=lambda r: r["game_index"])


@pytest.mark.parametrize("tau_decay", [0.9, 0.0])
def test_recording_changes_no_game_of_the_built_in_network(cuda_lib, tau_decay):
    w = om.init_weights(128, 7, 256, seed=4)
    on = selfplay(cuda_lib, w, True, tau_decay_rate=tau_decay)
    off = selfplay(cuda_lib, w, False, tau_decay_rate=tau_decay)
    assert [{k: v for k, v in r.items() if k != "visits"} for r in on] == off
    argmax_plies = 0
    for r in on:
        s, seen = osenv.INIT_STATE, set()
        for t, (m, v) in enumerate(zip(r["moves"], r["visits"])):
            if not v:                                                   # only the appended final capture has none
                assert t == r["n_plies"] - 1
                break
            d = dict(v)
            assert d.get(LABEL_OF[m], 0) > 0
            assert [l for l, _ in v] == sorted(d)
            # arg-max plies: tau = 0 and no repetition of the position (which would raise the temperature)
            if tau_decay == 0.0 and s not in seen:
                best = max(d.values())
                assert LABEL_OF[m] == min(l for l, n in v if n == best)
                argmax_plies += 1
            seen.add(s)
            s = osenv.step(s, m)
    assert tau_decay != 0.0 or argmax_plies > 500


def engine_games(cuda_lib, n_games, seed, slots=2500):
    w = om.init_weights(64, 2, 256, seed=seed)
    out = []
    for r in range((n_games + slots - 1) // slots):
        k = min(slots, n_games - len(out))
        eng = Engine(cuda_lib, "cuda", n_games=k, sims_per_move=8, leaves_per_round=4, nn_filters=64, nn_blocks=2,
                     max_game_length=120, seed=seed + r, enable_resign_rate=0.0, record_visits=True)
        eng.set_weights({kk: torch.as_tensor(v) for kk, v in w.items()})
        eng.reset()
        recs = []
        while len(recs) < k:
            eng.selfplay(target_games=k - len(recs), max_moves=0)
            recs += eng.drain_records()
        eng.close()
        out += [rd.record_to_play_data(x) for x in sorted(recs, key=lambda x: x["game_index"])[:k]]
    return out


def test_cuda_targets_equal_emulator_on_10000_selfplay_games(cuda_lib, cuda_env):
    games = rd.pack_play_games(engine_games(cuda_lib, 10000, seed=12), "selfplay", visits=True)
    ds = rd.replay_play_games(cuda_lib, "cuda", games, cuda_env.label_lut)
    emul = CzLib(EMUL)
    n = len(ds)
    idx = np.random.RandomState(0).permutation(n)[:50000]
    cpu = rd.replay_play_games(emul, "cpu", rd.PlayGames(games.boards, games.counts, games.codes, games.values, games.visits),
                               cuda_env.label_lut)
    step = 8192
    soft = 0
    for a in range(0, len(idx), step):
        ids = idx[a:a + step]
        g = ds.visit_targets(cuda_lib, torch.as_tensor(ids, device="cuda")).cpu()
        e = cpu.visit_targets(emul, torch.as_tensor(ids))
        assert torch.equal(g.view(torch.int32), e.view(torch.int32))
        soft += int(((g > 0).sum(1) > 1).sum())
    assert n > 200000 and soft > 20000


@pytest.mark.parametrize("in_planes", [14, 28])
def test_optimize_worker_same_on_host_and_device_paths_with_visit_targets(cuda_lib, tmp_path, in_planes, monkeypatch):
    records = engine_games(cuda_lib, 60, seed=3, slots=60)
    orig = OptimizeWorker.__init__
    monkeypatch.setattr(OptimizeWorker, "__init__", lambda self, *a, **k: orig(self, *a, **k, policy_target="visits"))
    h_hist, h_w = run_worker(tmp_path / "host", records, "host", in_planes)
    d_hist, d_w = run_worker(tmp_path / "device", records, "device", in_planes)
    assert len(h_hist) >= 4 and all(np.isfinite(r["loss"]) and np.isfinite(r["val_loss"]) for r in h_hist)
    assert h_hist == d_hist
    assert sorted(h_w) == sorted(d_w)
    for k in h_w:
        assert h_w[k].tobytes() == d_w[k].tobytes(), k
