"""CPU tier of the trainer: the float64 Keras restatement (tests/train_oracle.py) against central finite differences,
and OptimizeWorker's host loop (which files load, validation split, shuffle, partial batch, lr schedule, saved and
moved files) with the emulator's rules kernels and a recording fake step."""
import json
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import model as om
from oracle import senv as osenv
from tests import nn_checks as nc
from tests import train_oracle as to


@pytest.mark.parametrize("in_planes", [14, 28])
def test_oracle_gradients_match_finite_differences(in_planes):
    n = 4
    _, planes, _ = nc.positions(n, in_planes, seed=in_planes)
    w = om.init_weights(64, 1, 256, seed=in_planes, trained_like=True, spread=0.3, in_planes=in_planes)
    rng = np.random.RandomState(0)
    pol = np.zeros((n, om.N_LABELS), np.float32)
    pol[np.arange(n), rng.randint(0, om.N_LABELS, n)] = 1
    val = np.array([1, -1, 0, 1], np.float32)
    ref = to.fit_step(w, planes, pol, val, 1, 0.01)
    w64 = {k: torch.as_tensor(v, dtype=torch.float64) for k, v in w.items()}

    def loss(ws):
        return to.losses(ws, planes, pol, val, 1)[0].item()

    h = 1e-6
    for k, g in ref["grad"].items():
        flat = w64[k].reshape(-1)
        for i in rng.choice(flat.numel(), min(3, flat.numel()), replace=False):
            old = flat[i].item()
            flat[i] = old + h
            up = loss(w64)
            flat[i] = old - h
            dn = loss(w64)
            flat[i] = old
            fd = (up - dn) / (2 * h)
            gi = g.reshape(-1)[i].item()
            scale = g.abs().max().item()
            assert abs(fd - gi) <= 1e-6 * scale + 1e-4 * abs(gi), (k, int(i), fd, gi, scale)


def test_clipped_target_has_exactly_zero_policy_gradient():
    """Keras clips p^ to [1e-7, 1 - 1e-7]: a target label whose probability lies below passes no gradient at all."""
    _, planes, _ = nc.positions(8, seed=3)
    w = nc.well_conditioned_weights(64, 1, planes, seed=2, logit_std=1.0)
    wt = {k: torch.as_tensor(v, dtype=torch.float64).requires_grad_(not to.is_stat(k)) for k, v in w.items()}
    logits = to.forward_train(wt, planes, 1)[0]
    p = torch.softmax(logits.detach(), dim=1)                          # training mode: BN on the batch statistics
    lab = int(p[0].argmin())
    assert float(p[0, lab]) < 1e-8
    pol = np.zeros((8, om.N_LABELS), np.float32)
    pol[0, lab] = 1
    pol[1, int((p[1] - 1e-3).abs().argmin())] = 1                     # a label well inside the clip interval
    ce = to.keras_ce(logits, torch.as_tensor(pol, dtype=torch.float64))
    g0 = torch.autograd.grad(ce[0], wt["policy_out/bias"], retain_graph=True)[0]
    assert torch.count_nonzero(g0).item() == 0
    g1 = torch.autograd.grad(ce[1], wt["policy_out/bias"])[0]
    assert torch.count_nonzero(g1).item() > 0                       # an unclipped sample does pass gradient


def test_fit_host_loop_restatement():
    tr, va = to.validation_split(1000)
    assert (tr == np.arange(980)).all() and (va == np.arange(980, 1000)).all()
    assert to.make_batches(980, 256) == [(0, 256), (256, 512), (512, 768), (768, 980)]
    assert to.decide_learning_rate([(0, 0.01), (150000, 0.003), (400000, 0.0001)], 149999) == 0.01
    assert to.decide_learning_rate([(0, 0.01), (150000, 0.003), (400000, 0.0001)], 150000) == 0.003
    assert to.decide_learning_rate([(10, 0.01)], 0) is None


# ---------------------------------------------------------------------------------------------- OptimizeWorker host logic
class RecordingTrainer:
    """Stands in for train.Trainer: records every step's batch and lr, returns fixed losses."""

    def __init__(self, model, batch_size, device):
        self.model, self.batch_size = model, batch_size
        self.steps, self.validations = [], []

    def step(self, planes, policy, value, lr):
        assert len(planes) <= self.batch_size
        self.steps.append((planes.copy(), policy.copy(), value.copy(), lr))
        return np.array([1.0, 0.5, 0.5, 0.0])

    def validation_loss(self, planes, policy, value):
        self.validations.append(len(planes))
        return 1.0, 0.5, 0.5, 0.0

    def export(self):
        return {k: v + 1 for k, v in self.model.weights.items()}


def _game(rng, plies):
    from cczero_b200.records import record_to_play_data
    s, moves = osenv.INIT_STATE, []
    for _ in range(plies):
        lm = osenv.get_legal_moves(s)
        m = lm[rng.randint(len(lm))]
        moves.append(m)
        s = osenv.step(s, m)
    return record_to_play_data({"moves": moves, "value_red": 1})


def _config(tmp_path, **tc):
    d = str(tmp_path)
    rc = SimpleNamespace(data_dir=d, play_data_dir=os.path.join(d, "play_data"), play_data_filename_tmpl="play_%s.json",
                         model_best_config_path=os.path.join(d, "model", "best_config.json"),
                         model_best_weight_path=os.path.join(d, "model", "best_weight.npz"),
                         next_generation_config_path=os.path.join(d, "model", "ng", "ng_config.json"),
                         next_generation_weight_path=os.path.join(d, "model", "ng", "ng_weight.npz"))
    mc = SimpleNamespace(cnn_filter_num=64, res_layer_num=1, value_fc_size=32, l2_reg=1e-4, cnn_first_filter_size=5,
                         cnn_filter_size=3)
    t = dict(batch_size=16, epoch_to_checkpoint=2, dataset_size=100000, start_total_steps=0, load_data_steps=2,
             momentum=0.9, loss_weights=[1.0, 1.0], min_games_to_begin_learn=1, lr_schedules=[(0, 0.01), (4, 0.003)])
    t.update(tc)
    return SimpleNamespace(resource=rc, model=mc, trainer=SimpleNamespace(**t), opts=SimpleNamespace(new=False, has_history=False))


def test_optimize_worker_host_logic(tmp_path, emul_env):
    from cczero_b200.optimize import OptimizeWorker
    cfg = _config(tmp_path)
    os.makedirs(cfg.resource.play_data_dir)
    rng = np.random.RandomState(1)
    names = []
    for i, plies in enumerate([30, 33, 14]):
        p = os.path.join(cfg.resource.play_data_dir, f"play_2026010{i}-000000.000000.json")
        data = _game(rng, plies) + (_game(rng, 6) if i == 0 else [])     # file 0 holds two games back to back
        json.dump(data, open(p, "w"))
        names.append(p)
    np.random.seed(0)
    w = OptimizeWorker(cfg, env=emul_env, trainer_factory=RecordingTrainer)
    w.start()
    tr = w.trainer
    # load_step 2: files 0 and 1 first (36 + 33 samples), then file 2 (14 samples <= batch_size 16: no training on it,
    # reference behaviour), then no new files: the next generation is saved and the loop ends
    n = 36 + 33
    n_train = int(n * 0.98)
    per_epoch = [len(s[0]) for s in tr.steps]
    assert per_epoch == [16, 16, 16, 16, n_train - 64] * 2              # the final partial batch is kept
    assert tr.validations == [n - n_train] * 2                           # the last 2 % validate, once per epoch
    # each epoch visits every training sample exactly once, in a new order
    all_vals = [np.concatenate([s[2] for s in tr.steps[:5]]), np.concatenate([s[2] for s in tr.steps[5:]])]
    assert len(all_vals[0]) == n_train and len(all_vals[1]) == n_train
    first = np.concatenate([s[0] for s in tr.steps[:5]]).reshape(n_train, -1)
    second = np.concatenate([s[0] for s in tr.steps[5:]]).reshape(n_train, -1)
    assert not np.array_equal(first, second)
    assert sorted(map(bytes, first)) == sorted(map(bytes, second))
    # lr: 0.01 inside the fit (total_steps 0), then (69 // 16) * 2 = 8 steps >= 4 -> 0.003 for the next call
    assert {s[3] for s in tr.steps} == {0.01}
    assert w.opt.lr == 0.003
    # files: the trained ones moved to data/trained, file 2 stays (it was loaded but not trained on, and not moved)
    trained = sorted(os.listdir(os.path.join(cfg.resource.data_dir, "trained")))
    assert trained == sorted(os.path.basename(p) for p in names[:2])
    assert os.path.exists(names[2])
    assert os.path.exists(cfg.resource.model_best_weight_path) and os.path.exists(cfg.resource.next_generation_weight_path)
    z = np.load(cfg.resource.next_generation_weight_path)
    assert z["policy_out__bias"].shape == (om.N_LABELS,)
