"""The whole training step (cz_train_step through train.Trainer) against the float64 Keras restatement
(tests/train_oracle.py): gradients, updated weights and moving statistics, bit-reproducibility, the ABI's error codes,
a short learning run and the round trip trainer -> best model -> self-play engine -> evaluator."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import model as om
from tests import nn_checks as nc
from tests import train_oracle as to

pytestmark = pytest.mark.gpu


def config(filters, blocks, in_planes=14, pol_c=4, val_c=2, l2=1e-4, lr_schedules=((0, 0.01),), batch_size=256):
    mc = SimpleNamespace(cnn_filter_num=filters, res_layer_num=blocks, value_fc_size=256, l2_reg=l2, input_depth=in_planes,
                         policy_channels=pol_c, value_channels=val_c, cnn_first_filter_size=5, cnn_filter_size=3)
    tc = SimpleNamespace(momentum=0.9, loss_weights=[1.0, 1.0], batch_size=batch_size, epoch_to_checkpoint=1,
                         lr_schedules=list(lr_schedules), start_total_steps=0, min_games_to_begin_learn=1, load_data_steps=100,
                         dataset_size=100000, cleaning_processes=1)
    return SimpleNamespace(model=mc, trainer=tc)


def model_for(cfg, weights):
    from cczero_b200.model import CChessModel
    m = CChessModel(cfg)
    m.weights = {k: np.asarray(v, np.float32) for k, v in weights.items()}
    m.model = m
    return m


def batch(n, in_planes=14, seed=0, values=None):
    _, planes, _ = nc.positions(n, in_planes, seed)
    rng = np.random.RandomState(seed + 1)
    pol = np.zeros((n, om.N_LABELS), np.float32)
    pol[np.arange(n), rng.randint(0, om.N_LABELS, n)] = 1
    val = rng.choice([-1.0, 0.0, 1.0], n).astype(np.float32) if values is None else values
    return planes.astype(np.float32), pol, val


# Whole-step bounds.  The gradients of these nets are extremely sensitive to any rounding: rounding only the tensor-core
# operands to fp16 (activations, weights, scaled conv-output gradients), with everything else in float64, already moves
# them by 1-10 % (relative Frobenius) in 7- and 10-block towers and by up to a few percent in 1-block nets — the BN
# backward subtracts the gradient's projections on the batch mean and on xhat, which cancels most of it in every layer.
# The GPU perturbs the same operands in the same places (plus fp32 sums, which flip some fp16 roundings the other way),
# so each gradient's distance to float64 is bounded by three times the distance those fp16 operands alone open in
# float64, plus TOL (measured on an H100: at most 0.71x of that bound).  The distance to the fp16-operand
# float64 run is printed too: about 2e-4 on 1-block nets, where that emulation is faithful.  A wrong kernel (a lost tap,
# a transposed operand, a missing mean term) moves gradients by O(1), and the stage tests prove their bounds reject those.
TOL = 5e-3


def check_grads(tr, w, planes, pol, val, blocks, lr):
    ref = to.fit_step(w, planes, pol, val, blocks, lr, device="cuda")
    ref16 = to.fit_step(w, planes, pol, val, blocks, lr, device="cuda", fp16_operands=True)
    rows = []
    for k, g in ref["grad"].items():
        got = tr.grad(k)
        e16, e, gap = nc.rel_frobenius(got, ref16["grad"][k]), nc.rel_frobenius(got, g), nc.rel_frobenius(ref16["grad"][k], g)
        rows.append((k, e16, e, gap))
    worst16 = max(rows, key=lambda r: r[1])
    worst = max(rows, key=lambda r: r[2] / (3 * r[3] + TOL))
    print(f"worst vs fp16-operand float64: {worst16[0]} {worst16[1]:.3g}; vs float64: {worst[0]} {worst[2]:.3g} (gap {worst[3]:.3g})")
    bad = [r for r in rows if not r[2] <= 3 * r[3] + TOL]
    assert not bad, bad
    return ref, ref16


@pytest.mark.parametrize("filters,blocks", [(128, 7), (192, 10)])
def test_whole_step_matches_float64(cuda_lib, filters, blocks):
    from cczero_b200.train import Trainer
    n = 256
    planes, pol, val = batch(n, seed=filters)
    w = nc.well_conditioned_weights(filters, blocks, planes[:64], seed=blocks)
    cfg = config(filters, blocks, batch_size=n)
    tr = Trainer(model_for(cfg, w), n, "cuda")
    lr = 0.01
    losses = tr.step(planes, pol, val, lr)
    ref, ref16 = check_grads(tr, w, planes, pol, val, blocks, lr)
    # The update on the GPU's own gradients, in fp32 from a zero velocity: v = -lr (g + 2 l2 K), w' = w + v; a few fp32
    # roundings of |w| and of lr (|g| + 2 l2 |K|).  Moving statistics against the fp16-operand float64 run (the forward's
    # batch statistics differ by fp32 sums, times 0.01).
    l2 = cfg.model.l2_reg
    for k, w0 in w.items():
        w0 = torch.as_tensor(w0, dtype=torch.float64)
        if to.is_stat(k):
            r = ref16["weights"][k].cpu()
            assert (tr.weights[k].double().cpu() - r).abs().max().item() <= 1e-4 * r.abs().max().item() + 1e-6, k
            continue
        g = tr.grad(k).double().cpu()
        l2x2 = 2 * l2 if to.is_reg(k) else 0.0
        v_ref = -lr * (g + l2x2 * w0)
        v_mag = lr * (g.abs() + l2x2 * w0.abs())

        def check_v(got, r, v_mag=v_mag, k=k):
            nc.check_close(got, r, v_mag * 2.0 ** -21 / nc.BETA, out="fp32", what=f"velocity {k}")

        check_v(tr.velocity[k].double().cpu(), v_ref)
        nc.check_close(tr.weights[k].double().cpu(), w0 + v_ref, (w0.abs() * 2.0 ** -22 + v_mag * 2.0 ** -21) / nc.BETA,
                       out="fp32", what=f"weight {k}")
        if k.startswith("res1_conv1"):
            nc.assert_rejects(check_v, tr.velocity[k].double().cpu(), v_ref, [
                nc.Mutation("L2 gradient l2 K instead of 2 l2 K", lambda g_, r: -lr * (g + l2 * w0))])
    np.testing.assert_allclose(losses[1:3], ref["losses"][1:3], rtol=2e-3)
    np.testing.assert_allclose(losses[3], ref["losses"][3], rtol=1e-5)
    tr.close()


def test_step_is_bit_reproducible(cuda_lib):
    from cczero_b200.train import Trainer
    n = 256
    planes, pol, val = batch(n, seed=5)
    w = om.init_weights(64, 2, 256, seed=4)
    cfg = config(64, 2, batch_size=n)
    a, b = Trainer(model_for(cfg, w), n, "cuda"), Trainer(model_for(cfg, w), n, "cuda")
    for _ in range(2):
        la, lb = a.step(planes, pol, val, 0.01), b.step(planes, pol, val, 0.01)
        assert np.array_equal(la, lb)
    for k in a.weights:
        assert torch.equal(a.weights[k], b.weights[k]), k
    for k in a.velocity:
        assert torch.equal(a.velocity[k], b.velocity[k]), k
    a.close(); b.close()


@pytest.mark.parametrize("filters,in_planes,heads,n", [(64, 28, (4, 2), 7), (128, 14, (2, 4), 1), (64, 14, (32, 4), 33)])
def test_step_configurations_match_float64(cuda_lib, filters, in_planes, heads, n):
    """Head widths (4,2), (2,4), (32,4), 14 and 28 planes, batches 1 .. 33: gradients of a 1-block net (first-conv wgrad
    and head gradients included) against float64."""
    from cczero_b200.train import Trainer
    planes, pol, val = batch(n, in_planes, seed=n)
    w = om.init_weights(filters, 1, 256, seed=n, trained_like=True, spread=0.3, in_planes=in_planes, policy_filters=heads[0],
                        value_filters=heads[1])
    cfg = config(filters, 1, in_planes, heads[0], heads[1], batch_size=max(n, 8))
    tr = Trainer(model_for(cfg, w), max(n, 8), "cuda")
    tr.step(planes, pol, val, 0.02)
    _, ref16 = check_grads(tr, w, planes, pol, val, 1, 0.02)
    for k in ref16["weights"]:
        if k.endswith("moving_mean") or k.endswith("moving_variance"):       # batch statistics of fp32 sums, times 0.01
            r = ref16["weights"][k]
            e = (tr.weights[k].double() - r).abs().max().item()
            assert e <= 1e-5 * r.abs().max().item() + 1e-6, (k, e)
    tr.close()


def test_clipped_target_passes_no_policy_gradient(cuda_lib):
    """A target label whose probability is below Keras's clip (1e-7) contributes no gradient: policy_out/bias gets exactly
    0 (the CE without the clip would give p - onehot)."""
    from cczero_b200.train import Trainer
    planes, pol, val = batch(8, seed=3)
    w = nc.well_conditioned_weights(64, 1, planes, seed=2, logit_std=1.0)
    wt = {k: torch.as_tensor(v, dtype=torch.float64) for k, v in w.items()}
    logits = to.forward_train(wt, planes, 1)[0]                       # training mode: BN on the batch statistics
    p = torch.softmax(logits, dim=1)
    pol[:] = 0
    for i in range(8):                                                  # every label below the clip
        pol[i, int(p[i].argmin())] = 1
    assert float(p.min(dim=1).values.max()) < 1e-8
    cfg = config(64, 1, batch_size=8)
    tr = Trainer(model_for(cfg, w), 8, "cuda")
    tr.step(planes, pol, val, 0.01)
    g = tr.grad("policy_out/bias")
    unclipped = (p - torch.as_tensor(pol, dtype=torch.float64)).sum(0) / 8

    def check_zero(got, r):
        assert torch.count_nonzero(got).item() == 0, "policy gradient of a clipped target"

    check_zero(g, None)
    nc.assert_rejects(check_zero, g.cpu(), g.cpu(), [nc.Mutation("CE without the clip", lambda g_, r: unclipped.clone())])
    tr.close()


def test_abi_misuse_returns_error_codes(cuda_lib):
    from cczero_b200.lib import CzError, CzTrainConfig
    from cczero_b200.train import Trainer
    w = om.init_weights(64, 1, 256, seed=1)
    tr = Trainer(model_for(config(64, 1, batch_size=4), w), 4, "cuda")
    out = torch.empty(10, device="cuda")
    with pytest.raises(CzError, match=r"\(-1\).*no trainable tensor"):
        tr.lib.call("cz_train_read_grad", tr._h, b"nosuch_layer/kernel", C.c_void_p(out.data_ptr()), 10)
    with pytest.raises(CzError, match=r"\(-1\).*elements"):
        tr.lib.call("cz_train_read_grad", tr._h, b"policy_out/bias", C.c_void_p(out.data_ptr()), 10)
    planes, pol, val = batch(5, seed=1)
    with pytest.raises(CzError, match=r"\(-1\).*batch 5"):
        tr.step(planes, pol, val, 0.01)
    cfg = CzTrainConfig()
    cfg.struct_bytes = C.sizeof(CzTrainConfig)
    cfg.filters, cfg.blocks, cfg.in_planes, cfg.policy_channels, cfg.value_channels, cfg.value_fc, cfg.max_batch = 96, 1, 14, 4, 2, 256, 4
    with pytest.raises(CzError, match=r"\(-5\)"):
        tr.lib.call("cz_train_workspace_bytes", C.byref(cfg), C.byref(C.c_uint64(0)))
    # a parameter list without one tensor
    from cczero_b200.train import _descs
    partial = {k: v for k, v in tr.weights.items() if not k.startswith("value_out")}
    with pytest.raises(CzError, match=r"\(-1\).*value_out"):
        tr.lib.call("cz_train_set_params", tr._h, _descs(partial), len(partial), tr._vd, len(tr.velocity))
    tr.close()


def selfplay_samples(cuda_lib, cuda_env, n_games=64, seed=1, max_game_length=40):
    """Seeded engine self-play with a random 64x2 net -> play-data records and their training tensors."""
    from cczero_b200.engine import Engine
    from cczero_b200.records import expanding_data, record_to_play_data
    w = om.init_weights(64, 2, 256, seed=seed)
    eng = Engine(cuda_lib, "cuda", n_games=n_games, sims_per_move=8, leaves_per_round=4, nn_filters=64, nn_blocks=2,
                 max_game_length=max_game_length, seed=seed, enable_resign_rate=0.0)
    eng.set_weights({k: torch.as_tensor(v) for k, v in w.items()})
    eng.reset()
    recs = []
    while len(recs) < n_games:
        eng.selfplay(target_games=n_games - len(recs), max_moves=0)
        recs += eng.drain_records()
    eng.close()
    recs = sorted(recs, key=lambda r: r["game_index"])[:n_games]         # games finish in a timing-dependent order
    data = [record_to_play_data(r) for r in recs]
    t = [expanding_data(d, cuda_env) for d in data]
    return data, tuple(np.concatenate([x[i] for x in t]) for i in range(3))


def test_it_learns_like_float64(cuda_lib, cuda_env):
    """A 64x2 net on ~1k self-play positions: the GPU's loss curve follows float64 step by step, and the loss falls."""
    from cczero_b200.train import Trainer
    _, (planes, pol, val) = selfplay_samples(cuda_lib, cuda_env)
    planes, pol, val = planes[:1024], pol[:1024], val[:1024]
    n, bs, steps, lr = len(planes), 128, 20, 0.02
    w0 = om.init_weights(64, 2, 256, seed=7)
    cfg = config(64, 2, batch_size=bs)
    tr = Trainer(model_for(cfg, w0), bs, "cuda")
    rng = np.random.RandomState(0)
    order = [rng.permutation(n)[:bs] for _ in range(steps)]
    gpu = [tr.step(planes[i], pol[i], val[i], lr)[0] for i in order]
    curves = {}
    for emulate in (False, True):
        w, v, c = dict(w0), None, []
        for i in order:
            r = to.fit_step(w, planes[i], pol[i], val[i], 2, lr, velocity=v, device="cuda", fp16_operands=emulate)
            w = {k: x.cpu().numpy() for k, x in r["weights"].items()}
            v = {k: x.cpu().numpy() for k, x in r["velocity"].items()}
            c.append(r["losses"][0])
        curves[emulate] = np.array(c)
    ref, ref16, gpu = curves[False], curves[True], np.array(gpu)
    # Training at lr 0.02 with momentum on 128-position batches is chaotic: rounding only the tensor-core operands to
    # fp16 in float64 (ref16) drifts from float64 by up to ~0.5 % of the loss within 20 steps.  The GPU's run is another
    # such perturbation; per step it stays within 5x the largest drift fp16 operands alone caused up to that step, plus
    # 2e-3 of the loss, and ends within 5 % of float64's loss (measured on an H100: at most 0.26x of the per-step bound;
    # after 20 steps 6.294 against float64's 6.309, from 8.486).
    env = np.maximum.accumulate(np.abs(ref16 - ref))
    tol = 5 * env + 2e-3 * np.abs(ref)
    print("loss curve gpu / float64 / fp16-operand float64:", np.c_[gpu, ref, ref16][[0, 9, 19]].tolist(), "max dev / tol",
          float((np.abs(gpu - ref) / tol).max()))
    assert (np.abs(gpu - ref) <= tol).all()
    assert abs(gpu[-1] - ref[-1]) <= 0.05 * ref[-1]
    assert gpu[-5:].mean() < 0.9 * gpu[:5].mean()                      # it learns
    tr.close()


def test_round_trip_into_selfplay_and_arena(cuda_lib, cuda_env, tmp_path):
    """OptimizeWorker trains on the play-data files self-play wrote and saves the best model; CChessModelAPI hot-reloads
    it; the reloaded engine's forward matches float64 on the exported weights; the arena plays best vs next generation."""
    import os
    from cczero_b200 import evaluator
    from cczero_b200.api import CChessModelAPI
    from cczero_b200.model import CChessModel
    from cczero_b200.optimize import OptimizeWorker
    from cczero_b200.records import write_play_data
    data, _ = selfplay_samples(cuda_lib, cuda_env, n_games=16, seed=3, max_game_length=30)
    d = str(tmp_path)
    cfg = config(64, 2, batch_size=64)
    cfg.resource = SimpleNamespace(data_dir=d, play_data_dir=os.path.join(d, "play_data"), play_data_filename_tmpl="play_%s.json",
                                   model_best_config_path=os.path.join(d, "model", "best_config.json"),
                                   model_best_weight_path=os.path.join(d, "model", "best_weight.npz"),
                                   next_generation_config_path=os.path.join(d, "model", "ng", "ng_config.json"),
                                   next_generation_weight_path=os.path.join(d, "model", "ng", "ng_weight.npz"))
    cfg.trainer.load_data_steps = 100
    cfg.opts = SimpleNamespace(new=False, has_history=False)
    for i in range(0, len(data), 4):                                    # nb_game_in_file = 4
        write_play_data(cfg.resource.play_data_dir, sum(data[i:i + 4], []))
    start = CChessModel(cfg).build(seed=5)
    start.save(cfg.resource.model_best_config_path, cfg.resource.model_best_weight_path)
    served = CChessModel(cfg)
    assert served.load(cfg.resource.model_best_config_path, cfg.resource.model_best_weight_path)
    api = CChessModelAPI(cfg, served, lib=cuda_lib, device="cuda", max_batch=64)
    api._ensure_engine()
    w = OptimizeWorker(cfg, device="cuda")
    w.start()
    assert w.history and all(np.isfinite(h["loss"]) for h in w.history)
    assert os.path.exists(cfg.resource.next_generation_weight_path)
    old = served.digest
    api.try_reload_model()
    assert served.digest != old
    best = CChessModel(cfg)
    assert best.load(cfg.resource.model_best_config_path, cfg.resource.model_best_weight_path)
    for k, v in best.weights.items():
        assert np.array_equal(served.weights[k], v), k
    _, planes, _ = nc.positions(16, seed=4)
    pol, val = api.engine.nn_forward_planes(torch.as_tensor(planes, device="cuda"))
    ref_p, ref_v = om.forward(best.weights, planes, 2)
    assert np.abs(pol.cpu().numpy() - ref_p).max() < 1e-3 and np.abs(val.cpu().numpy() - ref_v).max() < 1e-3
    api.close()
    api.engine.close()
    ng = CChessModel(cfg)
    assert ng.load(cfg.resource.next_generation_config_path, cfg.resource.next_generation_weight_path)
    cfg.play = SimpleNamespace(simulation_num_per_move=8, search_threads=4, c_puct=1.5, noise_eps=0.0, tau_decay_rate=0.9,
                               max_game_length=20, max_processes=1)
    cfg.eval = SimpleNamespace(game_num=2)
    ew = evaluator.EvaluateWorker(cfg, best, ng, n_games=2, concurrent_games=2, lib=cuda_lib, device="cuda", playouts=None)
    total, *_ = ew.start()
    ew.close()
    assert 0 <= total <= 2
    w.trainer.close()
