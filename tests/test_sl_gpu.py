"""Supervised learning on the GPU: cz_sl_replay on the product library (fixture parity, CUDA == emulator on 10 000
seeded games), device-built batches, the fused Keras Adam update (bit-exact against a float32 restatement fed the GPU's
own gradients, mutation checks, float64 learning curve, determinism, SGD unchanged, error codes) and both workers end to
end."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from cczero_b200 import sl_data as sd
from cczero_b200.lib import CzLib, CzTensorDesc
from oracle import model as om
from oracle import senv as osenv
from tests import adam_oracle as ao
from tests import train_oracle as to
from tests.test_sl_replay import ROOT, check_replay, fixture
from tests.test_sl_workers import config as sl_config, write_csv, write_json
from tests.test_train_gpu import batch, config, model_for

pytestmark = pytest.mark.gpu
EMUL = os.path.join(ROOT, "tests", "simt_emul", "libcz_emul.so")


def test_replay_matches_reference_cuda(cuda_lib):
    check_replay(cuda_lib, "cuda", fixture())


def synthetic_games(n, seed):
    """Seeded records exercising every branch: plausible WXF spellings (many illegal or unresolvable) and digit moves."""
    rng = np.random.RandomState(seed)
    letters = np.array(list("KAEHRCPkaehrcpBNbn.x"))
    cols = np.array(list("123456789+-0"))
    movs = np.array(list("+-.=x"))
    dests = np.array(list("1234567890"))
    wxf, og = [], []
    for _ in range(n):
        k = rng.randint(0, 60)
        plies = [(letters[rng.randint(len(letters))] + cols[rng.randint(len(cols))] + movs[rng.randint(len(movs))] +
                  dests[rng.randint(len(dests))]).encode() for _ in range(k)]
        wxf.append((plies, [1 if i % 2 == 0 else -1 for i in range(k)]))
        og.append(([bytes(rng.randint(48, 58, 4).astype(np.uint8)) for _ in range(k)], [1 if i % 2 == 0 else -1 for i in range(k)]))
    return wxf, og


def test_replay_cuda_equals_emulator_on_10000_games(cuda_lib):
    emul = CzLib(EMUL)
    wxf, og = synthetic_games(10000, 3)
    b0 = np.stack([sd.start_board()] * len(wxf))
    for mode, games in ((sd.WXF, wxf), (sd.ONEGREEN, og)):
        a = sd.replay(cuda_lib, "cuda", b0, [p for p, _ in games], [s for _, s in games], mode)
        b = sd.replay(emul, "cpu", b0, [p for p, _ in games], [s for _, s in games], mode)
        assert (a.game == b.game).all()
        assert torch.equal(a.labels.cpu(), b.labels) and torch.equal(a.boards.cpu(), b.boards)
        assert (a.game[:, 0] > 0).sum() > 1000                          # the replays do get somewhere


def fixture_dataset(cuda_lib):
    data = fixture()
    games = [([(int(r["turn"]), r["move"]) for r in g["rows"] if r["side"] == "red"],
              [(int(r["turn"]), r["move"]) for r in g["rows"] if r["side"] == "black"], g["winner"]) for g in data["wxf"]]
    rep, wins, keep, _ = sd.replay_wxf_games(cuda_lib, "cuda", games)
    return sd.build_dataset(rep, wins), data


def test_device_batch_matches_host_planes_and_step(cuda_lib, cuda_env):
    from cczero_b200.train import Trainer
    ds, data = fixture_dataset(cuda_lib)
    ref = [r for g in data["wxf"] if not g["ref"]["raised"] for r in g["ref"]["records"]]
    idx = np.random.RandomState(1).permutation(len(ds))[:256]
    planes, policy, value = ds.batch(cuda_env, idx)
    hp = np.stack([osenv.state_to_planes(ref[i][0]) for i in idx]).astype(np.float32)
    hpol = np.zeros((len(idx), om.N_LABELS), np.float32)
    hpol[np.arange(len(idx)), [ref[i][1] for i in idx]] = 1
    hval = np.array([ref[i][2] for i in idx], np.float32)
    assert (planes.cpu().numpy() == hp).all() and (policy.cpu().numpy() == hpol).all() and (value.cpu().numpy() == hval).all()
    w0 = om.init_weights(64, 2, 256, seed=4)
    outs = []
    for feed in ((planes, policy, value), (hp, hpol, hval)):
        tr = Trainer(model_for(config(64, 2, batch_size=256), w0), 256, "cuda", optimizer="adam")
        tr.step(*feed, 1e-2)
        outs.append(tr.export())
        tr.close()
    assert all((outs[0][k] == outs[1][k]).all() for k in outs[0])


def adam_check(tr, w, m, v, lr, l2, iterations, mutate=None):
    """float32 restatement of one k_adam launch fed the GPU's own gradients; True when weights and moments agree bit for bit."""
    ok = True
    for k in tr.adam_m:
        g = tr.grad(k).cpu().numpy()
        reg = to.is_reg(k) or (mutate == "l2_on_bn" and (k.endswith("/gamma") or k.endswith("/beta")))
        it = 0 if mutate == "reset" else iterations
        if mutate == "no_bias_correction":
            ww, mm, vv = ao.adam_update_f32(w[k], g, m[k], v[k], lr, it, 2 * np.float32(l2), reg)
            a = np.float32(lr)
            f = np.float32
            mm = (f(ao.B1) * m[k] + (f(1) - f(ao.B1)) * ((g + f(2 * np.float32(l2)) * w[k]) if reg else g)).astype(f)
            ww = (w[k] - (a * mm) / (np.sqrt(vv) + f(ao.EPS))).astype(f)
        elif mutate == "eps_in_sqrt":
            ww, mm, vv = ao.adam_update_f32(w[k], g, m[k], v[k], lr, it, 2 * np.float32(l2), reg)
            a = np.float32(lr * (np.sqrt(1.0 - ao.B2 ** (it + 1)) / (1.0 - ao.B1 ** (it + 1))))
            ww = (w[k] - (a * mm) / np.sqrt(vv + np.float32(ao.EPS))).astype(np.float32)
        else:
            ww, mm, vv = ao.adam_update_f32(w[k], g, m[k], v[k], lr, it, 2 * np.float32(l2), reg)
        ok &= ww.tobytes() == tr.weights[k].cpu().numpy().tobytes()
        ok &= mm.tobytes() == tr.adam_m[k].cpu().numpy().tobytes()
        ok &= vv.tobytes() == tr.adam_v[k].cpu().numpy().tobytes()
    return ok


@pytest.mark.parametrize("filters,blocks", [(64, 2), (128, 7)])
def test_adam_is_bit_exact_and_mutations_fail(cuda_lib, filters, blocks):
    from cczero_b200.train import Trainer
    cfg = config(filters, blocks, batch_size=64)
    tr = Trainer(model_for(cfg, om.init_weights(filters, blocks, 256, seed=2)), 64, "cuda", optimizer="adam")
    lr, l2 = 1e-2, cfg.model.l2_reg
    assert tr.iterations == 0
    for s in range(3):
        planes, pol, val = batch(64, seed=10 + s)
        snap = lambda d: {k: x.cpu().numpy().copy() for k, x in d.items()}
        w, m, v = snap(tr.weights), snap(tr.adam_m), snap(tr.adam_v)
        tr.step(planes, pol, val, lr)
        assert tr.iterations == s + 1
        assert adam_check(tr, w, m, v, lr, l2, s)
        muts = ["no_bias_correction", "eps_in_sqrt", "l2_on_bn"] + (["reset"] if s > 0 else [])
        for mut in muts:
            assert not adam_check(tr, w, m, v, lr, l2, s, mutate=mut), mut
    tr.close()


def test_adam_learns_like_float64(cuda_lib, cuda_env):
    """20 Adam steps (lr 3e-3) of a 64x2 net on fixture SL positions follow the float64 Adam of tests/adam_oracle.py."""
    from cczero_b200.train import Trainer
    ds, _ = fixture_dataset(cuda_lib)
    bs, steps, lr = 128, 20, 3e-3
    w0 = om.init_weights(64, 2, 256, seed=7)
    tr = Trainer(model_for(config(64, 2, batch_size=bs), w0), bs, "cuda", optimizer="adam")
    rng = np.random.RandomState(0)
    order = [rng.permutation(len(ds))[:bs] for _ in range(steps)]
    feeds = [tuple(x.cpu().numpy() for x in ds.batch(cuda_env, i)) for i in order]
    gpu = np.array([tr.step(*f, lr)[0] for f in feeds])
    curves = {}
    for emulate in (False, True):
        w, c = {k: np.asarray(x, np.float64) for k, x in w0.items()}, []
        st = ao.AdamState.zeros_like(w)
        for f in feeds:
            loss, w = ao.fit_step_adam(w, st, *f, 2, lr, device="cuda", fp16_operands=emulate)
            c.append(loss[0])
        curves[emulate] = np.array(c)
    ref, ref16 = curves[False], curves[True]
    env = np.maximum.accumulate(np.abs(ref16 - ref))
    tol = 5 * env + 2e-3 * np.abs(ref)
    print("adam loss curve gpu / float64 / fp16-operand float64:", np.c_[gpu, ref, ref16][[0, 9, 19]].tolist(),
          "max dev / tol", float((np.abs(gpu - ref) / tol).max()))
    assert (np.abs(gpu - ref) <= tol).all()
    assert gpu[-5:].mean() < 0.9 * gpu[:5].mean()
    tr.close()


def test_adam_determinism_and_sgd_unchanged(cuda_lib):
    from cczero_b200.train import Trainer
    cfg = config(64, 2, batch_size=64)
    w0 = om.init_weights(64, 2, 256, seed=3)
    feeds = [batch(64, seed=20 + s) for s in range(2)]

    def run(**kw):
        tr = Trainer(model_for(cfg, w0), 64, "cuda", **kw)
        for f in feeds:
            tr.step(*f, 1e-2)
        out = tr.export()
        tr.close()
        return out

    a, b = run(optimizer="adam"), run(optimizer="adam")
    assert all(a[k].tobytes() == b[k].tobytes() for k in a)
    s0, s1 = run(), run(optimizer="sgd")
    assert all(s0[k].tobytes() == s1[k].tobytes() for k in s0)
    assert any(a[k].tobytes() != s0[k].tobytes() for k in a)


def test_adam_abi_misuse(cuda_lib):
    from cczero_b200.train import Trainer, _descs
    cfg = config(64, 1, batch_size=8)
    tr = Trainer(model_for(cfg, om.init_weights(64, 1, 256, seed=1)), 8, "cuda")
    rc = cuda_lib.raw("cz_train_adam_iterations")(tr._h, C.byref(C.c_int64(0)))
    assert rc == -3                                                           # SGD trainer
    m = {k: torch.zeros_like(v) for k, v in tr.velocity.items()}
    short = dict(m)
    short.pop(next(iter(short)))
    d_full, d_short = _descs(m), _descs(short)
    f = cuda_lib.raw("cz_train_set_adam")
    assert f(tr._h, d_short, len(short), d_full, len(m), 0.9, 0.999, 1e-8) == -1          # a missing moment
    bad = dict(m)
    k0 = next(iter(bad))
    bad[k0] = torch.zeros(bad[k0].numel() + 1, device="cuda")
    d_bad = _descs(bad)
    assert f(tr._h, d_full, len(m), d_bad, len(bad), 0.9, 0.999, 1e-8) == -1               # a mis-sized moment
    assert f(tr._h, d_full, len(m), d_full, len(m), 1.0, 0.999, 1e-8) == -1                # beta_1 out of range
    # a trainer without parameters
    ws = torch.zeros(tr.workspace.numel(), dtype=torch.uint8, device="cuda")
    h = C.c_void_p(0)
    cuda_lib.call("cz_train_create", C.byref(tr.cfg), C.c_void_p(ws.data_ptr()), C.c_uint64(ws.numel()),
                  C.c_void_p(torch.cuda.current_stream().cuda_stream), C.byref(h))
    assert f(h, d_full, len(m), d_full, len(m), 0.9, 0.999, 1e-8) == -3
    cuda_lib.raw("cz_train_destroy")(h)
    tr.close()


def end_to_end(tmp_path, onegreen, cuda_lib, seed=0):
    from cczero_b200 import sl, sl_onegreen
    from cczero_b200.model import CChessModel
    data = fixture()
    cfg = sl_config(tmp_path, batch_size=64, game_step=20)
    cfg.model.value_fc_size = 256
    cfg.opts.new = False                                     # start from a seeded model on the sl_best paths
    CChessModel(cfg).build(seed=5).save(cfg.resource.sl_best_config_path, cfg.resource.sl_best_weight_path)
    if onegreen:
        write_json(cfg, data["onegreen"])
    else:
        write_csv(cfg, data["wxf"])
    np.random.seed(seed)
    if onegreen:
        sl_onegreen.start(cfg, 3)
    else:
        sl.start(cfg)
    assert os.path.exists(cfg.resource.sl_best_weight_path) and os.path.exists(cfg.resource.sl_best_config_path)
    m = CChessModel(cfg)
    assert m.load(cfg.resource.sl_best_config_path, cfg.resource.sl_best_weight_path)
    return m


@pytest.mark.parametrize("onegreen", [False, True])
def test_workers_end_to_end(tmp_path, cuda_lib, cuda_env, onegreen):
    from cczero_b200.engine import Engine
    from tests import search_checks as sc
    a = end_to_end(tmp_path / "a", onegreen, cuda_lib)
    b = end_to_end(tmp_path / "b", onegreen, cuda_lib)
    from cczero_b200.model import CChessModel, engine_net_kwargs
    assert all(a.weights[k].tobytes() == b.weights[k].tobytes() for k in a.weights)        # a second run is identical
    start = CChessModel(a.config).build(seed=5).weights
    assert any(not np.array_equal(a.weights[k], start[k]) for k in start)                   # it trained
    states = [osenv.INIT_STATE] + sc.midgame_states(7, 1)
    eng = Engine(cuda_lib, "cuda:0", n_games=8, sims_per_move=16, leaves_per_round=2, **engine_net_kwargs(a.config.model))
    eng.set_weights({k: torch.as_tensor(v) for k, v in a.weights.items()})
    pol, val = eng.nn_forward_boards(cuda_env.boards_from_states(states))
    ref_p, ref_v = om.forward(a.weights, np.stack([osenv.state_to_planes(s) for s in states]), 1)
    eng.close()
    assert np.abs(pol.cpu().numpy() - ref_p).max() < 1e-3 and np.abs(val.cpu().numpy() - ref_v).max() < 1e-3
