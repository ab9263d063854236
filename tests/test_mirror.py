"""Left-right mirror symmetry (x -> 8 - x) on the emulator build of the rules kernels and the oracle: the label mirror M,
cz_env_mirror on the fixture boards, SlDataset.batch's mirror flags against a host restatement, and the training
workers' augment="mirror" (both OptimizeWorker data paths hand the trainer the same batches; no extra random numbers
without it)."""
import numpy as np
import pytest
import torch

from cczero_b200 import records as rd
from cczero_b200 import sl
from cczero_b200.env import StaticEnv, board_to_state, state_to_board, u16_to_move
from cczero_b200.lib import CzLib
from cczero_b200.optimize import OptimizeWorker, make_batches, validation_split
from oracle import senv as osenv
from tests.test_play_replay import RecordingTrainer, playout, run_worker
from tests.test_sl_workers import EMUL, config as sl_config, write_csv
from tests.test_sl_replay import fixture
from tests.test_train_host import _config
from tests.test_visit_records import with_visits


@pytest.fixture(scope="module")
def env(emul_lib):
    return StaticEnv(emul_lib, "cpu")


def msq(sq):
    return sq + 8 - 2 * (sq % 9)


def mirror_move(m):
    return '%d%s%d%s' % (8 - int(m[0]), m[1], 8 - int(m[2]), m[3])


def host_mirror_policy(policy, flags, m):
    out = policy.copy()
    for l in range(policy.shape[1]):
        out[flags, l] = policy[flags, m[l]]
    return out


# ------------------------------------------------------------------------------------------------ labels
def test_mirror_labels(env):
    m = env.mirror_labels.astype(np.int64)
    assert m.shape == (2086,) and (m[m] == np.arange(2086)).all()
    assert (m == np.arange(2086)).sum() == 90
    for l, s in enumerate(env.labels):
        assert env.labels[m[l]] == mirror_move(s)
        assert (m[l] == l) == (s[0] == '4' and s[2] == '4')
    assert [env.labels[x] for x in m] == [mirror_move(s) for s in osenv.ActionLabelsRed]
    lut = env.label_lut.reshape(90, 90).astype(np.int64)
    f, t = np.nonzero(lut >= 0)
    assert len(f) == 2086
    assert (lut[[msq(x) for x in f], [msq(x) for x in t]] == m[lut[f, t]]).all()


# ------------------------------------------------------------------------------------------------ boards
@pytest.fixture(scope="module")
def fixture_boards(env, golden_env):
    states = [r["state"] for r in golden_env["rows"]]
    return states, env.to_dev(np.stack([state_to_board(s) for s in states]))


def test_board_mirror_on_fixture_boards(env, fixture_boards):
    states, b = fixture_boards
    assert len(states) == 2145
    mb = env.mirror(b)
    host = b.numpy().copy()
    host[:, :90] = host[:, :90].reshape(-1, 10, 9)[:, :, ::-1].reshape(-1, 90)
    assert (mb.numpy() == host).all()
    assert (env.mirror(mb).numpy() == b.numpy()).all()                       # an involution
    assert (env.planes_batch(mb).numpy() == env.planes_batch(b).numpy()[..., ::-1]).all()
    mv, cnt = env.movegen_batch(b)
    mmv, mcnt = env.movegen_batch(mb)
    assert (cnt == mcnt).all()
    lut, m = env.label_lut, env.mirror_labels
    for i in range(len(states)):
        a = [u16_to_move(v) for v in mv[i, :int(cnt[i])].numpy().view(np.uint16)]
        c = [u16_to_move(v) for v in mmv[i, :int(cnt[i])].numpy().view(np.uint16)]
        assert sorted(mirror_move(x) for x in a) == sorted(c)
        for x in a:
            k = lut[(int(x[1]) * 9 + int(x[0])) * 90 + int(x[3]) * 9 + int(x[2])]
            y = mirror_move(x)
            if k >= 0:
                assert m[k] == lut[(int(y[1]) * 9 + int(y[0])) * 90 + int(y[3]) * 9 + int(y[2])]
    d, _ = env.done_batch(b, need_check=True)
    md, _ = env.done_batch(mb, need_check=True)
    assert (d[:, :3] == md[:, :3]).all()


def test_board_mirror_agrees_with_the_oracle(env, fixture_boards):
    states, b = fixture_boards
    mb = env.mirror(b).numpy()
    for i in range(0, len(states), 5):
        ms = board_to_state(mb[i])
        assert sorted(osenv.get_legal_moves(ms)) == sorted(mirror_move(x) for x in osenv.get_legal_moves(states[i]))
        assert list(osenv.done(ms, need_check=True))[:2] == list(osenv.done(states[i], need_check=True))[:2]


def test_flagged_mirror_leaves_other_rows_byte_identical(env, fixture_boards):
    _, b = fixture_boards
    b = b.clone()
    b[:, 90:] = torch.arange(6, dtype=torch.uint8) + 1                       # pad bytes travel with the row
    flags = torch.from_numpy(np.random.RandomState(5).randint(0, 2, len(b)).astype(np.uint8))
    out = env.mirror(b, flags).numpy()
    keep = flags.numpy() == 0
    assert keep.sum() > 500 and (~keep).sum() > 500
    assert out[keep].tobytes() == b.numpy()[keep].tobytes()
    assert (out[~keep] == env.mirror(b).numpy()[~keep]).all()
    assert (out[:, 90:] == b.numpy()[:, 90:]).all()


# ------------------------------------------------------------------------------------------------ SlDataset.batch
def _dataset(env, visits):
    rng = np.random.RandomState(11)
    games = [playout(rng, 30), playout(rng, 12, value=-1), playout(rng, 21)]
    if visits:
        games = [with_visits(g, rng, every=1 + i % 2) for i, g in enumerate(games)]
    packed = rd.pack_play_games([g for d in games for g in rd.split_games(d) if len(g) > 1], "test", visits=visits)
    return rd.replay_play_games(env.lib, env.device, packed, env.label_lut)


@pytest.mark.parametrize("visits", [False, True])
@pytest.mark.parametrize("history", [False, True])
def test_dataset_batch_mirror_equals_host_restatement(env, visits, history):
    ds = _dataset(env, visits)
    idx = np.random.RandomState(2).permutation(len(ds))[:40]
    flags = np.random.RandomState(3).randint(0, 2, len(idx))
    f = flags.astype(bool)
    p, pol, v = (t.numpy() for t in ds.batch(env, idx, history))
    mp, mpol, mv = (t.numpy() for t in ds.batch(env, idx, history, mirror=flags))
    assert mp.shape[1] == (28 if history else 14)
    want_p = p.copy()
    want_p[f] = p[f][..., ::-1]                                               # history planes mirrored with their position
    assert mp.tobytes() == want_p.tobytes()
    assert mpol.tobytes() == host_mirror_policy(pol, f, env.mirror_labels).tobytes()
    assert mv.tobytes() == v.tobytes()
    if not visits:
        lab = ds.labels.numpy()[idx].astype(np.int64)
        assert (mpol.argmax(1) == np.where(f, env.mirror_labels[lab], lab)).all()
    if history:
        assert p[:, 14:].any()


# ------------------------------------------------------------------------------------------------ workers
def _mirror_rows(plain, aug, m):
    """Each row of the augmented batch is the plain row or its mirror; returns how many are mirrored."""
    (p, pol, v), (ap, apol, av) = plain[:3], aug[:3]
    assert v.tobytes() == av.tobytes()
    mirrored = 0
    for i in range(len(p)):
        if ap[i].tobytes() == p[i].tobytes() and apol[i].tobytes() == pol[i].tobytes():
            continue
        assert ap[i].tobytes() == p[i][..., ::-1].tobytes() and apol[i].tobytes() == pol[i][m].tobytes()
        mirrored += 1
    return mirrored


@pytest.mark.parametrize("history", [False, True])
def test_optimize_worker_mirror_same_on_both_paths(env, tmp_path, monkeypatch, history):
    rng = np.random.RandomState(9)
    files = [(f"play_2026010{i}-000000.000000.json", playout(rng, int(rng.randint(10, 40)), value=int(rng.choice([-1, 1]))))
             for i in range(6)]
    orig = OptimizeWorker.__init__
    runs = {}
    for aug in (None, "mirror"):
        monkeypatch.setattr(OptimizeWorker, "__init__", lambda self, *a, **k: orig(self, *a, **k, augment=aug))
        runs[aug] = {path: run_worker(tmp_path / f"{path}_{aug}", files, env, path, history, load_data_steps=4, batch_size=12)
                     for path in ("host", "device")}
    h, d = runs["mirror"]["host"], runs["mirror"]["device"]
    assert len(h["steps"]) > 4 and len(h["steps"]) == len(d["steps"])
    for a, b in zip(h["steps"] + h["validations"], d["steps"] + d["validations"]):
        for x, y in zip(a, b):
            if isinstance(x, np.ndarray):
                assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes()
            else:
                assert x == y
    plain = runs[None]["host"]
    for a, b in zip(plain["validations"], h["validations"]):                  # the validation batch is never mirrored
        assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
    # the first epoch's shuffle comes before any flag is drawn: the same rows, about half of them mirrored
    mirrored = _mirror_rows(plain["steps"][0], h["steps"][0], env.mirror_labels)
    assert 0 < mirrored < len(h["steps"][0][0])


def test_optimize_worker_rejects_unknown_augment(tmp_path, env):
    with pytest.raises(ValueError):
        OptimizeWorker(_config(tmp_path), env=env, augment="flip")


def _fit_worker(tmp_path, env, dataset, augment):
    w = OptimizeWorker(_config(tmp_path), env=env, trainer_factory=RecordingTrainer, dataset=dataset, augment=augment)
    w.model = w.load_model()
    w.compile_model()
    return w


@pytest.mark.parametrize("dataset", ["host", "device"])
@pytest.mark.parametrize("augment", [None, "mirror"])
def test_fit_random_numbers(env, tmp_path, dataset, augment):
    """Without augment `fit` draws only its shuffles; with it, one randint of the epoch's length after each shuffle."""
    data = playout(np.random.RandomState(4), 60)
    if dataset == "host":
        x, pol, v = (np.concatenate(a) for a in zip(*[rd.expanding_data(g, env, False) for g in rd.split_games(data)]))
        n = len(x)
    else:
        ds = rd.replay_play_games(env.lib, env.device, rd.pack_play_games(rd.split_games(data), "test"), env.label_lut)
        n = len(ds)
    w = _fit_worker(tmp_path, env, dataset, augment)
    np.random.seed(21)
    if dataset == "host":
        w.fit(x, pol, v, 16, 3)
    else:
        w.fit_dataset(ds, 16, 3)
    after = np.random.get_state()
    np.random.seed(21)
    train_idx, _ = validation_split(n)
    for _ in range(3):
        order = train_idx.copy()
        np.random.shuffle(order)
        if augment:
            np.random.randint(0, 2, len(order))
    want = np.random.get_state()
    assert after[0] == want[0] and (after[1] == want[1]).all() and after[2:] == want[2:]
    assert len(w.trainer.steps) == 3 * len(make_batches(len(train_idx), 16))


class _Trainer:
    instances = []

    def __init__(self, model, batch_size, device, optimizer="sgd"):
        self.model, self.steps, self.val = model, [], []
        _Trainer.instances.append(self)

    def step(self, planes, policy, value, lr):
        self.steps.append((planes.numpy().copy(), policy.numpy().copy(), value.numpy().copy()))
        return np.array([1.0, 0.5, 0.5, 0.0])

    def validation_loss(self, planes, policy, value):
        self.val.append((planes.numpy().copy(), np.array(policy), np.array(value)))
        return 1.0, 0.5, 0.5, 0.0

    def export(self):
        return self.model.weights


def test_sl_worker_mirror(tmp_path, monkeypatch):
    games = fixture()["wxf"]
    monkeypatch.setattr(sl, "save_as_sl_best_model", lambda m: None)
    runs = {}
    for aug in (None, "mirror"):
        cfg = sl_config(tmp_path / str(aug), batch_size=64, game_step=len(games))
        write_csv(cfg, games)
        w = sl.SupervisedWorker(cfg, trainer_factory=_Trainer, device="cpu", lib=CzLib(EMUL), augment=aug)
        np.random.seed(0)
        w.start()
        runs[aug] = w.trainer
    plain, aug = runs[None], runs["mirror"]
    assert len(plain.steps) == len(aug.steps) > 1
    for a, b in zip(plain.val, aug.val):
        assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
    m = StaticEnv(CzLib(EMUL), "cpu").mirror_labels
    mirrored = sum(_mirror_rows(a, b, m) for a, b in zip(plain.steps, aug.steps))
    total = sum(len(s[0]) for s in aug.steps)
    assert 0.3 * total < mirrored < 0.7 * total
