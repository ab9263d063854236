"""Control flow of the supervised workers (cczero_b200.sl / sl_onegreen) against worker/sl.py and worker/sl_onegreen.py,
on the emulator's rules kernels with a recording fake trainer: chunking by sl_game_step, the `> batch_size` gate, the
dataset carried over or cleared, one save per trained chunk to the sl_best paths, Adam's lr, one trainer for the run,
`skip`, skipped games, and the 28-plane rejection."""
import json
import os
from types import SimpleNamespace

import numpy as np
import pytest

from cczero_b200 import sl, sl_onegreen
from cczero_b200.lib import CzLib
from tests.test_sl_replay import ROOT, fixture

EMUL = os.path.join(ROOT, "tests", "simt_emul", "libcz_emul.so")


class RecordingTrainer:
    instances = []

    def __init__(self, model, batch_size, device, optimizer="sgd"):
        self.model, self.batch_size, self.optimizer = model, batch_size, optimizer
        self.steps, self.val = [], []
        RecordingTrainer.instances.append(self)

    def step(self, planes, policy, value, lr):
        self.steps.append((tuple(planes.shape), float(lr), policy.argmax(1).numpy().copy(), value.numpy().copy()))
        return np.array([1.0, 0.5, 0.5, 0.0])

    def validation_loss(self, planes, policy, value):
        self.val.append(len(planes))
        return 1.0, 0.5, 0.5, 0.0

    def export(self):
        return self.model.weights


def config(tmp_path, batch_size=16, game_step=10, in_planes=14):
    d = str(tmp_path)
    mc = SimpleNamespace(cnn_filter_num=64, res_layer_num=1, value_fc_size=32, l2_reg=1e-4, input_depth=in_planes,
                         policy_channels=4, value_channels=2, cnn_first_filter_size=5, cnn_filter_size=3)
    tc = SimpleNamespace(batch_size=batch_size, sl_game_step=game_step, epoch_to_checkpoint=1, start_total_steps=0,
                         loss_weights=[1.0, 1.0], dataset_size=100000)
    rc = SimpleNamespace(sl_best_config_path=os.path.join(d, "model", "sl_best_config.json"),
                         sl_best_weight_path=os.path.join(d, "model", "sl_best_weight.npz"),
                         sl_data_gameinfo=os.path.join(d, "sl", "gameinfo.csv"), sl_data_move=os.path.join(d, "sl", "moves.csv"),
                         sl_onegreen=os.path.join(d, "sl", "onegreen.json"))
    return SimpleNamespace(model=mc, trainer=tc, resource=rc, opts=SimpleNamespace(new=True, light=True))


def write_csv(cfg, games):
    os.makedirs(os.path.dirname(cfg.resource.sl_data_gameinfo), exist_ok=True)
    with open(cfg.resource.sl_data_gameinfo, "w", encoding="utf-8") as f:
        f.write("gameID,winner\n" + "".join(f"{g['id']},{g['winner']}\n" for g in games))
    with open(cfg.resource.sl_data_move, "w", encoding="utf-8") as f:
        f.write("gameID,turn,side,move\n" + "".join(f"{r['gameID']},{r['turn']},{r['side']},{r['move']}\n"
                                                     for g in games for r in g["rows"]))


def write_json(cfg, games):
    os.makedirs(os.path.dirname(cfg.resource.sl_onegreen), exist_ok=True)
    with open(cfg.resource.sl_onegreen, "w", encoding="utf-8") as f:
        json.dump([{k: g[k] for k in ("init", "move_list", "result", "title", "url")} for g in games], f, ensure_ascii=False)


def ref_chunks(games, step, batch_size, skip=0):
    """The reference's loop on the fixture's expected records: per chunk, the positions loaded and whether it trains."""
    out, carried = [], 0
    for i in range(skip, len(games), step):
        carried += sum(len(g["ref"]["records"]) for g in games[i:i + step] if not g["ref"]["raised"])
        train = carried > batch_size
        out.append((carried, train))
        if train:
            carried = 0
    return out


def run(worker, monkeypatch):
    saves = []
    monkeypatch.setattr(sl, "save_as_sl_best_model", lambda m: saves.append(m.config.resource.sl_best_weight_path))
    RecordingTrainer.instances = []
    return saves


def test_wxf_worker_control_flow(tmp_path, monkeypatch):
    games = fixture()["wxf"]
    cfg = config(tmp_path, batch_size=150, game_step=7)
    write_csv(cfg, games)
    w = sl.SupervisedWorker(cfg, trainer_factory=RecordingTrainer, device="cpu", lib=CzLib(EMUL))
    saves = run(w, monkeypatch)
    np.random.seed(0)
    w.start()
    assert len(RecordingTrainer.instances) == 1                         # one compile: Adam's iterations run on
    tr = RecordingTrainer.instances[0]
    assert tr.optimizer == "adam" and all(s[1] == 1e-2 for s in tr.steps)
    chunks = ref_chunks(games, 7, 150)
    trained = [n for n, t in chunks if t]
    assert len(saves) == 1 + len(trained)                              # the fresh model, then one save per trained chunk
    assert all(p == cfg.resource.sl_best_weight_path for p in saves)
    # per trained chunk: batches over the first 98 % of its positions, the last one partial, and one validation pass
    want = []
    for n in trained:
        ntr = int(n * 0.98)
        want += [min(150, ntr - a) for a in range(0, ntr, 150)]
    assert [s[0][0] for s in tr.steps] == want
    assert tr.val == [n - int(n * 0.98) for n in trained]
    assert w.skipped + w.failed == sum(1 for g in games if g["ref"]["raised"])
    assert len(w.dataset) == (chunks[-1][0] if not chunks[-1][1] else 0)   # an untrained tail stays queued


def test_onegreen_worker_skip_and_lr(tmp_path, monkeypatch):
    games = fixture()["onegreen"]
    cfg = config(tmp_path, batch_size=100, game_step=6)
    write_json(cfg, games)
    w = sl_onegreen.SupervisedWorker(cfg, trainer_factory=RecordingTrainer, device="cpu", lib=CzLib(EMUL))
    saves = run(w, monkeypatch)
    np.random.seed(0)
    w.games = None
    w.model = w.load_model()
    with open(cfg.resource.sl_onegreen, encoding="utf-8") as f:
        w.games = json.load(f)
    w.training(skip=5)
    tr = RecordingTrainer.instances[0]
    assert tr.optimizer == "adam" and all(s[1] == 0.003 for s in tr.steps)
    norm = [dict(g, ref=dict(g["ref"], raised=g["ref"]["raised"] or g["ref"]["dropped"])) for g in games]
    chunks = ref_chunks(norm, 6, 100, skip=5)
    trained = [n for n, t in chunks if t]
    assert len(saves) == 1 + len(trained)
    assert sum(s[0][0] for s in tr.steps) == sum(int(n * 0.98) for n in trained)


def test_history_network_is_rejected(tmp_path, monkeypatch):
    cfg = config(tmp_path, in_planes=28)
    w = sl.SupervisedWorker(cfg, trainer_factory=RecordingTrainer, device="cpu", lib=CzLib(EMUL))
    run(w, monkeypatch)
    w.model = w.load_model()
    with pytest.raises(ValueError, match="28"):
        w.compile_model()


def test_build_policy_is_the_reference_label(tmp_path):
    w = sl.SupervisedWorker(config(tmp_path), device="cpu", lib=CzLib(EMUL))
    p = w.build_policy("0001", flip=False)
    assert p.sum() == 1 and w._env().labels[int(p.argmax())] == "0001"
    q = w.build_policy("0001", flip=True)
    assert w._env().labels[int(q.argmax())] == "8988"
    with pytest.raises(KeyError):
        w.build_policy("0000", flip=False)
