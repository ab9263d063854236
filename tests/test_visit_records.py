"""Root visit counts recorded by the on-device game loop (cz_config.record_visits, emulator build of the same kernel source)
against the restated reference loop's calc_policy; the play-data format with visits; the visit-count training targets
on the host (records.expanding_data) and on the device (cz_visit_targets via SlDataset.batch), bit for bit; input
validation; OptimizeWorker with policy_target="visits" on both data paths; and the two-rank gather of the pairs."""
import json
import os
from collections import deque

import numpy as np
import pytest
import torch

from cczero_b200 import records as rd
from cczero_b200.engine import Engine
from cczero_b200.env import StaticEnv
from cczero_b200.optimize import OptimizeWorker
from oracle import player as op
from oracle import selfplay as osp
from oracle import senv as osenv
from tests.search_checks import eval_planes
from tests.test_play_replay import CountingLib, RecordingTrainer, playout, run_worker, write
from tests.test_train_host import _config

LABEL_OF = {m: i for i, m in enumerate(osenv.ActionLabelsRed)}


def engine(lib, device, n_games, sims, k, seed, max_game_length, tau_decay, use_history=False, record_visits=True, resign=-0.6,
           **kw):
    return Engine(lib, device, n_games=n_games, sims_per_move=sims, leaves_per_round=k, noise_mode=1, noise_eps=0.0,
                  c_puct=1.5, tau_decay_rate=tau_decay, max_game_length=max_game_length, resign_threshold=resign,
                  enable_resign_rate=0.5, min_resign_turn=4, seed=seed, max_nodes_per_game=sims * 2 * max_game_length + 64,
                  use_history=use_history, record_visits=record_visits, **kw)


def device_games(lib, device, n_games, sims, k, seed, want, max_game_length, tau_decay, use_history=False, record_visits=True,
                 resign=-0.6):
    eng = engine(lib, device, n_games, sims, k, seed, max_game_length, tau_decay, use_history, record_visits, resign)
    eng.reset()
    recs = []
    for _ in range(4 * max_game_length * (want // n_games + 2)):
        eng.search_external(eval_planes, None)
        if eng.play_move():
            recs += eng.drain_records()
        if len(recs) >= want:
            break
    assert int(eng.counters()[4]) == 0
    eng.close()
    return recs


def restated_visits(monkeypatch, pc, seed, n_games, r, max_game_length, use_history):
    """The restated loop's game of record r, with calc_policy's counts (no_act zeroed, n > 0) of every searched ply."""
    log = []

    class Recorder(op.OraclePlayer):
        def calc_policy(self, state, turns, no_act):
            node = self.tree[state]
            log.append(sorted((self.move_lookup[m], a.n) for m, a in node.a.items()
                              if a.n > 0 and not (no_act and m in no_act)))
            return super().calc_policy(state, turns, no_act)

    monkeypatch.setattr(osp, "OraclePlayer", Recorder)
    slot, started = r["game_index"] % n_games, r["game_index"] // n_games
    ref = osp.play_game(pc, op.fake_evaluate_states_hist if use_history else op.fake_evaluate_states,
                        osp.DeviceDraws(seed, 0, slot, started, LABEL_OF), max_game_length=max_game_length,
                        enable_resign_rate=0.5, use_history=use_history)
    return ref, log


def check_visits(monkeypatch, recs, n_games, sims, k, seed, max_game_length, tau_decay, use_history=False, resign=-0.6):
    pc = op.PlayConfig(simulation_num_per_move=sims, search_threads=k, c_puct=1.5, noise_eps=0.0, dirichlet_alpha=0.2,
                       tau_decay_rate=tau_decay, virtual_loss=3, resign_threshold=resign, min_resign_turn=4)
    kinds = set()
    for r in recs:
        ref, log = restated_visits(monkeypatch, pc, seed, n_games, r, max_game_length, use_history)
        assert r["moves"] == ref["moves"]
        resigned = bool(r["flags"] & 1)
        searched = len(log) - (1 if resigned else 0)             # a resign ply has counts but no move
        assert searched in (r["n_plies"], r["n_plies"] - 1)
        want = log[:searched] + [[]] * (r["n_plies"] - searched)  # the appended final king capture: no pairs
        assert r["visits"] == want, r["game_index"]
        for v, m in zip(r["visits"][:searched], r["moves"]):
            assert LABEL_OF[m] in dict(v)
        kinds.add("resign" if resigned else "capture" if searched < r["n_plies"] else "other")
    return kinds


CONFIGS = [dict(n_games=3, sims=20, k=4, seed=11, want=6, max_game_length=25, tau_decay=0.9),
           dict(n_games=2, sims=12, k=1, seed=3, want=3, max_game_length=14, tau_decay=0.0),
           dict(n_games=2, sims=10, k=16, seed=4, want=2, max_game_length=18, tau_decay=0.99),
           dict(n_games=2, sims=20, k=4, seed=5, want=3, max_game_length=25, tau_decay=0.9, use_history=True),
           dict(n_games=3, sims=10, k=4, seed=7, want=4, max_game_length=14, tau_decay=0.9, resign=0.9)]   # resigns


def test_emul_recorded_visits_equal_restated_calc_policy(emul_lib, monkeypatch):
    """Items 1 and 2: the pairs of every ply equal calc_policy's counts integer-exact (K = 1, K > sims, tau-decay 0 and
    0.99, history planes), and the same seed without recording plays the same records."""
    kinds = set()
    for c in CONFIGS:
        c = dict(c)
        want = c.pop("want")
        recs = device_games(emul_lib, "cpu", want=want, **c)
        plain = device_games(emul_lib, "cpu", want=want, record_visits=False, **c)
        assert [{k: v for k, v in r.items() if k != "visits"} for r in recs] == plain
        assert all("visits" not in r for r in plain)
        kinds |= check_visits(monkeypatch, recs, **c)
    assert {"resign", "capture"} <= kinds, kinds


def test_emul_workspace_grows_only_with_the_flag_and_arena_rejected(emul_lib):
    from cczero_b200.lib import CzError
    on, off = (engine(emul_lib, "cpu", 4, 8, 4, 1, 10, 0.9, record_visits=v) for v in (True, False))
    assert on.workspace_bytes > off.workspace_bytes
    with pytest.raises(CzError, match="record_visits"):
        Engine(emul_lib, "cpu", n_games=4, sims_per_move=8, max_game_length=10, arena=True, record_visits=True)
    with pytest.raises(CzError, match="record_visits"):
        off.visits_layout()
    on.close()
    off.close()


def test_emul_ring_overrun_keeps_correct_pairs(emul_lib, monkeypatch):
    """Item 3: driving cz_play_move past the ring without draining counts the dropped records; the kept ones carry the
    pairs of their own game."""
    from cczero_b200.lib import CzError
    c = dict(n_games=40, sims=2, k=2, seed=5, max_game_length=1, tau_decay=0.9)
    eng = engine(emul_lib, "cpu", **c)
    eng.reset()
    with pytest.raises(CzError, match="dropped"):
        for _ in range(8):
            eng.search_external(eval_planes, None)
            eng.play_move()
    assert int(eng.counters()[3]) > 0
    recs = eng.drain_records()
    assert len(recs) == 80
    eng.close()
    check_visits(monkeypatch, recs, **c)


# ------------------------------------------------------------------------------------------------ format and targets
def visit_list(rng, move, big=False):
    """A flat [l0, n0, ...] list holding the move's label and a few others, ascending labels."""
    labs = {LABEL_OF[move]} | set(rng.choice(2086, rng.randint(0, 12), replace=False).tolist())
    hi = 2 ** 32 - 1 if big else 900
    return [x for lab in sorted(labs) for x in (int(lab), int(rng.randint(1, hi)))]


def with_visits(data, rng, every=1, big=False):
    """Third elements on a share of the plies (never on the last one: the final-capture form)."""
    out = [data[0]]
    for i, it in enumerate(data[1:]):
        last = i == len(data) - 2
        out.append([it[0], it[1], visit_list(rng, it[0], big)] if (not last and i % every == 0) else list(it))
    return out


@pytest.fixture(scope="module")
def env(emul_lib):
    return StaticEnv(emul_lib, "cpu")


def test_play_data_format_with_visits():
    rec = {"moves": ["7747", "7062", "1219"], "value_red": -1, "visits": [[(5, 3), (40, 7)], [(2, 1)], []]}
    assert rd.record_to_play_data(rec) == [osenv.INIT_STATE, ["7747", -1, [5, 3, 40, 7]], ["7062", 1, [2, 1]], ["1219", -1]]


def test_visits_file_reads_like_the_file_without_them(env, tmp_path):
    """Item 4: with policy_target="move" a file with visits gives exactly the arrays of the file without them."""
    rng = np.random.RandomState(1)
    games = [playout(rng, 20), playout(rng, 9, value=-1)]
    data = games[0] + games[1]
    vis = with_visits(games[0], rng, every=2) + with_visits(games[1], rng)
    for hist in (False, True):
        a = [rd.expanding_data(g, env, hist) for g in rd.split_games(data)]
        b = [rd.expanding_data(g, env, hist) for g in rd.split_games(vis)]
        for x, y in zip(a, b):
            assert all(u.tobytes() == v.tobytes() for u, v in zip(x, y))
    ga, gb = rd.load_play_file(write(tmp_path / "a.json", data)), rd.load_play_file(write(tmp_path / "b.json", vis))
    assert all((getattr(ga, k) == getattr(gb, k)).all() for k in ("boards", "counts", "codes", "values"))


def host_targets(data, env, hist):
    out = [rd.expanding_data(g, env, hist, policy_target="visits") for g in rd.split_games(data) if len(g) > 1]
    return tuple(np.concatenate([o[i] for o in out]) for i in range(3))


def device_targets(data, env, hist):
    games = [g for g in rd.split_games(data) if len(g) > 1]
    parts = [rd.replay_play_games(env.lib, env.device, rd.pack_play_games(gs, "test", visits=True), env.label_lut)
             for gs in (games[:2], games[2:])]                       # extend() joins the CSR columns
    ds = parts[0].extend(parts[1])
    idx = np.random.RandomState(0).permutation(len(ds))
    p, pol, v = (t.cpu().numpy() for t in ds.batch(env, idx, hist))
    inv = np.argsort(idx)
    return p[inv], pol[inv], v[inv]


@pytest.mark.parametrize("hist", [False, True])
def test_device_targets_equal_host_expansion(env, hist):
    """Item 5: several games per file, plies with and without visits, final captures, counts up to 2^32 - 1."""
    rng = np.random.RandomState(3)
    data = (with_visits(playout(rng, 25), rng) + with_visits(playout(rng, 7, value=-1), rng, every=3)
            + playout(rng, 5) + with_visits(playout(rng, 12), rng, big=True))
    h, d = host_targets(data, env, hist), device_targets(data, env, hist)
    for a, b in zip(h, d):
        assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
    assert h[0].shape[1] == (28 if hist else 14)
    soft = (h[1] > 0).sum(1) > 1
    assert soft.sum() > 20 and (~soft).sum() > 5                     # both kinds of rows
    assert np.abs(h[1].sum(1) - 1).max() < 1e-5


def test_target_is_the_float64_ratio_rounded_once(env):
    data = [osenv.INIT_STATE, ["7747", 1, [LABEL_OF["7747"], 1, 7, 2, 9, 3]]]
    _, pol, _ = host_targets(data, env, False)
    assert pol[0, LABEL_OF["7747"]] == np.float32(1 / 6) and pol[0, 7] == np.float32(2 / 6) and pol[0, 9] == np.float32(3 / 6)


BAD = [("x", "not a list"), ([1], "odd length"), ([1, 2.0], "a float"), ([[1, 2]], "nested"), ([True, 1], "a bool"),
       ([2086, 1], "label out of range"), ([-1, 1], "negative label"), ([5, 0], "n = 0"), ([5, -3], "n < 0"),
       ([5, 2 ** 32], "n beyond u32"), ([5, 1, 5, 2], "duplicate label"), ([5, 2 ** 70], "n beyond int64")]


@pytest.mark.parametrize("bad,why", BAD, ids=[w for _, w in BAD])
@pytest.mark.parametrize("path", ["host", "device"])
def test_malformed_visits_raise_before_any_launch(emul_lib, tmp_path, bad, why, path):
    """Item 6: the file and the move are named; nothing is launched."""
    lib = CountingLib(emul_lib)
    data = playout(np.random.RandomState(2), 6)
    data[4] = [data[4][0], data[4][1], bad]
    p = write(tmp_path / "play_bad.json", data)
    w = OptimizeWorker(_config(tmp_path), env=StaticEnv(lib, "cpu"), trainer_factory=RecordingTrainer, dataset=path, policy_target="visits")
    w.filenames = deque([p])
    with pytest.raises(ValueError) as e:
        w.fill_queue()
    assert p in str(e.value) and repr(data[4][0]) in str(e.value), why
    assert set(lib.calls) <= {"cz_action_labels"}, lib.calls       # the label table is a host copy, not a launch


def test_optimize_worker_same_on_both_paths_with_visit_targets(env, tmp_path, monkeypatch):
    """Item 7: recording trainers get identical batches (targets included) and validation sets on both paths."""
    rng = np.random.RandomState(7)
    files = []
    for i in range(6):
        data = with_visits(playout(rng, int(rng.randint(8, 40)), value=int(rng.choice([-1, 1]))), rng, every=1 + i % 2)
        if i % 3 == 0:
            data += playout(rng, int(rng.randint(1, 6)))
        files.append((f"play_2026010{i}-000000.000000.json", data))
    orig = OptimizeWorker.__init__
    monkeypatch.setattr(OptimizeWorker, "__init__", lambda self, *a, **k: orig(self, *a, **k, policy_target="visits"))
    runs = {path: run_worker(tmp_path / path, files, env, path, True, load_data_steps=4, batch_size=12)
            for path in ("host", "device")}
    h, d = runs["host"], runs["device"]
    assert len(h["steps"]) > 4 and len(h["steps"]) == len(d["steps"]) and len(h["validations"]) == len(d["validations"])
    soft = 0
    for a, b in zip(h["steps"] + h["validations"], d["steps"] + d["validations"]):
        for x, y in zip(a, b):
            if isinstance(x, np.ndarray):
                assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes()
            else:
                assert x == y
        soft += int(((a[1] > 0).sum(1) > 1).sum())
    assert soft > 0
    for k in ("lrs", "total_steps", "trained", "left", "history"):
        assert h[k] == d[k], k


# ------------------------------------------------------------------------------------------------ two ranks over gloo
def _worker(rank, world, port, emul_path, out):
    import sys
    import torch.distributed as dist
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from cczero_b200.engine import Engine
    from cczero_b200.lib import CzLib
    from cczero_b200 import records
    from tests.search_checks import eval_planes
    eng = Engine(CzLib(emul_path), "cpu", n_games=2, sims_per_move=12, leaves_per_round=4, noise_mode=1, noise_eps=0.25,
                 max_game_length=8, seed=3, rank=rank, max_nodes_per_game=2048, record_visits=True)
    eng.reset()
    finished = 0
    for _ in range(60):
        eng.search_external(eval_planes, None)
        finished += eng.play_move()
        if finished >= 2 + 2 * rank:
            break
    import ctypes as C
    ptr, used = C.c_void_p(0), C.c_uint64(0)
    eng.lib.call("cz_record_visits_buffer", eng._h, C.byref(ptr), C.byref(used))
    gathered, total = records.gather_records(eng, dist, world, clear=False)
    mine = eng.drain_records()
    out.put((rank, used.value, eng.visits_gathered_bytes, eng.visits_layout()[3], mine, gathered))
    eng.close()
    dist.destroy_process_group()


def test_two_ranks_gather_the_pairs(emul_lib):
    """Item 8: rank 0 decodes every rank's pairs equal to that rank's own drain; the heap bytes shipped per rank are the
    largest used length, not the worst case."""
    from tests.test_multiproc import _spawn
    (r0, u0, g0, cap0, mine0, gath0), (r1, u1, g1, cap1, mine1, gath1) = _spawn(_worker, (emul_lib.path,))
    assert gath1 is None and u0 != u1
    assert g0 == g1 == max(u0, u1) < cap0
    assert [rec for r, rec in gath0 if r == 0] == mine0 and [rec for r, rec in gath0 if r == 1] == mine1
    assert all(len(rec["visits"]) == rec["n_plies"] for rec in mine0 + mine1)
    assert sum(len(v) for rec in mine0 + mine1 for v in rec["visits"]) > 0
