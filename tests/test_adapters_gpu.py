"""Reference-facing drop-ins on the GPU: CChessModel / CChessModelAPI wire protocol, CChessPlayer with the built-in
network, SelfPlayWorker play-data files."""
import json
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import model as om
from oracle import player as op
from oracle import senv as osenv

pytestmark = pytest.mark.gpu


def _config(tmp, filters=64, blocks=2, sims=32, k=4):
    play = SimpleNamespace(simulation_num_per_move=sims, search_threads=k, c_puct=1.5, noise_eps=0.25, dirichlet_alpha=0.2,
                           tau_decay_rate=0.98, virtual_loss=3, resign_threshold=-0.92, min_resign_turn=20, max_game_length=12,
                           enable_resign_rate=0.5, max_processes=2)
    model = SimpleNamespace(cnn_filter_num=filters, res_layer_num=blocks, value_fc_size=256, cnn_first_filter_size=5,
                            cnn_filter_size=3, input_depth=14, l2_reg=1e-4)
    res = SimpleNamespace(play_data_dir=os.path.join(tmp, "play_data"), play_data_filename_tmpl="play_%s.json",
                          model_best_config_path=os.path.join(tmp, "model", "model_best_config.json"),
                          model_best_weight_path=os.path.join(tmp, "model", "model_best_weight.npz"))
    return SimpleNamespace(play=play, model=model, resource=res, opts=SimpleNamespace(evaluate=False),
                           play_data=SimpleNamespace(nb_game_in_file=1))


def test_model_api_serves_reference_wire_protocol(cuda_lib, tmp_path):
    """An oracle (reference-algorithm) player talks to CChessModelAPI over a Pipe exactly like player.py:108-143."""
    from cczero_b200.model import CChessModel
    cfg = _config(str(tmp_path))
    model = CChessModel(cfg).build(seed=4)
    model.save(cfg.resource.model_best_config_path, cfg.resource.model_best_weight_path)
    m2 = CChessModel(cfg)
    assert m2.load(cfg.resource.model_best_config_path, cfg.resource.model_best_weight_path)
    assert m2.digest == model.digest and set(m2.weights) == set(model.weights)
    pipe = m2.get_pipes()
    states = [osenv.INIT_STATE, osenv.step(osenv.INIT_STATE, "1219")]
    pipe.send([osenv.state_to_planes(s) for s in states])
    assert pipe.poll(60), f"prediction worker did not answer: {m2.api.last_error!r}"
    rets = pipe.recv()
    assert len(rets) == 2 and rets[0][0].shape == (2086,) and isinstance(rets[0][1], float)
    ref_p, ref_v = om.forward(model.weights, np.stack([osenv.state_to_planes(s) for s in states]), 2)
    for (p, v), rp, rv in zip(rets, ref_p, ref_v):
        assert np.abs(p - rp).max() < 1e-3 and abs(v - rv) < 1e-3

    # a reference-algorithm player searching through that pipe
    def evaluate(ss):
        pipe.send([osenv.state_to_planes(s) for s in ss])
        assert pipe.poll(60), f"prediction worker did not answer: {m2.api.last_error!r}"
        return pipe.recv()
    pl = op.OraclePlayer(op.PlayConfig(simulation_num_per_move=40, search_threads=4), evaluate)
    np.random.seed(0)
    a, pol = pl.action(osenv.INIT_STATE, 0)
    assert a in osenv.get_legal_moves(osenv.INIT_STATE) and abs(sum(pol) - 1) < 1e-9
    m2.close_pipes()


def test_player_with_builtin_network(cuda_lib, tmp_path):
    from cczero_b200.model import CChessModel
    from cczero_b200.player import CChessPlayer
    cfg = _config(str(tmp_path), sims=48, k=4)
    model = CChessModel(cfg).build(seed=2)
    np.random.seed(1)
    player = CChessPlayer(cfg, pipes=None, weights=model.torch_weights())
    state, turns = osenv.INIT_STATE, 0
    for _ in range(3):
        a, pol = player.action(state, turns)
        assert a in osenv.get_legal_moves(state)
        root = player.engine.root(0)
        assert root["sum_n"] >= 48 and sum(root["n"]) >= 40
        state = osenv.step(state, a)
        turns += 1
    player.close()


def test_selfplay_worker_writes_reference_records(cuda_lib, tmp_path):
    from cczero_b200.self_play import SelfPlayWorker
    cfg = _config(str(tmp_path), sims=16, k=4)
    w = SelfPlayWorker(cfg, concurrent_games=8, seed=3)
    v, turns, state, store = w.start_game(1, None)
    assert v in (-1, 0, 1) and turns > 0
    recs = w.play_games(4)
    assert len(recs) >= 4
    files = sorted(os.listdir(cfg.resource.play_data_dir)) if os.path.isdir(cfg.resource.play_data_dir) else []
    stored = [r for r in recs if not (r["flags"] & 4)]
    assert len(files) >= min(1, len(stored))
    for fn in files:
        data = json.load(open(os.path.join(cfg.resource.play_data_dir, fn)))
        assert data[0] == osenv.INIT_STATE
        s = data[0]
        val = data[1][1]
        for i, (m, vv) in enumerate(data[1:]):
            assert m in osenv.get_legal_moves(s), (fn, i, m)
            assert vv == val * (-1) ** i
            s = osenv.step(s, m)
    w.close()


def test_history_network_builtin_search_and_worker(cuda_lib, tmp_path):
    """use_history (28 planes): cz_search with the built-in network == the same search driven through cz_leaf_planes +
    cz_nn_forward (the planes an external CChessModelAPI would see); the self-play worker runs on such a network."""
    from cczero_b200.engine import Engine
    from cczero_b200.model import CChessModel
    from cczero_b200.self_play import SelfPlayWorker
    from tests.search_checks import game_history
    cfg = _config(str(tmp_path), sims=16, k=4)
    cfg.model.input_depth = 28
    model = CChessModel(cfg).build(seed=6)
    assert model.use_history and model.weights["input_conv-5-64/kernel"].shape == (5, 5, 28, 64)
    hists = [game_history(12, 3), None, game_history(2, 4)]
    states = [hists[0][-1], osenv.INIT_STATE, hists[2][-1]]

    def run(external):
        eng = Engine(cuda_lib, "cuda", n_games=3, sims_per_move=64, leaves_per_round=8, noise_mode=1, nn_filters=64, nn_blocks=2,
                     seed=5, use_history=True)
        eng.set_weights(model.torch_weights())
        eng.reset(states)
        opts = eng.make_opts(hist=hists)
        seen = []
        if external:
            def ev(planes):
                t = torch.as_tensor(planes).cuda()
                seen.append(t[:, 14:].abs().sum().item())
                p, v = eng.nn_forward_planes(t)
                return p.cpu().numpy(), v.cpu().numpy()
            eng.search_external(ev, opts)
        else:
            eng.search(opts)
        out = [(eng.root(g)["n"], eng.root(g)["w"]) for g in range(3)]
        assert int(eng.counters()[6]) == 0
        eng.close()
        return out, seen
    a, _ = run(False)                                     # device-driven loop (graphs, legal priors from logits)
    b, seen = run(True)                                   # host-driven, full softmax vectors through the reference-facing API
    assert a == b and sum(seen) > 0
    model.save(cfg.resource.model_best_config_path, cfg.resource.model_best_weight_path)
    w = SelfPlayWorker(cfg, concurrent_games=4, seed=3, use_history=True, model=model)
    recs = w.play_games(2)
    assert len(recs) >= 2 and all(r["n_plies"] > 0 for r in recs)
    w.close()


def test_search_loop_forms_agree(cuda_lib):
    """cz_search runs as one WHILE-graph launch, the production graph or, while cz_nn_profile is on, the profiled one (the
    same iteration with timestamp kernels around the tower); the first search of each runs its first iteration as plain
    launches.  Both give the per-game results of the Python loop over the public wave / forward / apply API."""
    from cczero_b200.engine import Engine
    from cczero_b200.model import CChessModel
    cfg = _config("/tmp", filters=64, blocks=2)
    weights = CChessModel(cfg).build(seed=9).torch_weights()

    def run(mode):
        eng = Engine(cuda_lib, "cuda", n_games=1024, sims_per_move=24, leaves_per_round=8, noise_mode=1, nn_filters=64,
                     nn_blocks=2, seed=5, max_nodes_per_game=512)
        eng.set_weights(weights)
        if mode == "profiled":
            eng.nn_profile(True)
        eng.reset()
        out = []
        for _ in range(3):
            if mode == "host":
                eng.search_begin(None)
                eng.run_waves(None, host_loop=True)
            else:
                eng.search(None)
            out.append([(eng.root(g)["n"], eng.root(g)["sum_n"]) for g in (0, 511, 512, 1023)])
            eng.play_move()
        sims = eng.sims_run().tolist()
        eng.close()
        return out, sims

    a, sa = run("while")
    b, sb = run("profiled")
    c, sc = run("host")
    assert a == b == c and sa == sb == sc


@pytest.mark.parametrize("arena", [False, True], ids=["one_network", "arena"])
def test_nn_profile_counts_every_bracketed_tower(cuda_lib, cuda_env, arena):
    """cz_nn_profile: while on, every range of every search iteration brackets its residual tower once (the profiled WHILE
    graph, on its first search and after), and so does every cz_nn_forward_boards; the flops are those towers' positions
    times their algorithmic flops, exactly.  Nothing accumulates while it is off."""
    from cczero_b200.engine import Engine
    from cczero_b200.model import CChessModel
    from tests import search_checks as chk
    filters, blocks, n_games = 64, 2, 64
    per_position = 2 * 90 * 9 * filters * filters * 2 * blocks
    weights = CChessModel(_config("/tmp", filters=filters, blocks=blocks)).build(seed=9).torch_weights()
    eng = Engine(cuda_lib, "cuda", n_games=n_games, sims_per_move=24, leaves_per_round=8, nn_filters=filters, nn_blocks=blocks,
                 seed=5, arena=arena)
    eng.set_weights(weights)
    if arena:
        eng.set_weights(weights, net=1)
    opts = eng.make_opts(active=[1] * n_games)
    boards = cuda_env.boards_from_states([osenv.INIT_STATE] + chk.midgame_states(9, 2))

    def search():
        eng.reset()
        eng.search(opts)

    search()                                              # the production graph
    eng.nn_forward_boards(boards)
    assert eng.nn_profile(True) == (0.0, 0, 0.0)
    for _ in range(2):                                    # the profiled graph's first search, then one launch of it
        c0 = eng.counters()
        search()
        c1 = eng.counters()
        ms, launches, flops = eng.nn_profile(True)
        waves, positions = int(c1[2] - c0[2]), int(c1[1] - c0[1])   # waves: one per range per iteration
        assert waves > 0 and launches == 2 * blocks * waves
        assert flops == positions * per_position and ms > 0
    eng.nn_forward_boards(boards)
    ms, launches, flops = eng.nn_profile(False)
    assert launches == 2 * blocks and flops == len(boards) * per_position and ms > 0
    search()
    eng.nn_forward_boards(boards)
    assert eng.nn_profile(False) == (0.0, 0, 0.0)
    eng.close()


def test_evaluator_arena_two_networks(cuda_lib, tmp_path):
    """worker/evaluator drop-in: two different networks, alternating colours, tallies add up."""
    from cczero_b200.evaluator import EvaluateWorker
    from cczero_b200.model import CChessModel
    cfg = _config(str(tmp_path), sims=24, k=4)
    cfg.play.tau_decay_rate = 0
    cfg.play.noise_eps = 0.2
    cfg.play.c_puct = 1
    cfg.eval = SimpleNamespace(game_num=2)
    bt, ng = CChessModel(cfg).build(seed=1), CChessModel(cfg).build(seed=2)
    w = EvaluateWorker(cfg, bt, ng, n_games=6, concurrent_games=4, seed=3, playouts=None)
    total, rw, rd, rf, bw, bd, bf = w.start()
    assert rw + rd + rf + bw + bd + bf == 6
    assert 0 <= total <= 6 and abs(total - (rw + bw + 0.5 * (rd + bd))) < 1e-9
    assert int(w.engine.counters()[6]) == 0
    w.close()
    # identical networks on both sides and no randomness: the same game is played from both colours
    cfg.play.noise_eps = 0
    w = EvaluateWorker(cfg, bt, bt, n_games=4, concurrent_games=4, seed=3, playouts=None)
    w.engine.selfplay(target_games=4, max_moves=0)
    recs = sorted(w.engine.drain_records(), key=lambda r: r["game_index"])
    assert recs[0]["moves"] == recs[1]["moves"] and recs[0]["value_red"] == recs[1]["value_red"]
    w.close()


def test_c3_shaped_builtin_search_equals_wave_apply(cuda_lib):
    """BASELINE configs[2] shape (1024 games x K = 8, 14 planes, 256x20 network, fp32 skip stream): the integrated
    `cz_search` (legal priors taken from the logits on the device) gives bit for bit the statistics of the same search driven
    from the host through cz_search_wave / cz_leaf_boards / cz_nn_forward_boards / cz_search_apply, i.e. through the full
    [n][2086] softmax vectors of the reference-facing network API (VERDICT r1 weak 1c).  Both WHILE graphs of the device loop
    are checked: `while` the production one, `profiled` (cz_nn_profile on) the one with timestamp kernels around the tower;
    each runs its first move's first iteration as plain launches and the rest as graph launches."""
    from cczero_b200.engine import Engine
    from cczero_b200.model import CChessModel
    from cczero_b200.records import RootStage
    cfg = _config("/tmp", filters=256, blocks=20)
    weights = CChessModel(cfg).build(seed=4).torch_weights()

    def run(mode):
        eng = Engine(cuda_lib, "cuda", n_games=1024, sims_per_move=40, leaves_per_round=8, noise_mode=1, nn_filters=256,
                     nn_blocks=20, seed=11, max_nodes_per_game=1024)
        eng.set_weights(weights)
        if mode == "profiled":
            eng.nn_profile(True)
        eng.reset()
        st = RootStage(eng)
        out = []
        for _ in range(2):                                   # second move: tree reuse + a different position per game
            if mode == "host":
                eng.search_begin(None)
                eng.run_waves(None, host_loop=True)
            else:
                eng.search(None)
            n, mv, cnt = eng.download_root_stats(st)
            roots = [eng.root(g) for g in (0, 1, 511, 512, 777, 1023)]
            out.append((n.clone(), mv.clone(), cnt.clone(), [(r["n"], r["w"], r["p"], r["sum_n"]) for r in roots]))
            eng.play_move()
        assert int(eng.counters()[6]) == 0
        eng.close()
        return out
    host, while_, profiled = run("host"), run("while"), run("profiled")
    for a in (while_, profiled):
        for (n0, m0, c0, r0), (n1, m1, c1, r1) in zip(host, a):
            assert torch.equal(n0, n1) and torch.equal(m0, m1) and torch.equal(c0, c1)
            assert r0 == r1                                  # N, W (f64), P (f32), sum_n of sampled roots, exactly
    assert int(host[1][0].sum()) > int(host[0][0].sum()) * 0.9
