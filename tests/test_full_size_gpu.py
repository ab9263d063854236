"""BASELINE.json configs[2] at FULL size (1024 concurrent games, 800 simulations per move, 256x20 network) through
size-independent properties: the oracle cannot run this size, so the checks are properties the search must have at any
size — replica agreement, size independence, visit conservation, determinism."""
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

G, SIMS, K, FILTERS, BLOCKS = 1024, 800, 8, 256, 20


def _weights():
    from cczero_b200.model import CChessModel
    cfg = SimpleNamespace(model=SimpleNamespace(cnn_filter_num=FILTERS, res_layer_num=BLOCKS, value_fc_size=256,
                                                cnn_first_filter_size=5, cnn_filter_size=3, input_depth=14))
    return CChessModel(cfg).build(seed=0).torch_weights()


def _engine(cuda_lib, n_games, weights, noise_eps):
    from cczero_b200.engine import Engine
    eng = Engine(cuda_lib, "cuda", n_games=n_games, sims_per_move=SIMS, leaves_per_round=K, noise_mode=1, noise_eps=noise_eps,
                 nn_filters=FILTERS, nn_blocks=BLOCKS, nn_value_fc=256, tau_decay_rate=0.9, seed=3)
    eng.set_weights(weights)
    eng.reset()
    return eng


def _roots(eng):
    from cczero_b200.records import RootStage
    st = RootStage(eng)
    n, moves, counts = eng.download_root_stats(st)
    return n.numpy().copy(), moves.numpy().copy(), counts.numpy().copy(), st.sims.numpy().copy()


def test_c3_full_size_replicas_agree_and_match_a_single_game(cuda_lib):
    """Root noise off: all 1024 games are the SAME search.  (a) every game's root statistics are bit-identical, (b) and
    identical to ONE game searched alone in its own engine — batch composition (8192 leaves per round vs 8) and the tile
    a position lands in must not leak into a game, (c) visits are conserved."""
    w = _weights()
    eng = _engine(cuda_lib, G, w, noise_eps=0.0)
    eng.search(None)
    n, moves, counts, sims = _roots(eng)
    assert int(eng.counters()[6]) == 0 and (sims == SIMS).all() and (counts == 44).all()
    assert (n == n[0]).all() and (moves == moves[0]).all()
    assert n[0, :44].sum() == SIMS - 1                      # the first simulation expands the root, the other 799 pass an edge
    r0, r511, r1023 = eng.root(0), eng.root(511), eng.root(1023)
    assert r0["w"] == r511["w"] == r1023["w"] and r0["p"] == r1023["p"]
    st = eng.search_stats()
    assert st["sims"] == G * SIMS and st["nodes_created"] + st["no_network"] == G * SIMS
    eng.close()
    one = _engine(cuda_lib, 1, w, noise_eps=0.0)
    one.search(None)
    r = one.root(0)
    assert r["n"] == r0["n"] and r["w"] == r0["w"] and r["p"] == r0["p"] and r["sum_n"] == r0["sum_n"] == SIMS
    one.close()


def test_c3_full_size_two_moves_conservation_and_determinism(cuda_lib):
    """With root noise and temperature sampling the games diverge after the first move.  Two identical runs must agree
    bit for bit (no race at full occupancy), every root conserves its visits, no error flag, no table reset."""
    w = _weights()

    def run():
        eng = _engine(cuda_lib, G, w, noise_eps=0.25)
        out = []
        for _ in range(2):
            eng.search(None)
            n, moves, counts, sims = _roots(eng)
            out.append((n, moves, counts, sims))
            for g in (0, 17, 1023):
                r = eng.root(g)
                assert sum(r["n"]) == r["sum_n"] - 1 and r["sum_n"] >= SIMS       # tree reuse keeps earlier visits
            eng.play_move()
        c = eng.counters()
        assert int(c[6]) == 0 and int(c[4]) == 0
        eng.close()
        return out
    a, b = run(), run()
    for x, y in zip(a, b):
        for u, v in zip(x, y):
            assert (u == v).all()
    n1, _, counts1, sims1 = a[1]
    assert (sims1 > 0).all() and (sims1 <= SIMS).all() and len({tuple(r) for r in n1[:64].tolist()}) > 8   # games did diverge
    for g in range(G):
        assert n1[g, :counts1[g]].sum() >= SIMS - 1
