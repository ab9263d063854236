"""Mirror-averaged leaf evaluation in the device search (cz_config.eval_mirror): the integrated search equals, bit for bit,
a host loop that evaluates every wave's leaves and their mirrors in ONE cz_nn_forward_boards and averages in torch float32
(production and profiled WHILE graphs, 14 and 28 planes, an arena of two networks, the c3 shape's 16 384-row batch); root
root priors and values are equivariant under the mirror; with the flag off the workspace and launches are the parent's."""
import ctypes as C

import numpy as np
import pytest
import torch

from cczero_b200.lib import CzConfig, CzError
from tests import search_checks as chk
from tests.test_adapters_gpu import _config

pytestmark = pytest.mark.gpu


def weights(filters, blocks, seed, hist=False):
    from cczero_b200.model import CChessModel
    cfg = _config("/tmp", filters=filters, blocks=blocks)
    cfg.model.input_depth = 28 if hist else 14
    return CChessModel(cfg).build(seed=seed).torch_weights()


def host_mirror_waves(eng, env):
    """cz_search_wave / cz_leaf_boards, one cz_nn_forward_boards on cat([b, Mb]), the average in float32, cz_search_apply."""
    m = torch.as_tensor(env.mirror_labels.astype(np.int64), device="cuda")
    while True:
        n, busy = eng.search_wave()
        if n > 0:
            b = eng.leaf_boards(n)
            mb = env.mirror(b.reshape(-1, 96)).reshape(b.shape)          # history engines: both boards of the record
            pol, val = eng.nn_forward_boards(torch.cat([b, mb]))
            eng.search_apply(((pol[:n] + pol[n:][:, m]) * 0.5).contiguous(), ((val[:n] + val[n:]) * 0.5).contiguous())
        if not busy:
            return


def run(cuda_lib, env, mode, n_games, k, filters, blocks, sims, hist=False, arena=False, moves=2, nets=None):
    from cczero_b200.engine import Engine
    from cczero_b200.records import RootStage
    eng = Engine(cuda_lib, "cuda", n_games=n_games, sims_per_move=sims, leaves_per_round=k, noise_mode=1, nn_filters=filters,
                 nn_blocks=blocks, seed=11, max_nodes_per_game=max(512, 24 * sims), use_history=hist, arena=arena,
                 eval_mirror=True)
    for i, w in enumerate(nets):
        eng.set_weights(w, net=i)
    if mode == "profiled":
        eng.nn_profile(True)
    eng.reset()
    st = RootStage(eng)
    out = []
    games = sorted({0, 1, n_games // 2 - 1, n_games // 2, n_games - 1})
    for _ in range(moves):
        if mode == "host":
            eng.search_begin(None)
            host_mirror_waves(eng, env)
        else:
            eng.search(None)
        n, mv, cnt = eng.download_root_stats(st)
        roots = [eng.root(g) for g in games]
        out.append((n.clone(), mv.clone(), cnt.clone(), [(r["n"], r["w"], r["p"], r["sum_n"]) for r in roots]))
        eng.play_move()
    assert int(eng.counters()[6]) == 0
    eng.close()
    return out


def assert_same(a, b):
    for (n0, m0, c0, r0), (n1, m1, c1, r1) in zip(a, b):
        assert torch.equal(n0, n1) and torch.equal(m0, m1) and torch.equal(c0, c1)
        assert r0 == r1                                      # N, W (f64), P (f32), sum_n of sampled roots, exactly


@pytest.mark.parametrize("hist", [False, True], ids=["14planes", "28planes"])
def test_integrated_equals_host_restatement(cuda_lib, cuda_env, hist):
    nets = [weights(64, 2, 4, hist)]
    host = run(cuda_lib, cuda_env, "host", 64, 8, 64, 2, 48, hist=hist, nets=nets)
    for mode in ("while", "profiled"):
        assert_same(host, run(cuda_lib, cuda_env, mode, 64, 8, 64, 2, 48, hist=hist, nets=nets))
    assert int(host[1][0].sum()) > 0


def test_arena_two_networks(cuda_lib, cuda_env):
    """Each range evaluates with its own network in the mirror form: both graphs agree, and the first range's games equal
    those of an arena with net 0 on both sides, the second range's those with net 1 on both sides (neither range's rows
    are overwritten by the other's mirrors)."""
    nets = [weights(64, 2, 4), weights(64, 2, 5)]
    a = run(cuda_lib, cuda_env, "while", 32, 4, 64, 2, 32, arena=True, nets=nets, moves=1)
    b = run(cuda_lib, cuda_env, "profiled", 32, 4, 64, 2, 32, arena=True, nets=nets, moves=1)
    assert_same(a, b)
    c = run(cuda_lib, cuda_env, "while", 32, 4, 64, 2, 32, arena=True, nets=[nets[0], nets[0]], moves=1)
    d = run(cuda_lib, cuda_env, "while", 32, 4, 64, 2, 32, arena=True, nets=[nets[1], nets[1]], moves=1)
    assert torch.equal(a[0][0][:16], c[0][0][:16]) and torch.equal(a[0][0][16:], d[0][0][16:])
    assert int(a[0][0][:16].sum()) > 0


def test_c3_shape_16384_rows(cuda_lib, cuda_env):
    """1024 games x K = 8 with eval_mirror: the network evaluates up to 16 384 rows per round."""
    nets = [weights(256, 20, 4)]
    host = run(cuda_lib, cuda_env, "host", 1024, 8, 256, 20, 40, nets=nets)
    assert_same(host, run(cuda_lib, cuda_env, "while", 1024, 8, 256, 20, 40, nets=nets))
    assert int(host[0][0].sum()) > 1024 * 30


def mirror_move(m):
    return '%d%s%d%s' % (8 - int(m[0]), m[1], 8 - int(m[2]), m[3])


@pytest.mark.parametrize("hist", [False, True], ids=["14planes", "28planes"])
def test_root_priors_and_values_are_equivariant(cuda_lib, cuda_env, hist):
    """Game 2i at P, game 2i+1 at M(P), no noise: the root's priors of mirrored moves agree to the renormalisation's
    rounding, and after the second simulation the visited (mirrored) child's N and W are equal bit for bit."""
    from cczero_b200.engine import Engine
    from cczero_b200.env import board_to_state, state_to_board
    states = chk.midgame_states(12, 3)
    boards = []
    for s in states:
        b = state_to_board(s)
        boards += [b, cuda_env.mirror(cuda_env.to_dev(b[None])).cpu().numpy()[0]]
    eng = Engine(cuda_lib, "cuda", n_games=len(boards), sims_per_move=2, leaves_per_round=1, noise_mode=0, noise_eps=0.0,
                 nn_filters=64, nn_blocks=2, seed=1, use_history=hist, eval_mirror=True)
    eng.set_weights(weights(64, 2, 7, hist))
    eng.reset([board_to_state(b) for b in boards])
    eng.search(None)
    checked = 0
    for i in range(len(states)):
        a, b = eng.root(2 * i), eng.root(2 * i + 1)
        pa = dict(zip(a["moves"], zip(a["p"], a["n"], a["w"])))
        pb = dict(zip(b["moves"], zip(b["p"], b["n"], b["w"])))
        assert sorted(mirror_move(m) for m in pa) == sorted(pb)
        if len(set(a["p"])) < len(a["p"]):
            continue                                         # tied priors: the visited child may differ by move order
        for m, (p, n, w) in pa.items():
            q, nb, wb = pb[mirror_move(m)]
            # the averaged network priors are equal bit for bit; the edge priors are then renormalised by a sequential
            # float32 sum in each position's own move order (player.py:272-284), which can differ in the last bits
            assert abs(p - q) <= 4 * np.spacing(np.float32(p))
            assert (n, w) == (nb, wb)                        # the visited child's mirror-averaged value, exactly
        checked += 1
    assert checked >= 6
    eng.close()


def _cfg(**kw):
    c = CzConfig()
    c.struct_bytes = C.sizeof(CzConfig)
    c.n_games, c.sims_per_move, c.leaves_per_round, c.virtual_loss = kw["games"], kw["sims"], kw["k"], 3
    c.max_nodes_per_game, c.max_edges_per_game, c.max_path, c.noise_mode = kw["nodes"], kw["nodes"] * 48, 128, 1
    c.max_game_length, c.max_plies = 100, 200
    c.nn_filters, c.nn_blocks, c.nn_value_fc = kw["filters"], kw["blocks"], 256
    c.c_puct, c.noise_eps, c.dirichlet_alpha, c.tau_decay_rate = 1.5, 0.25, 0.2, 0.98
    c.eval_mirror = kw.get("mirror", 0)
    return c


def workspace(lib, **kw):
    n = C.c_uint64(0)
    lib.call("cz_workspace_bytes", C.byref(_cfg(**kw)), C.byref(n))
    return n.value


C2 = dict(games=256, sims=200, k=8, nodes=4864, filters=128, blocks=7)
C3 = dict(games=1024, sims=800, k=8, nodes=19264, filters=256, blocks=20)
# cz_workspace_bytes of the commit before eval_mirror existed, for these two shapes
PARENT_WORKSPACE = {"c2": 1746739744, "c3": 24624495392}


@pytest.mark.parametrize("shape", ["c2", "c3"])
def test_workspace_off_is_the_parents_and_on_adds_the_mirror_buffers(cuda_lib, shape):
    kw = C2 if shape == "c2" else C3
    off = workspace(cuda_lib, **kw)
    assert off == PARENT_WORKSPACE[shape]
    on = workspace(cuda_lib, mirror=1, **kw)
    assert on > off
    # G*K more leaf board rows, the [2*G*K] value scratch and M, plus the network runtime's activations at twice the batch
    rows = kw["games"] * kw["k"]
    extra_tree = rows * 96 + 2 * rows * 4 + 2086 * 2
    assert extra_tree <= on - off


def test_launches_per_iteration_unchanged(cuda_lib):
    """cz_launch_count: launches per search-loop iteration (the slope between two searches of different length) and per
    search (the rest) are the same with and without the mirror form."""
    from cczero_b200.engine import Engine
    fits = {}
    for mirror in (False, True):
        eng = Engine(cuda_lib, "cuda", n_games=16, sims_per_move=24, leaves_per_round=4, nn_filters=64, nn_blocks=2, seed=5,
                     eval_mirror=mirror)
        eng.set_weights(weights(64, 2, 4))
        eng.reset()
        eng.search(None)                                     # first search: plain launches + capture
        pts = []
        for sims in (16, 64):
            eng.reset()
            l0, w0 = eng.launch_count(), int(eng.counters()[2])
            eng.search(eng.make_opts(sims_override=sims))
            pts.append((eng.launch_count() - l0, int(eng.counters()[2]) - w0))
        eng.close()
        (la, wa), (lb, wb) = pts
        assert wb > wa
        slope = (lb - la) // (wb - wa)
        assert slope * (wb - wa) == lb - la
        fits[mirror] = (slope, la - slope * wa)
    assert fits[False] == fits[True]


def test_create_rejects_eval_mirror_without_a_network(cuda_lib):
    from cczero_b200.engine import Engine
    with pytest.raises(CzError):
        Engine(cuda_lib, "cuda", n_games=4, sims_per_move=8, leaves_per_round=2, nn_filters=0, eval_mirror=True)
