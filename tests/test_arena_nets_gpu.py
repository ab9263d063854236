"""An arena engine evaluates each half of its slots with its own network: slots [0, n/2) with net 0, [n/2, n) with net 1.
With noise off the search is deterministic and a network's per-position arithmetic does not depend on the batch
(DESIGN.md §3.1), so every arena slot's root must equal, bit for bit, the root of a one-network engine that searched the
same position with that slot's network."""
import pytest
import torch

from oracle import model as om
from oracle import senv as osenv
from tests import search_checks as sc

pytestmark = pytest.mark.gpu

N_SLOTS, SIMS, K, FILTERS, BLOCKS, SEED = 64, 64, 8, 128, 2, 7


def _weights(seed):
    return {k: torch.as_tensor(v) for k, v in om.init_weights(FILTERS, BLOCKS, seed=seed, trained_like=True).items()}


def _engine(lib, **kw):
    from cczero_b200.engine import Engine
    return Engine(lib, "cuda", n_games=N_SLOTS, sims_per_move=SIMS, leaves_per_round=K, noise_eps=0.0, nn_filters=FILTERS,
                  nn_blocks=BLOCKS, seed=SEED, **kw)


def _search(eng, states):
    eng.reset(states)
    eng.search(eng.make_opts(active=[1] * N_SLOTS))
    assert int(eng.counters()[6]) == 0
    return [eng.root(g) for g in range(N_SLOTS)]


def _same(a, b):
    return a["moves"] == b["moves"] and a["p"] == b["p"] and a["n"] == b["n"] and a["w"] == b["w"]


@pytest.mark.parametrize("profiled", [False, True], ids=["while_graph", "profiled_graph"])
def test_arena_slot_ranges_search_with_their_own_network(cuda_lib, profiled):
    """Two searches per engine: the first runs its first iteration as plain launches, captures the WHILE graph and launches it;
    the second is one launch of that graph (with cz_nn_profile on, the profiled graph).  A third search after net 1 is
    reloaded with net 0's weights checks that the captured graph sees a reload."""
    wa, wb = _weights(1), _weights(2)
    positions = [[osenv.INIT_STATE] * (N_SLOTS // 2) + sc.midgame_states(N_SLOTS // 2, 3),
                 sc.midgame_states(N_SLOTS, 4)]

    def single(w):
        eng = _engine(cuda_lib)
        eng.set_weights(w)
        if profiled:
            eng.nn_profile(True)
        out = [_search(eng, s) for s in positions]
        eng.close()
        return out

    want_a, want_b = single(wa), single(wb)
    arena = _engine(cuda_lib, arena=True)
    arena.set_weights(wa, net=0)
    arena.set_weights(wb, net=1)
    if profiled:
        arena.nn_profile(True)
    got = [_search(arena, s) for s in positions]
    arena.set_weights(wa, net=1)
    reloaded = _search(arena, positions[1])
    arena.close()

    half = N_SLOTS // 2
    for i in range(len(positions)):
        for g in range(N_SLOTS):
            a, b = want_a[i][g], want_b[i][g]
            if len(a["moves"]) > 1:
                assert a["p"] != b["p"], (i, g)           # the two networks are told apart at every slot
            assert _same(got[i][g], a if g < half else b), (i, g)
    for g in range(N_SLOTS):
        assert _same(reloaded[g], want_a[1][g]), g
