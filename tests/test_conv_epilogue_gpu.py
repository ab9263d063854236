"""The residual convs' epilogue (k_igemm, dense layout) writes exactly the rows of the batch, and what it writes for a position
does not depend on where the position sits in the batch.

* Rows beyond the batch: a full-size forward first fills every row of the engine's buffers (conv1 output t, the tower output
  and its fp32 skip copy); a smaller batch then runs on the same engine, and the rows from its batch size up to the buffers'
  extent (what the tensor maps cover) must still hold the first forward's values, bit for bit.
* Batch offset: the same positions evaluated alone and behind a few other positions land at different places inside the
  128-pixel M tiles (a partial last tile in one run, a full tile in the other), so each position's outputs come from
  differently placed tiles.  Tower outputs, policy and value must agree bit for bit.

Cases: 256x20 (fp32 skip stream), 128x7 (fp16 skip), and a batch small enough for 64-column tiles; pixel counts are not
multiples of 128."""
import pytest
import torch

from oracle import model as om
from oracle import senv as osenv
from tests import nn_checks as nc
from tests.search_checks import midgame_states

pytestmark = pytest.mark.gpu

# (filters, blocks, positions, extra rows of the engine's buffers, positions in front of them in the offset run)
CASES = [(256, 20, 301, 37, 5), (128, 7, 301, 37, 5), (256, 20, 9, 7, 5)]


def _read(eng, n, c, s32):
    out = {"conv1": nc.read_act(eng, nc.LAST_CONV1, n, c), "tower": nc.read_act(eng, nc.TOWER_OUT, n, c)}
    if s32:
        out["tower32"] = nc.read_act(eng, nc.TOWER_OUT32, n, c)
    return out


@pytest.mark.parametrize("filters,blocks,n,extra,front", CASES, ids=lambda v: str(v))
def test_epilogue_rows_and_offsets(cuda_lib, cuda_env, filters, blocks, n, extra, front):
    from cczero_b200.engine import Engine
    n_max = n + extra
    s32 = blocks >= 10                                           # the engine's default skip stream precision
    w = om.init_weights(filters, blocks, 256, seed=filters + blocks, trained_like=True, spread=0.1)
    if n > 1024:                            # thousands of distinct positions: one oracle step each
        states, filler = nc.distinct_states(n, 21), nc.distinct_states(n_max, 22)
    else:
        states = [osenv.INIT_STATE] + midgame_states(n - 1, 21, lo=1, hi=120)
        filler = midgame_states(n_max, 22, lo=1, hi=120)
    ahead = midgame_states(front, 23, lo=1, hi=120)
    eng = Engine(cuda_lib, "cuda", n_games=n_max, sims_per_move=8, leaves_per_round=1, nn_filters=filters, nn_blocks=blocks,
                 nn_value_fc=256)
    try:
        eng.set_weights({k: torch.as_tensor(v) for k, v in w.items()})
        eng.nn_forward_boards(cuda_env.boards_from_states(filler))
        torch.cuda.synchronize()
        before = _read(eng, n_max, filters, s32)

        pol, val = eng.nn_forward_boards(cuda_env.boards_from_states(states))
        torch.cuda.synchronize()
        after = _read(eng, n_max, filters, s32)
        for k in before:
            assert torch.equal(after[k][n:], before[k][n:]), f"{k}: rows beyond the batch were written"

        pol2, val2 = eng.nn_forward_boards(cuda_env.boards_from_states(ahead + states))
        torch.cuda.synchronize()
        shifted = _read(eng, front + n, filters, s32)
    finally:
        eng.close()
    for k in after:
        assert torch.equal(shifted[k][front:], after[k][:n]), f"{k} depends on the position's place in the batch"
    assert torch.equal(pol2[front:], pol) and torch.equal(val2[front:], val)
    assert torch.isfinite(pol).all() and torch.isfinite(val).all()
