"""The 3x3 conv's halo-resident A operand (k_igemm conv mode) at the batch shapes that separate its cases.

An M tile of the full-width conv is 256 pixels when such tiles fill at least 8 waves of CTAs (C = 256 from 1500 boards,
C = 64 and 128 from 3001 on 132 SMs), else 128; its producer loads the tile's input rows plus 10 rows either side once, and every tap
reads them at a row offset, with taps that fall off the board pointed at a row of zeros.  Cases:

* pixel counts just below, at and just above a multiple of 256 (90 n is even: n = 91 + 128 k gives 256 j - 2, n = 128 k
  gives 256 j, n = 37 + 128 k gives 256 j + 2), so the last tile holds 254, 256 or 2 pixels, in both tile forms; and a
  single board, whose one tile's halo starts at row -10;
* every batch of more than two boards has boards that straddle a tile boundary.

Each run is checked against the float64 reference of tests/nn_checks.py, and the same boards run behind three others (every
board then sits at another place in its tile, or in another tile) must give the same bits.  A last case surrounds the boards
with boards of NaN inputs, in front of them and at the end of the batch, inside the partial last tile: a tap that reads a
neighbouring board's rows is one that falls off the board, so the NaN must never reach the checked boards' outputs."""
import ctypes as C

import pytest
import torch

from tests import nn_checks as nc
from tests.test_igemm_gpu import _conv_ref_and_scale

pytestmark = pytest.mark.gpu


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _conv(cuda_lib, x, w, bias, res, relu):
    """x, res: [B][C][10][9] (fp16 values), w: [C][C][3][3] -> the conv's fp16 output as [B][C][10][9]."""
    n, c = x.shape[0], x.shape[1]
    xs = x.permute(0, 2, 3, 1).contiguous().half()
    ws = w.permute(2, 3, 0, 1).reshape(9, c, c).contiguous().half()
    rs = res.permute(0, 2, 3, 1).contiguous().half() if res is not None else None
    out = torch.full((n, 10, 9, c), float("nan"), device="cuda", dtype=torch.half)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    cuda_lib.call("cz_igemm_conv3x3_dense", _p(xs), _p(ws), _p(bias), _p(rs), _p(out), n, c, int(relu), stream)
    torch.cuda.synchronize()
    return out.permute(0, 3, 1, 2)


def _inputs(n, c, seed, residual):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n, c, 10, 9, device="cuda", generator=g).half().float()
    w = (torch.randn(c, c, 3, 3, device="cuda", generator=g) * (1.0 / (3 * c ** 0.5))).half().float()
    bias = torch.randn(c, device="cuda", generator=g)
    res = torch.randn(n, c, 10, 9, device="cuda", generator=g).half().float() if residual else None
    return x, w, bias, res


CASES = ([(c, n) for c in (256, 128, 192) for n in (1, 37, 91, 128)]      # 128-pixel tiles
         + [(256, n) for n in (1627, 1536, 1573)] + [(c, n) for c in (128, 64) for n in (3035, 3072, 3109)])   # 256-pixel tiles


@pytest.mark.parametrize("c,n", CASES, ids=lambda v: str(v))
def test_halo_tiles_match_reference_and_offsets(cuda_lib, c, n):
    x, w, bias, res = _inputs(n + 3, c, 7 * n + c, residual=True)
    out = _conv(cuda_lib, x[3:], w, bias, res[3:], True)
    ref, scale = _conv_ref_and_scale(x[3:], w, bias, res[3:], True)
    nc.check_close(out, ref, scale, "fp16", what=f"conv3x3 halo tiles, {n} boards, C = {c}")
    shifted = _conv(cuda_lib, x, w, bias, res, True)
    assert torch.equal(shifted[3:], out), "a board's outputs depend on its place in the batch"


@pytest.mark.parametrize("c,n", [(256, 37), (256, 1573), (128, 3109)], ids=lambda v: str(v))
def test_off_board_taps_never_read_neighbours(cuda_lib, c, n):
    """n = 37 + 128 k: the last tile holds 2 pixels (128-pixel tiles at 37 boards, 256-pixel tiles at the larger batches)."""
    x, w, bias, _ = _inputs(n, c, 11 + c, residual=False)
    alone = _conv(cuda_lib, x[1:n - 2], w, bias, None, False)
    poisoned = x.clone()
    poisoned[0] = float("nan")
    poisoned[n - 2:] = float("nan")                              # the last two boards, 180 pixels up to the batch's end
    out = _conv(cuda_lib, poisoned, w, bias, None, False)
    assert torch.isfinite(out[1:n - 2]).all(), "NaN from a neighbouring board reached a checked board"
    assert torch.equal(out[1:n - 2], alone)
    assert torch.isnan(out[0]).any() and torch.isnan(out[n - 1]).any()
