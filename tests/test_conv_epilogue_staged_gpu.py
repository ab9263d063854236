"""The staged conv epilogue (k_igemm: a conv without a skip stream writes its fp16 output by TMA stores through shared
memory) against the register epilogue, at the batch shapes that separate them.

M tiles that lie wholly inside the batch take the staged path, the last, partial one keeps the register path.  The checks are
those of test_conv_epilogue_gpu.py (rows beyond the batch untouched, a position's outputs bit-identical wherever it sits in the
batch); the cases add

* 64 boards = 5760 pixels = 45 full tiles: no tile of the first run takes the register path, and the same positions behind
  5 others (a partial last tile, every position in a differently placed tile) must come out bit-identical, which makes the
  offset check an equality between the two epilogues;
* 377 boards = 265 full tiles and a partial one, more than two tiles per CTA on 132 SMs: the staging ring wraps inside a tile
  and across tiles while the previous tile's stores are still in flight;
* 1573 boards at C = 256 and 3109 at C = 128 (and the engine's 1610 and 3146 rows): 256-pixel M tiles, each consumer
  warpgroup storing two m64 blocks through its ring per tile, and a last tile of 2 pixels."""
import pytest

from tests.test_conv_epilogue_gpu import test_epilogue_rows_and_offsets as _check

pytestmark = pytest.mark.gpu

CASES = [(256, 20, 64, 37, 5), (128, 7, 64, 37, 5), (256, 20, 377, 37, 5), (128, 7, 377, 37, 5),
         (256, 20, 1573, 37, 5), (128, 7, 3109, 37, 5)]


@pytest.mark.parametrize("filters,blocks,n,extra,front", CASES, ids=lambda v: str(v))
def test_staged_epilogue_rows_and_offsets(cuda_lib, cuda_env, filters, blocks, n, extra, front):
    _check(cuda_lib, cuda_env, filters, blocks, n, extra, front)
