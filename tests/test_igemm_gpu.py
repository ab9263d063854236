"""wgmma implicit-GEMM kernel vs a plain PyTorch float64 reference of the same op, within the rounding bound of
tests/nn_checks.py (GPU only)."""
import ctypes as C

import pytest
import torch

from tests import nn_checks as nc

pytestmark = pytest.mark.gpu


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


@pytest.mark.parametrize("m,n_valid,n_pad,k,n_tile", [(128, 256, 256, 64, 256), (300, 2086, 2304, 384, 256),
                                                       (1000, 128, 128, 128, 128), (77, 192, 192, 192, 192)])
def test_dense_matches_torch(cuda_lib, m, n_valid, n_pad, k, n_tile):
    g = torch.Generator(device="cuda").manual_seed(m + k)
    a = (torch.randn(m, k, device="cuda", generator=g) * 0.5).half()
    w = torch.zeros(n_pad, k, device="cuda", dtype=torch.half)
    w[:n_valid] = (torch.randn(n_valid, k, device="cuda", generator=g) * 0.2).half()
    bias = torch.zeros(n_pad, device="cuda")
    bias[:n_valid] = torch.randn(n_valid, device="cuda", generator=g)
    out = torch.full((m, n_pad), float("nan"), device="cuda")
    cuda_lib.call("cz_igemm_dense", _p(a), _p(w), _p(bias), _p(out), m, n_valid, n_pad, k, n_tile, n_pad, _stream())
    torch.cuda.synchronize()
    a64, w64, b64 = a.double(), w.double()[:n_valid], bias.double()[:n_valid]
    ref, scale = a64 @ w64.t() + b64, a64.abs() @ w64.abs().t() + b64.abs()
    # fp16 products are exact in fp32; only the fp32 accumulation rounds (tests/nn_checks.py: BETA * S)
    nc.check_close(out[:, :n_valid], ref, scale, "fp32", what="igemm dense")


def _conv3x3_ref(x, w, bias):
    """Reference without cuDNN, in the dtype of x (float64 here): im2col (unfold) + one GEMM."""
    b, c = x.shape[0], x.shape[1]
    cols = torch.nn.functional.unfold(x, 3, padding=1)                    # [B, C*9, 90]
    out = torch.matmul(w.reshape(w.shape[0], -1), cols)                   # [B, C_out, 90]
    return out.reshape(b, w.shape[0], 10, 9) + bias.view(1, -1, 1, 1)


def _conv_ref_and_scale(x, w, bias, res, relu):
    """float64 reference of relu?(conv(x, w) + bias (+ res)) and its scale S (the same on absolute values)."""
    x, w, bias = x.double(), w.double(), bias.double()
    ref, scale = _conv3x3_ref(x, w, bias), _conv3x3_ref(x.abs(), w.abs(), bias.abs())
    if res is not None:
        ref, scale = ref + res.double(), scale + res.double().abs()
    return (ref.relu() if relu else ref), scale


@pytest.mark.parametrize("n_boards,c,residual,relu", [(1, 128, False, True), (5, 256, True, True), (29, 128, True, False),
                                                       (64, 256, False, False), (200, 192, True, True), (3, 64, True, True),
                                                       (1000, 256, True, True)])
def test_conv3x3_dense_im2col_matches_torch(cuda_lib, n_boards, c, residual, relu):
    """Dense NHWC activations through im2col-mode TMA (no separator rows, 128 useful pixels per tile)."""
    g = torch.Generator(device="cuda").manual_seed(n_boards * 1000 + c + 1)
    x = torch.randn(n_boards, c, 10, 9, device="cuda", generator=g).half().float()
    w = (torch.randn(c, c, 3, 3, device="cuda", generator=g) * (1.0 / (3 * c ** 0.5))).half().float()
    bias = torch.randn(c, device="cuda", generator=g)
    res = torch.randn(n_boards, c, 10, 9, device="cuda", generator=g).half().float() if residual else None
    xs = x.permute(0, 2, 3, 1).contiguous().half()                       # [B,10,9,C]
    ws = w.permute(2, 3, 0, 1).reshape(9, c, c).contiguous().half()
    rs = res.permute(0, 2, 3, 1).contiguous().half() if residual else None
    out = torch.full((n_boards, 10, 9, c), float("nan"), device="cuda", dtype=torch.half)
    cuda_lib.call("cz_igemm_conv3x3_dense", _p(xs), _p(ws), _p(bias), _p(rs), _p(out), n_boards, c, int(relu), _stream())
    torch.cuda.synchronize()
    ref, scale = _conv_ref_and_scale(x, w, bias, res, relu)
    nc.check_close(out.permute(0, 3, 1, 2), ref, scale, "fp16", what="igemm conv3x3 (dense, im2col)")
