"""Each stage of the training step against float64 on the GPU's own inputs to that stage (csrc/cz_train.cu building
blocks), with tests/nn_checks.py's bound |g - r| <= ALPHA ulp_out + BETA S (S = the reference on absolute values), and
a proof for every bound that it rejects a subtly wrong kernel (assert_rejects).

Gradient operands of the tensor-core convolutions are fp16 times a power of two 2^e with max|dy| 2^e in [2^14, 2^15);
the references below take exactly those operands (scaling is exact), so what is measured is the accumulation.

wgrad's K is the batch's pixel count, up to 368 640 at max_batch 4096, 160x the forward's 2304.  Each CTA accumulates
one contiguous split of at most ceil(chunks / splits) * 64 pixels in the wgmma fp32 accumulator, then <= 14 split
partials are summed in fp32 in a fixed order.  On 132 SMs that is about 13 200 pixels at batch 1024, C = 256 (7 splits),
and 52 700 at batch 4096, C = 256 (7 splits of 823 chunks; C = 64: 14 splits, 26 400 pixels).  The forward's BETA =
2^-16 carries a 5x margin over sqrt(K) 2^-24 S at K = 2304; the same argument at K = 52 700 gives sqrt(52 700) 2^-24 S =
2^-16.2 S for the accumulator and 14 * 2^-24 S = 2^-20.2 S for the ordered split sum, so WGRAD_BETA = 2^-13 keeps a
9x margin at the longest split the ABI allows (>10x up to batch 1024).  One board-edge column missing from a tap drops
about 1/9 of its terms (~0.1 S), far above it.
"""
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import nn_checks as nc

pytestmark = pytest.mark.gpu

WGRAD_BETA = 2.0 ** -13


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def scaled16(dy):
    """The fp16 operand the kernels build from an fp32 gradient, divided back: fp16(dy * 2^e) * 2^-e in float64."""
    m = dy.abs().max().item()
    e = 0 if m == 0 else 14 - (int(np.frexp(m)[1]) - 1)
    return (dy * 2.0 ** e).half().double() * 2.0 ** -e


def nchw(x, n, c):
    return x.reshape(n, 10, 9, c).permute(0, 3, 1, 2)


def wgrad_ref(x16, dy16, n, c):
    """float64 dW[kh][kw][ci][co] = sum_p dy[p][co] x[p + (kh-1, kw-1)][ci], and S on absolute values."""
    X, G = nchw(x16.double(), n, c), nchw(dy16, n, c)
    w = torch.nn.grad.conv2d_weight(X, (c, c, 3, 3), G, padding=1)
    s = torch.nn.grad.conv2d_weight(X.abs(), (c, c, 3, 3), G.abs(), padding=1)
    return w.permute(2, 3, 1, 0).contiguous(), s.permute(2, 3, 1, 0).contiguous()


WGRAD_CASES = [(64, 1), (64, 256), (128, 7), (192, 256), (256, 7), (256, 1024), (256, 4096), (64, 4096)]


@pytest.mark.parametrize("c,n", WGRAD_CASES)
def test_wgrad_matches_float64(cuda_lib, c, n):
    g = torch.Generator(device="cuda").manual_seed(c * 1000 + n)
    x16 = torch.relu(torch.randn(n * 90, c, device="cuda", generator=g)).half()
    dy = torch.randn(n * 90, c, device="cuda", generator=g) * 1e-4
    dw = torch.empty(3, 3, c, c, device="cuda")
    cuda_lib.call("cz_train_wgrad3x3", _p(x16), _p(dy), n, c, _p(dw), _stream())
    ref, s = wgrad_ref(x16, scaled16(dy.double()), n, c)

    def check(got, r):
        return nc.check_close(got, r, s * WGRAD_BETA / nc.BETA, out="fp32", what=f"wgrad C={c} n={n}")

    worst = check(dw, ref)
    X = nchw(x16.double(), n, c)
    Xcut = X.clone()
    Xcut[..., 8] = 0                                    # the last board column missing from every tap
    edge = torch.nn.grad.conv2d_weight(Xcut, (c, c, 3, 3), nchw(scaled16(dy.double()), n, c), padding=1).permute(2, 3, 1, 0)
    nc.assert_rejects(check, dw, ref, [
        nc.Mutation("transposed wgrad (co <-> ci)", lambda g_, r: g_.transpose(2, 3).contiguous()),
        nc.Mutation("one board-edge column missing", lambda g_, r: edge.clone()),
    ])
    print(f"wgrad C={c} n={n}: worst err/bound {worst:.3g}")


# the last three run the fp32-output conv on 256-pixel M tiles (two m64 blocks per consumer warpgroup) on 132 SMs
DGRAD_CASES = [(64, 7), (128, 256), (192, 1), (256, 1024), (256, 1573), (128, 3109), (64, 3035)]


@pytest.mark.parametrize("c,n", DGRAD_CASES)
def test_dgrad_matches_float64(cuda_lib, c, n):
    g = torch.Generator(device="cuda").manual_seed(7 * c + n)
    dy = torch.randn(n * 90, c, device="cuda", generator=g) * 3e-5
    w = torch.randn(3, 3, c, c, device="cuda", generator=g) * (1.0 / (3 * c ** 0.5))
    dx = torch.empty(n * 90, c, device="cuda")
    cuda_lib.call("cz_train_dgrad3x3", _p(dy), _p(w), n, c, _p(dx), _stream())
    w16 = w.half().double().permute(3, 2, 0, 1)                     # OIHW
    G = nchw(scaled16(dy.double()), n, c)
    ref = torch.nn.grad.conv2d_input((n, c, 10, 9), w16, G, padding=1)
    s = torch.nn.grad.conv2d_input((n, c, 10, 9), w16.abs(), G.abs(), padding=1)
    noflip = torch.nn.grad.conv2d_input((n, c, 10, 9), w16.flip(2, 3), G, padding=1)
    flat = lambda t: t.permute(0, 2, 3, 1).reshape(n * 90, c)

    def check(got, r):
        return nc.check_close(got, r, flat(s), out="fp32", what=f"dgrad C={c} n={n}")

    worst = check(dx, flat(ref))
    muts = [nc.Mutation("dgrad without the tap flip", lambda g_, r: flat(noflip).clone())]
    if nc.conv_tile_m(n, c, torch.cuda.get_device_properties(0).multi_processor_count) == 256:
        muts += nc.tile256_mutations()
    nc.assert_rejects(check, dx, flat(ref), muts)
    print(f"dgrad C={c} n={n}: worst err/bound {worst:.3g}")


BN_CASES = [(64, 1, False), (128, 7, True), (256, 256, True), (4, 1024, False), (2, 7, False), (32, 256, False)]


@pytest.mark.parametrize("c,n,skip", BN_CASES)
def test_bn_train_forward_backward_matches_float64(cuda_lib, c, n, skip):
    g = torch.Generator(device="cuda").manual_seed(c + 31 * n)
    rows = n * 90
    z = torch.randn(rows, c, device="cuda", generator=g) * 0.7 + 0.3
    gamma = 0.5 + torch.rand(c, device="cuda", generator=g)
    beta = torch.randn(c, device="cuda", generator=g) * 0.2
    sk = torch.relu(torch.randn(rows, c, device="cuda", generator=g)) if skip else None
    up = torch.randn(rows, c, device="cuda", generator=g) * 1e-3
    out, dz = torch.empty_like(z), torch.empty_like(z)
    mean, var, dgamma, dbeta = (torch.empty(c, device="cuda") for _ in range(4))
    cuda_lib.call("cz_train_bn", _p(z), rows, c, _p(gamma), _p(beta), _p(sk), _p(out), _p(mean), _p(var), _p(up), _p(dz),
                  _p(dgamma), _p(dbeta), _stream())
    Z = z.double().requires_grad_(True)
    m = Z.mean(0)
    v = Z.var(0, unbiased=False)
    xh = (Z - m) / torch.sqrt(v + 1e-3)
    y = xh * gamma.double() + beta.double() + (sk.double() if skip else 0)
    o = torch.relu(y)
    o.backward(up.double())
    mask = (y > 0).double()
    gm = up.double() * mask
    # Column sums run over <= 90 rows per chunk, <= 256 lanes and <= 1024 chunks, each stage in order in fp32: at most
    # about (90 + 256 + 1024) 2^-24 = 2^-13.6 of the sum of magnitudes.  K = 4 lifts BETA = 2^-16 to 2^-14 per unit of S (x4 more for the mean and variance),
    # with S = the magnitudes that enter (column sums of |.|, |z| + |mean| for everything normalised).
    K = 2 ** 2
    nc.check_close(mean, m.detach(), z.double().abs().mean(0) * K * 4, out="fp32", what="batch mean")
    nc.check_close(var, v.detach(), ((z.double().abs() + m.detach().abs()) ** 2).mean(0) * K * 4, out="fp32", what="batch var")
    rstd0 = 1 / torch.sqrt(v.detach() + 1e-3)
    zmag = (z.double().abs() + m.detach().abs()) * rstd0
    s_out = (zmag * gamma.double() + beta.double().abs() + (sk.double() if skip else 0)) * K
    nc.check_close(out, o.detach(), s_out, out="fp32", what="bn out")
    rstd = 1 / torch.sqrt(v.detach() + 1e-3)
    s_dz = gamma.double() * rstd * (gm.abs() + gm.abs().mean(0) + zmag * (gm.abs() * zmag).mean(0)) * K

    def check_dz(got, r):
        return nc.check_close(got, r, s_dz, out="fp32", what=f"bn dz C={c} n={n}")

    worst = check_dz(dz, Z.grad)
    nomean = gamma.double() * rstd * gm
    nc.assert_rejects(check_dz, dz, Z.grad, [nc.Mutation("BN backward without its mean terms", lambda g_, r: nomean.clone())])
    nc.check_close(dbeta, gm.sum(0), gm.abs().sum(0) * K, out="fp32", what="dbeta")
    nc.check_close(dgamma, (gm * xh.detach()).sum(0), (gm.abs() * zmag).sum(0) * K, out="fp32", what="dgamma")
    print(f"bn C={c} n={n} skip={skip}: worst dz err/bound {worst:.3g}")
