"""Every plain-CUDA stage of the training step (csrc/cz_train.cu, cz_train_step) against float64 on the GPU's own inputs to
that stage, read back with cz_train_read_buffer after one real step, with bounds derived from each kernel's summation order
at its launch geometry and a proof for every bound that it rejects a subtly wrong kernel (nc.assert_rejects).

The bound is the one of tests/nn_checks.py, |g - r| <= 1/2 ulp32(max(|g|, |r|)) + beta(k) S (+ propagated input error),
with S the reference evaluated on absolute values and

    beta(k) = MARGIN * sqrt(k) * 2^-24,   MARGIN = 8,

where k is the longest chain of ordered fp32 roundings that produces one output element: fused multiply-adds along one
K split of k_gemm plus the ordered sum of the splits, rows per lane + lanes + column chunks of a BN column sum, positions x
pixels per chunk + chunks of k_first_wgrad, pixels per CTA + splits of k_wgrad.  A round-to-nearest chain of k operations
errs by about sqrt(k) 2^-24 S; MARGIN = 8 covers the tail and, for the short chains (k <= 64), the worst case k 2^-24 S
too.  The launch geometry (splits, chunks, lanes) is restated from the host code below, asserted at the shapes that are
here to reach a path, and sets k: the bound at batch 4096 is derived, not tuned.

Where the step has overwritten a stage's pre-BN input z with dz, z is recomputed in float64 from the GPU's own inputs to
that conv and the conv's own bound is carried into the BN bound.  Tensor-core operands are rounded as the GPU rounds them
(fp16 activations and weights; scaled fp16 dz with the exponent its own max implies, which the step's scale slot must
hold).  ReLU masks come from the GPU's own post-ReLU output; fp16 outputs underflow, so an element of a conv1 output that
is 0 in fp16 while its float64 pre-activation lies within its bound of zero may take either mask.
"""
import ctypes as C
import math
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import model as om
from tests import nn_checks as nc
from tests import train_oracle as to

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
MARGIN = 8
N_LABELS = om.N_LABELS
BN_EPS = 1e-3

# cz_train_buffer (include/cczero_b200.h)
(PLANE_INDEX, BLOCK_OUT32, BLOCK_OUT16, CONV1_OUT16, BN_MEAN, BN_VAR, BN_DZ, POL_FEAT, VAL_FEAT, LOGITS, DLOGITS,
 VAL_HIDDEN_PRE, VAL_HIDDEN, DVAL_HIDDEN, VAL_PRE, DVAL_PRE, CE_ROWS, SE_ROWS, DPOL_FEAT, TRUNK_GRAD, SCALE_SLOTS) = range(21)


def beta(k):
    return MARGIN * math.sqrt(max(k, 1)) * U


# ---------------------------------------------------------------------------------------------- launch geometry (host code)
def gemm_splits(M, N, K):
    """cztrain::gemm: (splits, k per split) of k_gemm."""
    tiles = -(-M // 16) * -(-N // 16)
    splits = 1
    if tiles < 264 and K >= 2048:
        splits = min(528 // tiles, K // 256, 64)
        if splits * M * N > 64 * 70000:
            splits = 64 * 70000 // (M * N)
        splits = max(splits, 1)
    kps = (-(-K // splits) + 15) // 16 * 16
    return -(-K // kps), kps


def gemm_chain(M, N, K, extra=0):
    """Longest chain of one k_gemm output: fmas along a split, the ordered split sum, then bias / accumulate (extra)."""
    s, kps = gemm_splits(M, N, K)
    return min(kps, K) + (s if s > 1 else 0) + extra


def col_chunks(P):
    """cztrain::col_chunks: (chunks, rows per chunk) of the BN column sums."""
    ch = min(-(-P // 64), 1024)
    rows = -(-P // ch)
    return -(-P // rows), rows


def bn_chain(P, c):
    """k_bn_reduce: 256 / C lanes stride a chunk's rows, lanes then chunks are summed in order; then one division."""
    ch, rows = col_chunks(P)
    lanes = 256 // c
    return -(-rows // lanes) + lanes + ch + 1


def first_wgrad_geometry(n):
    """The step's k_first_wgrad launch: (chunks, positions per chunk)."""
    ch = min(-(-n // 64), 16)
    per = -(-n // ch)
    return -(-n // per), per


def wgrad_geometry(n, c):
    """cztrain::wgrad_launch: (splits, 64-pixel chunks per split)."""
    co_tiles = -(-c // 128)
    chunks = -(-n * 90 // 64)
    splits = max(min(torch.cuda.get_device_properties(0).multi_processor_count // (9 * co_tiles), 14, chunks), 1)
    per = -(-chunks // splits)
    return -(-chunks // per), per


# ---------------------------------------------------------------------------------------------- checks
class Report:
    def __init__(self, case):
        self.case, self.rows = case, []

    def check(self, what, got, ref, S, k, extra=0.0, mutations=()):
        """|g - r| <= 1/2 ulp32 + beta(k) S + k 2^-150 + extra, then every mutation must be rejected by the same bound.
        k 2^-150: in the subnormal range each of the k roundings may lose half the spacing 2^-149 absolutely."""
        got, ref = nc._f64(got), nc._f64(ref)
        S = nc._f64(S) if torch.is_tensor(S) else torch.full_like(ref, float(S))

        def chk(g, r):
            e = 0.5 * nc.ulp32(torch.maximum(g.abs(), r.abs())) + k * 2.0 ** -150 + extra
            return nc.check_close(g, r, S * (beta(k) / nc.BETA), out="fp32", extra=e, what=f"{self.case}: {what}")

        worst = chk(got, ref)
        # a mutation that leaves this output unchanged at this shape (a split the data leaves all zero) proves nothing:
        # it is skipped, and at least one must remain
        live = [m for m in mutations if not torch.equal(m(got, ref), got)]
        if mutations:
            assert live, f"{self.case}: {what}: every mutation leaves the output unchanged"
            nc.assert_rejects(chk, got, ref, live)
        self.rows.append((what, worst, len(live)))
        return worst

    def exact(self, what, got, ref):
        assert torch.equal(got, ref), f"{self.case}: {what} differs"
        self.rows.append((what, 0.0, 0))

    def print(self):
        for what, worst, nm in self.rows:
            print(f"{self.case:>18} | {what:<34} | worst err/bound {worst:.3g} | {nm} mutation(s) rejected")


def delta(name, d):
    """The kernel's output moved by d (= the reference of a wrong kernel minus the right reference)."""
    return nc.Mutation(name, lambda g, r: g + d)


def add_term(S, k):
    """One extra average term S / k in the output with the largest S (a dropped or duplicated k-block)."""
    def fn(g, r):
        d = torch.zeros_like(g).reshape(-1)
        i = int(S.reshape(-1).argmax())
        d[i] = S.reshape(-1)[i] / k
        return g + d.reshape(g.shape)
    return nc.Mutation("one average term added", fn)


def rows_of_flat(x, n, c):
    """Keras Flatten order [n][c * 90 + pix] -> BN rows [n * 90][c]."""
    return x.reshape(n, c, 90).permute(0, 2, 1).reshape(n * 90, c)


def flat_of_rows(x, n, c):
    return x.reshape(n, 90, c).permute(0, 2, 1).reshape(n, c * 90)


def nchw(x, n, c):
    return x.reshape(n, 10, 9, c).permute(0, 3, 1, 2)


def pix(x):
    n, c = x.shape[:2]
    return x.permute(0, 2, 3, 1).reshape(n * 90, c)


def bn_apply(z, zb, mean, var, gamma, beta_, skip=None):
    """y = gamma (z - mean) rstd + beta (+ skip) on the GPU's own batch statistics: (y, S, propagated error of z).
    7 roundings: v + eps, sqrt, 1 / x, z - mean, * rstd, the fma, + skip."""
    rstd = 1 / torch.sqrt(var + BN_EPS)
    y = gamma * (z - mean) * rstd + beta_
    S = gamma.abs() * (z.abs() + mean.abs()) * rstd + beta_.abs()
    if skip is not None:
        y, S = y + skip, S + skip.abs()
    return y, S, gamma.abs() * rstd * zb


def bn_backward(z, zb, mean, var, gamma, up, up_err, mask, amb=0.0):
    """dz of BN (training mode) under ReLU mask `mask`, from upstream `up` (error up_err); (dz, S, propagated error).
    Elements where amb = 1 may take either mask: their masked upstream is uncertain by |up|."""
    P = z.shape[0]
    rstd = 1 / torch.sqrt(var + BN_EPS)
    xh = (z - mean) * rstd
    xb = rstd * zb + 4 * U * xh.abs()
    g, ge = up * mask, up_err * torch.maximum(mask, torch.as_tensor(amb, dtype=up.dtype, device=up.device)) + up.abs() * amb
    sg, sgx = g.sum(0), (g * xh).sum(0)
    f = gamma * rstd
    dz = f * (g - sg / P - xh * sgx / P)
    ag, ax = g.abs(), xh.abs()
    S = f.abs() * (ag + ag.sum(0) / P + ax * (ag * ax).sum(0) / P)
    err = f.abs() * (ge + ge.sum(0) / P + ax * (ge * ax).sum(0) / P + xb * sgx.abs() / P + ax * (ag * xb).sum(0) / P)
    return dz, S, err


# ---------------------------------------------------------------------------------------------- the step under test
CFG = SimpleNamespace


def config(filters, blocks, in_planes, heads, batch):
    pc, vc, H = heads
    mc = CFG(cnn_filter_num=filters, res_layer_num=blocks, value_fc_size=H, l2_reg=1e-4, input_depth=in_planes,
             policy_channels=pc, value_channels=vc, cnn_first_filter_size=5, cnn_filter_size=3)
    tc = CFG(momentum=0.9, loss_weights=[1.0, 1.25], batch_size=batch)
    return CFG(model=mc, trainer=tc)


_POSITIONS = {}


def positions(n, in_planes, seed):
    """n positions: up to 256 distinct seeded ones, larger batches draw from them in a seeded order."""
    key = (in_planes, seed)
    if key not in _POSITIONS:
        _POSITIONS[key] = nc.positions(256 if in_planes == 14 else 128, in_planes, seed)[1].astype(np.float32)
    base = _POSITIONS[key]
    if n <= len(base):
        return base[:n]
    return base[np.random.RandomState(seed + n).randint(0, len(base), n)]


SAT = float(np.float32(np.tanh(9.0)))              # a saturated tanh value target
VALUES = [0.37, -1.0, 0.0, 1.0, float(np.float32(np.tanh(3.0))), -SAT, float(np.float32(np.tanh(0.6)))]


def targets(n, logits, seed, sharp):
    """Rows cycle through one-hot, two soft (normalised Dirichlet over 5..60 labels, like visit distributions) and all-zero
    targets; with `sharp` the row whose float64 probability is closest to 1 targets that label (p > 1 - 1e-7)."""
    rng = np.random.RandomState(seed)
    pol = np.zeros((n, N_LABELS), np.float32)
    for i in range(n):
        kind = i % 4
        if kind == 0:
            pol[i, rng.randint(N_LABELS)] = 1
        elif kind in (1, 2):
            idx = rng.choice(N_LABELS, rng.randint(5, 61), replace=False)
            d = rng.dirichlet(np.full(len(idx), 0.3)).astype(np.float32)
            pol[i, idx] = d / d.sum(dtype=np.float32)
    sharp_row = None
    if sharp:
        p = torch.softmax(logits, 1)
        top = p.max(1)
        sharp_row = int((1 - top.values).argmin())
        assert 1 - top.values[sharp_row].item() < 1e-8, "no row sharp enough for the upper clip"
        for i in range(n):                  # on so sharp a net random labels lie below the clip: soft over the top 8
            idx = torch.argsort(p[i], descending=True)[:8].cpu().numpy()
            pol[i] = 0
            pol[i, idx] = rng.dirichlet(np.full(8, 0.3)).astype(np.float32)
        pol[sharp_row] = 0
        pol[sharp_row, int(top.indices[sharp_row])] = 1
    val = np.array([VALUES[i * 3 % len(VALUES)] for i in range(n)], np.float32)
    return pol, val, sharp_row


def read(tr, which, index=0, dtype=torch.float32):
    nb = C.c_int64(0)
    tr.lib.call("cz_train_read_buffer", tr._h, which, index, None, 0, C.byref(nb))
    out = torch.empty(nb.value, dtype=torch.uint8, device=tr.device)
    tr.lib.call("cz_train_read_buffer", tr._h, which, index, C.c_void_p(out.data_ptr()), out.numel(), C.byref(nb))
    return out.view(dtype)


# id, filters, blocks, in_planes, heads (policy channels, value channels, value_fc), batch, logit_std, paths to hit
CASES = [
    ("mini-b1", 64, 0, 14, (4, 2, 256), 1, 2.0, {"dFp_split"}),
    ("mini-b2-sharp", 64, 0, 14, (4, 2, 256), 2, 100.0, {"dFp_split"}),
    ("p28-b65", 64, 0, 28, (2, 4, 17), 65, 2.0, {"fw_chunks2", "dFp_split", "dWp_split"}),
    ("h111-b33", 128, 0, 14, (1, 1, 1), 33, 2.0, {"dWp_split"}),
    ("h32-b16", 64, 0, 14, (32, 4, 256), 16, 2.0, {"logits_split", "dFp_split"}),
    ("c256-b1000", 256, 0, 14, (4, 2, 256), 1000, 2.0, {"fw_partial", "bn_cap", "dWp_split"}),
    ("c64-b4096", 64, 0, 14, (4, 2, 256), 4096, 2.0, {"fw_256", "bn_cap", "value_split", "dbd_split", "dWp_split"}),
    ("1blk-c64-b7", 64, 1, 14, (4, 2, 256), 7, 2.0, {"dFp_split"}),
    ("1blk-c192-b256", 192, 1, 14, (4, 2, 256), 256, 2.0, {"dWp_split"}),
    ("10blk-c192-b1024", 192, 10, 14, (4, 2, 256), 1024, 2.0, {"bn_cap", "dWp_split"}),
    # 256-pixel conv tiles.  P = 1024 x 270 fills the last BN column chunk: a dropped last chunk then moves a batch
    # variance by 1/1024 of it, as at 10blk-c192-b1024, under the smaller conv bound of C = 128.  (At 1573 x 256 the last of
    # 1019 chunks holds 68 rows, and dropping it stays within the conv's propagated bound.)
    ("1blk-c128-b3072", 128, 1, 14, (4, 2, 256), 3072, 2.0, {"conv_m256", "bn_cap", "dWp_split"}),
]


def geometry_paths(n, C_, heads, blocks):
    """Which launch paths the restated geometry predicts for this shape."""
    pc, vc, H = heads
    pk, vk, P = pc * 90, vc * 90, n * 90
    paths = set()
    if blocks and nc.conv_tile_m(n, C_, torch.cuda.get_device_properties(0).multi_processor_count) == 256:
        paths.add("conv_m256")                      # the residual block's convs and dgrads on 256-pixel M tiles
    ch, per = first_wgrad_geometry(n)
    if ch == 2:
        paths.add("fw_chunks2")
    if ch == 16 and n % per:
        paths.add("fw_partial")
    if ch == 16 and per == 256:
        paths.add("fw_256")
    if -(-P // 64) > 1024:
        paths.add("bn_cap")
    if gemm_splits(n, N_LABELS, pk)[0] > 1:
        paths.add("logits_split")
    if gemm_splits(n, pk, N_LABELS)[0] > 1:
        paths.add("dFp_split")
    if all(gemm_splits(*s)[0] > 1 for s in ((H, 1, n), (1, 1, n), (vk, H, n), (1, H, n))):
        paths.add("value_split")
    if gemm_splits(1, N_LABELS, n)[0] > 1:
        paths.add("dbd_split")
    if gemm_splits(C_, pc, P)[0] > 1 and gemm_splits(C_, vc, P)[0] > 1:
        paths.add("dWp_split")
    return paths


def test_geometry_restatement_reaches_every_path():
    """The cases below reach every split / chunk path of the step's launch code (host-only arithmetic)."""
    hit = set()
    for _, c, blocks, _, heads, n, _, want in CASES:
        got = geometry_paths(n, c, heads, blocks)
        assert want <= got, (n, c, heads, want - got)
        hit |= got
    assert {"conv_m256", "fw_chunks2", "fw_partial", "fw_256", "bn_cap", "logits_split", "dFp_split", "value_split",
            "dbd_split", "dWp_split"} <= hit
    assert first_wgrad_geometry(1000) == (16, 63) and 1000 - 15 * 63 == 55
    assert first_wgrad_geometry(4096) == (16, 256)
    assert col_chunks(729 * 90)[0] <= 1024 < -(-729 * 90 // 64)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_train_step_stages_match_float64(cuda_lib, case):
    from cczero_b200.model import CChessModel
    from cczero_b200.train import Trainer
    cid, C_, L, ip, heads, n, logit_std, want = case
    pc, vc, H = heads
    pk, vk, P = pc * 90, vc * 90, n * 90
    assert want <= geometry_paths(n, C_, heads, L)
    dev = "cuda"
    seed = n + 7 * L + C_
    planes = positions(n, ip, seed % 5)
    w = nc.well_conditioned_weights(C_, L, planes[:64], seed=seed, logit_std=logit_std, in_planes=ip, policy_filters=pc,
                                    value_filters=vc, value_fc=H)
    w64 = {k: torch.as_tensor(v, dtype=torch.float64, device=dev) for k, v in w.items()}
    # batch statistics move the heads away from the moving-statistics scaling (a batch of 1 saturates tanh): rescale
    # policy_out and value_out so that the training-mode logits and value_pre have the same spread
    logits0, vpre0 = to.forward_train(w64, planes, L, device=dev)[:2]
    a, b = logit_std / logits0.std(dim=1).mean().item(), 0.5 / vpre0.abs().median().item()
    for k, f in (("policy_out/kernel", a), ("policy_out/bias", a), ("value_out/kernel", b), ("value_out/bias", b)):
        w[k] = (w[k].astype(np.float64) * f).astype(np.float32)
        w64[k] = torch.as_tensor(w[k], dtype=torch.float64, device=dev)
    logits0 = to.forward_train(w64, planes, L, device=dev)[0]
    pol, val, sharp_row = targets(n, logits0, seed, logit_std > 10)
    cfg = config(C_, L, ip, heads, n)
    model = CChessModel(cfg)
    model.weights = {k: np.asarray(v, np.float32) for k, v in w.items()}
    tr = Trainer(model, n, dev)
    lr = 0.01
    losses = tr.step(planes, pol, val, lr)
    R = Report(cid)

    def W(layer, weight):
        return w64[to._name(w64, layer, weight)]

    def f64(x):
        return x.to(torch.float64)

    def rd(which, index=0, dtype=torch.float32):
        return read(tr, which, index, dtype)

    X = torch.as_tensor(planes, dtype=torch.float64, device=dev)
    T = torch.as_tensor(pol, dtype=torch.float64, device=dev)
    Z = torch.as_tensor(val, dtype=torch.float64, device=dev)
    w_p, w_v = (float(np.float32(x)) for x in cfg.trainer.loss_weights)
    l2 = float(np.float32(cfg.model.l2_reg))

    # ------------------------------------------------------------------------------------------ first conv + input BN
    nb = ip // 14
    pl = rd(PLANE_INDEX, dtype=torch.int8).reshape(n, 2, 90)[:, :nb].long()
    occ = X.reshape(n, nb, 14, 90)
    want_pl = torch.where(occ.amax(2) > 0.5, occ.argmax(2), torch.full_like(occ[:, :, 0], -1).long())
    R.exact("plane index", pl, want_pl)
    Wf = W("input_conv", "kernel").permute(3, 2, 0, 1)                  # OIHW
    z0 = pix(F.conv2d(X, Wf, padding=2))
    k_first = 25 * nb                                                   # occupied taps, summed in order
    zb0 = beta(k_first) * pix(F.conv2d(X, Wf.abs(), padding=2))
    m0, v0 = f64(rd(BN_MEAN, 0)), f64(rd(BN_VAR, 0))

    def stats(j, z, zb, what):
        m, v = f64(rd(BN_MEAN, j)), f64(rd(BN_VAR, j))
        k = bn_chain(P, z.shape[1])
        ch, rows = col_chunks(P)
        last = slice((ch - 1) * rows, P)
        R.check(f"{what} mean", m, z.mean(0), z.abs().mean(0), k, zb.mean(0),
                [delta("last column chunk dropped", -z[last].sum(0) / P)])
        d = z - m
        R.check(f"{what} var", v, (d * d).mean(0), ((z.abs() + m.abs()) ** 2).mean(0), k + 2, (2 * d.abs() * zb + zb * zb).mean(0),
                [delta("last column chunk dropped", -(d[last] ** 2).sum(0) / P)])
        return m, v

    stats(0, z0, zb0, "input BN")
    g0, b0 = W("input_batchnorm", "gamma"), W("input_batchnorm", "beta")
    y0, Sy0, ey0 = bn_apply(z0, zb0, m0, v0, g0, b0)
    s0 = f64(rd(BLOCK_OUT32, 0).reshape(P, C_))
    Wedge = torch.zeros_like(Wf)
    Wedge[:, :, 2, 4] = Wf[:, :, 2, 4]                                  # tap (2, 4) reads the column two to the right
    Xedge = torch.zeros_like(X)
    Xedge[..., 8] = X[..., 8]
    muts = [delta("one board-edge tap missing", torch.relu(bn_apply(z0 - pix(F.conv2d(Xedge, Wedge, padding=2)), zb0, m0, v0,
                                                                       g0, b0)[0]) - torch.relu(y0))]
    if ip == 28:
        Xh = X.clone()
        Xh[:, 14:] = X[:, :14]
        muts.append(delta("history board read as board 0", torch.relu(bn_apply(pix(F.conv2d(Xh, Wf, padding=2)), zb0, m0, v0,
                                                                                   g0, b0)[0]) - torch.relu(y0)))
    R.check("first conv + BN + ReLU (s32[0])", s0, torch.relu(y0), Sy0, 7, ey0, muts)
    R.exact("a16[0] = fp16(s32[0])", rd(BLOCK_OUT16, 0, torch.float16).reshape(P, C_), s0.float().half())

    # ------------------------------------------------------------------------------------------ head 1x1 convs + BN, Flatten order
    SL = f64(rd(BLOCK_OUT32, L).reshape(P, C_))
    heads_fwd = {}
    for name, j, c, buf, conv, bn in (("policy", 2 * L + 1, pc, POL_FEAT, "policy_conv", "policy_batchnorm"),
                                      ("value", 2 * L + 2, vc, VAL_FEAT, "value_conv", "value_batchnorm")):
        Wc = W(conv, "kernel").reshape(C_, c)
        z = SL @ Wc
        zb = beta(gemm_chain(P, c, C_)) * (SL.abs() @ Wc.abs())
        m, v = stats(j, z, zb, f"{name} BN")
        y, Sy, ey = bn_apply(z, zb, m, v, W(bn, "gamma"), W(bn, "beta"))
        got = f64(rd(buf).reshape(n, c * 90))
        muts = [nc.Mutation("features shifted by one pixel", lambda g, r, c=c: torch.roll(g.reshape(n, c, 90), 1, 2).reshape(n, -1))]
        if c > 1:
            muts.append(nc.Mutation("pixel-major Flatten", lambda g, r, c=c: g.reshape(n, c, 90).transpose(1, 2).reshape(n, -1)))
        R.check(f"{name} features (Flatten order)", got, flat_of_rows(torch.relu(y), n, c), flat_of_rows(Sy, n, c), 7,
                flat_of_rows(ey, n, c), muts)
        heads_fwd[name] = (z, zb, m, v, got)
    Fp, Fv = heads_fwd["policy"][4], heads_fwd["value"][4]

    # ------------------------------------------------------------------------------------------ logits and value MLP
    Wd, bd = W("policy_out", "kernel"), W("policy_out", "bias")
    logits = f64(rd(LOGITS).reshape(n, N_LABELS))
    S_lg = Fp.abs() @ Wd.abs() + bd.abs()
    d_tile = torch.zeros_like(logits)
    d_tile[:, 2080:] = S_lg[:, 2080:] / pk
    R.check("logits", logits, Fp @ Wd + bd, S_lg, gemm_chain(n, N_LABELS, pk, 1),
            mutations=[delta("last 6 labels (partial 16-tile) off by one term", d_tile), delta("bias missing", -bd.expand(n, -1))])
    W1, b1, W2, b2 = W("value_dense", "kernel"), W("value_dense", "bias"), W("value_out", "kernel"), W("value_out", "bias")
    hpre = f64(rd(VAL_HIDDEN_PRE).reshape(n, H))
    R.check("value hidden before ReLU", hpre, Fv @ W1 + b1, Fv.abs() @ W1.abs() + b1.abs(), gemm_chain(n, H, vk, 1),
            mutations=[delta("bias missing", -b1.expand(n, -1))])
    hact = f64(rd(VAL_HIDDEN).reshape(n, H))
    R.exact("value hidden = relu(pre)", hact, torch.relu(hpre))
    vpre = f64(rd(VAL_PRE))
    R.check("value before tanh", vpre, (hact @ W2 + b2)[:, 0], (hact.abs() @ W2.abs() + b2.abs())[:, 0], gemm_chain(n, 1, H, 1),
            mutations=[delta("bias missing", -b2.expand(n))])

    # ------------------------------------------------------------------------------------------ losses and output gradients
    lm = logits - logits.max(1, keepdim=True).values
    p = torch.softmax(logits, 1)
    eps, hi = to.KERAS_EPS, to.KERAS_HI
    # relative error of the GPU's renormalised probability: expf (2 ulp) of an argument rounded once (|lm| u), a
    # 256-lane sum of <= 9 terms per lane and an 8-level tree (17), the reciprocal, the product, the renormalising sum (17)
    # and division: <= 64 u + |lm| u.
    rel = U * (64 + lm.abs())
    c = p.clamp(eps, hi)
    inside = (p >= eps) & (p <= hi) & (T != 0)
    near = (T != 0) & (((p - eps).abs() <= 2 * rel * eps) | ((p - hi).abs() <= 2 * rel))
    ce = f64(rd(CE_ROWS))
    ce_ref = -(T * torch.log(c)).sum(1)
    ce_err = 4 * (T.abs() * (rel + 20 * U * torch.log(c).abs())).sum(1)
    tl = (T * torch.log(c)).abs()
    i_ce, j_ce = divmod(int(tl.argmax()), N_LABELS)
    d_ce = torch.zeros_like(ce_ref)
    d_ce[i_ce] = (T * torch.log(c))[i_ce, j_ce]
    R.check("CE rows", ce, ce_ref, 0, 1, ce_err, [delta("one target term dropped", d_ce)])
    v = torch.tanh(vpre)
    ev = 2 * U * v.abs()                                                # tanhf: 2 ulp
    d = v - Z
    ed = ev + U * (v.abs() + Z.abs())
    se = f64(rd(SE_ROWS))
    R.check("SE rows", se, d * d, (v.abs() + Z.abs()) ** 2, 2, 2 * d.abs() * ed,
            [delta("value target sign flipped", (v + Z) ** 2 - d * d)])
    lo_gpu = torch.as_tensor(losses, dtype=torch.float64, device=dev)
    kb = -(-n // 256) + 8 + 1
    R.check("losses[1] = mean CE", lo_gpu[1:2], ce.mean().view(1), ce.abs().mean().view(1), kb,
            mutations=[delta("one row dropped", -ce.max().view(1) / n)])
    R.check("losses[2] = mean SE", lo_gpu[2:3], se.mean().view(1), se.abs().mean().view(1), kb,
            mutations=[delta("one row dropped", -se.max().view(1) / n)])
    kern = [k for k in w64 if to.is_reg(k)]
    l2_ref = l2 * sum((w64[k] ** 2).sum() for k in kern)
    k_l2 = max(-(-w64[k].numel() // 256) for k in kern) + 8 + len(kern) + 1
    share = {k: (l2 * (w64[k] ** 2).sum()).item() for k in kern}
    k_small = min((k for k in kern if share[k] > 1e-3 * l2_ref.item()), key=share.get)   # the smallest visible kernel
    R.check("losses[3] = L2", lo_gpu[3:4], l2_ref.view(1), l2_ref.view(1), k_l2,
            mutations=[delta(f"{k_small} left out", -torch.tensor([share[k_small]], dtype=torch.float64, device=dev))])
    tot = w_p * lo_gpu[1] + w_v * lo_gpu[2] + lo_gpu[3]
    R.check("losses[0] = total", lo_gpu[0:1], tot.view(1), (w_p * lo_gpu[1].abs() + w_v * lo_gpu[2].abs() + lo_gpu[3].abs()).view(1), 3,
            mutations=[delta("value weight 1", ((1 - w_v) * lo_gpu[2]).view(1))])

    # DLOGITS: Keras CE through renormalisation and softmax; dlog_j = w_p / n * p_j (u_j - A) with u_j = -t_j / c_j inside
    # the clip interval and A = sum u p.  Terms whose probability lies within its error of a clip edge may take either side.
    scale = w_p / n

    def dlog_ref(ins):
        u = torch.where(ins, -T / c, torch.zeros_like(T))
        A = (u * p).sum(1, keepdim=True)
        g = u - A
        return scale * p * (g - (g * p).sum(1, keepdim=True)), u
    ref_dl, u_in = dlog_ref(inside)
    ref_flip = dlog_ref(inside ^ near)[0]
    u_any = dlog_ref(inside | near)[1].abs()                          # error terms of either decision
    Aabs = (u_any * p).sum(1, keepdim=True)
    term = (u_any + Aabs) * (3 * rel + 20 * U)
    # + subnormal outputs: each of the <= 8 roundings of the product chain loses up to half the spacing 2^-149 absolutely
    dl_err = (4 * scale * p * (term + (p * term).sum(1, keepdim=True)) + (ref_flip - ref_dl).abs() +
              2.0 ** -149 * (4 + 2 * scale * (u_any + Aabs)))
    dlog = f64(rd(DLOGITS).reshape(n, N_LABELS))
    zero_rows = [i for i in range(n) if (T[i] == 0).all()] + ([sharp_row] if sharp_row is not None else [])

    def dlog_check(g, r):
        for i in zero_rows:
            assert torch.count_nonzero(g[i]).item() == 0, f"{cid}: DLOGITS row {i} must be exactly zero"
        return nc.check_close(g, r, torch.zeros_like(r), out="fp32", extra=dl_err + 0.5 * nc.ulp32(torch.maximum(g.abs(), r.abs())),
                              what=f"{cid}: DLOGITS")

    worst = dlog_check(dlog, ref_dl)
    # the A term is zero where every target term is clipped (a one-hot label below 1e-7); "no clip" then moves the row
    cands = [("soft-target term A missing", scale * p * u_in - ref_dl), ("no clip", dlog_ref(T != 0)[0] - ref_dl)]
    if sharp_row is not None:
        cands.append(("clip applied below only", dlog_ref((p >= eps) & (T != 0))[0] - ref_dl))
    muts = [delta(name, d) for name, d in cands if not torch.equal(dlog + d, dlog)]
    assert muts and (sharp_row is None or muts[-1].name == "clip applied below only")
    nc.assert_rejects(dlog_check, dlog, ref_dl, muts)
    R.rows.append(("DLOGITS", worst, len(muts)))
    if sharp_row is not None:
        assert p[sharp_row].max().item() > hi

    dvpre = f64(rd(DVAL_PRE))
    cv = 2 * w_v / n
    one_m = 1 - v * v
    dv_err = 2 * abs(cv) * (ed * one_m.abs() + d.abs() * (2 * v.abs() * ev + 2 * U * (1 + v * v)) + 4 * U * d.abs() * one_m.abs())
    R.check("DVAL_PRE", dvpre, cv * d * one_m, 0, 1, dv_err, [delta("(1 - v^2) missing", cv * d - cv * d * one_m)])
    dh = f64(rd(DVAL_HIDDEN).reshape(n, H))
    mask_h = (hpre > 0).double()
    dh_ref = mask_h * dvpre[:, None] * W2[:, 0]
    cands = [("ReLU mask missing", dvpre[:, None] * W2[:, 0] - dh_ref),
             ("ReLU mask one row off", (torch.roll(mask_h, 1, 0) - mask_h) * dvpre[:, None] * W2[:, 0])]
    muts = [delta(name, d) for name, d in cands if not torch.equal(dh + d, dh)]
    assert muts, "no hidden unit masked"
    R.check("DVAL_HIDDEN (masked)", dh, dh_ref, dh_ref.abs(), 1, mutations=muts)

    # ------------------------------------------------------------------------------------------ head weight gradients
    def grad(layer, weight):
        return f64(tr.grad(to._name(w64, layer, weight)))

    def sum_grad(what, got, A, B, M, N, K):
        """got = A^T B over K rows (k_gemm of M x N, K): check, rejecting the last K split dropped (or one term)."""
        ref, S = A.t() @ B, A.abs().t() @ B.abs()
        s, kps = gemm_splits(M, N, K)
        if s > 1:
            r0 = kps * (s - 1)
            muts = [delta(f"last of {s} K splits dropped", -(A[r0:].t() @ B[r0:]))]
        else:
            muts = [add_term(S, K)]
        return R.check(what, got.reshape(ref.shape), ref, S, gemm_chain(M, N, K), mutations=muts), s

    ones = torch.ones(n, 1, dtype=torch.float64, device=dev)
    split_seen = {}
    _, split_seen["dW2"] = sum_grad("dW2 (value_out kernel)", grad("value_out", "kernel"), hact, dvpre[:, None], H, 1, n)
    _, split_seen["db2"] = sum_grad("db2 (value_out bias)", grad("value_out", "bias"), ones, dvpre[:, None], 1, 1, n)
    gW1 = grad("value_dense", "kernel")
    ref1 = Fv.t() @ dh
    s1, kps1 = gemm_splits(vk, H, n)
    muts = [add_term(Fv.abs().t() @ dh.abs(), n)]
    if H > 1:
        muts.append(nc.Mutation("transposed dW1", lambda g, r: g.t().contiguous().reshape(vk, H)))
    if s1 > 1:
        muts.append(delta(f"last of {s1} K splits dropped", -(Fv[kps1 * (s1 - 1):].t() @ dh[kps1 * (s1 - 1):])))
    R.check("dW1 (value_dense kernel)", gW1, ref1, Fv.abs().t() @ dh.abs(), gemm_chain(vk, H, n), mutations=muts)
    split_seen["dW1"] = s1
    _, split_seen["db1"] = sum_grad("db1 (value_dense bias)", grad("value_dense", "bias"), ones, dh, 1, H, n)
    sum_grad("dWd (policy_out kernel)", grad("policy_out", "kernel"), Fp, dlog, pk, N_LABELS, n)
    _, split_seen["dbd"] = sum_grad("dbd (policy_out bias)", grad("policy_out", "bias"), ones, dlog, 1, N_LABELS, n)
    if "value_split" in want:
        assert all(split_seen[k] > 1 for k in ("dW2", "db2", "dW1", "db1")), split_seen
    if "dbd_split" in want:
        assert split_seen["dbd"] > 1

    # DPOL_FEAT = dlog Wd^T
    dFp = f64(rd(DPOL_FEAT).reshape(n, pk))
    s, kps = gemm_splits(n, pk, N_LABELS)
    S_dF = dlog.abs() @ Wd.abs().t()
    muts = [add_term(S_dF, N_LABELS)]
    if s > 1:
        muts.append(delta(f"last of {s} K splits dropped", -(dlog[:, kps * (s - 1):] @ Wd[:, kps * (s - 1):].t())))
    R.check("DPOL_FEAT", dFp, dlog @ Wd.t(), S_dF, gemm_chain(n, pk, N_LABELS), mutations=muts)
    if "dFp_split" in want:
        assert s > 1

    # ------------------------------------------------------------------------------------------ head BN backward (flat upstream)
    dFv = dh @ W1.t()
    dFv_err = beta(gemm_chain(n, vk, H)) * (dh.abs() @ W1.abs().t()) + 0.5 * nc.ulp32(dFv)
    dz_head = {}
    for name, j, cc, up, up_err, bn in (("policy", 2 * L + 1, pc, dFp, torch.zeros_like(dFp), "policy_batchnorm"),
                                        ("value", 2 * L + 2, vc, dFv, dFv_err, "value_batchnorm")):
        z, zb, m, var, feat = heads_fwd[name]
        gamma = W(bn, "gamma")
        mask = rows_of_flat((feat > 0).double(), n, cc)
        up_r, err_r = rows_of_flat(up, n, cc), rows_of_flat(up_err, n, cc)
        ref, S, err = bn_backward(z, zb, m, var, gamma, up_r, err_r, mask)
        got = f64(rd(BN_DZ, j).reshape(P, cc))
        shifted = rows_of_flat(torch.roll(up.reshape(n, cc, 90), 1, 2).reshape(n, -1), n, cc)
        muts = [delta("upstream shifted by one pixel", bn_backward(z, zb, m, var, gamma, shifted, err_r, mask)[0] - ref)]
        if cc > 1:
            muts.append(delta("upstream read in row order", bn_backward(z, zb, m, var, gamma, up.reshape(P, cc), err_r, mask)[0] - ref))
        R.check(f"{name} BN dz (BN_DZ[{j}])", got, ref, S, bn_chain(P, cc) + 6, err, muts)
        dz_head[name] = got

    # dWp, dWv = s32[L]^T dz
    for name, cc, conv in (("dWp", pc, "policy_conv"), ("dWv", vc, "value_conv")):
        dz = dz_head["policy" if name == "dWp" else "value"]
        _, s = sum_grad(f"{name} ({conv} kernel)", grad(conv, "kernel"), SL, dz, C_, cc, P)
        if "dWp_split" in want:
            assert s > 1, (name, s)

    Wp, Wv = W("policy_conv", "kernel").reshape(C_, pc), W("value_conv", "kernel").reshape(C_, vc)
    dzp, dzv = dz_head["policy"], dz_head["value"]
    G_ref = dzp @ Wp.t() + dzv @ Wv.t()
    S_G = dzp.abs() @ Wp.abs().t() + dzv.abs() @ Wv.abs().t()
    k_G = pc + vc + 1
    if L == 0:
        G = f64(rd(TRUNK_GRAD).reshape(P, C_))
        R.check("TRUNK_GRAD = dzp Wp^T + dzv Wv^T", G, G_ref, S_G, k_G, mutations=[delta("dzv Wv^T term missing", -(dzv @ Wv.t()))])
    else:
        # ------------------------------------------------------------------------------------------ last residual block
        i = L - 1
        Gb = beta(k_G) * S_G + 0.5 * nc.ulp32(G_ref)
        slots = rd(SCALE_SLOTS).reshape(2 * L + 1, 4)
        h16 = rd(CONV1_OUT16, i, torch.float16).reshape(P, C_)
        a16 = rd(BLOCK_OUT16, i, torch.float16).reshape(P, C_)
        s_prev = f64(rd(BLOCK_OUT32, i).reshape(P, C_))
        k_conv = 9 * C_

        def conv_z(x16, layer):
            Wk = W(layer, "kernel").float().half().double().permute(3, 2, 0, 1)
            Xn = nchw(f64(x16), n, C_)
            return pix(F.conv2d(Xn, Wk, padding=1)), beta(k_conv) * pix(F.conv2d(Xn.abs(), Wk.abs(), padding=1)), Wk

        z2, zb2, W2k = conv_z(h16, f"res{L}_conv2")
        m2, var2 = stats(2 * L, z2, zb2, f"res{L} BN2")
        mask2 = (SL > 0).double()                                      # s32[L] = relu(y2 + skip)
        ref2, S2, err2 = bn_backward(z2, zb2, m2, var2, W(f"res{L}_batchnorm2", "gamma"), G_ref, Gb, mask2)
        dz2 = f64(rd(BN_DZ, 2 * L).reshape(P, C_))
        R.check(f"res{L} conv2 BN dz", dz2, ref2, S2, bn_chain(P, C_) + 6, err2,
                [delta("upstream unmasked", bn_backward(z2, zb2, m2, var2, W(f"res{L}_batchnorm2", "gamma"), G_ref, Gb,
                                                        torch.ones_like(mask2))[0] - ref2)])

        def scale_slot(slot, dz, what):
            """{max |dz| (float bits), 2^e, 2^-e} with max |dz| 2^e in [2^14, 2^15), from the GPU's own dz."""
            mx = dz.abs().max().item()
            e = 0 if mx == 0 else 14 - (int(np.frexp(mx)[1]) - 1)
            R.exact(f"{what} scale slot", slots[slot, :3].cpu(), torch.tensor([mx, 2.0 ** e, 2.0 ** -e], dtype=torch.float32))
            return e

        e2 = scale_slot(2 * i + 1, dz2, f"res{L} conv2")
        dz2_16 = to._scaled16(dz2)
        sp, per = wgrad_geometry(n, C_)
        k_wg = per * 64 + sp

        def wgrad_check(what, x16, dz16, layer):
            Xn, Gn = nchw(f64(x16), n, C_), nchw(dz16, n, C_)
            ref = torch.nn.grad.conv2d_weight(Xn, (C_, C_, 3, 3), Gn, padding=1).permute(2, 3, 1, 0)
            S = torch.nn.grad.conv2d_weight(Xn.abs(), (C_, C_, 3, 3), Gn.abs(), padding=1).permute(2, 3, 1, 0)
            Xc = Xn.clone()
            Xc[..., 8] = 0
            edge = torch.nn.grad.conv2d_weight(Xc, (C_, C_, 3, 3), Gn, padding=1).permute(2, 3, 1, 0)
            R.check(what, grad(layer, "kernel"), ref, S, k_wg, mutations=[
                nc.Mutation("transposed wgrad", lambda g, r: g.transpose(2, 3).contiguous()),
                delta("one board-edge column missing", edge - ref)])

        wgrad_check(f"res{L} conv2 wgrad", h16, dz2_16, f"res{L}_conv2")
        D2 = pix(torch.nn.grad.conv2d_input((n, C_, 10, 9), W2k, nchw(dz2_16, n, C_), padding=1))
        D2b = beta(k_conv) * pix(torch.nn.grad.conv2d_input((n, C_, 10, 9), W2k.abs(), nchw(dz2_16.abs(), n, C_), padding=1))

        z1, zb1, W1k = conv_z(a16, f"res{L}_conv1")
        m1, var1 = stats(2 * L - 1, z1, zb1, f"res{L} BN1")
        g1 = W(f"res{L}_batchnorm1", "gamma")
        y1, Sy1, ey1 = bn_apply(z1, zb1, m1, var1, g1, W(f"res{L}_batchnorm1", "beta"))
        yb1 = beta(7) * Sy1 + ey1 + 0.5 * nc.ulp32(y1)

        def chk_h16(g, r):
            return nc.check_close(g, r, Sy1 * (beta(7) / nc.BETA), out="fp16", extra=ey1, what=f"{cid}: res{L} conv1 output (fp16)")
        R.rows.append((f"res{L} conv1 + BN + ReLU (h16)", chk_h16(f64(h16), torch.relu(y1)), 1))
        nc.assert_rejects(lambda g, r: chk_h16(g.reshape(P, C_), r), f64(h16).reshape(n, 90, C_), torch.relu(y1),
                          [nc.ShiftBlock(64)] + (nc.tile256_mutations() if "conv_m256" in want else []))
        y2, Sy2, ey2 = bn_apply(z2, zb2, m2, var2, W(f"res{L}_batchnorm2", "gamma"), W(f"res{L}_batchnorm2", "beta"), s_prev)
        R.check(f"res{L} output (s32[{L}])", SL, torch.relu(y2), Sy2, 7, ey2,
                [nc.Mutation("residual dropped from one channel",
                             lambda g, r: nc.DropResidual(s_prev.reshape(n, 90, C_))(g.reshape(n, 90, C_), r).reshape(P, C_))])
        sure = (f64(h16) > 0).double()
        amb = (h16 == 0) & (y1 + yb1 > 0)                              # fp16 underflow: either mask
        print(f"{cid}: {int(amb.sum())} conv1 outputs may take either ReLU mask (fp16 underflow)")
        ref1, S1, err1 = bn_backward(z1, zb1, m1, var1, g1, D2, D2b, sure, amb.double())
        dz1 = f64(rd(BN_DZ, 2 * L - 1).reshape(P, C_))
        R.check(f"res{L} conv1 BN dz", dz1, ref1, S1, bn_chain(P, C_) + 6, err1,
                [delta("upstream unmasked", bn_backward(z1, zb1, m1, var1, g1, D2, D2b, torch.ones_like(sure))[0] - ref1)])
        e1 = scale_slot(2 * i, dz1, f"res{L} conv1")
        dz1_16 = to._scaled16(dz1)
        wgrad_check(f"res{L} conv1 wgrad", a16, dz1_16, f"res{L}_conv1")
        if L == 1:
            D1 = pix(torch.nn.grad.conv2d_input((n, C_, 10, 9), W1k, nchw(dz1_16, n, C_), padding=1))
            S_D1 = pix(torch.nn.grad.conv2d_input((n, C_, 10, 9), W1k.abs(), nchw(dz1_16.abs(), n, C_), padding=1))
            G = f64(rd(TRUNK_GRAD).reshape(P, C_))
            tg = mask2 * G_ref + D1
            R.check("TRUNK_GRAD = masked G_1 + dgrad", G, tg, torch.zeros_like(tg), 1,
                    mask2 * Gb + beta(k_conv) * S_D1 + 0.5 * nc.ulp32(G_ref), [
                        delta("skip path unmasked", (1 - mask2) * G_ref),
                        delta("dgrad contribution not unscaled", D1 * (2.0 ** e1 - 1))])
    # ------------------------------------------------------------------------------------------ input BN backward, first wgrad
    G = f64(rd(TRUNK_GRAD).reshape(P, C_))
    mask0 = (s0 > 0).double()
    ref0, S0, err0 = bn_backward(z0, zb0, m0, v0, g0, G, torch.zeros_like(G), mask0)
    dz0 = f64(rd(BN_DZ, 0).reshape(P, C_))
    R.check("input BN dz (BN_DZ[0])", dz0, ref0, S0, bn_chain(P, C_) + 6, err0,
            [delta("BN backward without its mean terms", g0 / torch.sqrt(v0 + BN_EPS) * G * mask0 - ref0)])
    Pl = X                                                              # PLANE_INDEX equals the input planes (checked above)
    ch, per = first_wgrad_geometry(n)
    if "fw_chunks2" in want:
        assert ch == 2
    if "fw_partial" in want:
        assert (ch, per, n - (ch - 1) * per) == (16, 63, 55)
    if "fw_256" in want:
        assert (ch, per) == (16, 256)
    Dn = nchw(dz0, n, C_)
    shape = (C_, ip, 5, 5)
    ref_fw = torch.nn.grad.conv2d_weight(Pl, shape, Dn, padding=2)
    S_fw = torch.nn.grad.conv2d_weight(Pl, shape, Dn.abs(), padding=2)
    b0_last = (ch - 1) * per
    tap24 = (torch.arange(25, device=dev).reshape(1, 1, 5, 5) == 2 * 5 + 4).double()     # tap (2, 4), column 8 squares
    muts = [delta("one tap's board edge missing", (-torch.nn.grad.conv2d_weight(Xedge, shape, Dn, padding=2) * tap24)
                  .permute(2, 3, 1, 0))]
    if ch > 1:
        muts.append(delta("last position chunk dropped", -torch.nn.grad.conv2d_weight(Pl[b0_last:], shape, Dn[b0_last:], padding=2)
                          .permute(2, 3, 1, 0)))
    R.check("first-conv wgrad", grad("input_conv", "kernel"), ref_fw.permute(2, 3, 1, 0), S_fw.permute(2, 3, 1, 0), per * 90 + ch,
            mutations=muts)

    # ------------------------------------------------------------------------------------------ update
    mom = float(np.float32(cfg.trainer.momentum))
    lr32 = float(np.float32(lr))
    for k in w64:
        if to.is_stat(k):
            continue
        g = f64(tr.grad(k)).reshape(w64[k].shape)
        l2x2 = 2 * l2 if to.is_reg(k) else 0.0
        v_ref = mom * 0.0 - lr32 * (g + l2x2 * w64[k])
        v_S = lr32 * (g.abs() + l2x2 * w64[k].abs())
        vel = f64(tr.velocity[k])
        muts = [delta("L2 missing", lr32 * l2x2 * w64[k])] if k.startswith("value_dense") and to.is_reg(k) else []
        if muts or k.startswith("input_conv"):
            R.check(f"SGD velocity {k}", vel, v_ref, v_S, 4, mutations=muts or [add_term(v_S, 1)])
        else:
            R.check(f"SGD velocity {k}", vel, v_ref, v_S, 4)
        R.check(f"SGD weight {k}", f64(tr.weights[k]), w64[k] + vel, w64[k].abs() + vel.abs(), 1,
                mutations=[delta("velocity not added", -vel)] if k.startswith("input_conv") else ())
    cm = float(np.float32(1) - np.float32(0.99))
    for j, layer in enumerate(["input_batchnorm"] + [f"res{b}_batchnorm{c}" for b in range(1, L + 1) for c in (1, 2)] +
                              ["policy_batchnorm", "value_batchnorm"]):
        bm, bv = f64(rd(BN_MEAN, j)), f64(rd(BN_VAR, j))
        for stat, batch_stat in (("moving_mean", bm), ("moving_variance", bv)):
            m_old = W(layer, stat)
            ref = m_old - (m_old - batch_stat) * cm
            # three fp32 roundings (m - b, * c, m - .), each within 2^-24 of S: the worst case, not beta(3)
            S_m = m_old.abs() + (m_old.abs() + batch_stat.abs()) * cm
            muts = [delta("momentum 0.9 instead of 0.99", -(m_old - batch_stat) * (0.1 - cm))]
            unbiased = bv * cm / (P - 1)
            if stat == "moving_variance" and (unbiased > 4 * U * S_m + nc.ulp32(ref)).any():
                # visible in fp32 only up to batch ~500: beyond, var / (P - 1) * 0.01 is below one ulp of the average
                muts.append(delta("moving variance unbiased", unbiased))
            R.check(f"moving {stat} {layer}", f64(tr.weights[to._name(w64, layer, stat)]), ref, 0, 1, 3 * U * S_m,
                    mutations=muts)
    R.print()
    tr.close()


def test_read_buffer_errors(cuda_lib):
    """cz_train_read_buffer: CZ_ERR_STATE before the first step; CZ_ERR_ARG for an unknown buffer, an index out of range
    and a destination that is too small."""
    from cczero_b200.lib import CzError
    from cczero_b200.model import CChessModel
    from cczero_b200.train import Trainer
    cfg = config(64, 1, 14, (4, 2, 256), 4)
    model = CChessModel(cfg)
    model.weights = om.init_weights(64, 1, 256, seed=1)
    tr = Trainer(model, 4, "cuda")
    nb = C.c_int64(0)
    with pytest.raises(CzError, match=r"\(-3\)"):
        tr.lib.call("cz_train_read_buffer", tr._h, LOGITS, 0, None, 0, C.byref(nb))
    planes = positions(3, 14, 0)
    pol = np.zeros((3, N_LABELS), np.float32)
    pol[:, 5] = 1
    tr.step(planes, pol, np.zeros(3, np.float32), 0.01)
    tr.lib.call("cz_train_read_buffer", tr._h, LOGITS, 0, None, 0, C.byref(nb))
    assert nb.value == 3 * N_LABELS * 4                                  # the last step's batch, not max_batch
    tr.lib.call("cz_train_read_buffer", tr._h, BN_DZ, 4, None, 0, C.byref(nb))
    assert nb.value == 3 * 90 * 2 * 4                                    # 2L + 2 = the value BN (2 channels)
    tr.lib.call("cz_train_read_buffer", tr._h, SCALE_SLOTS, 0, None, 0, C.byref(nb))
    assert nb.value == 3 * 4 * 4
    for which, index in ((21, 0), (-1, 0), (BN_DZ, 5), (BLOCK_OUT32, 2), (CONV1_OUT16, 1), (LOGITS, 1), (BN_MEAN, -1)):
        with pytest.raises(CzError, match=r"\(-1\)"):
            tr.lib.call("cz_train_read_buffer", tr._h, which, index, None, 0, C.byref(nb))
    out = torch.empty(3 * N_LABELS - 1, device="cuda")
    with pytest.raises(CzError, match=r"\(-1\).*bytes"):
        tr.lib.call("cz_train_read_buffer", tr._h, LOGITS, 0, C.c_void_p(out.data_ptr()), out.numel() * 4, C.byref(nb))
    tr.close()
