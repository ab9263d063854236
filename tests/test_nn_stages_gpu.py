"""Every kernel of the network forward against a float64 reference of the same operation, one stage at a time.

The reference of a stage is "teacher-forced": it takes the GPU's own input to that stage (read back with
cz_nn_read_buffer) and the operands the GPU folded (oracle.model.folded_operands), so each kernel's error is measured
alone and must stay within rounding (tests/nn_checks.py: ALPHA * ulp_out + BETA * S).  A 1-block tower exposes every
buffer: x = first conv, t = conv1, y = tower output.  Deep towers are compared end to end, and their heads
teacher-forced on the deep tower's own output.  Every check also proves, on corrupted copies of the GPU output, that it
would have failed on a subtly wrong kernel.

The cases cover the branches of the kernels: C = 64 (no N-split) .. 256; n = 1 (one partial M tile), 9 (64-column
N-split tiles, one position per k_heads block), 64 and 301 (full-width tiles, partial last M tile, 4 positions per
k_heads block with one position in the last block); fp32 skip stream on and off; head widths (4, 2), (2, 4) and (32, 4)
(K = 8640 in the policy GEMM, > 48 KB of shared memory in k_heads); 14 and 28 input planes; and 1536 to 3109 distinct
positions, where the residual convs run 256-pixel M tiles with full, nearly empty and nearly full last tiles.  Together
the cases reach every conv kernel instance launch_igemm can choose and every epilogue form of each."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import model as om
from oracle import senv as osenv
from tests import nn_checks as nc

pytestmark = pytest.mark.gpu

# (filters, blocks, positions, fp32 skip stream (None = auto: fp32 from 10 blocks), policy channels, value channels, planes)
ONE_BLOCK = [
    (64, 1, 9, False, 4, 2, 14),
    (64, 1, 301, True, 4, 2, 28),
    (128, 1, 1, False, 4, 2, 14),
    (128, 1, 9, True, 2, 4, 14),
    (128, 1, 301, True, 4, 2, 14),
    (192, 1, 64, False, 32, 4, 28),
    (192, 1, 301, True, 2, 4, 14),
    (256, 1, 9, True, 4, 2, 28),
    (256, 1, 64, False, 32, 4, 14),
    (256, 1, 301, False, 4, 2, 14),
    # 256-pixel M tiles (two m64 blocks per consumer warpgroup) on 132 SMs; the last tile holds 90 n mod 256 pixels
    (256, 1, 1573, True, 4, 2, 14),        # 2
    (256, 1, 1536, False, 4, 2, 14),       # 0: no partial tile
    (256, 1, 1627, True, 2, 4, 14),        # 254
    (128, 1, 3109, False, 4, 2, 14),       # 2
    (128, 1, 3072, True, 4, 2, 14),        # 0
    (64, 1, 3035, False, 4, 2, 14),        # 254
    (64, 1, 3109, True, 4, 2, 14),         # 2
]
DEEP = [(192, 10, 64, None, 4, 2, 14), (256, 20, 64, None, 4, 2, 14)]
ALL = ONE_BLOCK + DEEP

# Relative Frobenius error of the fp16 TOWER_OUT of the deep well-conditioned nets against the float64 tower from the
# boards (fp32 skip stream, the default from 10 blocks).  Measured on one H100 80GB HBM3 (SXM, 400 W power limit):
# 5.0e-4 (192x10), 6.4e-4 (256x20); fp16 rounding of the output alone is ~2.8e-4.
DEEP_TOWER_REL = {10: 1.5e-3, 20: 2e-3}


def _id(case):
    c, b, n, s32, pc, vc, planes = case
    return f"{c}x{b}-n{n}-{'auto' if s32 is None else ('f32' if s32 else 'f16')}skip-h{pc}.{vc}-p{planes}"


class Run:
    """One forward of a case on the GPU with every buffer read back, its operands and its float64 reference."""

    def __init__(self, case, cuda_lib, cuda_env):
        from cczero_b200.engine import Engine
        c, blocks, n, s32, pc, vc, in_planes = case
        self.c, self.blocks, self.n, self.pc = c, blocks, n, pc
        self.s32 = blocks >= 10 if s32 is None else s32
        if n > 1024:                                       # one ply per position: thousands of distinct positions in seconds
            states = nc.distinct_states(n, seed=c + n)
            planes, hist = np.stack([osenv.state_to_planes(s) for s in states]), [None] * n
        else:
            states, planes, hist = nc.positions(n, in_planes, seed=c + n)
        self.planes = torch.from_numpy(planes).cuda()
        self.w = nc.well_conditioned_weights(c, blocks, planes, seed=c + blocks + pc, device="cuda", in_planes=in_planes,
                                             policy_filters=pc, value_filters=vc)
        self.fo = om.folded_operands(self.w, in_planes)
        self.st = om.forward_stages(self.w, planes, blocks, device="cuda")
        eng = Engine(cuda_lib, "cuda", n_games=n, sims_per_move=8, leaves_per_round=1, nn_filters=c, nn_blocks=blocks,
                     nn_value_fc=256, nn_fp32_skip=s32, use_history=in_planes == 28, nn_policy_channels=pc, nn_value_channels=vc)
        try:
            eng.set_weights({k: torch.as_tensor(v) for k, v in self.w.items()})
            pol, val = eng.nn_forward_boards(nc.boards(cuda_env, states, hist, in_planes))
            torch.cuda.synchronize()
            launches = eng.launch_count()
            self.policy, self.value = pol, val
            if blocks == 1:
                self.first = nc.read_act(eng, nc.FIRST_OUT, n, c)
                self.first32 = nc.read_act(eng, nc.FIRST_OUT32, n, c) if self.s32 else None
            self.conv1 = nc.read_act(eng, nc.LAST_CONV1, n, c)
            self.tower = nc.read_act(eng, nc.TOWER_OUT, n, c)
            self.tower32 = nc.read_act(eng, nc.TOWER_OUT32, n, c) if self.s32 else None
            self.pol_feat = nc.read_buffer(eng, nc.POL_FEAT, n).view(torch.float16)
            self.logits = nc.read_buffer(eng, nc.LOGITS, n).view(torch.float32)
            self.stats = nc.read_buffer(eng, nc.STATS, n).view(torch.float32).reshape(n, nc.KPOLN // 256, 2)
            assert eng.launch_count() == launches            # reading buffers launches nothing
        finally:
            eng.close()
        self.heads_in = self.tower32 if self.s32 else self.tower       # what k_heads read
        self.feat_ref, self.feat_scale, self.vpre_ref, self.vpre_scale = nc.heads_ref(self.heads_in, self.fo)

    def pol_segments(self):
        return nc.split_pol_feat(self.pol_feat, self.fo["pol_k1"])

    def pol_features(self):
        """GPU policy features decoded as hi + lo, channel-major [n][pol_c * 90]."""
        hi, lo, _ = self.pol_segments()
        return (hi.double() + lo.double())[:, :self.pc * 90]


# Every stage test of a case checks the same forward.  A run of more than 1024 positions holds float64 stage tensors of
# a few hundred MB each, so at most one of those is kept: the parametrizations are module-scoped, which makes pytest run
# all the tests of one case back to back.
_runs = {}
BIG = 1024


def _run(case, cuda_lib, cuda_env):
    if case not in _runs:
        if case[2] > BIG:
            for k in [k for k in _runs if k[2] > BIG]:
                del _runs[k]
            torch.cuda.empty_cache()
        _runs[case] = Run(case, cuda_lib, cuda_env)
    return _runs[case]


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _conv_mutations(r):
    """The 256-pixel tiles' own row placements on top of the checks every case runs."""
    return nc.tile256_mutations() if nc.conv_tile_m(r.n, r.c, _sms()) == 256 else []


def _report(stage, case, value):
    print(f"\n[nn-stage] {stage:<14} {_id(case):<36} {value:.3g}")


def conv_forms(case, sms):
    """(kernel instance N_TILE x M_TILE, epilogue form) of the residual convs of a 1-block case, restated from cz_nn.cu and
    k_igemm: conv1 (no skip) leaves its full M tiles by the staged epilogue and a partial last tile from registers; conv2
    adds the skip stream in registers, fp16 or fp32 (then also writing the fp32 copy out32)."""
    c, _, n, s32, *_ = case
    tm = nc.conv_tile_m(n, c, sms)
    inst = f"{nc.conv_tile_n(c, nc.use_n_split(n, c, sms))}x{tm}"
    forms = {"fp32 skip + out32" if s32 else "fp16 skip"}
    if n * 90 >= tm:
        forms.add("staged")
    if n * 90 % tm:
        forms.add("register, no skip")
    return {(inst, f) for f in forms}


def test_cases_cover_both_conv_paths(cuda_lib):
    """The residual convs take the N-split small-batch path or the full-width one depending on the SM count, and 128- or
    256-pixel M tiles; the 1-block cases above run both paths for C = 128 and C = 256 on this device, and every conv kernel
    instance launch_igemm can choose with every epilogue form."""
    sms = _sms()
    for c in (128, 256):
        assert {nc.use_n_split(n, c, sms) for (cc, _, n, *_rest) in ALL if cc == c} == {True, False}, (c, sms)
    assert any(nc.use_n_split(n, c, sms) for (c, _, n, *_r) in ONE_BLOCK) and any(n > 2 * sms for (_, _, n, *_r) in ALL)
    reached = set().union(*(conv_forms(case, sms) for case in ONE_BLOCK))
    for inst, form in sorted(reached):
        print(f"\n[nn-stage] reached {inst:<8} {form}")
    instances = {"64x128", "64x256", "128x128", "128x256", "192x128"}
    forms = {"staged", "register, no skip", "fp16 skip", "fp32 skip + out32"}
    assert {(i, f) for i in instances for f in forms} <= reached, sorted({(i, f) for i in instances for f in forms} - reached)
    assert {i for i, _ in reached} == instances


@pytest.mark.parametrize("case", ONE_BLOCK, ids=_id, scope="module")
def test_first_conv(cuda_lib, cuda_env, case):
    """k_conv_first: 5x5 conv of the one-hot planes (gathered from packed boards) + BN + ReLU, fp32 sums, fp16 out."""
    r = _run(case, cuda_lib, cuda_env)
    ref, s = nc.first_conv_ref(r.planes, r.fo, "cuda")
    check = lambda g, rf: nc.check_close(g, rf, s, "fp16", what="FIRST_OUT")
    _report("first_conv", case, check(r.first, ref))
    nc.assert_rejects(check, r.first, ref, [nc.AddTerm(s, 25), nc.ShiftBlock()])
    if r.s32:
        _report("first_conv32", case, nc.check_close(r.first32, ref, s, "fp32", what="FIRST_OUT32"))
        assert torch.equal(r.first, r.first32.half())      # fp16 output = RN(fp32 output), bit for bit


@pytest.mark.parametrize("case", ONE_BLOCK, ids=_id, scope="module")
def test_conv1(cuda_lib, cuda_env, case):
    """k_igemm conv1 of the block (BN + ReLU) on the GPU's first-conv output."""
    r = _run(case, cuda_lib, cuda_env)
    ref, s = nc.res_conv_ref(r.first, r.fo, 0)
    check = lambda g, rf: nc.check_close(g, rf, s, "fp16", what="LAST_CONV1")
    _report("conv1", case, check(r.conv1, ref))
    nc.assert_rejects(check, r.conv1, ref, [nc.AddTerm(s, 9 * r.c), nc.ShiftBlock()] + _conv_mutations(r))


@pytest.mark.parametrize("case", ONE_BLOCK, ids=_id, scope="module")
def test_conv2_with_skip(cuda_lib, cuda_env, case):
    """k_igemm conv2 (BN, + skip from the first conv in fp16 or fp32, ReLU; fp32 copy for the next block) on the GPU's conv1."""
    r = _run(case, cuda_lib, cuda_env)
    skip = (r.first32 if r.s32 else r.first).double()
    ref, s = nc.res_conv_ref(r.conv1, r.fo, 1, skip)
    check = lambda g, rf: nc.check_close(g, rf, s, "fp16", what="TOWER_OUT")
    _report("conv2", case, check(r.tower, ref))
    nc.assert_rejects(check, r.tower, ref, [nc.AddTerm(s, 9 * r.c), nc.ShiftBlock(), nc.DropResidual(skip)] + _conv_mutations(r))
    if r.s32:
        _report("conv2_32", case, nc.check_close(r.tower32, ref, s, "fp32", what="TOWER_OUT32"))
        assert torch.equal(r.tower, r.tower32.half())


@pytest.mark.parametrize("case", DEEP, ids=_id, scope="module")
def test_deep_tower_end_to_end(cuda_lib, cuda_env, case):
    """The whole residual tower of a deep net from the boards: relative Frobenius error against the float64 tower."""
    r = _run(case, cuda_lib, cuda_env)
    ref = nc.to_pix(r.st["out"][-1])
    e = nc.rel_frobenius(r.tower, ref)
    _report("tower_rel", case, e)
    if r.tower32 is not None:
        _report("tower32_rel", case, nc.rel_frobenius(r.tower32, ref))
    assert e < DEEP_TOWER_REL[r.blocks], e


@pytest.mark.parametrize("case", ALL, ids=_id, scope="module")
def test_heads_policy_features(cuda_lib, cuda_env, case):
    """k_heads: 1x1 policy conv + BN + ReLU in fp32, Keras Flatten (c * 90 + pix), split into fp16 [hi | lo | hi]."""
    r = _run(case, cuda_lib, cuda_env)
    hi, lo, hi2 = r.pol_segments()
    assert torch.equal(hi2.view(torch.int16), hi.view(torch.int16))
    pol_in = r.pc * 90
    for seg in (hi, lo, hi2):
        assert (seg[:, pol_in:].view(torch.int16) == 0).all()           # K padding is exactly +0
    assert (lo.double().abs() <= nc.ulp16(hi) / 2).all()
    got = (hi.double() + lo.double())[:, :pol_in].reshape(r.n, r.pc, 90).permute(0, 2, 1)
    check = lambda g, rf: nc.check_close(g, rf, r.feat_scale, "hilo", what="POL_FEAT")
    _report("pol_feat", case, check(got, r.feat_ref))
    nc.assert_rejects(check, got, r.feat_ref, [nc.AddTerm(r.feat_scale, r.c, "hilo"), nc.ShiftBlock()])


@pytest.mark.parametrize("case", ALL, ids=_id, scope="module")
def test_heads_value(cuda_lib, cuda_env, case):
    """k_heads value MLP (1x1 conv + BN + ReLU, Dense + ReLU, Dense, tanh), compared before tanh as atanh(value); tanhf's
    two ulps are stretched by 1 / (1 - v^2) there."""
    r = _run(case, cuda_lib, cuda_env)
    v = r.value.double()
    got = torch.atanh(v)
    extra = 2 * nc.ulp32(v) / (1 - v * v)
    check = lambda g, rf: nc.check_close(g, rf, r.vpre_scale, "fp32", extra=extra, what="value (atanh)")
    _report("value", case, check(got, r.vpre_ref))
    nc.assert_rejects(check, got, r.vpre_ref, [nc.AddTerm(r.vpre_scale, 256, "fp32")])


@pytest.mark.parametrize("case", ALL, ids=_id, scope="module")
def test_policy_gemm_split_precision(cuda_lib, cuda_env, case):
    """The policy Dense on wgmma as one split-precision GEMM ([x_hi | x_lo | x_hi] . [w_hi | w_hi | w_lo]) against the
    float64 product with the UNSPLIT fp32 kernel: within BETA * S with no extra slack, i.e. fp32 accuracy."""
    r = _run(case, cuda_lib, cuda_env)
    ref, s = nc.policy_gemm_ref(r.pol_features(), r.w)
    got = r.logits[:, :nc.N_LABELS]
    check = lambda g, rf: nc.check_close(g, rf, s, "fp32", what="LOGITS")
    _report("policy_gemm", case, check(got, ref))
    nc.assert_rejects(check, got, ref, [nc.SwapLabels(), nc.ScaleLastTile(0.99), nc.AddTerm(s, r.pc * 90, "fp32")])


def _check_stats(stats, logits):
    """Epilogue row statistics per 256-label tile: max over the tile's valid labels (bit for bit the max of the logits it
    wrote) and sum exp(x - max) within 1e-5 relative; returns the worst relative error of the sums."""
    worst = 0.0
    for t in range(stats.shape[1]):
        cols = logits[:, 256 * t:min(nc.N_LABELS, 256 * (t + 1))]
        mx = cols.max(dim=1).values
        assert torch.equal(stats[:, t, 0], mx), f"tile {t}: max"
        ref = torch.exp(cols.double() - mx.double()[:, None]).sum(dim=1)
        worst = max(worst, nc.check_rel(stats[:, t, 1], ref, 1e-5, what=f"tile {t}: sum exp"))
    return worst


@pytest.mark.parametrize("case", ALL, ids=_id, scope="module")
def test_gemm_row_stats(cuda_lib, cuda_env, case):
    r = _run(case, cuda_lib, cuda_env)
    logits = r.logits[:, :nc.N_LABELS]
    _report("row_stats", case, _check_stats(r.stats, logits))

    def last_sum(g, _):
        g[:, -1, 1] *= 0.99
        return g

    def last_max(g, _):
        m = g[:, -1, 0].float()
        g[:, -1, 0] = torch.nextafter(m, torch.full_like(m, -np.inf)).double()
        return g
    check = lambda g, lg: _check_stats(g.float(), lg.float())
    nc.assert_rejects(check, r.stats, logits, [nc.Mutation("last tile's sum x 0.99", last_sum),
                                               nc.Mutation("last tile's max one ulp low", last_max)])


@pytest.mark.parametrize("case", ALL, ids=_id, scope="module")
def test_softmax(cuda_lib, cuda_env, case):
    """k_softmax (finishing the epilogue's statistics) against the float64 softmax of the GPU's logits."""
    r = _run(case, cuda_lib, cuda_env)
    ref = torch.softmax(r.logits[:, :nc.N_LABELS].double(), dim=1)
    assert (r.policy.double().sum(dim=1) - 1).abs().max().item() <= 1e-5
    check = lambda g, rf: nc.check_rel(g, rf, 1e-5, what="policy")
    _report("softmax", case, check(r.policy, ref))
    nc.assert_rejects(check, r.policy, ref, [nc.SwapLabels(), nc.ScaleLastTile(0.99)])


def test_read_buffer_error_paths(cuda_lib):
    """Refusals are return codes, checked on the host: nothing is read out of bounds."""
    from cczero_b200.engine import Engine
    fn = cuda_lib.raw("cz_nn_read_buffer")
    rb = C.c_int64(0)
    dst = torch.empty(1 << 20, dtype=torch.uint8, device="cuda")
    p = C.c_void_p(dst.data_ptr())
    eng = Engine(cuda_lib, "cuda", n_games=4, sims_per_move=8, leaves_per_round=1, nn_filters=64, nn_blocks=2, nn_fp32_skip=False)
    try:
        h = eng._h
        rows = {nc.LAST_CONV1: 90 * 64 * 2, nc.TOWER_OUT: 90 * 64 * 2, nc.POL_FEAT: 3 * 384 * 2, nc.LOGITS: 2304 * 4, nc.STATS: 9 * 8}
        for which, row in rows.items():
            assert fn(h, which, 4, None, 0, C.byref(rb)) == 0 and rb.value == row, which
        assert fn(h, nc.FIRST_OUT, 1, p, dst.numel(), C.byref(rb)) == -3          # overwritten by block 2: CZ_ERR_STATE
        assert fn(h, nc.FIRST_OUT32, 1, p, dst.numel(), C.byref(rb)) == -3
        assert fn(h, nc.TOWER_OUT32, 1, p, dst.numel(), C.byref(rb)) == -3        # no fp32 skip stream
        assert fn(h, 8, 1, p, dst.numel(), C.byref(rb)) == -1                     # unknown buffer: CZ_ERR_ARG
        assert fn(h, -1, 1, p, dst.numel(), C.byref(rb)) == -1
        assert fn(h, nc.LOGITS, 5, p, dst.numel(), C.byref(rb)) == -1             # more rows than the max batch
        assert fn(h, nc.LOGITS, 4, p, 4 * 2304 * 4 - 1, C.byref(rb)) == -1       # destination one byte short
        assert fn(h, nc.LOGITS, 4, p, 4 * 2304 * 4, C.byref(rb)) == 0
    finally:
        eng.close()
    eng = Engine(cuda_lib, "cuda", n_games=2, sims_per_move=8, leaves_per_round=1, nn_filters=64, nn_blocks=1, nn_fp32_skip=True)
    try:
        for which, row in ((nc.FIRST_OUT, 90 * 64 * 2), (nc.FIRST_OUT32, 90 * 64 * 4), (nc.TOWER_OUT32, 90 * 64 * 4)):
            assert eng.lib.raw("cz_nn_read_buffer")(eng._h, which, 2, None, 0, C.byref(rb)) == 0 and rb.value == row
    finally:
        eng.close()
