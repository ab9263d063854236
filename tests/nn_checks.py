"""Shared checks of the network kernels against float64 references (used by test_nn_stages_gpu.py, test_nn_gpu.py and
test_igemm_gpu.py; the pure-host parts are exercised on the CPU by test_nn_checks.py).

One definition of "within rounding" for every kernel output g against its float64 reference r:

    |g - r| <= ALPHA * ulp_out(max(|r|, |g|)) + BETA * S

  ulp_out  the spacing of the output format at that magnitude: the fp16 ulp (floored at 2^-24, the subnormal spacing) for
           fp16 outputs, 0 for fp32 outputs, the fp16 ulp of the lo half for hi+lo split pairs.
  S        the same float64 reference evaluated on absolute values (|inputs|, |weights|, |bias|, |residual|): the magnitude
           of the terms that were summed, which is what sets an output's accumulation error.
  ALPHA    1/2: one final round-to-nearest into the output format.
  BETA     2^-16: fp32 accumulation of up to 2304 (9 taps x 256 channels) fp16 x fp16 products, each exact in fp32.  A
           round-to-nearest accumulator errs by about 2^-24 * S in practice; even a truncating one stays near
           sqrt(K) * 2^-24 * S (K = 2304: about 2^-18.4 * S), ~5x under BETA.  One dropped or duplicated average term is
           S / K, about 4e-4 * S = 2^-11.2 * S, ~30x above BETA: that is the kind of bug the bound is there to catch.
  A folded BN shift beta - mean * scale enters S as |beta| + |mean * scale|: nvcc may contract it into an FMA, which
  moves it by half an fp32 ulp of mean * scale, more than an ulp of the shift where the two cancel.

The mutations below corrupt a kernel output slightly, the way a wrong kernel would, and `assert_rejects` proves that a
check fails on each of them: a bound that passes everything proves nothing.
"""
import ctypes as C

import numpy as np
import torch

from oracle import model as om
from oracle import senv as osenv

ALPHA = 0.5
BETA = 2.0 ** -16
N_LABELS = om.N_LABELS
LAST_TILE = slice(2048, N_LABELS)            # the partial 9th N tile of the policy GEMM (256-column tiles)

# cz_nn_buffer (include/cczero_b200.h)
FIRST_OUT, FIRST_OUT32, LAST_CONV1, TOWER_OUT, TOWER_OUT32, POL_FEAT, LOGITS, STATS = range(8)
KPOLN = 2304                                  # logits row: 2086 labels padded to 9 tiles of 256


def use_n_split(n, c, sms):
    """cz_nn.cu use_n_split: the residual convs run as 64-column tiles when the M tiles x C / 64 fit one wave of CTAs."""
    return c > 64 and (n * 90 + 127) // 128 * (c // 64) <= sms


def conv_tile_n(c, split=False):
    """cz_nn.cu conv_tile_n: the conv's N tile."""
    return 64 if split else 128 if c == 256 else c


def conv_tile_m(n, c, sms):
    """cz_nn.cu conv_tile_m of the full-width conv (and of the trainer's convs, which never split): 256-pixel M tiles once
    they fill 8 waves of CTAs, else 128; C = 192 and the 64-column small-batch form stay at 128."""
    if use_n_split(n, c, sms) or c == 192:
        return 128
    return 256 if (n * 90 + 255) // 256 * (c // conv_tile_n(c)) >= 8 * sms else 128


def _f64(x):
    if isinstance(x, np.ndarray):
        x = torch.from_numpy(x)
    return x.to(torch.float64)


def ulp16(x):
    """Spacing of fp16 numbers at |x| (2^-24 below the normal range)."""
    x = _f64(x).abs().clamp(min=2.0 ** -14, max=65504.0)
    _, e = torch.frexp(x)                     # x = m * 2^e, m in [0.5, 1)
    return torch.ldexp(torch.ones_like(x), (e - 11).to(torch.int32))


def ulp32(x):
    x = _f64(x).abs().clamp(min=2.0 ** -126)
    _, e = torch.frexp(x)
    return torch.ldexp(torch.ones_like(x), (e - 24).to(torch.int32))


def bound(got, ref, scale, out="fp16", extra=0.0):
    """ALPHA * ulp_out(max(|r|, |g|)) + BETA * S (+ extra)."""
    got, ref, scale = _f64(got), _f64(ref), _f64(scale)
    mag = torch.maximum(got.abs(), ref.abs())
    if out == "fp16":
        u = ulp16(mag)
    elif out == "hilo":                       # hi + lo fp16 pair: lo = RN16(f - hi), |f - hi| <= ulp16(f) / 2
        u = ulp16(mag * 2.0 ** -11)
    elif out == "fp32":
        u = torch.zeros_like(mag)
    else:
        raise ValueError(out)
    return ALPHA * u + BETA * scale + extra


def check_close(got, ref, scale, out="fp16", extra=0.0, what=""):
    """Asserts |g - r| <= bound elementwise; returns the worst err / bound (a number well under 1 is the healthy case)."""
    got, ref = _f64(got), _f64(ref)
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    assert torch.isfinite(got).all(), f"{what}: non-finite output"
    b = bound(got, ref, scale, out, extra)
    ratio = (got - ref).abs() / b
    worst = ratio.max().item()
    if not worst <= 1.0:
        i = np.unravel_index(int(ratio.argmax()), tuple(ratio.shape))
        raise AssertionError(f"{what}: |g - r| / bound = {worst:.3g} at {i}: g = {got[i].item():.9g}, r = {ref[i].item():.9g}, "
                             f"bound = {b[i].item():.3g}; {int((ratio > 1).sum())} of {ratio.numel()} elements out")
    return worst


def check_rel(got, ref, tol, what=""):
    """Asserts |g - r| <= tol * |r| elementwise; returns the worst relative error."""
    got, ref = _f64(got), _f64(ref)
    assert got.shape == ref.shape and torch.isfinite(got).all(), what
    rel = ((got - ref).abs() / ref.abs()).max().item()
    assert rel <= tol, f"{what}: relative error {rel:.3g} > {tol:g}"
    return rel


def rel_frobenius(got, ref):
    got, ref = _f64(got), _f64(ref)
    return (torch.linalg.vector_norm(got - ref) / torch.linalg.vector_norm(ref)).item()


# ---------------------------------------------------------------------------------------------- mutations of an output
# Each is called as m(got, ref) on float64 tensors and returns a corrupted copy of `got`.  Conv-like outputs are
# [n][pixels][channels], label outputs [n][labels].

class SwapLabels:
    """Two labels of position 0 trade places (a label-order bug): the ones at the 25th and 75th percentile of the reference."""
    name = "swap two labels"

    def __call__(self, got, ref):
        order = torch.argsort(ref[0, :N_LABELS])
        i, j = order[N_LABELS // 4].item(), order[3 * N_LABELS // 4].item()
        assert ref[0, i] != ref[0, j]
        g = got.clone()
        g[0, i], g[0, j] = got[0, j], got[0, i]
        return g


class ScaleLastTile:
    """The partial last N tile (labels 2048..2085) scaled by `f` (a wrong bound on the last tile's columns)."""
    name = "scale the last partial N tile by 0.99"

    def __init__(self, f=0.99):
        self.f = f

    def __call__(self, got, ref):
        g = got.clone()
        g[:, LAST_TILE] *= self.f
        return g


class AddTerm:
    """One extra average-sized term S / k in one output (a dropped or duplicated tap / channel / k-block); the element is
    the one where such a term is easiest to see, which is where a real kernel bug would be seen first."""
    name = "add one weight term"

    def __init__(self, scale, k, out="fp16"):
        self.scale, self.k, self.out = _f64(scale), k, out

    def __call__(self, got, ref):
        term = self.scale.to(got.device) / self.k
        i = int((term / bound(got, ref, self.scale.to(got.device), self.out)).argmax())
        g = got.clone().reshape(-1)
        g[i] += term.reshape(-1)[i]
        return g.reshape(got.shape)


class ShiftBlock:
    """One `width`-channel block of position 0 read one pixel off (a wrong im2col / TMA coordinate)."""
    name = "shift one 64-channel block by one pixel"

    def __init__(self, width=64):
        self.width = width

    def __call__(self, got, ref):
        w = min(self.width, got.shape[2])
        best, g_best = -1.0, None
        for c0 in range(0, got.shape[2], w):
            g = got.clone()
            g[0, :, c0:c0 + w] = torch.roll(got[0, :, c0:c0 + w], 1, dims=0)
            d = (g - got).abs().max().item()
            if d > best:
                best, g_best = d, g
        return g_best


class DropResidual:
    """The skip connection missing from one output channel (the one with the largest skip): out = relu(out - skip).  Exact
    for a ReLU output with a non-negative skip: where the output is 0 so is the output without the skip."""
    name = "drop the residual from one channel"

    def __init__(self, skip):
        self.skip = _f64(skip)

    def __call__(self, got, ref):
        skip = self.skip.to(got.device)
        ch = int(skip.amax(dim=(0, 1)).argmax())
        g = got.clone()
        g[..., ch] = (got[..., ch] - skip[..., ch]).clamp(min=0)
        return g


class Mutation:
    """Any other corruption: fn(got, ref) -> corrupted copy."""

    def __init__(self, name, fn):
        self.name, self.fn = name, fn

    def __call__(self, got, ref):
        return self.fn(got.clone(), ref)


class SwapTileRows:
    """Inside one 256-pixel M tile, pixel rows [a, a + 64) and [b, b + 64) trade places: a = 0, b = 64 is a consumer
    warpgroup storing its two m64 blocks in swapped order; a = 64, b = 128 is a store row of cw * 64 instead of
    cw * MB * 64.  The tile is the full one whose two blocks differ most in the reference.  Outputs with one pixel per row
    and channels last: [n][90][C] or [n * 90][C]."""

    def __init__(self, a, b):
        self.a, self.b = a, b
        self.name = f"swap pixel rows {a}..{a + 63} and {b}..{b + 63} of a 256-pixel tile"

    def __call__(self, got, ref):
        c = got.shape[-1]
        rows = got.reshape(-1, c)
        tiles = rows.shape[0] // 256
        assert tiles >= 1, "no full 256-pixel tile"
        r = ref.reshape(-1, c)[:tiles * 256].reshape(tiles, 256, c)
        d = (r[:, self.a:self.a + 64] - r[:, self.b:self.b + 64]).abs().amax(dim=(1, 2))
        a, b = 256 * int(d.argmax()) + self.a, 256 * int(d.argmax()) + self.b
        g = rows.clone()
        g[a:a + 64], g[b:b + 64] = rows[b:b + 64], rows[a:a + 64]
        return g.reshape(got.shape)


def tile256_mutations():
    """The row placements a 256-pixel tile (two m64 blocks per consumer warpgroup) can get wrong."""
    return [SwapTileRows(0, 64), SwapTileRows(64, 128)]


def assert_rejects(check, got, ref, mutations):
    """`check(got, ref)` raises AssertionError on every mutated copy of `got`; returns the mutation names."""
    got, ref = _f64(got), _f64(ref)
    for m in mutations:
        bad = m(got, ref)
        assert not torch.equal(bad, got), m.name
        try:
            check(bad, ref)
        except AssertionError:
            continue
        raise AssertionError(f"check accepted a corrupted output: {m.name}")
    return [m.name for m in mutations]


# ---------------------------------------------------------------------------------------------- teacher-forced references
# Activations are [n][90][C] (pixel = row * 9 + column, the kernels' layout); the reference of a stage takes the GPU's own
# input to that stage and the operands the GPU folded (om.folded_operands), and returns (reference, S).

def to_nchw(x):
    n, _, c = x.shape
    return x.reshape(n, 10, 9, c).permute(0, 3, 1, 2)


def to_pix(x):
    n, c = x.shape[:2]
    return x.permute(0, 2, 3, 1).reshape(n, 90, c)


def conv_ref(x, w_oihw, shift, shift_abs, skip=None):
    """relu(conv(x, w) + shift (+ skip)) and its scale; x [n][in][10][9], w [out][in][k][k] ("same" padding); outputs [n][90][out]."""
    pad = w_oihw.shape[-1] // 2
    r = torch.nn.functional.conv2d(x, w_oihw, padding=pad) + shift.view(1, -1, 1, 1)
    s = torch.nn.functional.conv2d(x.abs(), w_oihw.abs(), padding=pad) + shift_abs.view(1, -1, 1, 1)
    r, s = to_pix(r), to_pix(s)
    if skip is not None:
        r, s = r + skip, s + skip.abs()
    return r.clamp(min=0), s


def first_conv_ref(planes, fo, device):
    w = torch.from_numpy(fo["w_first"].astype(np.float64)).permute(3, 2, 0, 1).to(device)        # HWIO -> OIHW
    t = lambda a: torch.from_numpy(a).to(device, torch.float64)
    return conv_ref(_f64(planes).to(device), w, t(fo["shift_first"]), t(fo["shift_first_abs"]))


def res_conv_ref(x, fo, layer, skip=None):
    """Residual conv `layer` (2 * block + j) on GPU activations x [n][90][C]."""
    w = torch.from_numpy(fo["w_conv"][layer].astype(np.float64)).to(x.device)          # [tap][co][ci]
    c = w.shape[1]
    w = w.reshape(3, 3, c, c).permute(2, 3, 0, 1)
    t = lambda a: torch.from_numpy(a).to(x.device, torch.float64)
    return conv_ref(to_nchw(_f64(x)), w, t(fo["shift_conv"][layer]), t(fo["shift_conv_abs"][layer]), skip)


def heads_ref(x, fo):
    """k_heads on tower output x [n][90][C]: (policy features [n][90][pol_c], their scale, value_pre [n], its scale)."""
    dev = x.device
    t = lambda a: torch.from_numpy(np.asarray(a, np.float64)).to(dev)
    x = _f64(x)
    wh, sh = t(fo["wh"]), t(fo["shifth"])
    pre, s = x @ wh.T + sh, x.abs() @ wh.abs().T + t(fo["shifth_abs"])
    feat = pre.clamp(min=0)
    pc = fo["pol_c"]
    vin = feat[..., pc:].permute(0, 2, 1).flatten(1)                  # Keras Flatten of channels_first: c * 90 + pix
    svin = s[..., pc:].permute(0, 2, 1).flatten(1)
    wv1, bv1, wv2, bv2 = t(fo["wv1"]), t(fo["bv1"]), t(fo["wv2"]), t(fo["bv2"])
    h, sh_ = (vin @ wv1 + bv1).clamp(min=0), svin @ wv1.abs() + bv1.abs()
    v, sv = (h @ wv2 + bv2)[:, 0], (sh_ @ wv2.abs() + bv2.abs())[:, 0]
    return feat[..., :pc], s[..., :pc], v, sv


def policy_gemm_ref(feat, w):
    """policy_out on features [n][pol_c * 90] (channel-major) with the UNSPLIT fp32 kernel: (logits [n][2086], scale)."""
    k = om._find(w, "policy_out", "kernel", torch.float64, feat.device)
    b = om._find(w, "policy_out", "bias", torch.float64, feat.device)
    feat = _f64(feat)
    return feat @ k + b, feat.abs() @ k.abs() + b.abs()


def split_pol_feat(pf, pol_k1):
    """POL_FEAT rows [hi | lo | hi] fp16 -> (hi, lo, hi again)."""
    return pf[:, :pol_k1], pf[:, pol_k1:2 * pol_k1], pf[:, 2 * pol_k1:3 * pol_k1]


# ---------------------------------------------------------------------------------------------- test nets and positions

def well_conditioned_weights(filters, blocks, planes, seed=0, logit_std=2.0, value_pre=0.5, device="cpu", value_fc=256, **kw):
    """om.init_weights(trained_like=True, spread=0.3) with policy_out rescaled so that the per-row standard deviation of the
    float64 logits on `planes` averages `logit_std`, and value_out rescaled so that the median |value_pre| is `value_pre`:
    probabilities spread over several orders of magnitude and values on the steep part of tanh, where a kernel error
    is visible instead of hidden under a near-uniform 2086-way softmax or tanh's flat tails."""
    w = om.init_weights(filters, blocks, value_fc, seed=seed, trained_like=True, spread=0.3, **kw)
    st = om.forward_stages(w, planes, blocks, device=device)
    a = logit_std / st["logits"].std(dim=1).mean().item()
    b = value_pre / st["value_pre"].abs().median().item()
    for name, f in (("policy_out/kernel", a), ("policy_out/bias", a), ("value_out/kernel", b), ("value_out/bias", b)):
        w[name] = (w[name].astype(np.float64) * f).astype(np.float32)
    return w


def positions(n, in_planes=14, seed=0):
    """n positions (the initial one first) as (states, planes [n][in_planes][10][9], history board per position or None).
    28 planes: random playouts of 0..40 plies, so histories both shorter than 5 entries (empty history planes) and longer."""
    from tests.search_checks import game_history, midgame_states
    if in_planes == 14:
        states = [osenv.INIT_STATE] + midgame_states(n - 1, seed, lo=1, hi=120)
        return states, np.stack([osenv.state_to_planes(s) for s in states]), [None] * n
    hists = [None] + [game_history(i % 41, seed * 1000 + i) for i in range(1, n)]
    states = [h[-1] if h else osenv.INIT_STATE for h in hists]
    planes = np.stack([osenv.state_history_to_planes(s, h) for s, h in zip(states, hists)])
    return states, planes, [h[-5] if h and len(h) >= 5 else None for h in hists]


def distinct_states(n, seed):
    """n distinct positions, the initial one first, that are not over: every ply of seeded random playouts of up to 120
    plies.  One oracle step per position (positions() replays a whole playout per position), so thousands take seconds."""
    rng = np.random.RandomState(seed)
    out, seen = [osenv.INIT_STATE], {osenv.INIT_STATE}
    while len(out) < n:
        s = osenv.INIT_STATE
        for _ in range(120):
            lm = osenv.get_legal_moves(s)
            s = osenv.step(s, lm[rng.randint(len(lm))])
            if osenv.done(s)[0]:
                break
            if s not in seen:
                seen.add(s)
                out.append(s)
                if len(out) == n:
                    break
    return out[:n]


def boards(cuda_env, states, history, in_planes):
    """Packed boards for cz_nn_forward_boards: [n][96], or [n][192] = (board, history board) pairs with 28 planes."""
    b = cuda_env.boards_from_states(states)
    if in_planes == 14:
        return b
    pairs = torch.zeros((len(states), 2, 96), dtype=torch.uint8, device=b.device)
    pairs[:, 0] = b
    for i, h in enumerate(history):
        if h is not None:
            pairs[i, 1] = cuda_env.boards_from_states([h])[0]
    return pairs.reshape(len(states), 192)


# ---------------------------------------------------------------------------------------------- the buffer accessor

def read_buffer(eng, which, n):
    """cz_nn_read_buffer: the first n rows of an intermediate buffer of the engine's last forward, as raw bytes [n][row]."""
    rb = C.c_int64(0)
    eng.lib.call("cz_nn_read_buffer", eng._h, which, n, None, 0, C.byref(rb))
    out = torch.empty((n, rb.value), dtype=torch.uint8, device=eng.device)
    eng.lib.call("cz_nn_read_buffer", eng._h, which, n, C.c_void_p(out.data_ptr()), out.numel(), C.byref(rb))
    return out


def read_act(eng, which, n, c):
    """FIRST_OUT / LAST_CONV1 / TOWER_OUT (fp16) or their fp32 copies as [n][90][C]."""
    dt = torch.float32 if which in (FIRST_OUT32, TOWER_OUT32) else torch.float16
    return read_buffer(eng, which, n).view(dt).reshape(n, 90, c)
