"""The search's network forward at its fixed launch shapes, with the batch size on the device, against the same forward
at a host-known batch and against float64.

In the search, nn_forward_leaves sizes every launch (conv tiles, grids, k_heads blocking) for n_max = G * K rows (twice
that with eval_mirror) and the kernels read the actual leaf count from the device.  At G = 1001, K = 8 the residual convs
therefore run 256-pixel M tiles (two m64 blocks per consumer warpgroup) over the 1001 leaves, whose last tile holds 234
pixels; at G = 401, C = 128 it holds 250; a single active game puts one board in a 256-pixel launch, one partial tile
whose halo starts at row -10.  sims_per_move = 1 and no noise: the only leaves are the roots, and k_scan_block's
exclusive scan in game order puts game g (the g-th active game) in leaf row g, its mirror in row n_dev + g.

Each shape runs three forwards on one engine: nn_forward_boards on n_max distinct boards (every row of every buffer
written), then a search from roots A (plain launches, then the WHILE graph is captured), then a search from roots B
(evaluated inside the WHILE graph, ending with the body run of n_dev = 0 that stops the loop).  After it

* the leaf rows of FIRST_OUT, LAST_CONV1, TOWER_OUT (and the fp32 copies), POL_FEAT, LOGITS and STATS are bit-identical
  to a second engine's nn_forward_boards on the same boards (its own launch shapes, from its own batch), and within the
  float64 stage bounds of tests/nn_checks.py;
* every row from the leaves up to the launch shape's extent still holds the first forward's bits;
* each root's priors are the float64 softmax of the GPU's own logits over the legal moves (mirror-averaged), renormalised.
"""
import numpy as np
import pytest
import torch

from oracle import model as om
from oracle import senv as osenv
from tests import nn_checks as nc

pytestmark = pytest.mark.gpu

K = 8
PC, VC = 4, 2
SOFTMAX_REL = 1e-5                    # test_nn_stages_gpu.py::test_softmax: a GPU probability against the float64 softmax
U = 2.0 ** -24

# id, filters, fp32 skip stream, games, the one active game (None = all)
SHAPES = [("c256-f32skip-g1001", 256, True, 1001, None),
          ("c128-f16skip-g401", 128, False, 401, None),
          ("c256-f32skip-g1001-one-board", 256, True, 1001, 500)]

BUFFERS = {"first": nc.FIRST_OUT, "first32": nc.FIRST_OUT32, "conv1": nc.LAST_CONV1, "tower": nc.TOWER_OUT,
           "tower32": nc.TOWER_OUT32, "pol_feat": nc.POL_FEAT, "logits": nc.LOGITS, "stats": nc.STATS}
_STATES = {}


def _states(n):
    """n distinct positions (cached per count: both mirror forms of a shape use the same ones)."""
    if n not in _STATES:
        _STATES[n] = nc.distinct_states(n, seed=n)
    return _STATES[n]


def _read_all(eng, n, s32):
    return {k: nc.read_buffer(eng, b, n) for k, b in BUFFERS.items() if s32 or k not in ("first32", "tower32")}


def _engine(cuda_lib, w, c, s32, games, k, mirror=False):
    from cczero_b200.engine import Engine
    eng = Engine(cuda_lib, "cuda", n_games=games, sims_per_move=1, leaves_per_round=k, noise_eps=0.0, nn_filters=c, nn_blocks=1,
                 nn_value_fc=256, nn_fp32_skip=s32, nn_policy_channels=PC, nn_value_channels=VC, eval_mirror=mirror)
    eng.set_weights({name: torch.as_tensor(v) for name, v in w.items()})
    return eng


def _report(what, shape, mirror, value):
    print(f"\n[nn-device-batch] {what:<14} {shape}{'-mirror' if mirror else '':<8} {value:.3g}")


def _check_stages(b, planes, w, c, s32, sid, mirror):
    """The stage checks of test_nn_stages_gpu.py on rows read back from the search's forward: each within its float64
    bound on the GPU's own input, and each bound rejecting a subtly wrong kernel (with 256-pixel tiles: the two row
    placements that tile can get wrong)."""
    n = planes.shape[0]
    fo = om.folded_operands(w, 14)
    act = lambda k: b[k].view(torch.float32 if k.endswith("32") else torch.float16).reshape(n, 90, c)
    first, conv1, tower = act("first"), act("conv1"), act("tower")
    tile_muts = nc.tile256_mutations() if n * 90 >= 256 else []

    ref, s = nc.first_conv_ref(planes, fo, "cuda")
    _report("first_conv", sid, mirror, nc.check_close(first, ref, s, "fp16", what="FIRST_OUT"))
    if s32:
        nc.check_close(act("first32"), ref, s, "fp32", what="FIRST_OUT32")
        assert torch.equal(first, act("first32").half())

    ref, s = nc.res_conv_ref(first, fo, 0)
    check = lambda g, rf: nc.check_close(g, rf, s, "fp16", what="LAST_CONV1")
    _report("conv1", sid, mirror, check(conv1, ref))
    nc.assert_rejects(check, conv1, ref, [nc.AddTerm(s, 9 * c), nc.ShiftBlock()] + tile_muts)

    skip = (act("first32") if s32 else first).double()
    ref, s = nc.res_conv_ref(conv1, fo, 1, skip)
    check = lambda g, rf: nc.check_close(g, rf, s, "fp16", what="TOWER_OUT")
    _report("conv2", sid, mirror, check(tower, ref))
    nc.assert_rejects(check, tower, ref, [nc.AddTerm(s, 9 * c), nc.ShiftBlock(), nc.DropResidual(skip)] + tile_muts)
    if s32:
        _report("conv2_32", sid, mirror, nc.check_close(act("tower32"), ref, s, "fp32", what="TOWER_OUT32"))
        assert torch.equal(tower, act("tower32").half())

    feat_ref, feat_scale, _, _ = nc.heads_ref(act("tower32") if s32 else tower, fo)
    hi, lo, _ = nc.split_pol_feat(b["pol_feat"].view(torch.float16), fo["pol_k1"])
    got = (hi.double() + lo.double())[:, :PC * 90]
    _report("pol_feat", sid, mirror, nc.check_close(got.reshape(n, PC, 90).permute(0, 2, 1), feat_ref, feat_scale, "hilo",
                                                     what="POL_FEAT"))
    ref, s = nc.policy_gemm_ref(got, w)
    logits = b["logits"].view(torch.float32)[:, :nc.N_LABELS]
    _report("policy_gemm", sid, mirror, nc.check_close(logits, ref, s, "fp32", what="LOGITS"))


def _root_priors(eng, games, logits, mirror, mirror_labels):
    """Per evaluated game: (GPU root priors, float64 reference, reference without the renormalisation, reference with the
    mirror row read at the unmirrored labels, legal move count)."""
    lookup = {m: i for i, m in enumerate(osenv.ActionLabelsRed)}
    n = len(games)
    p64 = torch.softmax(logits[:, :nc.N_LABELS].double(), dim=1).cpu()
    out = []
    for i, g in enumerate(games):
        r = eng.root(g)
        lab = torch.tensor([lookup[m] for m in r["moves"]])
        p = p64[i, lab]
        wrong = p
        if mirror:
            pm = p64[n + i]
            p, wrong = 0.5 * (p + pm[torch.from_numpy(mirror_labels[lab.numpy()].astype(np.int64))]), 0.5 * (p + pm[lab])
        out.append((torch.tensor(r["p"], dtype=torch.float64), p / p.sum(), p, wrong / wrong.sum(), len(lab)))
    return out


@pytest.mark.parametrize("mirror", [False, True], ids=["plain", "mirror"])
@pytest.mark.parametrize("shape", SHAPES, ids=[s[0] for s in SHAPES])
def test_search_forward_at_device_batch(cuda_lib, cuda_env, shape, mirror):
    sid, c, s32, G, one = shape
    f = 2 if mirror else 1
    n_rows = f * G * K                                      # the launch shape's extent
    leaves = 1 if one is not None else G
    rows = f * leaves                                       # rows the searches write
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert nc.conv_tile_m(n_rows, c, sms) == 256, "the search's convs must run 256-pixel tiles"
    assert (rows * 90) % 256 and (one is not None or rows * 90 > 256)  # a partial last tile behind full ones, or one board

    states = _states(n_rows + 2 * G)
    filler, roots_a, roots_b = states[:n_rows], states[n_rows:n_rows + G], states[n_rows + G:]
    games = [one] if one is not None else list(range(G))
    boards = cuda_env.boards_from_states([roots_b[g] for g in games])
    if mirror:
        boards = torch.cat([boards, cuda_env.mirror(boards)])
    planes = cuda_env.planes_batch(boards)
    w = nc.well_conditioned_weights(c, 1, planes.cpu().numpy(), seed=c + G, device="cuda", policy_filters=PC,
                                    value_filters=VC)

    eng = _engine(cuda_lib, w, c, s32, G, K, mirror)
    try:
        eng.nn_forward_boards(cuda_env.boards_from_states(filler))
        torch.cuda.synchronize()
        before = _read_all(eng, n_rows, s32)
        opts = (lambda: eng.make_opts(active=[1 if g == one else 0 for g in range(G)])) if one is not None else (lambda: None)
        for roots in (roots_a, roots_b):
            eng.reset(roots)
            eng.search(opts())
        torch.cuda.synchronize()
        after = _read_all(eng, n_rows, s32)
        assert int(eng.counters()[6]) == 0
        priors = _root_priors(eng, games, after["logits"][:rows].view(torch.float32), mirror, cuda_env.mirror_labels)
    finally:
        eng.close()

    ref_eng = _engine(cuda_lib, w, c, s32, rows, 1)
    try:
        ref_eng.nn_forward_boards(boards)
        torch.cuda.synchronize()
        alone = _read_all(ref_eng, rows, s32)
    finally:
        ref_eng.close()
    for k in after:
        assert torch.equal(after[k][:rows], alone[k]), f"{k}: the search's rows differ from the host-batch forward"
        assert torch.equal(after[k][rows:], before[k][rows:]), f"{k}: rows beyond the search's leaves were written"
    del before, alone

    _check_stages({k: v[:rows] for k, v in after.items()}, planes, w, c, s32, sid, mirror)

    worst, rejected = 0.0, 0
    for got, ref, unnorm, wrong, L in priors:
        tol = 2 * (SOFTMAX_REL + 2 * U) + (L + 1) * U       # both probabilities, the mirror average, the float32 sum, the division
        check = lambda g, r, tol=tol: nc.check_rel(g, r, tol, what="root priors")
        worst = max(worst, check(got, ref) / tol)
        muts = [nc.Mutation("priors not renormalised", lambda g, r, u=unnorm: u.clone())]
        if mirror:
            muts.append(nc.Mutation("mirror row read at the unmirrored labels", lambda g, r, x=wrong: x.clone()))
        live = [m for m in muts if not torch.equal(m(got, ref), got)]     # a single legal move is its own renormalisation
        rejected += len(nc.assert_rejects(check, got, ref, live))
    assert rejected >= len(priors)
    _report("root_priors/tol", sid, mirror, worst)
