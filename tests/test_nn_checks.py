"""Host-side checks of the float64 network oracle and of the helpers in tests/nn_checks.py (no GPU needed)."""
import numpy as np
import pytest
import torch

from oracle import model as om
from tests import nn_checks as nc


@pytest.fixture(scope="module")
def planes41():
    return nc.positions(41, 14, seed=3)[1]        # the positions test_nn_gpu.py evaluates


@pytest.mark.parametrize("filters,blocks,trained,spread", [
    (128, 7, False, 0), (128, 7, True, 0.3), (192, 10, True, 0.3), (256, 20, False, 0), (256, 3, True, 1.0),
    (192, 10, True, 1.0)])
def test_forward_stages_fp64_matches_fp32_forward(planes41, filters, blocks, trained, spread):
    """The float64 restatement agrees with the fp32 one (same operations, one definition) to fp32 rounding."""
    w = om.init_weights(filters, blocks, 256, seed=filters + blocks, trained_like=trained, spread=spread)
    p32, v32 = om.forward(w, planes41, blocks)
    st = om.forward_stages(w, planes41, blocks)
    assert st["logits"].dtype == torch.float64 and len(st["out"]) == len(st["conv1"]) == blocks
    assert np.abs(st["policy"].numpy() - p32).max() < 1e-5
    assert np.abs(st["value"].numpy() - v32).max() < 1e-5
    assert np.abs(st["log_policy"].numpy() - np.log(p32)).max() < 1e-4
    assert torch.equal(st["value"], torch.tanh(st["value_pre"]))
    assert torch.allclose(st["log_policy"].exp(), st["policy"], rtol=1e-12, atol=0)


@pytest.mark.parametrize("filters,blocks,in_planes,pc,vc", [(64, 1, 14, 4, 2), (128, 3, 28, 2, 4), (64, 2, 14, 32, 4)])
def test_well_conditioned_nets_reach_their_targets(filters, blocks, in_planes, pc, vc):
    _, planes, _ = nc.positions(41, in_planes, seed=5)
    w = nc.well_conditioned_weights(filters, blocks, planes, seed=1, in_planes=in_planes, policy_filters=pc, value_filters=vc)
    st = om.forward_stages(w, planes, blocks)
    assert abs(st["logits"].std(dim=1).mean().item() - 2.0) < 1e-3
    assert abs(st["value_pre"].abs().median().item() - 0.5) < 1e-3
    lp = st["log_policy"]
    assert (lp.max(dim=1).values - lp.min(dim=1).values).min().item() > np.log(1e4)     # several orders of magnitude
    assert st["value"].abs().max().item() < 0.999                                      # off tanh's flat tails


@pytest.fixture(scope="module")
def small_net():
    states, planes, _ = nc.positions(9, 14, seed=2)
    w = nc.well_conditioned_weights(64, 1, planes, seed=4)
    return w, planes, om.folded_operands(w), om.forward_stages(w, planes, 1)


def test_folded_operands_restate_the_network(small_net):
    """The operand replica computes the same network: fp16 folding moves a conv output by at most 2^-11 * S, the fp32
    heads by fp32 rounding only; layouts (tap order, [c_out][c_in], Flatten order, the [hi | hi | lo] split) are right."""
    w, planes, fo, st = small_net
    first, s = nc.first_conv_ref(planes, fo, "cpu")
    assert ((first - nc.to_pix(st["first"])).abs() <= 2.0 ** -11 * s + 1e-12).all()
    c1, s1 = nc.res_conv_ref(first, fo, 0)
    assert ((c1 - nc.to_pix(st["conv1"][0])).abs() <= 2.0 ** -10 * s1 + 1e-9).all()
    x = nc.to_pix(st["out"][-1])
    feat, sf, vpre, sv = nc.heads_ref(x, fo)
    pf = st["pol_feat"].reshape(len(planes), fo["pol_c"], 90).permute(0, 2, 1)
    assert ((feat - pf).abs() <= 2.0 ** -20 * sf).all()
    assert ((vpre - st["value_pre"]).abs() <= 2.0 ** -18 * sv).all()
    logits, sl = nc.policy_gemm_ref(st["pol_feat"], w)
    assert torch.allclose(logits, st["logits"], rtol=0, atol=1e-12)
    k1 = fo["pol_k1"]
    hi, hi2, lo = (fo["w_pol"][:, i * k1:(i + 1) * k1].astype(np.float64) for i in range(3))
    assert np.array_equal(hi, hi2) and fo["w_pol"].shape == (2304, 3 * k1)
    kern = om._array(w, "policy_out", "kernel").T.astype(np.float64)
    assert (np.abs(hi[:2086, :360] + lo[:2086, :360] - kern) <= 2.0 ** -22 * np.abs(kern) + 2.0 ** -25).all()
    assert not hi[2086:].any() and not hi[:, 360:].any() and not lo[:, 360:].any()


def test_every_mutation_is_rejected_on_the_reference_itself(small_net):
    """Each corruption in nn_checks.py, applied to the float64 reference, fails the check the GPU tests use."""
    w, planes, fo, st = small_net
    first, s0 = nc.first_conv_ref(planes, fo, "cpu")
    c1, s1 = nc.res_conv_ref(first, fo, 0)
    y, s2 = nc.res_conv_ref(c1, fo, 1, first)
    for ref, s, k, extra in ((first, s0, 25, []), (c1, s1, 9 * 64, []), (y, s2, 9 * 64, [nc.DropResidual(first)])):
        check = lambda g, r, s=s: nc.check_close(g, r, s, "fp16")
        assert check(ref, ref) == 0.0
        nc.assert_rejects(check, ref, ref, [nc.AddTerm(s, k), nc.ShiftBlock()] + extra)
    feat, sf, vpre, sv = nc.heads_ref(y, fo)
    check = lambda g, r: nc.check_close(g, r, sf, "hilo")
    nc.assert_rejects(check, feat, feat, [nc.AddTerm(sf, 64, "hilo"), nc.ShiftBlock()])
    check = lambda g, r: nc.check_close(g, r, sv, "fp32")
    nc.assert_rejects(check, vpre, vpre, [nc.AddTerm(sv, 256, "fp32")])
    logits, sl = nc.policy_gemm_ref(feat.permute(0, 2, 1).flatten(1), w)
    check = lambda g, r: nc.check_close(g, r, sl, "fp32")
    nc.assert_rejects(check, logits, logits, [nc.SwapLabels(), nc.ScaleLastTile(0.99), nc.AddTerm(sl, 360, "fp32")])
    p = torch.softmax(logits, dim=1)
    nc.assert_rejects(lambda g, r: nc.check_rel(g, r, 1e-5), p, p, [nc.SwapLabels(), nc.ScaleLastTile(0.99)])


def test_bound_arithmetic():
    assert nc.ulp16(torch.tensor([1.0, 1.5, 2.0, 0.0, 2.0 ** -20, 1000.0])).tolist() == \
        [2.0 ** -10, 2.0 ** -10, 2.0 ** -9, 2.0 ** -24, 2.0 ** -24, 0.5]
    assert nc.ulp32(torch.tensor([1.0, 3.0])).tolist() == [2.0 ** -23, 2.0 ** -22]
    # half an fp16 ulp on an output of 1 passes, a full one fails; S adds BETA * S
    one = torch.ones(1, dtype=torch.float64)
    nc.check_close(one + 2.0 ** -11, one, torch.zeros(1), "fp16")
    with pytest.raises(AssertionError):
        nc.check_close(one + 2.0 ** -10, one, torch.zeros(1), "fp16")
    nc.check_close(one + 2.0 ** -10, one, torch.full((1,), 2.0 ** 5), "fp16")
    nc.check_close(one + 2.0 ** -16, one, torch.ones(1), "fp32")
    with pytest.raises(AssertionError):
        nc.check_close(one + 2.0 ** -15, one, torch.ones(1), "fp32")


def test_read_buffer_is_unsupported_in_the_emulation_build(emul_lib):
    assert emul_lib.raw("cz_nn_read_buffer")(None, nc.LOGITS, 1, None, 0, None) == -5     # CZ_ERR_UNSUPPORTED


def test_conv_tile_restatement():
    """256-pixel M tiles from 1500 boards at C = 256 and from 3001 at C = 64 and 128 on 132 SMs; never at C = 192 or in
    the 64-column small-batch form."""
    for c, first in ((256, 1500), (128, 3001), (64, 3001)):
        assert nc.conv_tile_m(first - 1, c, 132) == 128 and nc.conv_tile_m(first, c, 132) == 256, c
    assert nc.conv_tile_m(20000, 192, 132) == 128
    assert nc.use_n_split(9, 256, 132) and nc.conv_tile_m(9, 256, 132) == 128
    assert not nc.use_n_split(20000, 64, 132)


def test_distinct_states_are_distinct_and_live():
    states = nc.distinct_states(500, seed=1)
    assert len(set(states)) == 500 and states[0] == nc.osenv.INIT_STATE
    assert not any(nc.osenv.done(s)[0] for s in states)
    assert states == nc.distinct_states(500, seed=1) and states != nc.distinct_states(500, seed=2)


def test_tile_row_swaps_are_rejected_on_the_reference_itself(small_net):
    """Both 256-pixel tile mutations move rows of a conv output far outside the bound (9 boards = 3 full tiles)."""
    w, planes, fo, st = small_net
    first, s0 = nc.first_conv_ref(planes, fo, "cpu")
    c1, s1 = nc.res_conv_ref(first, fo, 0)
    check = lambda g, r: nc.check_close(g, r, s1, "fp16")
    assert nc.assert_rejects(check, c1, c1, nc.tile256_mutations()) == [m.name for m in nc.tile256_mutations()]
    flat = c1.reshape(-1, c1.shape[-1])
    bad = nc.SwapTileRows(0, 64)(flat, flat)
    assert torch.equal(bad.reshape(c1.shape), nc.SwapTileRows(0, 64)(c1, c1))
    moved = (bad != flat).any(dim=1).nonzero().flatten().tolist()       # rows 0..127 of one tile, nothing else
    assert moved and moved[0] % 256 == 0 and set(moved) <= set(range(moved[0], moved[0] + 128))
