"""The keep-bit readouts of dropout_bits.py without a GPU: through the CPU simulation of the kernel arithmetic they
recover the oracle's mask exactly at every shape the GPU test runs (the readout values survive the bf16 roundings and
the 1 / n_i normaliser), a defective mask is reported at its first wrong (row, key), and the simulation stays inside
the dropout error bounds of attn_bounds.py at the shapes of the dropout cases in test_attention_bounds_gpu.py."""
import re

import pytest
import torch

import attn_bounds as AB
import dropout_bits as DB
from oracle import philox

SITE = 4 * 5 + 1


@pytest.mark.parametrize("c", DB.CASES, ids=[c["name"] for c in DB.CASES])
def test_simulated_readouts_recover_the_mask(c):
    keep, vis = DB.oracle_keep(c, SITE), DB.visible(c)
    for kind in DB.KINDS:
        DB.read_simulated(kind, c, keep).check(f"{c['name']} {kind}", keep, vis)


def _expect_first(kind, c, bad_keep):
    """The readout of a kernel drawing bad_keep fails at the first visible pair where bad_keep and the oracle differ."""
    keep, vis = DB.oracle_keep(c, SITE), DB.visible(c)
    diff = (bad_keep != keep) & vis[:, None]
    assert bool(diff.any()), "the defect changes no visible bit at this shape"
    first = tuple(int(i) for i in diff.nonzero()[0])
    with pytest.raises(AssertionError, match=re.escape(f"first at (seq, head, row, key) {first}:")):
        DB.read_simulated(kind, c, bad_keep).check(kind, keep, vis)


@pytest.mark.parametrize("kind", DB.KINDS)
def test_one_flipped_bit_is_reported(kind):
    """One keep bit flipped at a late visible pair (the last sequence and head, a key past 64 tiles of 64)."""
    c = dict(DB.case("flip", 64, 129, 129, mask=AB.MASK_CAUSAL), p=0.1)
    bad = DB.oracle_keep(c, SITE).clone()
    bad[1, 2, 128, 70] = ~bad[1, 2, 128, 70]
    _expect_first(kind, c, bad)


@pytest.mark.parametrize("kind", DB.KINDS)
@pytest.mark.parametrize("defect,sq,skv,mask", [
    ("s_kv_row", 63, 129, AB.MASK_NONE), ("s_kv_row", 129, 65, AB.MASK_NONE),
    ("head_seq_swap", 65, 65, AB.MASK_CAUSAL), ("words_1_2", 63, 63, AB.MASK_NONE),
    ("last_tile_shift", 15, 257, AB.MASK_NONE), ("last_tile_shift", 129, 129, AB.MASK_CAUSAL)])
def test_defective_masks_are_reported(kind, defect, sq, skv, mask):
    c = dict(DB.case(defect, 80, sq, skv, mask=mask), p=0.3)
    _expect_first(kind, c, DB.defect_keep(defect, c, SITE))


# the dropout cases of test_attention_bounds_gpu.py: (hd, s_q, s_kv, n, mask, mask_block, total_rows)
BOUND_SHAPES = [(64, 129, 129, 2, AB.MASK_CAUSAL, 0, 0), (96, 63, 129, 2, AB.MASK_NONE, 0, 0),
                (64, 1, 70, 2, AB.MASK_NONE, 0, 0), (64, 100, 100, 3, AB.MASK_CAUSAL, 0, 250),
                (80, 129, 129, 2, AB.MASK_CAUSAL, 0, 0), (128, 70, 200, 2, AB.MASK_NONE, 0, 0),
                (64, 80, 80, 3, AB.MASK_BLOCK, 20, 0), (128, 130, 130, 2, AB.MASK_CAUSAL, 0, 0),
                (96, 96, 96, 3, AB.MASK_BLOCK, 24, 0), (88, 80, 80, 3, AB.MASK_BLOCK, 8, 0),
                (80, 7, 1000, 2, AB.MASK_NONE, 0, 0), (96, 15, 257, 2, AB.MASK_NONE, 0, 0)]


@pytest.mark.parametrize("hd,sq,skv,n,mask,mb,total", BOUND_SHAPES)
@pytest.mark.parametrize("p", [0.1, 0.3])
def test_simulation_inside_dropout_bounds(hd, sq, skv, n, mask, mb, total, p):
    """With the oracle's Philox mask and scale, the simulated forward and backward (isolated and chained) stay inside
    the bounds that the GPU dropout cases use."""
    H = 2
    g = torch.Generator().manual_seed(hd + sq + skv)
    q, k, v, do = (torch.randn(n, H, s, hd, generator=g).to(torch.bfloat16).double() for s in (sq, skv, skv, sq))
    c = dict(DB.case("bounds", hd, sq, skv, n=n, H=H, mask=mask, mask_block=mb, total_rows=total), p=p)
    vis = DB.visible(c)
    m = DB.oracle_keep(c, SITE).double() * philox.scale(p)
    scale = hd ** -0.5
    ref = AB.reference(q, k, v, vis, scale, do, mult=m)
    rows, keys = vis.any(-1)[:, None], vis.any(-2)[:, None]
    e_o, e_lse = AB.fwd_bounds(q, k, v, scale, ref)
    o, lse = AB.simulate_fwd(q, k, v, vis, scale, mult=m)
    assert AB.worst_ratio(o, ref["O"], e_o, rows[..., None]) <= 1
    assert AB.worst_ratio(lse, ref["lse"], e_lse, rows) <= 1
    lse_ref = ref["lse"].float().masked_fill(~rows, 0.0)
    for o_in, l_in, e in ((ref["O"].to(torch.bfloat16).double(), lse_ref, (None, None)), (o, lse, (e_o, e_lse))):
        dq, dk, dv = AB.simulate_bwd(q, k, v, o_in, l_in, do, vis, scale, mult=m)
        e_dq, e_dk, e_dv = AB.bwd_bounds(q, k, v, do, scale, ref, *e)
        assert AB.worst_ratio(dq, ref["dQ"], e_dq, rows[..., None]) <= 1
        assert AB.worst_ratio(dk, ref["dK"], e_dk, keys[..., None]) <= 1
        assert AB.worst_ratio(dv, ref["dV"], e_dv, keys[..., None]) <= 1


# ---------------------------------------------------------------------------------- the oracle's threshold and scale
# p -> (fl32(p) as mantissa * 2^e, floor(fl32(p) * 2^32), 1.0f / (1.0f - fl32(p)) as an fp32 hex literal)
FP32_DROP = [(0.1, 13421773 * 2.0 ** -27, 13421773 << 5, "0x1.1c71c8p+0"),
             (0.15, 5033165 * 2.0 ** -25, 5033165 << 7, "0x1.2d2d2cp+0"),
             (0.3, 5033165 * 2.0 ** -24, 5033165 << 8, "0x1.6db6dcp+0"),
             (0.5, 0.5, 1 << 31, "0x1p+1"),
             (1e-7, 14073749 * 2.0 ** -47, 429, "0x1.000002p+0"),         # 14073749 / 2^15 = 429.497...
             (0.999, 16760439 * 2.0 ** -24, 16760439 << 8, "0x1.f401a6p+9")]


@pytest.mark.parametrize("p,p32,thresh,scale", FP32_DROP)
def test_threshold_and_scale_follow_the_fp32_p(p, p32, thresh, scale):
    """The kernels receive p as an fp32 (drop_state, philox.cuh): the threshold is floor(fl32(p) * 2^32) and the
    scale 1.0f / (1.0f - fl32(p)) in fp32, not the double p's."""
    assert float(torch.tensor(p, dtype=torch.float32)) == p32
    assert philox.threshold(p) == thresh
    assert philox.scale(p) == float.fromhex(scale)


def test_threshold_saturates():
    assert philox.threshold(1.0) == 0xFFFFFFFF and philox.threshold(0.0) == 0
    assert philox.threshold(1.0 - 2.0 ** -25) == 0xFFFFFFFF        # fl32 rounds it to 1


def test_scale_differs_from_rounding_the_double_quotient():
    """At p = 0.15, fl32(1 / (1 - fl32(p))) is one ulp above the kernels' fp32 quotient."""
    p32 = float(torch.tensor(0.15, dtype=torch.float32))
    f32 = float(torch.tensor(1.0 / (1.0 - p32), dtype=torch.float32))
    assert f32 - philox.scale(0.15) == 2.0 ** -23


def test_witness_of_the_double_threshold():
    """Seed 0x1234567812345, offset 7, site 9, row 6350, column 9906: the Philox word 429496732 lies between the
    double p's threshold (kept) and the fp32 p's (dropped); the kernels drop it."""
    w = philox.words(0x1234567812345, 7, 9, [6350], 9912)
    assert int(w[0, 9906]) == 429496732
    assert int(0.1 * 2.0 ** 32) <= 429496732 < philox.threshold(0.1)
    keep = philox.keep_mask(0x1234567812345, 7, 9, [6350], 9912, 0.1)
    assert not keep[0, 9906] and keep[0, :9906].mean() > 0.85
