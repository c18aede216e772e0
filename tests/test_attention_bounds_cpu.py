"""The float64 attention reference and its error bounds (attn_bounds.py), checked without a GPU: the explicit
gradients equal autograd's, a CPU simulation of the kernel arithmetic stays inside the bounds, and the same
simulation with one injected defect does not."""
import math

import pytest
import torch

import attn_bounds as AB
from oracle import philox

bf16 = torch.bfloat16

# (name, n_seq, s_q, s_kv, mask, mask_block, total_rows, kv_count): one of every mask the ABI has
MASKS = [
    ("none", 2, 70, 70, AB.MASK_NONE, 0, 0, None),
    ("causal", 2, 70, 70, AB.MASK_CAUSAL, 0, 0, None),
    ("offset_causal", 2, 21, 86, AB.MASK_CAUSAL, 0, 0, None),
    ("block", 2, 40, 40, AB.MASK_BLOCK, 8, 0, None),
    ("kv_count", 2, 5, 90, AB.MASK_NONE, 0, 0, 67),
    ("ragged_total_rows", 3, 50, 50, AB.MASK_CAUSAL, 0, 121, None),
    ("ragged_block", 2, 48, 48, AB.MASK_BLOCK, 12, 84, None),
]


def _inputs(n, sq, skv, hd=32, H=2, seed=0, sigma=1.0):
    g = torch.Generator().manual_seed(seed)
    q, k, v, do = (_bf(torch.randn(n, H, s, hd, generator=g) * sigma) for s in (sq, skv, skv, sq))
    return q, k, v, do


def _bf(x):
    return x.to(bf16).double()


@pytest.mark.parametrize("name,n,sq,skv,mask,mb,total,cnt", MASKS, ids=[m[0] for m in MASKS])
def test_explicit_gradients_match_autograd(name, n, sq, skv, mask, mb, total, cnt):
    q, k, v, do = _inputs(n, sq, skv, seed=1)
    vis = AB.visible(n, sq, skv, mask, mb, total, cnt)
    scale = 32 ** -0.5
    ref = AB.reference(q, k, v, vis, scale, do)
    qa, ka, va = (t.clone().requires_grad_() for t in (q, k, v))
    s = (scale * qa @ ka.transpose(-1, -2)).masked_fill(~vis[:, None], -math.inf)
    rows = vis.any(-1)[:, None, :, None]
    o = torch.where(rows, torch.softmax(s, -1).nan_to_num(0.0), torch.zeros_like(s)) @ va
    o.backward(do)
    assert torch.allclose(ref["O"], o.detach(), rtol=1e-12, atol=1e-12)
    for name_, got, want in (("dQ", ref["dQ"], qa.grad), ("dK", ref["dK"], ka.grad), ("dV", ref["dV"], va.grad)):
        assert torch.allclose(got, want, rtol=1e-10, atol=1e-12), name_
    lse = torch.logsumexp(s, -1)
    assert torch.equal(torch.isinf(lse), torch.isinf(ref["lse"]))
    fin = torch.isfinite(lse)
    assert torch.allclose(ref["lse"][fin], lse[fin], rtol=1e-12, atol=1e-12)


def test_seqmap_rows():
    """map_rows follows the ymp_seqmap formula: dense, shared-query, and the TimeSformer per-frame map with its cls
    prefix row (shared per clip on input, one per frame on output)."""
    assert torch.equal(AB.map_rows(AB.dense(5), 3, 5), torch.arange(15).view(3, 5))
    assert torch.equal(AB.map_rows(dict(outer_stride=0, pos_stride=1), 2, 4), torch.arange(4).expand(2, 4))
    B, N, T = 2, 3, 2
    m_in = dict(seq_div=T, outer_stride=N * T, inner_stride=1, pos_stride=T, n_prefix=1, prefix_base=B * N * T,
                prefix_stride=1, prefix_per_seq=0)
    r = AB.map_rows(m_in, B * T, N + 1)
    assert r[:, 0].tolist() == [12, 12, 13, 13]
    assert r[1, 1:].tolist() == [1, 3, 5] and r[2, 1:].tolist() == [6, 8, 10]
    assert AB.map_rows(dict(m_in, prefix_per_seq=1), B * T, N + 1)[:, 0].tolist() == [12, 13, 14, 15]


def test_visible_masks():
    v = AB.visible(1, 3, 5, AB.MASK_CAUSAL)[0]        # bottom-right aligned: query i sits at key i + 2
    assert v.sum(-1).tolist() == [3, 4, 5]
    v = AB.visible(2, 6, 6, AB.MASK_BLOCK, 3, total_rows=10)
    assert v[0].sum(-1).tolist() == [3] * 6 and v[1].sum(-1).tolist() == [3, 3, 3, 1, 0, 0]
    v = AB.visible(2, 1, 9, AB.MASK_NONE, kv_count=4)
    assert v.sum(-1).flatten().tolist() == [4, 4]


def _sim_ratios(q, k, v, do, vis, scale, defect=None):
    ref = AB.reference(q, k, v, vis, scale, do)
    e_o, e_lse = AB.fwd_bounds(q, k, v, scale, ref)
    o, lse = AB.simulate_fwd(q, k, v, vis, scale, defect)
    rows = vis.any(-1)[:, None]
    return ref, AB.worst_ratio(o, ref["O"], e_o, rows[..., None]), AB.worst_ratio(lse, ref["lse"], e_lse, rows)


@pytest.mark.parametrize("name,n,sq,skv,mask,mb,total,cnt", MASKS, ids=[m[0] for m in MASKS])
@pytest.mark.parametrize("sigma", [0.5, 2.0])
def test_simulation_inside_bounds(name, n, sq, skv, mask, mb, total, cnt, sigma):
    """The kernel arithmetic, simulated on the CPU, stays inside the forward and backward bounds (isolated backward
    from the reference O and lse, and chained from the simulated forward)."""
    hd = 32
    q, k, v, do = _inputs(n, sq, skv, hd=hd, seed=2, sigma=sigma)
    scale = hd ** -0.5
    vis = AB.visible(n, sq, skv, mask, mb, total, cnt)
    ref, r_o, r_lse = _sim_ratios(q, k, v, do, vis, scale)
    assert r_o <= 1 and r_lse <= 1, (r_o, r_lse)
    rows = vis.any(-1)[:, None, :, None]
    keys = vis.any(-2)[:, None, :, None]
    lse_in = ref["lse"].float().masked_fill(~rows[..., 0], 0.0)
    for o_in, l_in, e in ((_bf(ref["O"]), lse_in, (None, None)),
                          (*AB.simulate_fwd(q, k, v, vis, scale), AB.fwd_bounds(q, k, v, scale, ref))):
        dq, dk, dv = AB.simulate_bwd(q, k, v, o_in, l_in, do, vis, scale)
        e_dq, e_dk, e_dv = AB.bwd_bounds(q, k, v, do, scale, ref, *e)
        assert AB.worst_ratio(dq, ref["dQ"], e_dq, rows) <= 1
        assert AB.worst_ratio(dk, ref["dK"], e_dk, keys) <= 1
        assert AB.worst_ratio(dv, ref["dV"], e_dv, keys) <= 1


@pytest.mark.parametrize("defect,mask,sq,skv", [
    ("causal_shift", AB.MASK_CAUSAL, 130, 130), ("causal_shift", AB.MASK_CAUSAL, 70, 200),
    ("drop_last_block", AB.MASK_NONE, 70, 130), ("drop_last_block", AB.MASK_NONE, 1, 257),
    ("lse_shift", AB.MASK_NONE, 64, 64), ("lse_shift", AB.MASK_CAUSAL, 130, 130)])
def test_simulated_defects_exceed_bounds(defect, mask, sq, skv):
    """One wrong key, a skipped key block or an lse off by log(2)/64 takes the simulation outside the bounds."""
    hd = 64
    q, k, v, do = _inputs(2, sq, skv, hd=hd, seed=3)
    vis = AB.visible(2, sq, skv, mask)
    _, r_o, r_lse = _sim_ratios(q, k, v, do, vis, hd ** -0.5, defect)
    assert max(r_o, r_lse) > 1, (r_o, r_lse)
    if defect == "lse_shift":
        assert r_lse > 1 and r_o <= 1


def test_geometric_values_expose_a_late_causal_leak():
    """With V growing geometrically along the keys, a causal boundary off by one key only for rows past 64 (the
    second query tile) is still outside the O bound: the leak probe of the GPU tests does not depend on early rows."""
    hd, S = 64, 200
    q, k, v, do = _inputs(1, S, S, hd=hd, seed=4)
    r = math.exp(min(0.2, 30.0 / S))
    v = _bf(v.abs().clamp(min=0.5) * r ** torch.arange(S, dtype=torch.float64)[:, None])
    vis = AB.visible(1, S, S, AB.MASK_CAUSAL)
    ref = AB.reference(q, k, v, vis, hd ** -0.5)
    e_o, _ = AB.fwd_bounds(q, k, v, hd ** -0.5, ref)
    leak = vis | (torch.arange(S)[None, :, None] >= 64) & torch.roll(vis, 1, dims=-1) & (torch.arange(S) > 0)
    o, _ = AB.simulate_fwd(q, k, v, leak, hd ** -0.5)
    o_ok, _ = AB.simulate_fwd(q, k, v, vis, hd ** -0.5)
    assert AB.worst_ratio(o_ok, ref["O"], e_o) <= 1
    late = (torch.arange(S) >= 64)[None, None, :, None]
    assert AB.worst_ratio(o, ref["O"], e_o, late) > 1


def _mult(n, H, sq, skv, p, seed):
    g = torch.Generator().manual_seed(seed)
    keep = torch.rand(n, H, sq, skv, generator=g) >= p
    return keep.double() * philox.scale(p)


@pytest.mark.parametrize("mask,sq,skv", [(AB.MASK_CAUSAL, 70, 70), (AB.MASK_NONE, 33, 97)])
@pytest.mark.parametrize("p", [0.1, 0.5])
def test_dropout_simulation_inside_bounds(mask, sq, skv, p):
    """Dropout on the probabilities (O = (P o M) V, lse of the undropped P): the simulated kernel arithmetic with a
    keep mask stays inside the forward and backward bounds taken with the same multiplier, isolated and chained."""
    hd, n, H = 32, 2, 2
    q, k, v, do = _inputs(n, sq, skv, hd=hd, seed=4)
    scale = hd ** -0.5
    vis = AB.visible(n, sq, skv, mask)
    m = _mult(n, H, sq, skv, p, 5)
    ref = AB.reference(q, k, v, vis, scale, do, mult=m)
    e_o, e_lse = AB.fwd_bounds(q, k, v, scale, ref)
    o, lse = AB.simulate_fwd(q, k, v, vis, scale, mult=m)
    assert AB.worst_ratio(o, ref["O"], e_o) <= 1 and AB.worst_ratio(lse, ref["lse"], e_lse) <= 1
    for o_in, l_in, e in ((_bf(ref["O"]), ref["lse"].float(), (None, None)), (o, lse, (e_o, e_lse))):
        dq, dk, dv = AB.simulate_bwd(q, k, v, o_in, l_in, do, vis, scale, mult=m)
        e_dq, e_dk, e_dv = AB.bwd_bounds(q, k, v, do, scale, ref, *e)
        for got, want, b in ((dq, ref["dQ"], e_dq), (dk, ref["dK"], e_dk), (dv, ref["dV"], e_dv)):
            assert AB.worst_ratio(got, want, b) <= 1


def test_dropout_wrong_mask_exceeds_bounds():
    """The forward with another draw of the same keep probability is far outside the bounds of the right mask."""
    hd, n, H, sq = 32, 2, 2, 70
    q, k, v, do = _inputs(n, sq, sq, hd=hd, seed=4)
    vis = AB.visible(n, sq, sq, AB.MASK_CAUSAL)
    ref = AB.reference(q, k, v, vis, hd ** -0.5, do, mult=_mult(n, H, sq, sq, 0.1, 5))
    e_o, _ = AB.fwd_bounds(q, k, v, hd ** -0.5, ref)
    o, _ = AB.simulate_fwd(q, k, v, vis, hd ** -0.5, mult=_mult(n, H, sq, sq, 0.1, 6))
    assert AB.worst_ratio(o, ref["O"], e_o) > 1
