"""Float64 attention reference and per-element error bounds for the fused attention kernels.

Used by test_attention_bounds_gpu.py (kernel vs reference) and test_attention_bounds_cpu.py (the reference against
autograd, the bounds against a CPU simulation of the kernel arithmetic).  Pure torch: runs on any device.

Notation (one sequence, one head; i a query row, j a key, d a head-dim column; all inputs are the bf16 values the
kernels read, held exactly in float64):
    S_ij = scale * q_i . k_j,   P = softmax_j(S) over the visible keys,   O = P V,   lse_i = log sum_j exp(S_ij)
    dP = dO V^T,   delta_i = sum_d dO_id O_id,   dS = P o (dP - delta),   dQ = scale dS K,   dK = scale dS^T Q,
    dV = P^T dO
u = 2^-8 is the bf16 unit roundoff.  An fp32 sum of n terms is off by at most n * 2^-23 times the sum of their
magnitudes (2^-23 rather than 2^-24 so that truncating tensor-core accumulation is covered too).  Every bound is
multiplied by one safety factor C.

Forward.  The kernels accumulate q.k in fp32, so the scaled score is off by
    ds_ij = hd * 2^-23 * scale * sum_d |q_id| |k_jd|,
and exp(S + ds) = exp(S)(1 + ds): each P_ij is off by a relative ds_ij <= ds_i = max_j ds_ij, in the numerator and in
the normaliser, so O moves by at most 2 ds_i (P|V|) with (P|V|)_id = sum_j P_ij |V_jd| (>= |O_id|).  P is rounded to
bf16 before P V while the normaliser l sums the fp32 P: another u (P|V|).  The fp32 accumulations of P V and of l
over n <= 2^13 keys, and the rounding of the exponent argument (|arg| 2^-24 relative, |arg| < 128 where P does not
underflow), stay below a second u (P|V|).  exp2f / ex2.approx and the fp32 rescaling products are within 2^-20.  O
is finally rounded to bf16: u |O|.  2^-24 absolute covers underflow to zero.
    |O - O_ref| <= C [(2u + 2 ds_i + 2^-20) (P|V|) + u |O_ref|] + 2^-24
lse = m scale + log l with m the largest raw score.  l carries the relative error of the P_ij (ds_i plus the
exponent evaluation) and of its own fp32 summation over the n_i visible keys (n_i 2^-24; this term is missing from
a bound written as 2^-20 |lse| alone, and dominates it for long key ranges).  m scale and log l are each rounded
once; they can cancel, so their rounding is bounded by 2^-20 (1 + |lse| + max_j |S_ij|) rather than by |lse|:
    |lse - lse_ref| <= C [ds_i + (n_i + 4) 2^-24 + 2^-20 (1 + |lse_ref| + max_j |S_ij|)]

Backward (the kernels recompute P = exp(S - lse) in fp32 from the given lse).
    eP_ij   = ds_ij + 2^-20 (1 + |lse_i| + |S_ij|) + E_lse,i          relative error of the fp32 P
              (E_lse: the bound on the lse the backward was given; 0 when it is the reference's)
    dV      = P^T dO with P rounded to bf16 and fp32 accumulation (the second u, as in the forward), dV rounded to bf16:
              E_dV = C [((2u + eP) o P)^T |dO| + u |dV_ref|] + 2^-24
    dP      accumulated in fp32 over hd:  E_dP = hd 2^-23 (|dO| |V|^T)
    delta   is rowsum(dO o O) over the bf16 O the kernel is given (the tensor-core kernels) or rowsum(P o dP) (the
            warp-per-sequence kernel); the bound is the sum of both derivations:
              E_delta = (u + hd 2^-23) (|dO| . |O_ref|) + |dO| . E_O + sum_j P (eP |dP| + E_dP) + n_i 2^-24 sum_j P |dP|
              (E_O: the bound on the O the backward was given; 0 when it is the bf16-rounded reference)
    dS      = P o (dP - delta) from the fp32 P (u if a kernel used the bf16 P), rounded to bf16 for the dQ / dK products:
              E_dS = P o [(u + eP) |dP - delta| + E_dP + E_delta] + u |dS_ref|
    dQ      = scale dS K, fp32 accumulation over the keys (u, as above), rounded to bf16:
              E_dQ = C [scale (E_dS |K| + u |dS| |K|) + u |dQ_ref|] + 2^-24
    dK      = the same with dS^T and |Q|.

Dropout on the probabilities (mult M = keep / (1 - p), exact in float64; lse stays that of the undropped P):
O = (P o M) V, dP = M o (dO V^T), dV = (P o M)^T dO, and delta = rowsum(dO o O) = sum_j P_ij dP_ij still.  The kernels
scale each kept P_ij by one fp32 product (one more u32, inside the 2^-20 term), so every bound above holds with P o M
in place of P in (P|V|) and in E_dV, and E_dP multiplied by M.
"""
import math

import torch

U = 2.0 ** -8          # bf16 unit roundoff
G32 = 2.0 ** -23       # fp32 accumulation, per term
EXP = 2.0 ** -20       # exponent / logarithm evaluation
TINY = 2.0 ** -24      # absolute floor (underflow)
C = 2.0                # the one safety factor of the whole suite

MASK_NONE, MASK_CAUSAL, MASK_BLOCK = 0, 1, 2


# ---------------------------------------------------------------------------------- seqmaps
def map_rows(m, n_seq, S):
    """Row index of position i of sequence s under a seqmap (ymp.h: ymp_seqmap), as an int64 [n_seq, S] tensor.
    `m` is a dict with the ymp_seqmap fields (missing ones are 0; seq_div defaults to 1)."""
    g = lambda k, d=0: int(m.get(k, d))
    div = max(1, g("seq_div", 1))
    s = torch.arange(n_seq, dtype=torch.int64)[:, None]
    i = torch.arange(S, dtype=torch.int64)[None, :]
    outer, inner = s // div, s % div
    npre = g("n_prefix")
    reg = outer * g("outer_stride") + inner * g("inner_stride") + (i - npre) * g("pos_stride", 1)
    pre = g("prefix_base") + (s if g("prefix_per_seq") else outer) * g("prefix_stride") + i
    return torch.where(i < npre, pre, reg)


def dense(S):
    return dict(seq_div=1, outer_stride=S, pos_stride=1)


# ---------------------------------------------------------------------------------- masks
def lengths(n_seq, s_q, s_kv, total_rows=0, kv_count=None):
    """Per-sequence number of existing query rows and keys: total_rows cuts the last sequences short (dense packed
    sequences, s_q == s_kv), kv_count (the device-side key count) bounds every key range."""
    sq = torch.full((n_seq,), s_q, dtype=torch.int64)
    skv = torch.full((n_seq,), s_kv if kv_count is None else min(s_kv, kv_count), dtype=torch.int64)
    if total_rows:
        left = total_rows - torch.arange(n_seq, dtype=torch.int64) * s_q
        sq = torch.minimum(sq, left)
        skv = torch.minimum(skv, left)
    return sq, skv


def visible(n_seq, s_q, s_kv, mask, mask_block=0, total_rows=0, kv_count=None):
    """[n_seq, s_q, s_kv] bool: query i of sequence s sees key j.  Causal with s_q < s_kv is bottom-right aligned
    (query i at key position i + s_kv - s_q); rows that do not exist see nothing."""
    sq, skv = lengths(n_seq, s_q, s_kv, total_rows, kv_count)
    i = torch.arange(s_q)[None, :, None]
    j = torch.arange(s_kv)[None, None, :]
    vis = (i < sq[:, None, None]) & (j < skv[:, None, None])
    if mask == MASK_CAUSAL:
        vis = vis & (j <= i + (s_kv - s_q))
    elif mask == MASK_BLOCK:
        vis = vis & (i // mask_block == j // mask_block)
    return vis


# ---------------------------------------------------------------------------------- reference
def reference(q, k, v, vis, scale, dout=None, mult=None):
    """Explicit-formula float64 attention.  q [n,H,sq,hd], k/v [n,H,skv,hd], vis [n,sq,skv] bool, dout like q, mult
    [n,H,sq,skv] the dropout multiplier keep / (1 - p) or None.
    Returns a dict with O, lse, P, S (scaled scores, 0 where masked) and, with dout, dP, delta, dS, dQ, dK, dV.
    Rows that see no key get O = 0, lse = -inf, P = 0."""
    q, k, v = q.double(), k.double(), v.double()
    vm = vis[:, None].to(q.device)
    S = scale * (q @ k.transpose(-1, -2))
    Sm = S.masked_fill(~vm, -math.inf)
    lse = torch.logsumexp(Sm, -1)
    P = torch.exp(Sm - lse[..., None]).nan_to_num(0.0)
    Pm = P if mult is None else P * mult.double()
    r = dict(S=S.masked_fill(~vm, 0.0), P=P, Pm=Pm, mult=mult, O=Pm @ v, lse=lse, vis=vm)
    if dout is not None:
        do = dout.double()
        dP = do @ v.transpose(-1, -2)
        if mult is not None:
            dP = dP * mult.double()
        delta = (do * r["O"]).sum(-1)
        dS = P * (dP - delta[..., None])
        r.update(dP=dP, delta=delta, dS=dS, dQ=scale * dS @ k, dK=scale * dS.transpose(-1, -2) @ q,
                 dV=Pm.transpose(-1, -2) @ do)
    return r


def _score_err(q, k, scale, vm):
    hd = q.shape[-1]
    return (hd * G32 * scale) * (q.double().abs() @ k.double().abs().transpose(-1, -2)) * vm


def fwd_bounds(q, k, v, scale, ref):
    """Per-element bounds on |O - O_ref| and |lse - lse_ref| (module docstring)."""
    vm = ref["vis"]
    ds = _score_err(q, k, scale, vm)
    ds_i = ds.amax(-1)
    pv = ref.get("Pm", ref["P"]) @ v.double().abs()
    e_o = C * ((2 * U + 2 * ds_i[..., None] + EXP) * pv + U * ref["O"].abs()) + TINY
    n_i = vm.sum(-1).double()
    s_max = ref["S"].abs().amax(-1)
    e_lse = C * (ds_i + (n_i + 4) * 2.0 ** -24 + EXP * (1 + ref["lse"].abs() + s_max))
    return e_o, e_lse


def bwd_bounds(q, k, v, dout, scale, ref, e_o=None, e_lse=None):
    """Per-element bounds on |dQ - dQ_ref|, |dK - dK_ref|, |dV - dV_ref| (module docstring).  e_o / e_lse: bounds on
    the O and lse the backward was given (None: the reference's, O rounded to bf16)."""
    vm = ref["vis"]
    hd = q.shape[-1]
    q, k, v, do = q.double(), k.double(), v.double(), dout.double()
    P, lse = ref["P"], ref["lse"].masked_fill(~vm.any(-1), 0.0)
    eP = (_score_err(q, k, scale, vm) + EXP * (1 + lse.abs()[..., None] + ref["S"].abs())) * vm
    if e_lse is not None:
        eP = eP + e_lse.masked_fill(~vm.any(-1), 0.0)[..., None] * vm
    e_dv = C * ((((2 * U + eP) * ref.get("Pm", P)).transpose(-1, -2) @ do.abs()) + U * ref["dV"].abs()) + TINY
    e_dp = hd * G32 * (do.abs() @ v.abs().transpose(-1, -2))
    if ref.get("mult") is not None:
        e_dp = e_dp * ref["mult"].double()
    dP, delta = ref["dP"], ref["delta"]
    n_i = vm.sum(-1).double()
    pdp = (P * dP.abs()).sum(-1)
    e_delta = (U + hd * G32) * (do.abs() * ref["O"].abs()).sum(-1) + (P * (eP * dP.abs() + e_dp)).sum(-1) \
        + n_i * 2.0 ** -24 * pdp
    if e_o is not None:
        e_delta = e_delta + (do.abs() * e_o).sum(-1)
    dS = ref["dS"]
    e_ds = P * ((U + eP) * (dP - delta[..., None]).abs() + e_dp + e_delta[..., None]) + U * dS.abs()
    e_dq = C * (scale * (e_ds @ k.abs() + U * dS.abs() @ k.abs()) + U * ref["dQ"].abs()) + TINY
    e_dk = C * (scale * (e_ds.transpose(-1, -2) @ q.abs() + U * dS.abs().transpose(-1, -2) @ q.abs())
                + U * ref["dK"].abs()) + TINY
    return e_dq, e_dk, e_dv


# ---------------------------------------------------------------------------------- kernel arithmetic on the CPU
def _bf16(x):
    return x.to(torch.bfloat16).float()


def simulate_fwd(q, k, v, vis, scale, defect=None, mult=None):
    """The forward kernels' arithmetic in fp32: raw scores accumulated in fp32, the scale folded into the exponent
    (exp2 of s * scale * log2e - m * scale * log2e), P rounded to bf16 before P V, the normaliser summed from the
    fp32 P, O rounded to bf16, lse = m * scale + log(l).
    defect: None | "causal_shift" (each row also sees the next key) | "drop_last_block" (the last 64-key block of
    every sequence is skipped) | "lse_shift" (lse off by log(2) / 64)."""
    q, k, v = q.float(), k.float(), v.float()
    vm = vis[:, None]
    if defect == "causal_shift":
        vm = vm | torch.roll(vm, 1, dims=-1) & (torch.arange(vm.shape[-1]) > 0)
    elif defect == "drop_last_block":
        last = (vis.sum(-1).amax(-1) - 1).clamp(min=0) // 64 * 64            # [n]: first key of the last block
        vm = vm & (torch.arange(vm.shape[-1])[None, None, None, :] < last[:, None, None, None])
    sl2 = torch.tensor(scale * 1.4426950408889634, dtype=torch.float32)
    s = (q @ k.transpose(-1, -2)).masked_fill(~vm, -math.inf)
    m = s.amax(-1, keepdim=True)
    ms = torch.where(torch.isinf(m), torch.zeros_like(m), m * sl2)
    p = torch.exp2(s * sl2 - ms)
    l = p.sum(-1, keepdim=True)
    pd = p if mult is None else p * mult.float()          # dropout: each kept probability scaled by 1 / (1 - p)
    o = _bf16((_bf16(pd) @ v) / torch.where(l > 0, l, torch.ones_like(l)))
    lse = (m * torch.tensor(scale, dtype=torch.float32) + torch.log(l)).squeeze(-1)
    if defect == "lse_shift":
        lse = lse + math.log(2) / 64
    return o, lse


def simulate_bwd(q, k, v, o, lse, dout, vis, scale, mult=None):
    """The tensor-core backward's arithmetic in fp32 from the given bf16 O and fp32 lse: P = exp2(s * scale * log2e -
    lse * log2e), dP = dO V^T, delta = rowsum(dO o O), dS = P o (dP - delta) rounded to bf16, dQ = scale dS K,
    dK = scale dS^T Q, dV = bf16(P)^T dO, each rounded to bf16.  With a dropout multiplier M, dP is M o dO V^T and
    dV = bf16(P o M)^T dO."""
    q, k, v, o, do = q.float(), k.float(), v.float(), o.float(), dout.float()
    vm = vis[:, None]
    sl2 = torch.tensor(scale * 1.4426950408889634, dtype=torch.float32)
    lse2 = torch.where(vm.any(-1), lse.float(), torch.full_like(lse.float(), math.inf)) * 1.4426950408889634
    s = (q @ k.transpose(-1, -2)).masked_fill(~vm, -math.inf)
    p = torch.exp2(s * sl2 - lse2[..., None])
    dp = do @ v.transpose(-1, -2)
    pd = p
    if mult is not None:
        dp, pd = dp * mult.float(), p * mult.float()
    delta = (do * o).sum(-1, keepdim=True)
    ds = _bf16(p * (dp - delta))
    sc = torch.tensor(scale, dtype=torch.float32)
    dq = _bf16((ds @ k) * sc)
    dk = _bf16((ds.transpose(-1, -2) @ q) * sc)
    dv = _bf16(_bf16(pd).transpose(-1, -2) @ do)
    return dq, dk, dv


def worst_ratio(got, want, bound, where=None):
    """max |got - want| / bound over the elements selected by `where` (all by default); nan anywhere counts as inf."""
    err = (got.double() - want.double()).abs() / bound
    err = torch.where(torch.isnan(err), torch.full_like(err, math.inf), err)
    if where is not None:
        err = err[where.expand_as(err)]
    return float(err.max()) if err.numel() else 0.0
