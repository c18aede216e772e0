"""Float64 references and per-element error bounds for the LayerNorm, cross-entropy, reduction and optimizer kernels
(csrc/layernorm.cu, csrc/misc.cu, csrc/optim.cu), and a CPU simulation of their fp32 arithmetic.

Used by test_misc_bounds_gpu.py (kernel vs reference) and test_misc_bounds_cpu.py (the references against torch, the
bounds against the simulation).  Pure torch.  u = 2^-8 (bf16), u32 = 2^-24 (fp32), C = 2 and TINY = 2^-100 as in
gemm_bounds.py: every bound below is C [...] + TINY.  Inputs are the bf16 / fp32 values the kernels read, held exactly
in float64.  Grid sizes follow the host code; `sms` is the device's SM count.

Summation.  A sum evaluated along any order in which each term meets at most h roundings is within h u32 sum|x_i| of
the exact sum (each rounding is relative to a partial sum, at most sum|x_i|).  Adding an exact zero does not round.
k atomic adds onto x0 cost k u32 (|x0| + sum|x_i|) in any order.

LayerNorm forward (ln_fwd_kernel: lane-sequential sums over 8 ceil(D/256) elements, a 5-level butterfly, two-pass
variance, rsqrtf): the LayerNorm bound of gemm_bounds.py with n = D (a sum is at most D/32 + 5 <= D + 1 roundings
deep): mean C e_mean, rstd C e_rstd rstd, y layernorm_bound (an fp32 y rounds once, u32 |y|, a bf16 y u |y|).  A
padding slot (in_rows -1) is a bf16 zero row with mean = rstd = 0, exactly.

LayerNorm backward (ln_bwd_kernel), from statistics (mu, rs): xh = (x - mu) rs, gy = dy gamma (exact: a product of two
bf16), s1 = mean(gy), s2 = mean(gy xh), dx = rs (gy - s1 - xh s2) + add.  The row sums are h = 8 ceil(D/256) + 5
roundings deep and end with a division; fl(xh) is 2 u32 off and the product with gy rounds once:
    E1 = (h + 1) u32 sum|gy| / D,   E2 = (h + 4) u32 sum|gy xh| / D,   S = |gy| + |s1| + |xh s2|,
    e_dx = rs (E1 + |xh| E2 + 8 u32 S) + u32 (|dx - add| + |add|) [add]
(xh s2 costs 3 u32, the two subtractions and the product with rs 5 u32 of S).  Chained to the forward's own statistics
(off by e_mean and e_rstd rs), xh moves by Dxh = e_mean rs + |xh| e_rstd and dx by
    e_stat = e_rstd |dx - add| + rs (|s2| Dxh + |xh| mean(|gy| Dxh)).
bf16 dx: C [(1 + u) e + u |dx|].  dx_drop = fl(dx_fp32 k) on kept elements, 0 elsewhere, k = fl32(1/(1-p)):
    C [(1 + u) k e + u32 k |dx| + u |dx_drop|].
dgamma += sum_r dy xh, dbeta += sum_r dy: each thread sums the rows_w = ceil(rows / 8B) rows its warp visits in order,
the 8 warps of a block are summed in order, and each of the B = min(ceil(rows/8), sms (D <= 1024 ? 3 : 2)) blocks adds
one atomic:
    e_dgamma = (rows_w + 9 + B) u32 sum|dy xh| + B u32 |dgamma0|   (+ sum|dy| Dxh chained),
    e_dbeta  = (rows_w + 6 + B) u32 sum|dy| + B u32 |dbeta0|.

Cross-entropy forward (ce_fwd_kernel, 256 threads per row): per thread an online (max, sum) over 8-element vectors and
the ragged tail, then a 5-level butterfly and an 8-warp merge of (m, s) pairs; lse = M + logf(S), M the exact row max.
__expf(a) = ex2.approx(fl(a log2e)) is EX2_REL relative plus u32 |a| for each of a's own rounding, the product and the
fp32 log2e.  A term x_j meets its own exp and every rescaling on its way into S; the rescalings' arguments are the
increases of the running max, which add up to at most M - x_j, and there are at most nv + 12 of them (nv: the thread's
vectors and tail elements; n_t: its elements).  With p_j = exp(x_j - M) / S:
    e_S / S = (13 + nv) EX2_REL + 6 u32 sum_j p_j (M - x_j) + (n_t + 3 nv + 41) u32 + V 2^-126 / S,
    e_lse   = e_S / S + 2 u32 |log S| + u32 |lse|      (logf is the accurate libm function: no fast math),
    e_loss  = e_lse + u32 |loss|                        (absolute: a confident row's loss cancels to ~0).
Backward from a given fp32 lse l: dlogit = g (exp(x - l) - [label]), bf16, with q = exp(x - l):
    C [|g| q (EX2_REL + 3 u32 |x - l| + e_l) + u32 |g| |q - 1| [label] + (u32 + u) |dlogit| + |g| 2^-126],
e_l = e_lse when l is the kernel's own lse, else 0.  Rows with g = 0 are exact zeros.

colsum (colsum_kernel): with the host's (gx, splits, rpb), warp w of a split sums rows r0 + w + 8k in order, the block
sums its 8 warps in order, and each split adds one atomic:
    e = (ceil(rpb / 8) + 6) u32 sum|x| + splits u32 (|out0| + sum|x|).
group_reduce: out = bf16(fl(fl(sum_t x) scale)):  C [((T - 1) u32 sum|x| + u32 |sum x|) |scale| + (u32 + u) |out|].
Broadcast: bf16(fl(x scale)), exactly.
sumsq (sumsq_kernel, B = min(n/4/256 + 1, 8 sms) blocks): per thread k = ceil(n/4 / 256B) four-element groups (4
roundings each) added in order, the tail (2), a 5-level butterfly, the 3-level 8-lane shuffle and one atomic per block:
    e = (k + 14 + B) u32 sum g^2 + B u32 |out0|.

AdamW (adamw_kernel) against the float64 step on the fp32 values of every input and hyperparameter; bc1 and bc2 are
1 - beta^t from the fp32 betas (by-value step) or the given fp32 values (hyper):
    clip: sqrtf, * grad_scale, + 1e-6f, /, *: 6 u32 relative (fminf is 1-Lipschitz);  ge = g coef: eg = 7 u32.
    host powf: bc = fl(1 - powf(beta, t)) is e_bc = (2 u32 beta^t + u32 bc) / bc relative (0 with hyper).
    m' = b1 m + (1-b1) ge:          e_m = (1-b1) |ge| (eg + 2 u32) + 2 u32 (b1 |m| + (1-b1) |ge|)
    v' = b2 v + (1-b2) ge^2:        e_v = (1-b2) ge^2 (2 eg + 3 u32) + 2 u32 v'
    d = sqrtf(v') rsqrtf(bc2) + eps:  e_d = sqrt(v'/bc2) (e_v / 2v' + 2 u32 + 2^-22 + e_bc2 / 2) + u32 d
    q = (lr / bc1) m' / d:          e_q = |q| (e_bc1 + 3 u32 + e_d / d) + (lr / bc1) e_m / d
    w' = w (1 - lr wd) - q:         e_w = 3 u32 |w| + e_q + u32 |w'|
param must equal bf16(master) bit for bit.
"""
import math

import torch

from gemm_bounds import C, EX2_REL, TINY, U, U32, layernorm_bound, layernorm_stat_errors  # noqa: F401
from gemm_bounds import worst_ratio  # noqa: F401

LN_WARPS = 8
CE_THREADS = 256
SMS_H100 = 132
LOG2E32 = float(torch.tensor(math.log2(math.e), dtype=torch.float32))
CLIP_EPS32 = float(torch.tensor(1e-6, dtype=torch.float32))


def f32(x):
    """x rounded to fp32, as a Python float (a hyperparameter the kernel receives by value)."""
    return float(torch.tensor(x, dtype=torch.float32))


def _cdiv(a, b):
    return -(-a // b)


# ---------------------------------------------------------------------------------- host grid formulas
def ln_fwd_blocks(rows, sms):
    return min(_cdiv(rows, LN_WARPS), sms * 8)


def ln_bwd_blocks(rows, D, sms, wgrad=True):
    return min(_cdiv(rows, LN_WARPS), sms * ((3 if D <= 1024 else 2) if wgrad else 8))


def colsum_grid(R, Cc, sms):
    """(gx, splits, rows per split) of ymp_colsum."""
    gx = _cdiv(_cdiv(Cc, 8), 32)
    splits = max(1, min(_cdiv(R, 64), _cdiv(sms * 4, gx)))
    rpb = _cdiv(R, splits)
    return gx, _cdiv(R, rpb), rpb


def sumsq_blocks(n, sms):
    return min((n // 4 + 255) // 256 + 1, sms * 8)


# ---------------------------------------------------------------------------------- LayerNorm
def ln_fwd_reference(x, gamma, beta, eps):
    """(y, mean, rstd) in float64; x [rows, D] holds the rows the kernel normalises."""
    x = x.double()
    mean = x.mean(-1)
    rstd = 1.0 / torch.sqrt(x.var(-1, unbiased=False) + eps)
    y = (x - mean[:, None]) * rstd[:, None] * gamma.double() + beta.double()
    return y, mean, rstd


def ln_fwd_bounds(x, gamma, beta, eps, y_bf16=True):
    """(e_y, e_mean, e_rstd) per element / row."""
    e_mean, e_rstd = layernorm_stat_errors(x, eps)
    rstd = ln_fwd_reference(x, gamma, beta, eps)[2]
    return (layernorm_bound(x, gamma, beta, eps, out_bf16=y_bf16), C * e_mean[:, 0] + TINY,
            C * e_rstd[:, 0] * rstd + TINY)


def ln_row_depth(D):
    return 8 * _cdiv(D, 256) + 5


def ln_bwd_reference(dy, x, gamma, mean, rstd, add=None, dgamma0=None, dbeta0=None, keep=None, p=0.0):
    """float64 backward from the statistics (mean, rstd) [rows]: the given fp32 values, or the exact ones.  Returns a
    dict with dx (including add), dx_drop (keep: bool mask, p: dropout probability), dgamma / dbeta (added onto
    dgamma0 / dbeta0) and the intermediate terms the bounds use."""
    dy, x, g = dy.double(), x.double(), gamma.double()
    mu, rs = mean.double()[:, None], rstd.double()[:, None]
    D = x.shape[1]
    xh = (x - mu) * rs
    gy = dy * g
    s1 = gy.mean(-1, keepdim=True)
    s2 = (gy * xh).mean(-1, keepdim=True)
    dx0 = rs * (gy - s1 - xh * s2)
    dx = dx0 + add.double() if add is not None else dx0
    r = dict(dx=dx, dx0=dx0, xh=xh, gy=gy, s1=s1, s2=s2, rs=rs, dy=dy, add=add, D=D)
    if keep is not None:
        r["k"] = f32(1.0 / (1.0 - f32(p)))
        r["keep"] = keep
        r["dx_drop"] = torch.where(keep, dx * r["k"], torch.zeros_like(dx))
    if dgamma0 is not None:
        r["dgamma0"], r["dbeta0"] = dgamma0.double(), dbeta0.double()
        r["dgamma"] = r["dgamma0"] + (dy * xh).sum(0)
        r["dbeta"] = r["dbeta0"] + dy.sum(0)
    return r


def ln_bwd_bounds(ref, blocks, stat_err=None, rows=None):
    """Bounds on dx, dx_drop, dgamma, dbeta (module docstring).  blocks: the host's block count; stat_err = (e_mean,
    e_rstd) [rows, 1] of the forward when the statistics are the kernel's own (then ref holds the exact ones); rows: the
    launch's row count when it includes padding slots that ref leaves out."""
    D, rs, xh, gy, s1, s2, dx0 = ref["D"], ref["rs"], ref["xh"], ref["gy"], ref["s1"], ref["s2"], ref["dx0"]
    h = ln_row_depth(D)
    E1 = (h + 1) * U32 * gy.abs().sum(-1, keepdim=True) / D
    E2 = (h + 4) * U32 * (gy * xh).abs().sum(-1, keepdim=True) / D
    S = gy.abs() + s1.abs() + (xh * s2).abs()
    e = rs * (E1 + xh.abs() * E2 + 8 * U32 * S)
    if ref["add"] is not None:
        e = e + U32 * (dx0.abs() + ref["add"].double().abs())
    dxh = None
    if stat_err is not None:
        e_mean, e_rstd = stat_err
        dxh = e_mean * rs + xh.abs() * e_rstd
        e = e + e_rstd * dx0.abs() + rs * (s2.abs() * dxh + xh.abs() * (gy.abs() * dxh).mean(-1, keepdim=True))
    out = dict(dx=C * ((1 + U) * e + U * ref["dx"].abs()) + TINY)
    if "keep" in ref:
        k = ref["k"]
        b = C * ((1 + U) * k * e + U32 * k * ref["dx"].abs() + U * ref["dx_drop"].abs()) + TINY
        out["dx_drop"] = torch.where(ref["keep"], b, torch.full_like(b, TINY))
    if "dgamma" in ref:
        rows_w = _cdiv(rows or ref["dy"].shape[0], LN_WARPS * blocks)
        dy = ref["dy"]
        eg = (rows_w + 9 + blocks) * U32 * (dy * xh).abs().sum(0) + blocks * U32 * ref["dgamma0"].abs()
        if dxh is not None:
            eg = eg + (dy.abs() * dxh).sum(0)
        eb = (rows_w + 6 + blocks) * U32 * dy.abs().sum(0) + blocks * U32 * ref["dbeta0"].abs()
        out["dgamma"], out["dbeta"] = C * eg + TINY, C * eb + TINY
    return out


# ---------------------------------------------------------------------------------- cross-entropy
def ce_reference(x, labels):
    """(loss, lse) in float64 for logits x [rows, V] and int64 labels (clamped to [0, V) like the kernel)."""
    x = x.double()
    lse = torch.logsumexp(x, -1)
    lab = labels.clamp(0, x.shape[1] - 1)
    return lse - x.gather(1, lab[:, None])[:, 0], lse


def ce_thread_counts(V):
    """(n_t, nv): the most elements and (vectors + tail elements) one of the 256 threads handles."""
    nvec, tail = V // 8, V % 8
    per = _cdiv(nvec, CE_THREADS)
    t = 1 if tail else 0
    return 8 * per + t, per + t


def ce_fwd_bounds(x, labels):
    """(e_loss, e_lse) per row and the unscaled e_lse that a chained backward adds (module docstring)."""
    x = x.double()
    V = x.shape[1]
    n_t, nv = ce_thread_counts(V)
    loss, lse = ce_reference(x, labels)
    M = x.max(-1, keepdim=True).values
    w = torch.exp(x - M)
    S = w.sum(-1)
    spread = (w * (M - x)).sum(-1) / S
    eS = (13 + nv) * EX2_REL + 6 * U32 * spread + (n_t + 3 * nv + 41) * U32 + V * 2.0 ** -126 / S
    e_lse = eS + 2 * U32 * torch.log(S).abs() + U32 * lse.abs()
    e_loss = e_lse + U32 * loss.abs()
    return C * e_loss + TINY, C * e_lse + TINY, e_lse


def ce_bwd_reference(x, labels, lse, g):
    """g (exp(x - lse) - onehot) in float64 with the given lse [rows] and row gradients g [rows]."""
    x = x.double()
    q = torch.exp(x - lse.double()[:, None])
    lab = labels.clamp(0, x.shape[1] - 1)
    onehot = torch.zeros_like(q).scatter_(1, lab[:, None], 1.0)
    return g.double()[:, None] * (q - onehot), q, onehot


def ce_bwd_bounds(x, labels, lse, g, e_l=None):
    want, q, onehot = ce_bwd_reference(x, labels, lse, g)
    ga = g.double().abs()[:, None]
    el = 0.0 if e_l is None else e_l.double()[:, None]
    e = ga * q * (EX2_REL + 3 * U32 * (x.double() - lse.double()[:, None]).abs() + el) + U32 * ga * (q - 1).abs() * onehot \
        + (U32 + U) * want.abs() + ga * 2.0 ** -126
    return want, C * e + TINY


# ---------------------------------------------------------------------------------- reductions
def colsum_bound(x, out0, sms):
    R, Cc = x.shape
    _, splits, rpb = colsum_grid(R, Cc, sms)
    sa = x.double().abs().sum(0)
    return C * ((_cdiv(rpb, 8) + 6) * U32 * sa + splits * U32 * (out0.double().abs() + sa)) + TINY


def group_reduce_reference(x, G, T, scale):
    """out [G, C] = scale * sum_t x[g, t] (x [G*T, C]); scale is the fp32 value the kernel receives."""
    return x.double().view(G, T, -1).sum(1) * f32(scale)


def group_reduce_bound(x, G, T, scale):
    xs = x.double().view(G, T, -1)
    want = xs.sum(1) * f32(scale)
    e = ((T - 1) * U32 * xs.abs().sum(1) + U32 * xs.sum(1).abs()) * abs(f32(scale)) + (U32 + U) * want.abs()
    return C * e + TINY


def sumsq_bound(g, out0, sms):
    n = g.numel()
    B = sumsq_blocks(n, sms)
    k = _cdiv(n // 4, B * 256)
    return C * ((k + 14 + B) * U32 * (g.double() ** 2).sum() + B * U32 * abs(float(out0))) + TINY


# ---------------------------------------------------------------------------------- AdamW
def adamw_hyper(step, lr, beta1, beta2, weight_decay, hyper=None):
    """(lr, wd, bc1, bc2, e_bc1, e_bc2) as the kernel sees them, in float64: fp32 values, bias corrections exact from
    the fp32 betas (by value) or the given fp32 array (hyper), and the relative error of the host's powf."""
    if hyper is not None:
        h = [float(v) for v in hyper.float().cpu()]
        return h[0], h[1], h[2], h[3], 0.0, 0.0
    b1, b2 = f32(beta1), f32(beta2)
    p1, p2 = b1 ** step, b2 ** step
    bc1, bc2 = 1.0 - p1, 1.0 - p2
    return f32(lr), f32(weight_decay), bc1, bc2, (2 * U32 * p1 + U32 * bc1) / bc1, (2 * U32 * p2 + U32 * bc2) / bc2


def clip_coef(sumsq, grad_scale, max_norm):
    """The clip coefficient from the given fp32 sum of squares (NULL -> None or max_norm <= 0: no clipping)."""
    gs = f32(grad_scale)
    if sumsq is None or max_norm <= 0:
        return gs
    norm = math.sqrt(float(sumsq)) * gs
    return gs * min(1.0, f32(max_norm) / (norm + CLIP_EPS32))


def adamw_reference(master, grad, m, v, *, step, lr, beta1, beta2, eps, weight_decay, grad_scale=1.0, max_norm=0.0,
                    sumsq=None, hyper=None):
    """One AdamW step in float64 (torch.optim.AdamW's formula, decoupled decay).  Returns (w, m, v, coef, hyper)."""
    lr_, wd, bc1, bc2, _, _ = adamw_hyper(step, lr, beta1, beta2, weight_decay, hyper)
    b1, b2, ep = f32(beta1), f32(beta2), f32(eps)
    coef = clip_coef(sumsq, grad_scale, max_norm)
    ge = grad.double() * coef
    m1 = b1 * m.double() + (1 - b1) * ge
    v1 = b2 * v.double() + (1 - b2) * ge * ge
    w1 = master.double() * (1 - lr_ * wd) - (lr_ / bc1) * m1 / (torch.sqrt(v1) / math.sqrt(bc2) + ep)
    return w1, m1, v1


def adamw_bounds(master, grad, m, v, *, step, lr, beta1, beta2, eps, weight_decay, grad_scale=1.0, max_norm=0.0,
                 sumsq=None, hyper=None):
    """(e_master, e_m, e_v) per element (module docstring)."""
    lr_, wd, bc1, bc2, e_bc1, e_bc2 = adamw_hyper(step, lr, beta1, beta2, weight_decay, hyper)
    b1, b2, ep = f32(beta1), f32(beta2), f32(eps)
    clipped = sumsq is not None and max_norm > 0
    eg = (7 if clipped else 1) * U32
    w1, m1, v1 = adamw_reference(master, grad, m, v, step=step, lr=lr, beta1=beta1, beta2=beta2, eps=eps,
                                 weight_decay=weight_decay, grad_scale=grad_scale, max_norm=max_norm, sumsq=sumsq,
                                 hyper=hyper)
    ge = grad.double() * clip_coef(sumsq, grad_scale, max_norm)
    e_m = (1 - b1) * ge.abs() * (eg + 2 * U32) + 2 * U32 * (b1 * m.double().abs() + (1 - b1) * ge.abs())
    e_v = (1 - b2) * ge * ge * (2 * eg + 3 * U32) + 2 * U32 * v1
    sv = torch.sqrt(v1 / bc2)
    d = sv + ep
    rel_v = torch.where(v1 > 0, e_v / (2 * v1), torch.zeros_like(v1))
    e_d = sv * (rel_v + 2 * U32 + 2.0 ** -22 + e_bc2 / 2) + U32 * d
    step_sz = lr_ / bc1
    q = step_sz * m1 / d
    e_q = q.abs() * (e_bc1 + 3 * U32 + e_d / d) + step_sz * e_m / d
    e_w = 3 * U32 * master.double().abs() + e_q + U32 * w1.abs()
    return C * e_w + TINY, C * e_m + TINY, C * e_v + TINY


# ---------------------------------------------------------------------------------- kernel arithmetic on the CPU
def _fma(a, b, c):
    """fp32 fma: the product of two fp32 values is exact in float64, the sum is rounded (twice, harmlessly)."""
    return (a.double() * b.double() + c.double()).float()


def _ex2(x):
    """ex2.approx.ftz.f32 without its approximation error: 2^x rounded to fp32, results below 2^-126 flushed to 0."""
    r = torch.exp2(x.double()).float()
    return torch.where(r.abs() < 2.0 ** -126, torch.zeros_like(r), r)


def _expf(a):
    """__expf(a) = ex2.approx(fl(a log2e))."""
    return _ex2(a.float() * LOG2E32)


def _rsqrt(x):
    return (1.0 / torch.sqrt(x.double())).float()


def _bf16(x):
    return x.to(torch.bfloat16).float()


def _butterfly(s):
    """warp_sum over the last dimension (32 lanes): v += shfl_xor(v, o) for o = 16 .. 1; every lane ends equal."""
    idx = torch.arange(s.shape[-1])
    for o in (16, 8, 4, 2, 1):
        s = s + s[..., idx ^ o]
    return s[..., 0]


def _lane_view(x):
    """[rows, D] -> [rows, VPL, 32, 8]: element (j * 32 + lane) * 8 + e, zero-padded past D."""
    rows, D = x.shape
    vpl = _cdiv(D // 8, 32)
    pad = torch.zeros(rows, vpl * 256, dtype=x.dtype)
    pad[:, :D] = x
    return pad.view(rows, vpl, 32, 8)


def _row_sum(t):
    """The kernel's row sum of t [rows, D] in fp32: per lane over j then e in order, then the butterfly."""
    lv = _lane_view(t.float())
    acc = torch.zeros(lv.shape[0], 32)
    for j in range(lv.shape[1]):
        for e in range(8):
            acc = acc + lv[:, j, :, e]
    return _butterfly(acc)


def simulate_ln_fwd(x, gamma, beta, eps, y_bf16=True, defect=None):
    """(y, mean, rstd) with ln_fwd_kernel's fp32 arithmetic.  defect: None | "var_d_minus_1" | "no_eps" |
    "skip_last_vec" (the last 8-column vector of each row not stored: NaN, the sentinel of unwritten memory)."""
    x = x.float()
    D = x.shape[1]
    mu = _row_sum(x) / D
    d = x - mu[:, None]
    q = _row_sum(d * d)
    var = q / (D - 1 if defect == "var_d_minus_1" else D)
    rs = _rsqrt(var if defect == "no_eps" else var + torch.tensor(eps, dtype=torch.float32))
    y = _fma(d * rs[:, None], gamma.float(), beta.float())
    if y_bf16:
        y = _bf16(y)
    if defect == "skip_last_vec":
        y[:, D - 8:] = math.nan
    return y, mu, rs


def simulate_ln_bwd(dy, x, gamma, mean, rstd, add=None, dgamma0=None, dbeta0=None, keep=None, p=0.0, blocks=1,
                    seed=0, defect=None):
    """ln_bwd_kernel's fp32 arithmetic: dict with dx (bf16 values), dx_drop, dgamma, dbeta.  dgamma / dbeta: each
    warp's threads sum its rows in order, blocks sum their 8 warps in order, the block partials go onto dgamma0 / dbeta0
    in a shuffled order.  defect: None | "drop_block_dgamma" (block 0's partial never added) | "xh_s2_no_rs"."""
    dy, x, g = dy.float(), x.float(), gamma.float()
    rows, D = x.shape
    mu, rs = mean.float()[:, None], rstd.float()[:, None]
    xh = (x - mu) * rs
    gy = dy * g
    s1 = _row_sum(gy)[:, None] / D
    s2 = _row_sum(gy * xh)[:, None] / D
    t = (x - mu) * (1.0 if defect == "xh_s2_no_rs" else rs) * s2
    o = rs * (gy - s1 - t)
    if add is not None:
        o = o + add.float()
    r = dict(dx=_bf16(o))
    if keep is not None:
        k = torch.tensor(1.0, dtype=torch.float32) / (1.0 - torch.tensor(p, dtype=torch.float32))
        r["dx_drop"] = _bf16(torch.where(keep, o * k, torch.zeros_like(o)))
    if dgamma0 is not None:
        nw = LN_WARPS * blocks
        passes = _cdiv(rows, nw)
        for name, terms, init in (("dgamma", dy * xh, dgamma0), ("dbeta", dy, dbeta0)):
            pad = torch.zeros(passes * nw, D)
            pad[:rows] = terms
            acc = torch.zeros(nw, D)
            for k_ in range(passes):
                acc = acc + pad[k_ * nw:(k_ + 1) * nw]
            acc = acc.view(blocks, LN_WARPS, D)
            part = torch.zeros(blocks, D)
            for w in range(LN_WARPS):
                part = part + acc[:, w]
            out = init.float().clone()
            gen = torch.Generator().manual_seed(seed)
            for b in torch.randperm(blocks, generator=gen).tolist():
                if not (defect == "drop_block_dgamma" and b == 0):
                    out = out + part[b]
            r[name] = out
    return r


def simulate_ce_fwd(x, labels, defect=None):
    """(loss, lse) with ce_fwd_kernel's fp32 arithmetic.  defect: None | "skip_tail" (the V % 8 tail loop removed) |
    "label_plus_1" (the loss reads x[label + 1])."""
    x = x.float()
    rows, V = x.shape
    nvec = V // 8
    per = _cdiv(nvec, CE_THREADS)
    m = torch.full((rows, CE_THREADS), -math.inf)
    s = torch.zeros(rows, CE_THREADS)
    for k in range(per):
        v = k * CE_THREADS + torch.arange(CE_THREADS)
        act = v < nvec
        cols = (v.clamp(max=max(nvec - 1, 0))[:, None] * 8 + torch.arange(8)).view(-1)
        f = x[:, cols].view(rows, CE_THREADS, 8)
        mx = f.max(-1).values
        up = act & (mx > m)
        s = torch.where(up, s * _expf(m - mx), s)
        m = torch.where(up, mx, m)
        for e in range(8):
            s = torch.where(act, s + _expf(f[..., e] - m), s)
    if defect != "skip_tail":
        for c in range(nvec * 8, V):   # thread c - nvec * 8 (the tail is shorter than 256)
            t = c - nvec * 8
            xc = x[:, c]
            up = xc > m[:, t]
            s[:, t] = torch.where(up, s[:, t] * _expf(m[:, t] - xc) + 1.0, s[:, t] + _expf(xc - m[:, t]))
            m[:, t] = torch.where(up, xc, m[:, t])

    def merge(m1, s1, m2, s2):
        mn = torch.maximum(m1, m2)
        sn = torch.where(mn == -math.inf, torch.zeros_like(s1), s1 * _expf(m1 - mn) + s2 * _expf(m2 - mn))
        return mn, sn

    m, s = m.view(rows, 8, 32), s.view(rows, 8, 32)
    idx = torch.arange(32)
    for o in (16, 8, 4, 2, 1):
        m, s = merge(m, s, m[..., idx ^ o], s[..., idx ^ o])
    M, S = m[..., 0, 0], s[..., 0, 0]
    for w in range(1, 8):
        mn = torch.maximum(M, m[..., w, 0])
        S = S * _expf(M - mn) + s[..., w, 0] * _expf(m[..., w, 0] - mn)
        M = mn
    lse = M + torch.log(S.double()).float()
    lab = labels.clamp(0, V - 1)
    if defect == "label_plus_1":
        lab = (lab + 1).clamp(max=V - 1)
    return lse - x.gather(1, lab[:, None])[:, 0], lse


def simulate_colsum(x, out0, sms, seed=0, defect=None):
    """colsum_kernel's fp32 arithmetic.  defect: None | "drop_last_row" (the last row of every split not summed)."""
    x = x.float()
    R, Cc = x.shape
    _, splits, rpb = colsum_grid(R, Cc, sms)
    parts = []
    for sp in range(splits):
        r0, r1 = sp * rpb, min(R, (sp + 1) * rpb)
        if defect == "drop_last_row":
            r1 -= 1
        blk = torch.zeros(_cdiv(rpb, 8) * 8, Cc)
        blk[:r1 - r0] = x[r0:r1]
        blk = blk.view(-1, 8, Cc)       # [k, warp, C]: warp w takes rows r0 + w + 8k
        acc = torch.zeros(8, Cc)
        for k in range(blk.shape[0]):
            acc = acc + blk[k]
        part = torch.zeros(Cc)
        for w in range(8):
            part = part + acc[w]
        parts.append(part)
    out = out0.float().clone()
    for i in torch.randperm(splits, generator=torch.Generator().manual_seed(seed)).tolist():
        out = out + parts[i]
    return out


def simulate_sumsq(g, out0, sms, seed=0, defect=None):
    """sumsq_kernel's fp32 arithmetic.  defect: None | "no_tail" (the n % 4 elements not summed)."""
    g = g.float()
    n = g.numel()
    B = sumsq_blocks(n, sms)
    nt = B * 256
    n4 = n // 4
    k = _cdiv(n4, nt)
    v = torch.zeros(k * nt, 4)
    v[:n4] = g[:n4 * 4].view(n4, 4)
    acc = torch.zeros(nt)
    for i in range(k):
        c = v[i * nt:(i + 1) * nt]
        acc = acc + (((c[:, 0] * c[:, 0] + c[:, 1] * c[:, 1]) + c[:, 2] * c[:, 2]) + c[:, 3] * c[:, 3])
    if defect != "no_tail":
        for j in range(n4 * 4, n):
            t = j - n4 * 4
            acc[t] = acc[t] + g[j] * g[j]
    w = _butterfly(acc.view(B, 8, 32))           # [B, 8]
    idx = torch.arange(8)
    for o in (4, 2, 1):
        w = w + w[:, idx ^ o]
    out = torch.tensor(float(out0), dtype=torch.float32)
    for b in torch.randperm(B, generator=torch.Generator().manual_seed(seed)).tolist():
        out = out + w[b, 0]
    return out


def simulate_adamw(master, grad, m, v, *, step, lr, beta1, beta2, eps, weight_decay, grad_scale=1.0, max_norm=0.0,
                   sumsq=None, defect=None):
    """adamw_kernel's fp32 arithmetic (by-value hyperparameters, host powf).  Returns (master, m, v, param).
    defect: None | "bc2_not_sqrt" (1/bc2 where 1/sqrt(bc2) belongs)."""
    t32 = lambda a: torch.tensor(a, dtype=torch.float32)  # noqa: E731
    b1, b2, ep, gs = t32(beta1), t32(beta2), t32(eps), t32(grad_scale)
    coef = gs
    if sumsq is not None and max_norm > 0:
        norm = torch.sqrt(t32(float(sumsq))) * gs
        coef = coef * torch.clamp(t32(max_norm) / (norm + t32(1e-6)), max=1.0)
    bc1 = 1.0 - t32(float(b1) ** step)
    bc2 = 1.0 - t32(float(b2) ** step)
    lr_, wd = t32(lr), t32(weight_decay)
    stp = lr_ / bc1
    inv_bc2 = 1.0 / bc2 if defect == "bc2_not_sqrt" else _rsqrt(bc2)
    decay = 1.0 - lr_ * wd
    ge = grad.float() * coef
    m1 = _fma(b1, m.float(), (1.0 - b1) * ge)
    v1 = _fma(b2, v.float(), (1.0 - b2) * ge * ge)
    w1 = _fma(master.float(), decay, -(stp * m1 / _fma(torch.sqrt(v1), inv_bc2, ep)))
    return w1, m1, v1, w1.to(torch.bfloat16)
