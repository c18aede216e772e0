"""Float64 GEMM-epilogue reference and per-element error bounds for ymp_gemm, ymp_gemm_skinny and ymp_gemm_skinny_wide.

Used by test_gemm_bounds_gpu.py (kernel vs reference) and test_gemm_bounds_cpu.py (the reference against
torch.nn.functional, the bounds against a CPU simulation of the kernel arithmetic).  Pure torch: runs on any device.

Reference (ymp.h, in this order; all inputs are the bf16 / fp32 values the kernels read, held exactly in float64):
    acc = op(A) op(B)^T,   v = alpha acc + bias,   aux_out = act'(v) (act != NONE) or v,
    out = v * aux_in (aux_in given) or act(v),   out += residual[m % res_row_mod],
    D[store_row(m)] = out, or D += out (accumulate).
u = 2^-8 is the bf16 unit roundoff, u32 = 2^-24 the fp32 one.  Every bound is multiplied by one safety factor C.

Pre-activation v.  The tensor cores add one 16-wide product block per MMA step into the fp32 accumulator with at most
one rounding (possibly truncating: 2^-23 relative to the running magnitude) inside the block and one for the add, so
after S = ceil(K/16) steps split over `split` independent chains
    e_acc = (S + split) 2^-22 (|A||B|)_mn.
alpha costs one rounding (u32 |alpha acc|), the bias add one (u32 |v|).
    e_v = |alpha| e_acc + u32 |alpha acc| [alpha != 1] + u32 |v| [bias].

Activation.  act and act' are Lipschitz with L1 = sup|gelu'| < 1.13 and L2 = sup|gelu''| < 0.8 (both forms; the
CPU suite checks the constants on a grid), so the input error moves them by at most L1 e_v and L2 e_v.  On top of
that each has its own approximation error E(x), evaluated at the reference v:
  erf   Phi = 0.5 + xc Q(u), xc = clamp(x, PHI_ZERO_X, 4.5), u = min(x^2, 4.5^2); pdf = ex2(c1 x^2 + c0)
        (ptx.cuh: norm_cdf_pdf).  Below PHI_ZERO_X (= -4.5 - 8e-6) Phi is the constant PHI_FLOOR = 8.3e-10, so
        E_Phi(x) = Phi(x) + PHI_FLOOR                                   x < PHI_ZERO_X
                 = PHI_POLY_ERR + e_horner(clamp(x, +-4.5)) + Phi(-4.5) [x > 4.5]   otherwise
        (above 4.5 Phi keeps its value at 4.5, which is within Phi(-4.5) of Phi(x); between PHI_ZERO_X and -4.5 it falls
        linearly from its value at -4.5 to PHI_FLOOR).
        PHI_POLY_ERR bounds the polynomial in exact arithmetic on |x| <= 4.5 (checked on a dense grid by the CPU suite);
        e_horner is the running error bound of the fp32 Horner evaluation (each fma rounds once, u = fl(xc^2) once):
        e_j = |u| e_{j+1} + u32 |q_j| + |q_{j+1}| |u| u32,  e_Phi = |xc| e_0 + u32 |Phi|.
        The pdf is ex2.approx of fl(fl(x^2) c1 + c0): relative error EX2_REL of the instruction plus ln2 |arg| 2u32 of
        the argument, flushed to zero below 2^-126:  E_pdf = pdf (EX2_REL + ln2 (|arg| + 2) 2 u32) + 2^-126.
        E_gelu  = |x| E_Phi + u32 |gelu|,   E_gelu' = E_Phi + |x| E_pdf + u32 (|Phi| + |x pdf|).
  tanh  t = tanh.approx(k x (1 + 0.044715 x^2)).  The PTX ISA documents a maximum relative error of about 2^-11 for
        tanh.approx.f32; TANH_REL = 2^-10.9 is used.  The argument carries 4 roundings: (1 - t^2) |arg| 4 u32.
        dt = TANH_REL |t| + (1 - t^2) |arg| 4 u32.  0.5 x (1 + t) has 1 + t exact where it cancels (Sterbenz), so
        E_gelu  = 0.5 |x| dt + 3 u32 |gelu|          (relative to gelu this is large for -5 < x < -2, where 1 + t is small)
        E_gelu' = (|x t du| + 0.5) dt + 4 u32 (|x du| + 1 + |gelu'|),  du = k (1 + 3 0.044715 x^2).
aux_out is stored in bf16:  e_aux = C [L2 e_v + E_gelu'(v) + u |act'(v)|]   (act = NONE: C [e_v + u |v|]).

Output.  aux_in:  e = e_v |aux_in| + u32 |v aux_in|;  act: e = L1 e_v + E_gelu(v) + u32 |act(v)|;  none: e = e_v.
The residual add rounds once (u32 |out|).  Accumulation adds `split` partials to D atomically in any order: each add
rounds relative to the running sum, split u32 (|D0| + |alpha| |A||B|).  A bf16 store adds u |out|.  2^-100 absolute
covers results that underflow.
    e_out = C [e + u32 |out| [residual] + split u32 (|D0| + |alpha||A||B|) [accumulate] + u |out| [bf16]] + 2^-100

LayerNorm of an fp32 row y (two-pass statistics over n = N columns, rsqrt.approx):
    e_mean = (n + 1) u32 mean|y|,   relative error of var + eps: e_var = ((n + 4) u32 var + e_mean^2) / (var + eps)
    (the sum of squares of the deviations from the computed mean is off by n e_mean^2 at most),
    e_rstd = 0.5 e_var + 2^-22 (rsqrt.approx) + 2 u32,
    e_ln   = C [|gamma| (e_mean rstd + |z| (e_rstd + 2 u32)) + u32 |gamma z| + u |ln|] + 2^-100,  z = (y - mean) rstd.
"""
import math

import torch

from attn_bounds import worst_ratio  # noqa: F401  (same definition: max |got - want| / bound, nan counts as inf)

U = 2.0 ** -8           # bf16 unit roundoff
U32 = 2.0 ** -24        # fp32 unit roundoff
G22 = 2.0 ** -22        # one tensor-core accumulation step, per unit of |A||B|
TINY = 2.0 ** -100      # absolute floor (underflow)
C = 2.0                 # the one safety factor of the whole suite

ACT_NONE, ACT_GELU_ERF, ACT_GELU_TANH = 0, 1, 2

# ptx.cuh, norm_cdf_pdf: Q(u) = sum_j PHI_COEF[9 - j] u^j (Horner from the first entry), pdf = ex2(c1 x^2 + c0)
PHI_COEF = (-1.6543631001e-12, 1.9532824653e-10, -1.0287317553e-08, 3.2170341066e-07, -6.7323919166e-06,
            1.0108823657e-04, -1.1397043329e-03, 9.8841767687e-03, -6.6411978624e-02, 3.9892175804e-01)
EX2_C1, EX2_C0 = -0.72134752044, -1.32574806474
CLAMP = 4.5
PHI_ZERO_X = -4.5000081062316895   # ptx.cuh: lower clamp of x in Phi
PHI_FLOOR = 8.3e-10     # |0.5 + PHI_ZERO_X Q(4.5^2)| in the kernel's fp32 arithmetic (checked by the CPU suite)
PHI_POLY_ERR = 4.5e-6   # sup over |x| <= 4.5 of |0.5 + x Q(x^2) - Phi(x)| in exact arithmetic (fp32 coefficients)
EX2_REL = 2.0 ** -21    # ex2.approx.f32 relative error (documented as a few ulp; taken generously)
TANH_REL = 2.0 ** -10.9
TANH_K, TANH_A, TANH_DA = 0.79788456, 0.044715, 0.134145   # the kernel's fp32 constants
L1, L2 = 1.13, 0.8      # Lipschitz constants of gelu and gelu' (both forms)


def _f32(x):
    return torch.tensor(x, dtype=torch.float32).double().item()


PHI_COEF32 = tuple(_f32(c) for c in PHI_COEF)


# ---------------------------------------------------------------------------------- exact activations
def ndtr(x):
    return 0.5 * torch.erfc(-x / math.sqrt(2.0))


def npdf(x):
    return torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


def act_ref(x, act):
    """act(x) in float64: x Phi(x) (erf) or Megatron's tanh form with its exact constants."""
    x = x.double()
    if act == ACT_GELU_ERF:
        return x * ndtr(x)
    if act == ACT_GELU_TANH:
        return 0.5 * x * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (x + TANH_A * x ** 3)))
    return x


def dact_ref(x, act):
    """act'(x) in float64."""
    x = x.double()
    if act == ACT_GELU_ERF:
        return ndtr(x) + x * npdf(x)
    if act == ACT_GELU_TANH:
        k = math.sqrt(2.0 / math.pi)
        t = torch.tanh(k * (x + TANH_A * x ** 3))
        return 0.5 * (1.0 + t) + 0.5 * x * (1.0 - t * t) * k * (1.0 + 3.0 * TANH_A * x * x)
    return torch.ones_like(x)


def phi_poly(x):
    """The kernel's Phi in exact arithmetic (float64, fp32 coefficients), with its clamps."""
    x = x.double()
    xc = x.clamp(PHI_ZERO_X, CLAMP)
    u = (x * x).clamp(max=CLAMP * CLAMP)
    q = torch.full_like(x, PHI_COEF32[0])
    for c in PHI_COEF32[1:]:
        q = q * u + c
    return 0.5 + xc * q


# ---------------------------------------------------------------------------------- reference
def res_rows(M, res_row_mod=0):
    r = torch.arange(M, dtype=torch.int64)
    return r % res_row_mod if res_row_mod else r


def store_rows(M, d_row_block=0, d_row_stride=0):
    """Row of D that result row m is stored to (ymp.h: d_row_block / d_row_stride)."""
    r = torch.arange(M, dtype=torch.int64)
    return (r // d_row_block) * d_row_stride + r % d_row_block if d_row_block else r


def reference(a, b, *, alpha=1.0, bias=None, act=ACT_NONE, aux_in=None, residual=None, res_row_mod=0, d0=None):
    """The whole epilogue in float64.  a [M, K], b [N, K] (op() already applied), bias [N], aux_in [M, N], residual
    [R, N] read at row m % res_row_mod, d0 [M, N] the D rows an accumulating call adds to.  Returns a dict with acc,
    absab = |A||B|, v (pre-activation), aux (what aux_out holds), out (what D holds afterwards) and the inputs."""
    a, b = a.double(), b.double()
    M = a.shape[0]
    acc = a @ b.T
    absab = a.abs() @ b.abs().T
    v = alpha * acc
    if bias is not None:
        v = v + bias.double()[None, :]
    aux = dact_ref(v, act) if act else v
    out = v * aux_in.double() if aux_in is not None else act_ref(v, act)
    res = None
    if residual is not None:
        res = residual.double()[res_rows(M, res_row_mod).to(residual.device)]
        out = out + res
    if d0 is not None:
        out = d0.double() + out
    return dict(acc=acc, absab=absab, v=v, aux=aux, out=out, alpha=alpha, bias=bias, act=act, aux_in=aux_in,
                residual=res, d0=d0)


# ---------------------------------------------------------------------------------- bounds
def _horner_err(xc):
    """Running error bound of the kernel's fp32 Horner evaluation of Phi at xc (module docstring)."""
    u = xc * xc
    q = torch.full_like(xc, PHI_COEF32[0])
    e = torch.zeros_like(xc)
    for c in PHI_COEF32[1:]:
        qn = q * u + c
        e = u.abs() * e + U32 * qn.abs() + q.abs() * u.abs() * U32
        q = qn
    phi = 0.5 + xc * q
    return xc.abs() * e + U32 * phi.abs()


def act_err(x, act):
    """(E_act, E_act'): the activation's own approximation error at float64 pre-activation x (module docstring)."""
    x = x.double()
    ax = x.abs()
    if act == ACT_GELU_ERF:
        xc = x.clamp(-CLAMP, CLAMP)
        phi = ndtr(x)
        e_phi = torch.where(x < PHI_ZERO_X, phi + PHI_FLOOR,
                            PHI_POLY_ERR + _horner_err(xc) + torch.where(x > CLAMP, ndtr(torch.tensor(-CLAMP)),
                                                                          torch.zeros_like(x)))
        pdf = npdf(x)
        arg = x * x * abs(EX2_C1) + abs(EX2_C0)
        e_pdf = pdf * (EX2_REL + math.log(2.0) * (arg + 2.0) * 2 * U32) + 2.0 ** -126
        e_act = ax * e_phi + U32 * (x * phi).abs()
        e_dact = e_phi + ax * e_pdf + U32 * (phi + ax * pdf)
        return e_act, e_dact
    if act == ACT_GELU_TANH:
        arg = TANH_K * x * (1.0 + TANH_A * x * x)
        t = torch.tanh(arg)
        dt = TANH_REL * t.abs() + (1.0 - t * t) * arg.abs() * 4 * U32
        du = TANH_K * (1.0 + TANH_DA * x * x)
        e_act = 0.5 * ax * dt + 3 * U32 * act_ref(x, act).abs()
        e_dact = (ax * t.abs() * du + 0.5) * dt + 4 * U32 * (ax * du + 1.0 + dact_ref(x, act).abs())
        return e_act, e_dact
    z = torch.zeros_like(x)
    return z, z


def bounds(ref, K, *, split=1, out_bf16=True):
    """Per-element bounds (e_out, e_aux) on |D - ref['out']| and |aux_out - ref['aux']| (module docstring).  split: the
    number of independently accumulated K chains (K-splits of ymp_gemm, K slices of the skinny kernels)."""
    absab, v, act = ref["absab"], ref["v"], ref["act"]
    al = abs(ref["alpha"])
    steps = -(-K // 16)
    e = (steps + split) * G22 * al * absab
    if ref["alpha"] != 1.0:
        e = e + U32 * (al * ref["acc"]).abs()
    if ref["bias"] is not None:
        e = e + U32 * v.abs()
    e_act, e_dact = act_err(v, act)
    if act:
        e_aux = L2 * e + e_dact + U * ref["aux"].abs()
    else:
        e_aux = e + U * v.abs()
    if ref["aux_in"] is not None:
        pre = v * ref["aux_in"].double()
        e_out = e * ref["aux_in"].double().abs() + U32 * pre.abs()
    elif act:
        pre = act_ref(v, act)
        e_out = L1 * e + e_act + U32 * pre.abs()
    else:
        pre, e_out = v, e
    if ref["residual"] is not None:
        pre = pre + ref["residual"]
        e_out = e_out + U32 * pre.abs()
    if ref["d0"] is not None:
        e_out = e_out + split * U32 * (ref["d0"].double().abs() + al * absab)
    if out_bf16:
        e_out = e_out + U * ref["out"].abs()
    return C * e_out + TINY, C * e_aux + TINY


def skinny_slices(N, K):
    """K slices per CTA of ymp_gemm_skinny / ymp_gemm_skinny_wide, as the host picks them (gemv.cu): up to 8 (4 for
    N > 4096), doubled while every slice keeps at least 128 columns.  Each slice is its own accumulation chain (the
    `split` of bounds())."""
    ks, ks_max = 1, 8 if N <= 4096 else 4
    while ks < ks_max and K // (2 * ks) >= 128:
        ks *= 2
    return ks


def layernorm_reference(y, gamma, beta, eps):
    """float64 LayerNorm of each row of y (the kernel's own fp32 result); returns (ln, z, rstd, mean|y|, sigma)."""
    y = y.double()
    mean = y.mean(-1, keepdim=True)
    var = ((y - mean) ** 2).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    z = (y - mean) * rstd
    return z * gamma.double() + beta.double(), z, rstd, y.abs().mean(-1, keepdim=True), var.sqrt()


def layernorm_stat_errors(y, eps):
    """(e_mean, e_rstd) per row, before the safety factor: the absolute error of the fp32 mean and the relative error of
    the fp32 rstd (module docstring).  The variance error is taken relative to var + eps, which is what rstd sees."""
    n = y.shape[-1]
    y = y.double()
    var = y.var(-1, unbiased=False, keepdim=True)
    e_mean = (n + 1) * U32 * y.abs().mean(-1, keepdim=True)
    e_var = ((n + 4) * U32 * var + e_mean ** 2) / (var + eps)
    return e_mean, 0.5 * e_var + 2.0 ** -22 + 2 * U32


def layernorm_bound(y, gamma, beta, eps, out_bf16=True):
    """Per-element bound on the error of a LayerNorm of the fp32 rows y against the float64 LN(y) (module docstring;
    an fp32 output rounds once, u32 |ln|, instead of u |ln|)."""
    ln, z, rstd, _, _ = layernorm_reference(y, gamma, beta, eps)
    e_mean, e_rstd = layernorm_stat_errors(y, eps)
    g = gamma.double().abs()
    e = g * (e_mean * rstd + z.abs() * (e_rstd + 2 * U32)) + U32 * (g * z).abs() + (U if out_bf16 else U32) * ln.abs()
    return C * e + TINY


# ---------------------------------------------------------------------------------- kernel arithmetic on the CPU
def _bf16(x):
    return x.to(torch.bfloat16).float()


def _fma(a, b, c):
    """fp32 fma: the product of two fp32 values is exact in float64, the sum is rounded (twice, harmlessly)."""
    return (a.double() * b.double() + c.double()).float()


def _ex2(x):
    """ex2.approx.ftz.f32 without its approximation error: 2^x rounded to fp32, results below 2^-126 flushed to 0."""
    r = torch.exp2(x.double()).float()
    return torch.where(r.abs() < 2.0 ** -126, torch.zeros_like(r), r)


def simulate_act(x, act, *, defect=None, tanh_sign=1.0):
    """(act(x), act'(x)) with the kernel's fp32 arithmetic (ptx.cuh: gelu_erf_both / gelu_tanh_both).
    defect "erf_old_clamp": x clamped to +-4.5 for Phi and for the pdf (the arithmetic before the tails were fixed:
    Phi and the pdf keep their values at -4.5 below it).  tanh_sign: tanh.approx's error is modelled as t (1 + tanh_sign TANH_REL)."""
    x = x.float()
    if act == ACT_GELU_ERF:
        if defect == "erf_old_clamp":
            xc = x.clamp(-CLAMP, CLAMP)
            xx = u = xc * xc
        else:
            xc = x.clamp(PHI_ZERO_X, CLAMP)
            xx = x * x
            u = xx.clamp(max=CLAMP * CLAMP)
        e = _ex2(_fma(xx, torch.tensor(EX2_C1), torch.tensor(EX2_C0)))
        q = torch.full_like(x, PHI_COEF[0])
        for c in PHI_COEF[1:]:
            q = _fma(q, u, torch.tensor(c))
        cdf = _fma(xc, q, torch.tensor(0.5))
        return x * cdf, _fma(x, e, cdf)
    if act == ACT_GELU_TANH:
        k = torch.tensor(TANH_K, dtype=torch.float32)
        arg = (k * x) * _fma(torch.tensor(TANH_A, dtype=torch.float32) * x, x, torch.tensor(1.0))
        t = (torch.tanh(arg.double()) * (1.0 + tanh_sign * TANH_REL)).float()
        du = k * _fma(torch.tensor(TANH_DA, dtype=torch.float32) * x, x, torch.tensor(1.0))
        hp = 0.5 * (1.0 + t)
        return x * hp, _fma(0.5 * x * (1.0 - t * t), du, hp)
    return x, torch.ones_like(x)


def simulate(a, b, *, alpha=1.0, bias=None, act=ACT_NONE, aux_in=None, residual=None, res_row_mod=0, d0=None,
             split=1, out_bf16=True, defect=None, tanh_sign=1.0, seed=0):
    """ymp_gemm's arithmetic in fp32 on the CPU: the product accumulated one 16-wide k step at a time (each step's
    block sum rounded to fp32 once, then added), `split` chains over 64-wide k-blocks as the host divides them, the
    epilogue in fp32 with bf16 stores, and an accumulating call's partials added to D0 in a shuffled order.
    Returns (D, aux_out).  defect: None | "drop_k16_mid" | "drop_k16_tail" (one k step skipped) | "bias_last_quad"
    (the last quad of every row reads the bias one column to the left) | "bias_twice" | "residual_row" (residual row
    off by one) | "aux_value" (aux_out holds act(v), not act'(v)) | "f32_as_bf16" (an fp32 output rounded to bf16) |
    "erf_old_clamp" (simulate_act)."""
    a, b = a.double(), b.double()
    M, K = a.shape
    N = b.shape[0]
    steps = -(-K // 16)
    kb_total = -(-K // 64)
    per = -(-kb_total // split)
    skip = {"drop_k16_mid": steps // 2, "drop_k16_tail": steps - 1}.get(defect, -1)
    parts = []
    for s0 in range(0, kb_total, per):
        acc = torch.zeros(M, N, dtype=torch.float32)
        for j in range(4 * s0, min(steps, 4 * (s0 + per))):
            if j != skip:
                acc = acc + (a[:, 16 * j:16 * j + 16] @ b[:, 16 * j:16 * j + 16].T).float()
        parts.append(acc)
    outs, aux = [], None
    for acc in parts:
        v = acc * alpha if alpha != 1.0 else acc
        if bias is not None:
            bb = bias.float()
            if defect == "bias_last_quad":
                last = (N - 1) // 4 * 4
                bb = bb.clone()
                bb[max(last, 1):] = bias.float()[max(last, 1) - 1:N - 1]
            v = v + bb
            if defect == "bias_twice":
                v = v + bb
        if aux_in is not None:
            o = v * aux_in.float()
        else:
            o, d = simulate_act(v, act, defect=defect, tanh_sign=tanh_sign)
            aux = _bf16(o if defect == "aux_value" else d) if act else _bf16(v)
        if residual is not None:
            r = res_rows(M, res_row_mod)
            if defect == "residual_row":
                r = (r + 1) % residual.shape[0]
            o = o + residual.float()[r]
        outs.append(o)
    if d0 is not None:  # accumulate: alpha only, no aux_out
        g = torch.Generator().manual_seed(seed)
        out, aux = d0.float().clone(), None
        for i in torch.randperm(len(outs), generator=g).tolist():
            out = out + outs[i]
    else:
        out = outs[0]
    if out_bf16 or defect == "f32_as_bf16":
        out = _bf16(out)
    return out, aux
