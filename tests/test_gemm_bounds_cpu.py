"""The float64 GEMM-epilogue reference and its error bounds (gemm_bounds.py), checked without a GPU: the reference
equals torch.nn.functional and autograd, the constants the bounds rest on hold, a CPU simulation of the kernel
arithmetic stays inside the bounds, and the same simulation with one injected defect does not."""
import pytest
import torch
import torch.nn.functional as F

import gemm_bounds as GB

bf16 = torch.bfloat16


def _bf(x):
    return x.to(bf16).double()


def _operands(M, N, K, sigma=1.0, seed=0):
    g = torch.Generator().manual_seed(seed)
    a = _bf(torch.randn(M, K, generator=g) * sigma)
    b = _bf(torch.randn(N, K, generator=g) * sigma)
    return a, b, g


def _bf16_values(limit=16.0, tails=(20.0, 50.0, 100.0)):
    """Every finite bf16 value with |x| <= limit, and +-tails."""
    v = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(bf16).double()
    v = v[torch.isfinite(v) & (v.abs() <= limit)]
    t = torch.tensor(tails, dtype=torch.float64)
    return torch.cat([v, t, -t])


@pytest.mark.parametrize("act", [GB.ACT_NONE, GB.ACT_GELU_ERF, GB.ACT_GELU_TANH])
def test_reference_matches_functional(act):
    """linear + gelu / gelu(tanh) and their autograd derivatives, the multiplier, residual broadcast, alpha and
    accumulation, to 1e-12."""
    M, N, K = 37, 29, 70
    a, b, g = _operands(M, N, K, seed=1)
    bias = _bf(torch.randn(N, generator=g))
    ref = GB.reference(a, b, bias=bias, act=act)
    v = F.linear(a, b, bias).requires_grad_()
    fn = {GB.ACT_NONE: lambda x: x, GB.ACT_GELU_ERF: F.gelu, GB.ACT_GELU_TANH: lambda x: F.gelu(x, approximate="tanh")}[act]
    y = fn(v)
    y.sum().backward()
    assert torch.allclose(ref["v"], v.detach(), rtol=1e-12, atol=1e-12)
    assert torch.allclose(ref["out"], y.detach(), rtol=1e-12, atol=1e-12)
    want_aux = v.grad if act else v.detach()
    assert torch.allclose(ref["aux"], want_aux, rtol=1e-12, atol=1e-12)
    # multiplier, residual table broadcast by row, alpha, accumulation into D0
    mul, res, d0 = _bf(torch.randn(M, N, generator=g)), torch.randn(5, N, generator=g).double(), torch.randn(M, N, generator=g).double()
    r = GB.reference(a, b, alpha=0.5, bias=bias, act=act, aux_in=mul, residual=res, res_row_mod=5, d0=d0)
    want = d0 + (0.5 * F.linear(a, b) + bias) * mul + res[torch.arange(M) % 5]
    assert torch.allclose(r["out"], want, rtol=1e-12, atol=1e-12)
    assert torch.equal(GB.store_rows(6, 2, 5), torch.tensor([0, 1, 5, 6, 10, 11]))


def test_bound_constants():
    """PHI_POLY_ERR bounds the kernel's Phi polynomial (exact arithmetic, fp32 coefficients) on |x| <= 4.5 and on to
    PHI_ZERO_X; L1 and L2 bound |gelu'| and |gelu''| of both forms."""
    x = torch.cat([torch.linspace(-GB.CLAMP, GB.CLAMP, 2_000_001, dtype=torch.float64),
                   torch.linspace(GB.PHI_ZERO_X, -GB.CLAMP, 101, dtype=torch.float64)])
    assert float((GB.phi_poly(x) - GB.ndtr(x)).abs().max()) <= GB.PHI_POLY_ERR
    g = torch.linspace(-40.0, 40.0, 800_001, dtype=torch.float64)
    for act in (GB.ACT_GELU_ERF, GB.ACT_GELU_TANH):
        gg = g.clone().requires_grad_()
        d = GB.dact_ref(gg, act)
        d.sum().backward()
        assert float(d.detach().abs().max()) <= GB.L1
        assert float(gg.grad.abs().max()) <= GB.L2
        # the derivative formula of the reference is the derivative of its activation
        ga = g[::97].clone().requires_grad_()
        GB.act_ref(ga, act).sum().backward()
        assert torch.allclose(ga.grad, GB.dact_ref(g[::97], act), rtol=1e-12, atol=1e-12)


def _act_ratios(x, act, defect=None, tanh_sign=1.0):
    a, d = GB.simulate_act(x, act, defect=defect, tanh_sign=tanh_sign)
    want, dwant = GB.act_ref(x, act), GB.dact_ref(x, act)
    e_act, e_dact = GB.act_err(x, act)
    r_act = GB.worst_ratio(a, want, GB.C * (e_act + GB.U32 * want.abs()) + GB.TINY)
    r_aux = GB.worst_ratio(d.to(bf16).float(), dwant, GB.C * (e_dact + GB.U * dwant.abs()) + GB.TINY)
    return r_act, r_aux


@pytest.mark.parametrize("act,tanh_sign", [(GB.ACT_GELU_ERF, 1.0), (GB.ACT_GELU_TANH, 1.0), (GB.ACT_GELU_TANH, -1.0)])
def test_activation_simulation_inside_bounds(act, tanh_sign):
    """Every bf16 value with |x| <= 16 and +-20, +-50, +-100 through the kernel's activation arithmetic: act(x) in
    fp32 and act'(x) stored in bf16 stay inside the activation bounds (part B of the GPU suite checks the device)."""
    r_act, r_aux = _act_ratios(_bf16_values(), act, tanh_sign=tanh_sign)
    assert r_act <= 1 and r_aux <= 1, (r_act, r_aux)


def test_phi_floor():
    """Below PHI_ZERO_X the kernel's fp32 Phi (0.5 + PHI_ZERO_X Q(4.5^2), Horner in fp32) is within PHI_FLOOR of 0, and
    PHI_ZERO_X lies within 1e-5 below -4.5 (no bf16 value lies between them)."""
    x = torch.tensor([GB.PHI_ZERO_X, -5.0, -100.0], dtype=torch.float32)
    cdf = GB.simulate_act(x, GB.ACT_GELU_ERF)[0] / x
    assert float(cdf.abs().max()) <= GB.PHI_FLOOR
    assert -4.5 - 1e-5 < GB.PHI_ZERO_X < -4.5


def test_old_erf_tails_exceed_bounds():
    """Phi and the pdf clamped at -4.5 (the erf-GELU before its tails were fixed: gelu(-10) = -9e-6, gelu'(-10) =
    -1.6e-4) are outside the bounds at x = -10, for gelu and for gelu'; the fixed arithmetic is inside."""
    x = torch.tensor([-10.0], dtype=torch.float64)
    r_act, r_aux = _act_ratios(x, GB.ACT_GELU_ERF, defect="erf_old_clamp")
    assert r_act > 1 and r_aux > 1, (r_act, r_aux)
    assert max(_act_ratios(x, GB.ACT_GELU_ERF)) <= 1


# (name, epilogue keyword arguments of reference / simulate, fp32 output)
EPILOGUES = [
    ("plain_bf16", dict(), False),
    ("plain_f32", dict(), True),
    ("alpha_bias", dict(alpha=0.5, bias=True), False),
    ("erf_aux", dict(bias=True, act=GB.ACT_GELU_ERF), False),
    ("tanh_aux", dict(bias=True, act=GB.ACT_GELU_TANH), False),
    ("aux_in", dict(aux_in=True), False),
    ("residual_f32_rowmod", dict(bias=True, residual=torch.float32, res_row_mod=7), True),
    ("residual_bf16", dict(bias=True, residual=bf16), False),
    ("accumulate_split3", dict(d0=True, split=3), True),
]


def _case(M, N, K, sigma, kw, seed):
    a, b, g = _operands(M, N, K, sigma, seed)
    kw = dict(kw)
    split = kw.pop("split", 1)
    if kw.pop("bias", False):
        kw["bias"] = _bf(torch.randn(N, generator=g))
    if kw.pop("aux_in", False):
        kw["aux_in"] = _bf(torch.randn(M, N, generator=g))
    if "residual" in kw:
        rows = kw.get("res_row_mod") or M
        kw["residual"] = (torch.randn(rows, N, generator=g) * 3).to(kw["residual"]).double()
    if kw.pop("d0", False):
        kw["d0"] = torch.randn(M, N, generator=g).float().double()
    return a, b, kw, split


def _ratios(M, N, K, sigma, kw, out_f32, seed=0, defect=None, sim_kw=None):
    a, b, kw, split = _case(M, N, K, sigma, kw, seed)
    ref = GB.reference(a, b, **kw)
    e_out, e_aux = GB.bounds(ref, K, split=split, out_bf16=not out_f32)
    out, aux = GB.simulate(a, b, **kw, split=split, out_bf16=not out_f32, defect=defect, seed=seed, **(sim_kw or {}))
    r_aux = GB.worst_ratio(aux, ref["aux"], e_aux) if aux is not None else 0.0
    return GB.worst_ratio(out, ref["out"], e_out), r_aux


@pytest.mark.parametrize("name,kw,out_f32", EPILOGUES, ids=[e[0] for e in EPILOGUES])
@pytest.mark.parametrize("sigma", [0.25, 1.0, 4.0])
@pytest.mark.parametrize("K", [8, 40, 200, 1032, 8192])
def test_simulation_inside_bounds(name, kw, out_f32, sigma, K):
    """The kernel arithmetic, simulated on the CPU, stays inside the bounds for every epilogue, at K from one partial
    k step to 8192 and operands from sigma 0.25 to 4 (pre-activations deep into both GELU tails)."""
    r_out, r_aux = _ratios(24, 43, K, sigma, kw, out_f32, seed=K)
    assert r_out <= 1 and r_aux <= 1, (r_out, r_aux)


@pytest.mark.parametrize("defect,name,K", [
    ("drop_k16_mid", "plain_f32", 200), ("drop_k16_tail", "plain_f32", 200), ("drop_k16_tail", "plain_f32", 8192),
    ("drop_k16_mid", "plain_bf16", 1032),
    ("bias_last_quad", "alpha_bias", 64), ("bias_twice", "alpha_bias", 64),
    ("residual_row", "residual_f32_rowmod", 64), ("residual_row", "residual_bf16", 64),
    ("aux_value", "erf_aux", 64), ("aux_value", "tanh_aux", 64),
    ("f32_as_bf16", "plain_f32", 64), ("f32_as_bf16", "accumulate_split3", 1032)])
def test_simulated_defects_exceed_bounds(defect, name, K):
    """A skipped k step (in the middle, at the K tail), the bias read one column off in the last (partial) quad or
    added twice, the residual row off by one, aux_out holding act(v) instead of act'(v), and an fp32 output rounded to
    bf16 each take the simulation outside the bounds (N = 43: the last quad holds three columns)."""
    kw, out_f32 = {e[0]: (e[1], e[2]) for e in EPILOGUES}[name]
    r_out, r_aux = _ratios(24, 43, K, 1.0, kw, out_f32, seed=7, defect=defect)
    assert max(r_out, r_aux) > 1, (r_out, r_aux)
    assert max(_ratios(24, 43, K, 1.0, kw, out_f32, seed=7)) <= 1
