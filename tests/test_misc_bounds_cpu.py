"""The float64 references and error bounds of misc_bounds.py, checked without a GPU: the references equal torch (layer_norm,
cross_entropy and their autograd, clip_grad_norm_ + AdamW), a CPU simulation of each kernel's fp32 arithmetic in its
summation order stays inside the bounds at the host's grid for 132 SMs, and the same simulation with one injected defect
does not.  The argument checks of the entry points are exercised in a child process that sees no GPU."""
import json
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

import misc_bounds as MB

bf16 = torch.bfloat16
SMS = MB.SMS_H100
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _bf(x):
    return x.to(bf16).double()


def _ln_inputs(rows, D, seed, x_f32=False):
    """Rows with random offsets and scales, an outlier in the last 8-column vector of every row, a constant row and a
    near-constant row (whose variance is far below eps: only eps keeps its rstd finite and correct)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, D, generator=g) * (0.5 + 2 * torch.rand(rows, 1, generator=g)) + 3 * torch.randn(rows, 1, generator=g)
    x[:, D - 8 + (seed % 8)] += 16
    if rows > 2:
        x[1] = 1.5
        x[2] = 0.75 + 2.0 ** -8 * (torch.arange(D) % 2)
    x = x.float().double() if x_f32 else _bf(x)
    gamma = _bf(1 + 0.5 * torch.randn(D, generator=g))
    beta = _bf(0.5 * torch.randn(D, generator=g))
    return x, gamma, beta, g


# ---------------------------------------------------------------------------------- references against torch
def test_layernorm_reference_matches_torch():
    x, gamma, beta, g = _ln_inputs(37, 136, 1)
    dy, add = _bf(torch.randn(37, 136, generator=g)), _bf(torch.randn(37, 136, generator=g))
    xt, gt, bt = x.clone().requires_grad_(), gamma.clone().requires_grad_(), beta.clone().requires_grad_()
    y = F.layer_norm(xt, (136,), gt, bt, 1e-5)
    (y * dy).sum().backward()
    ry, mean, rstd = MB.ln_fwd_reference(x, gamma, beta, 1e-5)
    assert torch.allclose(ry, y.detach(), rtol=1e-12, atol=1e-12)
    d0, b0 = torch.randn(136, generator=g).double(), torch.randn(136, generator=g).double()
    r = MB.ln_bwd_reference(dy, x, gamma, mean, rstd, add=add, dgamma0=d0, dbeta0=b0)
    assert torch.allclose(r["dx"], xt.grad + add, rtol=1e-12, atol=1e-12)
    assert torch.allclose(r["dgamma"], d0 + gt.grad, rtol=1e-12, atol=1e-12)
    assert torch.allclose(r["dbeta"], b0 + bt.grad, rtol=1e-12, atol=1e-12)


def test_cross_entropy_reference_matches_torch():
    g = torch.Generator().manual_seed(2)
    x = _bf(torch.randn(29, 1003, generator=g) * 4)
    labels = torch.randint(0, 1003, (29,), generator=g)
    gr = torch.randn(29, generator=g).double()
    xt = x.clone().requires_grad_()
    loss = F.cross_entropy(xt, labels, reduction="none")
    (loss * gr).sum().backward()
    rl, lse = MB.ce_reference(x, labels)
    assert torch.allclose(rl, loss.detach(), rtol=1e-12, atol=1e-12)
    assert torch.allclose(lse, torch.logsumexp(x, -1), rtol=1e-12, atol=1e-12)
    assert torch.allclose(MB.ce_bwd_reference(x, labels, lse, gr)[0], xt.grad, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("step,wd,clip", [(1, 0.0, 0.5), (3, 0.1, 100.0), (7, 0.05, 0.0)])
def test_adamw_reference_matches_torch(step, wd, clip):
    """clip_grad_norm_ then one torch.optim.AdamW step in float64 (after step - 1 earlier steps that set the state)."""
    g = torch.Generator().manual_seed(step)
    n = 1000
    lr, b1, b2, eps = MB.f32(1e-3), MB.f32(0.9), MB.f32(0.999), MB.f32(1e-8)
    p = torch.nn.Parameter(torch.randn(n, generator=g).double())
    opt = torch.optim.AdamW([p], lr=lr, betas=(b1, b2), eps=eps, weight_decay=MB.f32(wd))
    for _ in range(step - 1):
        p.grad = torch.randn(n, generator=g).double()
        opt.step()
    st = opt.state[p]
    w0 = p.detach().clone()
    m0 = st["exp_avg"].clone() if st else torch.zeros(n, dtype=torch.float64)
    v0 = st["exp_avg_sq"].clone() if st else torch.zeros(n, dtype=torch.float64)
    grad = torch.randn(n, generator=g).double() * 0.1
    sumsq = float((grad ** 2).sum())
    p.grad = grad.clone()
    if clip > 0:
        torch.nn.utils.clip_grad_norm_([p], clip)
    opt.step()
    w1, m1, v1 = MB.adamw_reference(w0, grad, m0, v0, step=step, lr=lr, beta1=b1, beta2=b2, eps=eps, weight_decay=wd,
                                    max_norm=clip, sumsq=sumsq)
    assert torch.allclose(m1, opt.state[p]["exp_avg"], rtol=1e-12, atol=1e-15)
    assert torch.allclose(v1, opt.state[p]["exp_avg_sq"], rtol=1e-12, atol=1e-15)
    assert torch.allclose(w1, p.detach(), rtol=1e-12, atol=1e-15)


# ---------------------------------------------------------------------------------- simulation inside the bounds
def _ln_fwd_ratios(rows, D, y_bf16, seed, defect=None, x_f32=False):
    x, gamma, beta, _ = _ln_inputs(rows, D, seed, x_f32)
    y, mu, rs = MB.simulate_ln_fwd(x, gamma, beta, 1e-5, y_bf16=y_bf16, defect=defect)
    wy, wm, wr = MB.ln_fwd_reference(x, gamma, beta, 1e-5)
    ey, em, er = MB.ln_fwd_bounds(x, gamma, beta, 1e-5, y_bf16=y_bf16)
    return MB.worst_ratio(y, wy, ey), MB.worst_ratio(mu, wm, em), MB.worst_ratio(rs, wr, er)


@pytest.mark.parametrize("D", [8, 136, 768, 1408, 2560, 4096])
@pytest.mark.parametrize("y_bf16", [True, False])
def test_ln_fwd_simulation_inside_bounds(D, y_bf16):
    r = _ln_fwd_ratios(9, D, y_bf16, seed=D, x_f32=not y_bf16)
    assert max(r) <= 1, r


def test_ln_fwd_simulation_three_passes():
    """3 passes of the forward grid (8 rows x 8 sms x 8 per pass)."""
    rows = 3 * MB.ln_fwd_blocks(10 ** 9, SMS) * MB.LN_WARPS + 5
    r = _ln_fwd_ratios(rows, 136, True, seed=5)
    assert max(r) <= 1, r


@pytest.mark.parametrize("defect,D,y_bf16", [("var_d_minus_1", 768, False), ("no_eps", 136, True),
                                             ("skip_last_vec", 1408, True)])
def test_ln_fwd_defects_exceed_bounds(defect, D, y_bf16):
    assert max(_ln_fwd_ratios(9, D, y_bf16, seed=3, defect=defect)) > 1
    assert max(_ln_fwd_ratios(9, D, y_bf16, seed=3)) <= 1


def _ln_bwd_case(rows, D, seed, chained=False, drop=False):
    x, gamma, beta, g = _ln_inputs(rows, D, seed)
    dy = _bf(torch.randn(rows, D, generator=g))
    dy[-1] *= 8                                 # the last row (of the last pass) carries an outlier row
    add = _bf(torch.randn(rows, D, generator=g))
    d0, b0 = torch.randn(D, generator=g).float().double(), torch.randn(D, generator=g).float().double()
    keep = torch.rand(rows, D, generator=g) >= 0.1 if drop else None
    if chained:
        _, mean, rstd = MB.simulate_ln_fwd(x, gamma, beta, 1e-5)
        ref_stats = MB.ln_fwd_reference(x, gamma, beta, 1e-5)[1:]
        stat_err = MB.layernorm_stat_errors(x, 1e-5)
    else:
        _, m64, r64 = MB.ln_fwd_reference(x, gamma, beta, 1e-5)
        mean, rstd = m64.float(), r64.float()
        ref_stats, stat_err = (mean, rstd), None
    return dict(dy=dy, x=x, gamma=gamma, add=add, d0=d0, b0=b0, keep=keep, mean=mean, rstd=rstd, ref_stats=ref_stats,
                stat_err=stat_err)


def _ln_bwd_ratios(rows, D, seed, chained=False, drop=False, defect=None):
    c = _ln_bwd_case(rows, D, seed, chained, drop)
    blocks = MB.ln_bwd_blocks(rows, D, SMS)
    sim = MB.simulate_ln_bwd(c["dy"], c["x"], c["gamma"], c["mean"], c["rstd"], add=c["add"], dgamma0=c["d0"],
                             dbeta0=c["b0"], keep=c["keep"], p=0.1, blocks=blocks, seed=seed, defect=defect)
    ref = MB.ln_bwd_reference(c["dy"], c["x"], c["gamma"], *c["ref_stats"], add=c["add"], dgamma0=c["d0"],
                              dbeta0=c["b0"], keep=c["keep"], p=0.1)
    b = MB.ln_bwd_bounds(ref, blocks, c["stat_err"])
    return {k: MB.worst_ratio(sim[k], ref[k], b[k]) for k in sim}


@pytest.mark.parametrize("D", [8, 136, 768, 1024, 2048, 4096])
@pytest.mark.parametrize("chained", [False, True])
def test_ln_bwd_simulation_inside_bounds(D, chained):
    r = _ln_bwd_ratios(33, D, seed=D, chained=chained, drop=D == 768)
    assert max(r.values()) <= 1, r


def test_ln_bwd_simulation_three_passes():
    """dgamma / dbeta carried over 3 passes of the weight-gradient grid (3168 rows per pass at D <= 1024)."""
    rows = 3 * MB.ln_bwd_blocks(10 ** 9, 768, SMS) * MB.LN_WARPS + 7
    r = _ln_bwd_ratios(rows, 768, seed=11)
    assert max(r.values()) <= 1, r


@pytest.mark.parametrize("defect,D", [("drop_block_dgamma", 768), ("xh_s2_no_rs", 136)])
def test_ln_bwd_defects_exceed_bounds(defect, D):
    rows = 3 * MB.ln_bwd_blocks(10 ** 9, D, SMS) * MB.LN_WARPS + 7 if defect == "drop_block_dgamma" else 33
    assert max(_ln_bwd_ratios(rows, D, seed=4, defect=defect).values()) > 1


def _ce_case(rows, V, seed, sigma=4.0):
    """Logits with row scales up to sigma, one row of equal logits, and for odd rows the row max and the label in the
    ragged tail."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, V, generator=g) * (1 + (sigma - 1) * torch.rand(rows, 1, generator=g))
    labels = torch.randint(0, V, (rows,), generator=g)
    x[0] = 0.5
    if V % 8:
        x[1::2, V - 1] = x[1::2].max(-1).values + 3
        labels[1::2] = V - 1 - (torch.arange(1, rows, 2) % (V % 8))
    return _bf(x), labels


def _ce_ratios(rows, V, seed, defect=None):
    x, labels = _ce_case(rows, V, seed)
    loss, lse = MB.simulate_ce_fwd(x, labels, defect=defect)
    wl, wlse = MB.ce_reference(x, labels)
    el, else_, _ = MB.ce_fwd_bounds(x, labels)
    return MB.worst_ratio(loss, wl, el), MB.worst_ratio(lse, wlse, else_)


@pytest.mark.parametrize("V", [8, 1000, 1003, 51200])
def test_ce_simulation_inside_bounds(V):
    r = _ce_ratios(24 if V == 51200 else 64, V, seed=V)
    assert max(r) <= 1, r


@pytest.mark.parametrize("defect", ["skip_tail", "label_plus_1"])
def test_ce_defects_exceed_bounds(defect):
    assert max(_ce_ratios(16, 1003, seed=5, defect=defect)) > 1


def _colsum_ratio(R, Cc, seed, defect=None):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(R, Cc, generator=g)
    _, splits, rpb = MB.colsum_grid(R, Cc, SMS)
    last = torch.arange(1, splits + 1) * rpb - 1
    x[last.clamp(max=R - 1)] *= 64              # large values in the last row of each split
    x = _bf(x)
    out0 = torch.randn(Cc, generator=g).float().double() * 10
    got = MB.simulate_colsum(x, out0, SMS, seed=seed, defect=defect)
    return MB.worst_ratio(got, out0 + x.sum(0), MB.colsum_bound(x, out0, SMS))


@pytest.mark.parametrize("R,Cc", [(50208, 96), (2, 12040), (16, 1001), (777, 770), (3000, 8)])
def test_colsum_simulation_inside_bounds(R, Cc):
    assert _colsum_ratio(R, Cc, seed=R) <= 1


def test_colsum_defect_exceeds_bounds():
    assert _colsum_ratio(3000, 770, seed=1, defect="drop_last_row") > 1


def _sumsq_ratio(n, seed, defect=None):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, generator=g)
    x[n - n % 4:] = 1000.0                    # outliers in the n % 4 tail
    out0 = 5.0
    got = MB.simulate_sumsq(x, out0, SMS, seed=seed, defect=defect)
    return MB.worst_ratio(got, out0 + (x.double() ** 2).sum(), MB.sumsq_bound(x, out0, SMS))


@pytest.mark.parametrize("n", [1, 3, 4097, 3 * 1081344 + 3])
def test_sumsq_simulation_inside_bounds(n):
    """3 * 1081344 + 3: three passes of the 8 sms x 256-thread x 4-element grid and a tail."""
    assert _sumsq_ratio(n, seed=n) <= 1


def test_sumsq_defect_exceeds_bounds():
    assert _sumsq_ratio(4097, seed=2, defect="no_tail") > 1


def _adamw_ratios(step, clip, wd, defect=None):
    g = torch.Generator().manual_seed(step)
    n = 20000
    w = torch.randn(n, generator=g).float().double()
    grad = (torch.randn(n, generator=g) * 10 ** (4 * torch.rand(n, generator=g) - 3)).float().double()
    grad[::97] = 0
    m = (torch.randn(n, generator=g) * 0.01).float().double() if step > 1 else torch.zeros(n, dtype=torch.float64)
    v = (torch.rand(n, generator=g) * 1e-4).float().double() if step > 1 else torch.zeros(n, dtype=torch.float64)
    sumsq = MB.f32(float((grad ** 2).sum()))
    kw = dict(step=step, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=wd, grad_scale=0.5, max_norm=clip,
              sumsq=sumsq)
    sw, sm, sv, sp = MB.simulate_adamw(w, grad, m, v, defect=defect, **kw)
    rw, rm, rv = MB.adamw_reference(w, grad, m, v, **kw)
    ew, em, ev = MB.adamw_bounds(w, grad, m, v, **kw)
    assert torch.equal(sp, sw.to(bf16))
    return MB.worst_ratio(sw, rw, ew), MB.worst_ratio(sm, rm, em), MB.worst_ratio(sv, rv, ev)


@pytest.mark.parametrize("step,clip,wd", [(1, 1.0, 0.0), (2, 1e6, 0.1), (50, 0.0, 0.05), (1000, 0.3, 0.1)])
def test_adamw_simulation_inside_bounds(step, clip, wd):
    r = _adamw_ratios(step, clip, wd)
    assert max(r) <= 1, r


def test_adamw_defect_exceeds_bounds():
    assert max(_adamw_ratios(1, 1.0, 0.1, defect="bc2_not_sqrt")) > 1


# ---------------------------------------------------------------------------------- argument checks
_ARGCHECK = r"""
import ctypes as C, json
from ymp import lib as L

A, BAD = 0x10000, 0x10002        # fake device addresses: 16-byte aligned, and not
res = []

def run(fn, st, what):
    rc = fn(C.byref(st), None)
    res.append([what, rc, L.lib.ymp_last_error().decode()])

def lnb(**kw):
    a = L.LayerNormBwdArgs()
    a.dy = a.x = a.gamma = a.mean = a.rstd = a.dx = A
    a.rows, a.D, a.ldx, a.lddy, a.ldadd = 4, 64, 64, 64, 64
    for k, v in kw.items():
        setattr(a, k, v)
    return a

for f in ("dy", "x", "gamma", "dx"):
    run(L._ln_bwd, lnb(**{f: BAD}), "ln_bwd misaligned " + f)
run(L._ln_bwd, lnb(add=BAD), "ln_bwd misaligned add")
run(L._ln_bwd, lnb(ldx=56), "ln_bwd ldx < D")
run(L._ln_bwd, lnb(lddy=56), "ln_bwd lddy < D")
run(L._ln_bwd, lnb(add=A, ldadd=56), "ln_bwd ldadd < D")

def grp(**kw):
    a = L.GroupArgs()
    a.in_, a.out, a.G, a.T, a.C, a.ld_in, a.ld_out, a.scale = A, A, 2, 3, 64, 64, 64, 1.0
    for k, v in kw.items():
        setattr(a, k, v)
    return a

for bc in (0, 1):
    run(L._group, grp(in_=BAD, broadcast=bc), "group misaligned in")
    run(L._group, grp(out=BAD, broadcast=bc), "group misaligned out")
    run(L._group, grp(ld_in=56, broadcast=bc), "group ld_in < C")
    run(L._group, grp(ld_out=56, broadcast=bc), "group ld_out < C")

def emb(**kw):
    a = L.EmbedArgs()
    a.ids, a.table, a.pos, a.out = A, A, A, A
    a.B, a.L, a.S, a.row_offset, a.hidden, a.vocab, a.ldo = 2, 3, 5, 1, 64, 100, 64
    for k, v in kw.items():
        setattr(a, k, v)
    return a

for f in ("table", "pos", "out"):
    run(L._embed, emb(**{f: BAD}), "embed misaligned " + f)
run(L._embed, emb(vocab=0), "embed vocab 0")
print(json.dumps(res))
"""

ARG_MESSAGES = {"ln_bwd misaligned": "ymp_layernorm_bwd: 16-byte alignment required",
                "ln_bwd ld": "ymp_layernorm_bwd: bad ld",
                "group misaligned": "ymp_group_reduce: 16-byte alignment required",
                "group ld": "ymp_group_reduce: bad ld",
                "embed misaligned": "ymp_embed_gather: 16-byte alignment required",
                "embed vocab": "ymp_embed_gather: vocab must be positive"}


def test_argument_checks_reject_misaligned_and_short_strides():
    """ymp_layernorm_bwd, ymp_group_reduce and ymp_embed_gather read and write 16-byte vectors: a misaligned pointer, a
    row stride below the width or an empty vocabulary is rejected with YMP_EINVAL before anything is launched.  Run in
    a child process that sees no GPU, so that a missing check cannot reach a device with the fake pointers."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="", PYTHONPATH=os.pathsep.join([os.path.join(ROOT, "youku-mplug_b200"), ROOT]))
    p = subprocess.run([sys.executable, "-c", _ARGCHECK], env=env, capture_output=True, text=True, timeout=120)
    assert p.returncode == 0, p.stderr
    res = json.loads(p.stdout.strip().splitlines()[-1])
    assert len(res) == 20
    for what, rc, msg in res:
        want = next(m for k, m in ARG_MESSAGES.items() if what.startswith(k))
        assert rc == -1 and msg == want, (what, rc, msg)
