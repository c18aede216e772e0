"""LayerNorm, cross-entropy, colsum, group reduce / broadcast, sumsq and AdamW element by element against the float64
references of misc_bounds.py with their derived per-element bounds; im2col, the embedding gather and ymp_dropout bit for
bit.

Inputs sit in wider buffers whose columns past the width, rows around the view and rows that no in_rows entry names hold
NaN (a read of any of them turns an output NaN); outputs go into buffers pre-filled with a NaN bit pattern and padded
to ld > width: every addressed element must come back finite and within its bound (or bit-exact), every other element
keep its pattern.  Inputs carry outliers where a dropped piece of work shows: the last 8-column vector of a row, the
last row of a grid pass, the row max and the label in the cross-entropy's ragged tail, the last row of each colsum
split, the n % 4 tail of sumsq.  Row and element counts reach 3 passes of each grid-stride loop on the device's SMs.
Set YMP_MISC_BOUNDS_REPORT=<file> to write the largest err / bound per kernel and tensor as JSON.
"""
import json
import math
import os

import numpy as np
import pytest
import torch

import misc_bounds as MB
from oracle import philox
from test_gemm_bounds_gpu import ROW0, SENT16, SENT32, Out, _in, _in_vec

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
f32 = torch.float32
EPS = 1e-5
SEED, OFFSET = 0x1234567812345, 7
RATIOS = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    path = os.environ.get("YMP_MISC_BOUNDS_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump(RATIOS, f, indent=1, sort_keys=True)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _check(key, got, want, bound):
    r = MB.worst_ratio(got, want, bound)
    RATIOS[key] = max(RATIOS.get(key, 0.0), r)
    if r > 1:
        err = ((got.double() - want.double()).abs() / bound).nan_to_num(math.inf)
        idx = int(err.flatten().argmax())
        raise AssertionError(f"{key}: err / bound = {r:.3g} at flat index {idx}: got {got.flatten()[idx].item():.8g}, "
                             f"want {want.flatten()[idx].item():.8g}, bound {bound.flatten()[idx].item():.3g}")


def _bits(t):
    return t.view({bf16: torch.int16, f32: torch.int32, torch.float16: torch.int16}[t.dtype])


def _same_bits(what, got, want):
    bad = _bits(got) != _bits(want.to(got.dtype))
    assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements differ, first at {bad.nonzero()[0].tolist()}"


def _rng(dev):
    return torch.tensor([SEED, OFFSET], dtype=torch.int64, device=dev)


def _keep(rows, cols, site, p, dev):
    return torch.from_numpy(philox.keep_mask(SEED, OFFSET, site, np.asarray(rows), cols, p)).to(dev)


# ---------------------------------------------------------------------------------- LayerNorm
def _ln_x(g, rows, D, dtype):
    """Row offsets and scales, an outlier in the last 8-column vector of every row and of the last row, a constant row
    and a near-constant row (variance far below eps)."""
    x = torch.randn(rows, D, device=g.device, generator=g) * (0.5 + 2 * torch.rand(rows, 1, device=g.device, generator=g)) \
        + 3 * torch.randn(rows, 1, device=g.device, generator=g)
    x[:, D - 8 + rows % 8] += 16
    x[-1] *= 4
    if rows > 2:
        x[1] = 1.5
        x[2] = 0.75 + 2.0 ** -8 * (torch.arange(D, device=g.device) % 2)
    return x.to(dtype)


def _affine(g, D):
    gamma = (1 + 0.5 * torch.randn(D, device=g.device, generator=g)).to(bf16)
    beta = (0.5 * torch.randn(D, device=g.device, generator=g)).to(bf16)
    return gamma, beta


def _ln_fwd_check(key, x, gamma, beta, y, mean, rstd, y_bf16):
    wy, wm, wr = MB.ln_fwd_reference(x, gamma, beta, EPS)
    ey, em, er = MB.ln_fwd_bounds(x, gamma, beta, EPS, y_bf16=y_bf16)
    _check(f"{key}.y_{'bf16' if y_bf16 else 'f32'}", y, wy, ey)
    _check(f"{key}.mean", mean, wm, em)
    _check(f"{key}.rstd", rstd, wr, er)


LN_D = [8, 136, 768, 1024, 1408, 2048, 2560, 4096]


@pytest.mark.parametrize("D", LN_D)
def test_layernorm_fwd(cuda, D):
    """x bf16 / fp32 -> y bf16 / fp32 at 1, 7 and 9 rows (VPL 3 / 8 / 16 instantiations, idle lanes at D < 256)."""
    from ymp import ops
    g = torch.Generator(device=cuda).manual_seed(D)
    for xdt in (bf16, f32):
        for ydt in (bf16, f32):
            for rows in (1, 7, 9):
                x = _ln_x(g, rows, D, xdt)
                gamma, beta = _affine(g, D)
                y = Out(cuda, rows, D, ydt)
                _, mean, rstd = ops.layernorm_fwd(_in(x), _in_vec(gamma), _in_vec(beta), EPS, out=y.view)
                _ln_fwd_check("ln_fwd", x, gamma, beta, y.check(f"D={D} {xdt}->{ydt} rows={rows}"), mean, rstd,
                              ydt == bf16)


def test_layernorm_fwd_three_passes(cuda):
    """50208 x 768 (the ViT's rows): at least 3 passes of the 8 x 8 sms-row grid on the device."""
    from ymp import ops
    rows, D = 50208, 768
    assert rows >= 3 * MB.ln_fwd_blocks(10 ** 9, _sms()) * MB.LN_WARPS
    g = torch.Generator(device=cuda).manual_seed(1)
    x = _ln_x(g, rows, D, bf16)
    gamma, beta = _affine(g, D)
    y = Out(cuda, rows, D, bf16)
    _, mean, rstd = ops.layernorm_fwd(_in(x), gamma, beta, EPS, out=y.view)
    _ln_fwd_check("ln_fwd", x, gamma, beta, y.check("50208 x 768"), mean, rstd, True)


def _key_rows(n, per, pad, dev):
    """The abstractor's key pattern: blocks of `per` rows, each followed by `pad` padding slots (-1)."""
    r = []
    for b in range(0, n, per):
        r += list(range(b, min(n, b + per))) + [-1] * pad
    return torch.tensor(r, dtype=torch.int32, device=dev)


@pytest.mark.parametrize("D", [136, 1408])
@pytest.mark.parametrize("pattern", ["keys", "subset"])
def test_layernorm_fwd_in_rows(cuda, D, pattern):
    """Output row r normalises x row in_rows[r]; -1 slots give bf16 zero rows with mean = rstd = 0, and x rows that no
    entry names hold NaN."""
    from ymp import ops
    g = torch.Generator(device=cuda).manual_seed(D + len(pattern))
    n = 40
    if pattern == "keys":
        rows = _key_rows(n, 9, 3, cuda)
    else:
        rows = torch.randperm(n, device=cuda, generator=g)[:23].to(torch.int32)
    for xdt in (bf16, f32):
        x = _ln_x(g, n, D, xdt)
        named = torch.zeros(n, dtype=torch.bool, device=cuda)
        named[rows[rows >= 0].long()] = True
        xp = x.clone()
        xp[~named] = math.nan
        gamma, beta = _affine(g, D)
        y = Out(cuda, rows.numel(), D, bf16)
        _, mean, rstd = ops.layernorm_fwd(_in(xp), gamma, beta, EPS, out=y.view, in_rows=rows)
        got = y.check(f"in_rows {pattern}")
        v = rows >= 0
        _ln_fwd_check("ln_fwd.in_rows", x[rows[v].long()], gamma, beta, got[v], mean[v], rstd[v], True)
        assert torch.equal(_bits(got[~v]), torch.zeros_like(_bits(got[~v]))), "padding slots must be zero rows"
        assert bool((mean[~v] == 0).all()) and bool((rstd[~v] == 0).all())


def _ln_bwd_run(cuda, g, key, rows, D, xdt, *, add=False, wgrad=False, drop=False, chained=False, int_dy=False,
                in_rows=None, nx=None):
    from ymp import ops
    nx = nx or rows
    x = _ln_x(g, nx, D, xdt)
    gamma, beta = _affine(g, D)
    irows = torch.arange(rows, device=cuda) if in_rows is None else in_rows.long()
    valid = irows >= 0
    xr = torch.zeros(rows, D, device=cuda, dtype=xdt)
    xr[valid] = x[irows[valid]]
    if int_dy:
        dy = torch.randint(-2, 3, (rows, D), device=cuda, generator=g).to(bf16)
    else:
        dy = torch.randn(rows, D, device=cuda, generator=g).to(bf16)
        dy[-1] *= 8
    xp = x.clone()
    if in_rows is not None:
        named = torch.zeros(nx, dtype=torch.bool, device=cuda)
        named[irows[valid]] = True
        xp[~named] = math.nan
    if chained:
        _, mean, rstd = ops.layernorm_fwd(_in(xp), gamma, beta, EPS, in_rows=in_rows, rows=rows,
                                          out=torch.empty(rows, D, device=cuda, dtype=bf16))
        _, m64, r64 = MB.ln_fwd_reference(xr, gamma, beta, EPS)
        stat_err = MB.layernorm_stat_errors(xr, EPS)
    else:
        _, m64, r64 = MB.ln_fwd_reference(xr, gamma, beta, EPS)
        mean, rstd = m64.float(), r64.float()
        m64, r64, stat_err = mean, rstd, None
    kw = {}
    addv = None
    if add:
        addv = torch.randn(nx, D, device=cuda, generator=g).to(bf16)
        kw["add"] = _in(addv)
    d0 = b0 = None
    if wgrad:
        if int_dy:
            d0 = torch.randint(-50, 50, (D,), device=cuda, generator=g).float()
        else:
            d0 = torch.randn(D, device=cuda, generator=g) * 10
        b0 = d0.flip(0).clone()
        dg, db = Out(cuda, 1, D, f32, init=d0[None]), Out(cuda, 1, D, f32, init=b0[None])
        kw["dgamma"], kw["dbeta"] = dg.view[0], db.view[0]
    dx = Out(cuda, nx, D, bf16)
    p, site = 0.1, 7
    dxd = None
    if drop:
        dxd = Out(cuda, nx, D, bf16)
        kw["drop"], kw["dx_drop"] = ops.Drop(_rng(cuda), site, p), dxd.view
    ops.layernorm_bwd(_in(dy), _in(xp), _in_vec(gamma), mean, rstd, in_rows=in_rows, dx=dx.view, **kw)
    rows_sel = irows[valid]
    keep = _keep(rows_sel.cpu().numpy(), D, site, p, cuda) if drop else None
    ref = MB.ln_bwd_reference(dy[valid], xr[valid], gamma, m64[valid], r64[valid],
                              add=addv[rows_sel] if add else None, keep=keep, p=p,
                              dgamma0=d0, dbeta0=b0)
    blocks = MB.ln_bwd_blocks(rows, D, _sms(), wgrad)
    se = None if stat_err is None else (stat_err[0][valid], stat_err[1][valid])
    b = MB.ln_bwd_bounds(ref, blocks, se, rows=rows)
    # dx rows are x rows: rows_sel in output-row order (Out.check returns them in that order)
    _check("ln_bwd.dx" + (".chained" if chained else ""), dx.check(key + " dx", rows_sel), ref["dx"], b["dx"])
    if drop:
        _check("ln_bwd.dx_drop", dxd.check(key + " dx_drop", rows_sel), ref["dx_drop"], b["dx_drop"])
    if wgrad:
        _check("ln_bwd.dgamma" + (".chained" if chained else ""), dg.check(key + " dgamma")[0], ref["dgamma"], b["dgamma"])
        gb = db.check(key + " dbeta")[0]
        if int_dy:
            _same_bits(key + " dbeta (integer dy)", gb, ref["dbeta"])
        _check("ln_bwd.dbeta", gb, ref["dbeta"], b["dbeta"])


# (add, trainable affine, dx_drop, chained to the kernel's own statistics)
LN_BWD_CASES = [(False, False, False, False), (True, True, False, False), (True, False, True, False),
                (False, True, False, True), (True, True, True, True)]


@pytest.mark.parametrize("D", LN_D)
def test_layernorm_bwd(cuda, D):
    """Every combination row of LN_BWD_CASES with x bf16 and fp32, at 9 rows (and 7 for the plain case)."""
    g = torch.Generator(device=cuda).manual_seed(100 + D)
    for xdt in (bf16, f32):
        for add, wgrad, drop, chained in LN_BWD_CASES:
            for rows in ((7, 9) if not (add or wgrad or drop or chained) else (9,)):
                _ln_bwd_run(cuda, g, f"D={D} {xdt} add={add} wgrad={wgrad} drop={drop} chained={chained} rows={rows}",
                            rows, D, xdt, add=add, wgrad=wgrad, drop=drop, chained=chained)


@pytest.mark.parametrize("D,xdt", [(768, bf16), (2048, f32)])
def test_layernorm_bwd_three_passes(cuda, D, xdt):
    """dgamma / dbeta carried over 3 passes of the weight-gradient grid (8 x 3 or 2 x sms rows per pass), then the same
    with integer dy, where dbeta must be bit-exact."""
    g = torch.Generator(device=cuda).manual_seed(D)
    rows = 3 * MB.ln_bwd_blocks(10 ** 9, D, _sms()) * MB.LN_WARPS + 7
    _ln_bwd_run(cuda, g, f"3 passes D={D}", rows, D, xdt, add=True, wgrad=True, chained=True)
    _ln_bwd_run(cuda, g, f"3 passes D={D} integer dy", rows, D, xdt, wgrad=True, int_dy=True)


def test_layernorm_bwd_in_rows(cuda):
    """The backward of a gathered forward: dx rows in_rows[r] only, -1 slots skipped, rows never named untouched."""
    g = torch.Generator(device=cuda).manual_seed(5)
    rows = _key_rows(40, 9, 3, cuda)
    for drop in (False, True):
        _ln_bwd_run(cuda, g, f"in_rows drop={drop}", rows.numel(), 1408, bf16, add=True, wgrad=True, drop=drop,
                    in_rows=rows, nx=40)


# ---------------------------------------------------------------------------------- cross-entropy
def _ce_logits(g, rows, V):
    """Row scales sigma from 1 to 8, a row of equal logits, and in odd rows the row max and the label in the ragged
    tail (V % 8 != 0)."""
    dev = g.device
    x = torch.randn(rows, V, device=dev, generator=g) * (1 + 7 * torch.rand(rows, 1, device=dev, generator=g))
    labels = torch.randint(0, V, (rows,), device=dev, generator=g)
    x[0] = 0.5
    if V % 8:
        x[1::2, V - 1] = x[1::2].max(-1).values + 3
        labels[1::2] = V - 1 - (torch.arange(1, rows, 2, device=dev) % (V % 8))
    return x.to(bf16), labels


# (V, rows, logits as a view with ld > V)
CE_CASES = [(8, 7, True), (1000, 1, False), (1000, 300, True), (1003, 257, True), (1003, 2000, True),
            (51200, 2048, True)]


@pytest.mark.parametrize("V,rows,padded", CE_CASES)
def test_cross_entropy(cuda, V, rows, padded):
    """loss and lse against float64 (absolute bounds), then the backward from the reference lse out of place and chained
    to the kernel's own lse in place; rows with g = 0 are exact zeros, columns past V untouched."""
    from ymp import ops
    g = torch.Generator(device=cuda).manual_seed(V + rows)
    x, labels = _ce_logits(g, rows, V)
    xin = _in(x) if padded else x.clone()
    loss, lse = ops.ce_fwd(xin, labels)
    el, else_, e_lse = MB.ce_fwd_bounds(x, labels)
    wl, wlse = MB.ce_reference(x, labels)
    _check("ce_fwd.loss", loss, wl, el)
    _check("ce_fwd.lse", lse, wlse, else_)
    gr = torch.randn(rows, device=cuda, generator=g)
    gr[::5] = 0
    zero = gr == 0
    # out of place, from the reference lse rounded to fp32
    l32 = wlse.float()
    xin2 = _in(x)
    d = Out(cuda, rows, V, bf16)
    ops.ce_bwd(xin2, labels, l32, gr, dlogits=d.view)
    want, bound = MB.ce_bwd_bounds(x, labels, l32, gr)
    got = d.check(f"ce_bwd V={V}")
    _check("ce_bwd.dlogits", got, want, bound)
    assert torch.equal(_bits(got[zero]), torch.zeros_like(_bits(got[zero])))
    assert torch.equal(_bits(xin2), _bits(x)), "out-of-place backward wrote its input"
    # in place, chained to the kernel's lse
    buf = _in(x)
    ops.ce_bwd(buf, labels, lse, gr)
    want, bound = MB.ce_bwd_bounds(x, labels, lse, gr, e_l=e_lse)
    _check("ce_bwd.dlogits.chained", buf, want, bound)
    assert torch.equal(_bits(buf[zero]), torch.zeros_like(_bits(buf[zero])))
    full = buf.as_strided((ROW0 + rows + 3, buf.stride(0)), (buf.stride(0), 1), buf.storage_offset() - ROW0 * buf.stride(0))
    pad = torch.ones_like(full, dtype=torch.bool)
    pad[ROW0:ROW0 + rows, :V] = False
    assert bool(torch.isnan(full[pad]).all()), "in-place backward wrote outside the logits"


# ---------------------------------------------------------------------------------- colsum
def _colsum_in(g, R, Cc, kind, exact):
    """x [R, Cc] as a view: 'padded' of a NaN buffer with ld = rounded width + 8, 'rounded' with ld = the rounded width
    (the columns up to it hold NaN and are read and discarded), 'slice' a column slice of a wider finite buffer."""
    dev = g.device
    if exact:
        x = torch.randint(-2, 3, (R, Cc), device=dev, generator=g).float()
    else:
        x = torch.randn(R, Cc, device=dev, generator=g)
        _, splits, rpb = MB.colsum_grid(R, Cc, _sms())
        x[(torch.arange(1, splits + 1, device=dev) * rpb - 1).clamp(max=R - 1)] *= 64
    x = x.to(bf16)
    if kind == "padded":
        return x, _in(x)
    rw = (Cc + 7) // 8 * 8
    if kind == "rounded":
        base = torch.full((R, rw), math.nan, device=dev, dtype=bf16)
        base[:, :Cc] = x
        return x, base[:, :Cc]
    base = torch.randn(R, 3 * Cc, device=dev, generator=g).to(bf16)
    base[:, Cc:2 * Cc] = x
    return x, base[:, Cc:2 * Cc]


# (R, C, layout): a bias gradient, the ViT's position / temporal table (2 x N T D), the abstractor's B x Q D, ragged C
COLSUM = [(50208, 768, "padded"), (2, 1204224, "padded"), (8, 90112, "padded"), (300, 770, "rounded"),
          (1000, 1001, "rounded"), (4096, 768, "slice"), (65, 8, "padded")]


@pytest.mark.parametrize("R,Cc,kind", COLSUM)
def test_colsum(cuda, R, Cc, kind):
    """Integer inputs onto an integer out: bit-exact; Gaussian inputs with large last rows of each split onto a
    non-zero out: within the bound; out past C untouched."""
    from ymp import ops
    g = torch.Generator(device=cuda).manual_seed(R + Cc)
    for exact in (True, False):
        x, xin = _colsum_in(g, R, Cc, kind, exact)
        out0 = torch.randint(-100, 100, (Cc,), device=cuda, generator=g).float() if exact else \
            torch.randn(Cc, device=cuda, generator=g) * 10
        out = Out(cuda, 1, Cc, f32, init=out0[None])
        ops.colsum(xin, out.view[0])
        got = out.check(f"colsum {R}x{Cc}")[0]
        want = out0.double() + x.double().sum(0)
        if exact:
            _same_bits(f"colsum {R}x{Cc} integers", got, want)
        else:
            _check("colsum", got, want, MB.colsum_bound(x, out0, _sms()))


# ---------------------------------------------------------------------------------- group reduce / broadcast
@pytest.mark.parametrize("G,T,Cc", [(4, 8, 768), (3, 16, 1408), (130, 4, 64)])
def test_group_reduce(cuda, G, T, Cc):
    """The mean over frames (scale 1/T) and the plain sum (scale 1) within the bound, and the broadcast back bit-exact,
    with strided rows in and out."""
    from ymp import ops
    g = torch.Generator(device=cuda).manual_seed(G * T)
    x = torch.randn(G * T, Cc, device=cuda, generator=g).to(bf16)
    x[T - 1::T] *= 16                        # the last frame of each group
    for scale in (1.0 / T, 1.0):
        out = Out(cuda, G, Cc, bf16)
        ops.group_reduce(_in(x), G, T, out.view, scale=scale)
        _check("group_reduce", out.check(f"group_reduce scale={scale}"), MB.group_reduce_reference(x, G, T, scale),
               MB.group_reduce_bound(x, G, T, scale))
        y = torch.randn(G, Cc, device=cuda, generator=g).to(bf16)
        ob = Out(cuda, G * T, Cc, bf16)
        ops.group_reduce(_in(y), G, T, ob.view, scale=scale, broadcast=True)
        want = (y.float() * torch.tensor(scale, dtype=f32, device=cuda)).to(bf16).repeat_interleave(T, 0)
        _same_bits(f"group broadcast scale={scale}", ob.check("group broadcast"), want)


# ---------------------------------------------------------------------------------- embedding gather
@pytest.mark.parametrize("out_dtype", [bf16, f32])
@pytest.mark.parametrize("with_pos", [True, False])
def test_embed_gather(cuda, out_dtype, with_pos):
    """table[clamp(id)] + pos[row_offset + l], bit-exact, into rows b S + row_offset + l only; ids below 0 and past
    the vocabulary clamp; table and pos rows the call must not read hold NaN."""
    from ymp import ops
    g = torch.Generator(device=cuda).manual_seed(3 + with_pos)
    B, Ln, S, off, H, vocab = 3, 7, 12, 4, 768, 1000
    tb = torch.full((vocab + 4, H), math.nan, device=cuda, dtype=bf16)
    table = tb[2:2 + vocab]
    table.copy_(torch.randn(vocab, H, device=cuda, generator=g).to(bf16))
    ids = torch.randint(0, vocab, (B, Ln), device=cuda, generator=g)
    ids[0, 0], ids[1, 1], ids[2, 6] = -3, vocab + 5, vocab - 1
    pos = None
    want = table[ids.clamp(0, vocab - 1)].float()
    if with_pos:
        pb = torch.full((off + Ln + 4, H), math.nan, device=cuda, dtype=bf16)
        pos = pb[:off + Ln + 2]
        pos[off:off + Ln] = torch.randn(Ln, H, device=cuda, generator=g).to(bf16)
        want = want + pos[off:off + Ln].float()[None]
    out = Out(cuda, B * S, H, out_dtype)
    ops.embed_gather(ids, table, pos, out.view, S, off)
    rows = (torch.arange(B)[:, None] * S + off + torch.arange(Ln)[None]).reshape(-1)
    _same_bits("embed_gather", out.check("embed_gather", rows), want.reshape(B * Ln, H))


# ---------------------------------------------------------------------------------- im2col
def _patches(video, P):
    B, Cc, T, H, W = video.shape
    Hp, Wp = H // P, W // P
    return video.view(B, Cc, T, Hp, P, Wp, P).permute(0, 3, 5, 2, 1, 4, 6).reshape(B * Hp * Wp * T, Cc * P * P)


@pytest.mark.parametrize("shape,P", [((2, 3, 4, 32, 48), 16), ((1, 3, 2, 224, 224), 14), ((2, 3, 2, 28, 70), 14)],
                         ids=["vector-P16", "generic-P14-224", "generic-W70"])
def test_im2col(cuda, shape, P):
    """Bit-exact against the reshape.  The vector kernel (P, W multiples of 8) leaves columns [C P P, ldo) alone, the
    element kernel writes zeros there."""
    from ymp import ops
    g = torch.Generator(device=cuda).manual_seed(P)
    video = torch.randn(*shape, device=cuda, generator=g).to(bf16)
    want = _patches(video, P)
    rows, K = want.shape
    out = Out(cuda, rows, K, bf16)
    ops.im2col(video, P, out=out.view)
    vector = P % 8 == 0 and shape[-1] % 8 == 0
    if not vector:
        pad = out.base[ROW0:ROW0 + rows, K:]
        assert torch.equal(_bits(pad), torch.zeros_like(_bits(pad))), "padding columns must be zero"
        pad.view(torch.int16).fill_(SENT16)
    _same_bits(f"im2col P={P}", out.check(f"im2col P={P}"), want)


# ---------------------------------------------------------------------------------- sumsq
@pytest.mark.parametrize("n", [1, 3, 4097, 5 * 2 ** 20 + 3])
def test_sumsq(cuda, n):
    """Values in {-1, 0, 1}: bit-exact; Gaussian values with outliers in the n % 4 tail: within the bound; both onto a
    non-zero out.  5 * 2^20 + 3 takes more than 3 passes of the grid (8 sms blocks of 256 threads x 4 elements)."""
    from ymp import ops
    g = torch.Generator(device=cuda).manual_seed(n)
    for exact in (True, False):
        if exact:
            x = torch.randint(-1, 2, (n,), device=cuda, generator=g).float()
            out0 = 7.0
        else:
            x = torch.randn(n, device=cuda, generator=g)
            x[n - n % 4:] = 1000.0
            out0 = 3.25
        out = Out(cuda, 1, 1, f32, init=torch.tensor([[out0]], device=cuda))
        ops.sumsq(_in_vec(x), out.view[0])
        got = out.check(f"sumsq n={n}")[0]
        want = out0 + (x.double() ** 2).sum()
        if exact:
            _same_bits(f"sumsq n={n} integers", got, want[None])
        else:
            _check("sumsq", got, want[None], MB.sumsq_bound(x, out0, _sms())[None])


# ---------------------------------------------------------------------------------- AdamW
class Flat:
    """A flat [n] slice at `off` of a buffer pre-filled with a NaN bit pattern (16 more elements after it)."""

    def __init__(self, cuda, n, off, dtype, vals):
        sent, itype = (SENT32, torch.int32) if dtype == f32 else (SENT16, torch.int16)
        self.base = torch.full((off + n + 16,), sent, dtype=itype, device=cuda).view(dtype)
        self.view = self.base[off:off + n]
        self.view.copy_(vals)
        self.sent, self.itype, self.off, self.n = sent, itype, off, n

    def untouched_outside(self, what):
        b = self.base.view(self.itype)
        outside = torch.cat([b[:self.off], b[self.off + self.n:]])
        assert bool((outside == self.sent).all()), f"{what}: written outside the slice"


# (sumsq given, max_norm factor of the gradient norm (0: no clip), weight decay, hyper array, zero_grad, chained steps)
ADAMW_CASES = [(True, 0.25, 0.1, False, True, 3), (True, 4.0, 0.0, True, False, 1), (False, 0.0, 0.1, False, False, 1)]


@pytest.mark.parametrize("off", [0, 3], ids=["vector", "scalar"])
@pytest.mark.parametrize("with_sumsq,clip_f,wd,use_hyper,zero_grad,steps", ADAMW_CASES)
def test_adamw(cuda, off, with_sumsq, clip_f, wd, use_hyper, zero_grad, steps):
    """n = 5 * 2^20 + 3 on slices at offset 0 (vector path) and 3 (scalar path) of larger buffers: m, v and master
    within their bounds, param = bf16(master) bit for bit, grad zeroed or untouched, nothing outside the slices
    touched; clipping active, inactive and absent; the hyper array; three chained steps."""
    from ymp import ops
    n = 5 * 2 ** 20 + 3
    g = torch.Generator(device=cuda).manual_seed(off + steps + int(wd * 100))
    w = torch.randn(n, device=cuda, generator=g)
    master = Flat(cuda, n, off, f32, w)
    param = Flat(cuda, n, off, bf16, w.to(bf16))
    m = Flat(cuda, n, off, f32, torch.zeros(n, device=cuda))
    v = Flat(cuda, n, off, f32, torch.zeros(n, device=cuda))
    grad = Flat(cuda, n, off, f32, torch.zeros(n, device=cuda))
    hp = dict(lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8, weight_decay=wd, grad_scale=0.5)
    for step in range(1, steps + 1):
        gv = torch.randn(n, device=cuda, generator=g) * 10 ** (4 * torch.rand(n, device=cuda, generator=g) - 3)
        gv[::97] = 0
        grad.view.copy_(gv)
        s = (gv.double() ** 2).sum().float()
        st = torch.full((1,), float(s), device=cuda) if with_sumsq else None
        max_norm = clip_f * math.sqrt(float(s)) * 0.5
        hyper = None
        if use_hyper:
            hyper = torch.tensor([2e-3, wd, 1 - 0.9 ** 5, 1 - 0.999 ** 5], device=cuda, dtype=f32)
        w0, m0, v0, g0 = (t.view.clone() for t in (master, m, v, grad))
        ops.adamw(master.view, param.view, grad.view, m.view, v.view, step=step, max_grad_norm=max_norm, sumsq_t=st,
                  hyper=hyper, zero_grad=zero_grad, **hp)
        kw = dict(step=step, lr=hp["lr"], beta1=hp["beta1"], beta2=hp["beta2"], eps=hp["eps"], weight_decay=wd,
                  grad_scale=hp["grad_scale"], max_norm=max_norm, sumsq=float(s) if with_sumsq else None, hyper=hyper)
        rw, rm, rv = MB.adamw_reference(w0, g0, m0, v0, **kw)
        ew, em, ev = MB.adamw_bounds(w0, g0, m0, v0, **kw)
        path = "vector" if off == 0 else "scalar"
        _check(f"adamw.{path}.master", master.view, rw, ew)
        _check(f"adamw.{path}.m", m.view, rm, em)
        _check(f"adamw.{path}.v", v.view, rv, ev)
        _same_bits("adamw param", param.view, master.view.to(bf16))
        if zero_grad:
            assert torch.equal(_bits(grad.view), torch.zeros_like(_bits(grad.view))), "grad not zeroed"
        else:
            assert torch.equal(_bits(grad.view), _bits(g0)), "grad changed without zero_grad"
        for t, name in ((master, "master"), (param, "param"), (m, "m"), (v, "v"), (grad, "grad")):
            t.untouched_outside(f"adamw {name}")


# ---------------------------------------------------------------------------------- ymp_dropout
@pytest.mark.parametrize("dtype", [bf16, f32])
def test_dropout_values(cuda, dtype):
    """y = fl(x fl32(1/(1-p))) on kept elements and 0 elsewhere, bit for bit, with ld > cols on both sides."""
    from ymp import ops
    g = torch.Generator(device=cuda).manual_seed(9)
    R, Cc, p, site, row0 = 77, 1000, 0.1, 9, 1000
    x = torch.randn(R, Cc, device=cuda, generator=g).to(dtype)
    out = Out(cuda, R, Cc, dtype)
    ops.dropout(_in(x), ops.Drop(_rng(cuda), site, p), out=out.view, row0=row0)
    keep = _keep(np.arange(row0, row0 + R), Cc, site, p, cuda)
    k = torch.tensor(1.0, dtype=f32) / (1.0 - torch.tensor(p, dtype=f32))
    want = torch.where(keep, x.float() * k.to(cuda), torch.zeros(R, Cc, device=cuda)).to(dtype)
    _same_bits(f"dropout {dtype}", out.check(f"dropout {dtype}"), want)
