"""ymp_gemm, ymp_gemm_skinny and ymp_gemm_skinny_wide element by element: bit-exact where the arithmetic is exact, and
against the float64 reference of gemm_bounds.py with its derived per-element bounds everywhere else.

A. Exact-integer sweep.  Operands in {-2..2} make every partial sum an integer below 2^15, so the fp32 accumulation is
   exact in any order: an fp32 output must equal the float64 reference bit for bit, a bf16 output its round-to-nearest-
   even value.  Operands sit in wider buffers whose columns past K, past M / N and rows around the view hold NaN (a read
   of any of them turns an output NaN); outputs go into buffers pre-filled with a NaN bit pattern and padded to
   ld > N: every addressed element must come back exact, every other element keep its pattern.
B. Epilogue transfer function.  A single non-zero k column carries every bf16 value with |x| <= 16 and +-20, +-50,
   +-100, so the pre-activation is exact: act(x) and act'(x) against float64 within the activation bound, and the
   vector (full quads) and scalar (ragged N) epilogue paths, with and without aux_out, and the skinny kernels bit-equal.
C. Gaussian operands at the model's shapes: err / bound <= 1 for every element.
Set YMP_GEMM_BOUNDS_REPORT=<file> to write the largest err / bound per kernel, epilogue and tensor as JSON.
"""
import json
import math
import os

import pytest
import torch

import gemm_bounds as GB

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16

SENT16 = 0x7FA5          # bf16 NaN bit pattern of untouched output memory
SENT32 = 0x7FA0BEEF      # fp32 NaN bit pattern of untouched output memory
ROW0 = 2                 # rows of every buffer before the addressed view
RATIOS = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    path = os.environ.get("YMP_GEMM_BOUNDS_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump(RATIOS, f, indent=1, sort_keys=True)


def _ld(cols):
    return (cols + 7) // 8 * 8 + 8


def _in(vals):
    """vals (a bf16 / fp32 CUDA matrix) as a view of a wider buffer holding NaN everywhere else."""
    R, Cc = vals.shape
    base = torch.full((ROW0 + R + 3, _ld(Cc)), math.nan, dtype=vals.dtype, device=vals.device)
    base[ROW0:ROW0 + R, :Cc] = vals
    return base[ROW0:ROW0 + R, :Cc]


def _in_vec(vals):
    base = torch.full((vals.numel() + 16,), math.nan, dtype=vals.dtype, device=vals.device)
    base[:vals.numel()] = vals
    return base[:vals.numel()]


class Out:
    """An output view [rows, cols] inside a buffer pre-filled with a NaN bit pattern: ROW0 rows before it, 3 after,
    ld = _ld(cols) > cols."""

    def __init__(self, cuda, rows, cols, dtype, init=None):
        self.sent = SENT32 if dtype == torch.float32 else SENT16
        itype = torch.int32 if dtype == torch.float32 else torch.int16
        self.base = torch.full((ROW0 + rows + 3, _ld(cols)), self.sent, dtype=itype, device=cuda).view(dtype)
        self.view = self.base[ROW0:ROW0 + rows, :cols]
        if init is not None:
            self.view.copy_(init)
        self.itype = itype

    def check(self, what, rows=None):
        """The addressed rows (all by default) must hold finite values, every other element its pattern."""
        addr = torch.zeros(self.base.shape, dtype=torch.bool, device=self.base.device)
        r = torch.arange(self.view.shape[0], device=self.base.device) if rows is None else rows.to(self.base.device)
        addr[ROW0 + r, :self.view.shape[1]] = True
        bad = (self.base.view(self.itype) != self.sent) & ~addr
        assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements outside the output were written, first at " \
                                    f"{bad.nonzero()[0].tolist()} (buffer row, column)"
        got = self.base[addr]
        assert bool(torch.isfinite(got).all()), f"{what}: {int((~torch.isfinite(got)).sum())} addressed elements not " \
                                                f"written or not finite"
        return self.base[ROW0 + r][:, :self.view.shape[1]]


def _ints(g, *shape, dtype=bf16):
    return torch.randint(-2, 3, shape, generator=g, device=g.device).to(dtype)


def _exact(what, got, ref):
    """got (fp32 or bf16) equals the float64 integer reference rounded once to got's type."""
    want = ref.float().to(got.dtype)
    bad = got.view(torch.int16 if got.dtype == bf16 else torch.int32) != want.view(torch.int16 if got.dtype == bf16 else torch.int32)
    if bool(bad.any()):
        i = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} elements differ, first at {i}: got {got[i[0], i[1]].item()}, "
                             f"want {want[i[0], i[1]].item()}")


def _check(key, got, want, bound):
    r = GB.worst_ratio(got, want, bound)
    RATIOS[key] = max(RATIOS.get(key, 0.0), r)
    if r > 1:
        err = ((got.double() - want.double()).abs() / bound).nan_to_num(math.inf)
        idx = int(err.flatten().argmax())
        raise AssertionError(f"{key}: err / bound = {r:.3g} at flat index {idx}: got {got.flatten()[idx].item():.8g}, "
                             f"want {want.flatten()[idx].item():.8g}, bound {bound.flatten()[idx].item():.3g}")


# ---------------------------------------------------------------------------------- A. exact-integer sweep
# Epilogues cycled over the shapes so that each meets ragged M, N and K: (out dtype, bias, aux_out, aux_in,
# residual dtype, res_row_mod, alpha)
EXACT_EPILOGUES = [
    (torch.float32, True, True, False, None, 0, 1.0),
    (bf16, False, False, False, None, 0, 1.0),
    (bf16, True, False, True, bf16, 0, 1.0),
    (torch.float32, True, False, False, torch.float32, 3, 0.5),
    (bf16, True, True, False, torch.float32, 0, 0.5),
]


def _gemm_exact(cuda, g, M, N, K, a_t, b_t, tile_n, epi, what):
    from ymp import ops
    out_dtype, has_bias, has_aux, has_mul, res_dtype, mod, alpha = epi
    a = _ints(g, K, M) if a_t else _ints(g, M, K)
    b = _ints(g, K, N) if b_t else _ints(g, N, K)
    A = (a.t() if a_t else a).double()
    B = (b if b_t else b.t()).double()
    v = alpha * (A @ B)
    kw = {}
    if has_bias:
        bias = _ints(g, N)
        kw["bias"] = _in_vec(bias)
        v = v + bias.double()
    aux = Out(cuda, M, N, bf16) if has_aux else None
    if aux is not None:
        kw["aux_out"] = aux.view
    out_v = v
    if has_mul:
        mul = _ints(g, M, N)
        kw["aux_in"], kw["act"] = _in(mul), 1
        out_v = v * mul.double()
    if res_dtype is not None:
        res = _ints(g, mod or M, N, dtype=res_dtype) * 3
        kw["residual"], kw["res_row_mod"] = _in(res), mod
        out_v = out_v + res.double()[GB.res_rows(M, mod).to(cuda)]
    out = Out(cuda, M, N, out_dtype)
    ops.gemm(_in(a), _in(b), a_t=a_t, b_t=b_t, out=out.view, tile_n=tile_n, alpha=alpha, **kw)
    _exact(what, out.check(what), out_v)
    if aux is not None:
        _exact(what + " aux_out", aux.check(what + " aux_out"), v)


@pytest.mark.parametrize("tile_n", [0, 128, 256])
@pytest.mark.parametrize("a_t,b_t", [(False, False), (False, True), (True, False), (True, True)])
def test_gemm_exact_sweep(cuda, a_t, b_t, tile_n):
    """Every (M, N, K) of M in {1, 64, 127, 129, 200}, N in {8, 131, 250, 256, 300}, K in {8, 16, 40, 64, 72, 200}:
    ragged M and N tiles, N % 4 != 0 (the scalar tail inside a quad), K below one k-block and ragged K tails."""
    g = torch.Generator(device=cuda).manual_seed(1000 * a_t + 100 * b_t + tile_n)
    i = 0
    for M in (1, 64, 127, 129, 200):
        for N in (8, 131, 250, 256, 300):
            for K in (8, 16, 40, 64, 72, 200):
                epi = EXACT_EPILOGUES[i % len(EXACT_EPILOGUES)]
                i += 1
                _gemm_exact(cuda, g, M, N, K, a_t, b_t, tile_n, epi, f"M={M} N={N} K={K} epilogue {epi}")


def test_gemm_exact_many_waves(cuda):
    """M = 20000: many more tiles than SMs, with every epilogue."""
    g = torch.Generator(device=cuda).manual_seed(7)
    for j, epi in enumerate(EXACT_EPILOGUES):
        _gemm_exact(cuda, g, 20000, 300, 72, False, j % 2 == 1, (0, 128, 256)[j % 3], epi, f"M=20000 epilogue {epi}")


@pytest.mark.parametrize("a_t,b_t,tile_n", [(True, True, 0), (False, False, 256), (True, False, 128)])
def test_gemm_exact_split_k(cuda, a_t, b_t, tile_n):
    """K = 4096 accumulated into a non-zero fp32 buffer with split_k 1, 3, 7, 0 (the library's choice) and more
    splits than k-blocks, alpha 1 and 0.5: exact whatever the order of the atomic adds."""
    from ymp import ops
    g = torch.Generator(device=cuda).manual_seed(11)
    M, N, K = 200, 131, 4096
    for split in (1, 3, 7, 0, 100):
        for alpha in (1.0, 0.5):
            a = _ints(g, K, M) if a_t else _ints(g, M, K)
            b = _ints(g, K, N) if b_t else _ints(g, N, K)
            d0 = _ints(g, M, N, dtype=torch.float32) * 1000
            ref = d0.double() + alpha * ((a.t() if a_t else a).double() @ (b if b_t else b.t()).double())
            out = Out(cuda, M, N, torch.float32, init=d0)
            ops.gemm(_in(a), _in(b), a_t=a_t, b_t=b_t, out=out.view, accumulate=True, split_k=split, alpha=alpha,
                     tile_n=tile_n)
            what = f"split_k={split} alpha={alpha}"
            _exact(what, out.check(what), ref)


def test_gemm_exact_row_blocked_store(cuda):
    """d_row_block / d_row_stride: [B*Q] result rows land in a [B, S > Q] buffer; the rows between blocks and the
    aux_out rows (plain layout) are checked separately."""
    from ymp import ops
    g = torch.Generator(device=cuda).manual_seed(12)
    M, N, K, blk, stride = 200, 131, 72, 50, 64
    a, b, bias = _ints(g, M, K), _ints(g, N, K), _ints(g, N)
    res = _ints(g, 7, N)
    rows = GB.store_rows(M, blk, stride)
    v = a.double() @ b.double().t() + bias.double()
    for out_dtype in (bf16, torch.float32):
        out = Out(cuda, (M // blk - 1) * stride + blk, N, out_dtype)
        aux = Out(cuda, M, N, bf16)
        ops.gemm(_in(a), _in(b), bias=_in_vec(bias), residual=_in(res), res_row_mod=7, out=out.view, aux_out=aux.view,
                 d_row_block=blk, d_row_stride=stride)
        _exact("row-blocked D", out.check("row-blocked D", rows), v + res.double()[GB.res_rows(M, 7).to(cuda)])
        _exact("row-blocked aux_out", aux.check("aux_out"), v)


def test_gemm_exact_fused_im2col(cuda):
    """The patch embedding's fused im2col A operand at ragged M (144 = 128 + 16 rows: B = 3 clips, 3 x 2 patches,
    T = 8 frames), with a bias and a residual table broadcast by row."""
    from ymp import ops
    g = torch.Generator(device=cuda).manual_seed(13)
    Bc, Cc, T, H, W, P, N = 3, 2, 8, 48, 32, 16, 200
    video = _ints(g, Bc, Cc, T, H, W).contiguous()
    Hp, Wp = H // P, W // P
    patches = video.view(Bc, Cc, T, Hp, P, Wp, P).permute(0, 3, 5, 2, 1, 4, 6).reshape(Bc * Hp * Wp * T, Cc * P * P)
    M, K = patches.shape
    w, bias, table = _ints(g, N, K), _ints(g, N), _ints(g, 5 * T, N)
    ref = patches.double() @ w.double().t() + bias.double() + table.double()[GB.res_rows(M, 5 * T).to(cuda)]
    for out_dtype in (bf16, torch.float32):
        out = Out(cuda, M, N, out_dtype)
        ops.patch_embed_gemm(video, _in(w), P, bias=_in_vec(bias), residual=_in(table), res_row_mod=5 * T, out=out.view)
        _exact("fused im2col", out.check("fused im2col"), ref)


# skinny (M, K, N): K picks the K slices per CTA (128 -> 1, 256 -> 2, 512 -> 4, >= 1024 -> 8, capped at 4 for N > 4096)
SKINNY_KN = [(8, 16), (64, 72), (128, 131), (256, 250), (512, 8), (1024, 1000), (1024, 4104), (2048, 300)]
# (out dtype, bias, residual dtype, y2 row copy)
SKINNY_EPILOGUES = [(bf16, True, None, True), (torch.float32, False, torch.float32, False),
                    (bf16, True, bf16, False), (torch.float32, True, None, False)]


@pytest.mark.parametrize("M", [1, 3, 8, 9, 16, 17, 40, 64])
def test_skinny_exact_sweep(cuda, M):
    """ymp_gemm_skinny (M <= 8) and ymp_gemm_skinny_wide: every K-slice count, N % 8 != 0, strided x / w / y / residual,
    the bf16 y2 row copy at a device-side offset."""
    from ymp import ops
    g = torch.Generator(device=cuda).manual_seed(M)
    fns = [ops.gemm_skinny_wide] if M > 8 else [ops.gemm_skinny, ops.gemm_skinny_wide]
    for i, (K, N) in enumerate(SKINNY_KN):
        for fn in fns:
            out_dtype, has_bias, res_dtype, has_y2 = SKINNY_EPILOGUES[(i + M) % len(SKINNY_EPILOGUES)]
            x, w = _ints(g, M, K), _ints(g, N, K)
            ref = x.double() @ w.double().t()
            kw = {}
            if has_bias:
                bias = _ints(g, N)
                kw["bias"] = _in_vec(bias)
                ref = ref + bias.double()
            if res_dtype is not None:
                res = _ints(g, M, N, dtype=res_dtype) * 3
                kw["residual"] = _in(res)
                ref = ref + res.double()
            y2 = None
            if has_y2:
                ML, off = 5, 3
                y2 = Out(cuda, M * ML, N, bf16)
                kw.update(out2=y2.view, out2_row_stride=ML, out2_off=torch.tensor([off], device=cuda, dtype=torch.int64))
            out = Out(cuda, M, N, out_dtype)
            fn(_in(x), _in(w), out=out.view, **kw)
            what = f"{fn.__name__} M={M} K={K} N={N}"
            _exact(what, out.check(what), ref)
            if y2 is not None:
                got2 = y2.check(what + " y2", torch.arange(M) * ML + off)
                assert torch.equal(got2.view(torch.int16), out.view.view(torch.int16)), what + " y2"


# ---------------------------------------------------------------------------------- bias under accumulation
@pytest.mark.parametrize("split_k", [0, 1, 3])
def test_accumulate_rejects_bias(cuda, split_k):
    """Each K-split of an accumulating call adds its own partial to D, so a bias would be counted once per split:
    ymp_gemm rejects the combination and leaves D alone."""
    from ymp import lib, ops
    g = torch.Generator(device=cuda).manual_seed(3)
    a, b, bias = _ints(g, 256, 1024), _ints(g, 128, 1024), _ints(g, 128)
    d = torch.ones(256, 128, device=cuda)
    with pytest.raises(lib.YmpError, match="accumulate"):
        ops.gemm(a, b, bias=bias, out=d, accumulate=True, split_k=split_k)
    torch.cuda.synchronize()
    assert bool((d == 1).all())


# ---------------------------------------------------------------------------------- B. epilogue transfer function
def _transfer_values(cuda):
    v = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(bf16).float()
    v = v[torch.isfinite(v) & (v.abs() <= 16)]
    t = torch.tensor([20.0, 50.0, 100.0])
    return torch.cat([v, t, -t]).to(bf16).to(cuda)


@pytest.mark.parametrize("act", [GB.ACT_GELU_ERF, GB.ACT_GELU_TANH], ids=["erf", "tanh"])
def test_epilogue_transfer_function(cuda, act):
    from ymp import ops
    xs = _transfer_values(cuda)
    n, K = xs.numel(), 16
    a = torch.zeros(n, K, device=cuda, dtype=bf16)
    a[:, 0] = xs
    x64 = xs.double()
    want, dwant = GB.act_ref(x64, act), GB.dact_ref(x64, act)
    e_act, e_dact = GB.act_err(x64, act)
    bound = GB.C * (e_act + GB.U32 * want.abs()) + GB.TINY
    dbound = GB.C * (e_dact + GB.U * dwant.abs()) + GB.TINY
    name = {GB.ACT_GELU_ERF: "gelu_erf", GB.ACT_GELU_TANH: "gelu_tanh"}[act]
    outs = {}
    for N in (128, 65):     # tile_n = 128: N = 128 runs every quad on the vector path, N = 65 every one on the scalar
        b = torch.zeros(N, K, device=cuda, dtype=bf16)
        b[:, 0] = 1
        for with_aux in (True, False):
            out = Out(cuda, n, N, torch.float32)
            aux = Out(cuda, n, N, bf16) if with_aux else None
            ops.gemm(a, b, act=act, out=out.view, aux_out=aux.view if aux else None, tile_n=128)
            y = out.check(f"{name} N={N}")
            outs[(N, with_aux)] = y[:, :65]
            _check(f"gemm.{name}.act", y, want[:, None].expand(n, N), bound[:, None].expand(n, N))
            if aux is not None:
                d = aux.check(f"{name} aux N={N}")
                outs[(N, "aux")] = d[:, :65]
                _check(f"gemm.{name}.aux_out", d, dwant[:, None].expand(n, N), dbound[:, None].expand(n, N))
    ref_bits = outs[(128, True)].view(torch.int32)
    for key in ((128, False), (65, True), (65, False)):
        assert torch.equal(outs[key].view(torch.int32), ref_bits), f"{name}: path {key} differs from the vector path"
    assert torch.equal(outs[(65, "aux")].view(torch.int16), outs[(128, "aux")].view(torch.int16)), f"{name} aux_out"
    # the skinny kernels: the values along N (one row, and 16 identical rows of the wide kernel)
    w = torch.zeros(n, K, device=cuda, dtype=bf16)
    w[:, 0] = xs
    for fn, M in ((ops.gemm_skinny, 1), (ops.gemm_skinny_wide, 16)):
        x = torch.zeros(M, K, device=cuda, dtype=bf16)
        x[:, 0] = 1
        y = fn(x, w, act=act, out_dtype=torch.float32)
        _check(f"{fn.__name__}.{name}.act", y, want[None].expand(M, n), bound[None].expand(M, n))
        assert torch.equal(y.view(torch.int32), ref_bits[:, 0][None].expand(M, n)), f"{fn.__name__}: {name} bits"


# ---------------------------------------------------------------------------------- C. Gaussian operands, model shapes
# (name, M, N, K, a_t, b_t, epilogue): forward / dgrad / wgrad launches at the ViT (768), abstractor (1408) and
# GPT-3 1.3B / 2.7B (2048 / 2560) widths and the 51200-column LM head
GAUSS = [
    ("vit_qkv", 400, 2304, 768, False, False, dict(bias=True)),
    ("vit_fc1", 400, 3072, 768, False, False, dict(bias=True, act=GB.ACT_GELU_ERF, aux=True)),
    ("vit_fc2", 400, 768, 3072, False, False, dict(bias=True, residual=torch.float32, out=torch.float32)),
    ("vit_fc1_dgrad", 400, 3072, 768, False, True, dict(aux_in=True)),
    ("abstractor_fc1", 300, 5632, 1408, False, False, dict(bias=True, act=GB.ACT_GELU_ERF, aux=True)),
    ("abstractor_proj", 300, 1408, 1408, False, False, dict(bias=True, residual=bf16)),
    ("gpt13_h4h", 256, 8192, 2048, False, False, dict(bias=True, act=GB.ACT_GELU_TANH, aux=True)),
    ("gpt13_4hh", 256, 2048, 8192, False, False, dict(bias=True, residual=torch.float32, out=torch.float32)),
    ("gpt27_qkv", 256, 7680, 2560, False, False, dict(bias=True, alpha=0.5)),
    ("gpt27_dgrad", 256, 2560, 10240, False, True, dict()),
    ("lm_head", 96, 51200, 2048, False, False, dict(out=torch.float32)),
    ("wgrad_768", 768, 768, 4096, True, True, dict(accumulate=True)),
    ("wgrad_2048x8192", 2048, 8192, 1024, True, True, dict(accumulate=True)),
]


@pytest.mark.parametrize("name,M,N,K,a_t,b_t,epi", GAUSS, ids=[c[0] for c in GAUSS])
def test_gemm_gaussian_model_shapes(cuda, name, M, N, K, a_t, b_t, epi):
    from ymp import ops
    g = torch.Generator(device=cuda).manual_seed(M + N + K)
    sig = 2.0 * K ** -0.5      # pre-activations ~ N(0, 4): both GELU tails are reached
    a = torch.randn((K, M) if a_t else (M, K), device=cuda, generator=g).to(bf16)
    b = (torch.randn((K, N) if b_t else (N, K), device=cuda, generator=g) * sig).to(bf16)
    A, B = (a.t() if a_t else a), (b.t() if b_t else b)
    kw, rk = dict(a_t=a_t, b_t=b_t), {}
    if epi.get("bias"):
        rk["bias"] = kw["bias"] = torch.randn(N, device=cuda, generator=g).to(bf16)
    if epi.get("act"):
        rk["act"] = kw["act"] = epi["act"]
    if epi.get("aux_in"):
        rk["aux_in"] = kw["aux_in"] = torch.rand(M, N, device=cuda, generator=g).to(bf16)
        kw["act"] = GB.ACT_GELU_ERF
    if epi.get("residual") is not None:
        rk["residual"] = kw["residual"] = torch.randn(M, N, device=cuda, generator=g).to(epi["residual"])
    if "alpha" in epi:
        rk["alpha"] = kw["alpha"] = epi["alpha"]
    out_dtype = epi.get("out", bf16)
    split = 1
    if epi.get("accumulate"):
        out_dtype = torch.float32
        d0 = torch.randn(M, N, device=cuda, generator=g)
        rk["d0"], kw["out"], kw["accumulate"], kw["split_k"] = d0, d0.clone(), True, 0
        kb = -(-K // 64)
        split = min(64, kb)   # the library's choice is at most this
    if epi.get("aux"):
        kw["aux_out"] = torch.empty(M, N, device=cuda, dtype=bf16)
    out = ops.gemm(a, b, out_dtype=out_dtype, **kw)
    ref = GB.reference(A, B, **rk)
    e_out, e_aux = GB.bounds(ref, K, split=split, out_bf16=out_dtype == bf16)
    epi_name = "+".join(k for k in epi if k not in ("out",)) or "plain"
    _check(f"gemm.{name}({epi_name}).D", out, ref["out"], e_out)
    if epi.get("aux"):
        _check(f"gemm.{name}({epi_name}).aux_out", kw["aux_out"], ref["aux"], e_aux)


# (kernel, M, N, K, epilogue) at the decoding step's shapes
SKINNY_GAUSS = [
    ("gemm_skinny", 5, 6144, 2048, dict(bias=True)),
    ("gemm_skinny", 8, 8192, 2048, dict(bias=True, act=GB.ACT_GELU_TANH)),
    ("gemm_skinny", 1, 2560, 10240, dict(bias=True, residual=torch.float32, out=torch.float32)),
    ("gemm_skinny", 8, 51200, 2048, dict(out=torch.float32)),
    ("gemm_skinny", 4, 3072, 768, dict(bias=True, act=GB.ACT_GELU_ERF)),
    ("gemm_skinny_wide", 40, 7680, 2560, dict(bias=True, residual=bf16)),
    ("gemm_skinny_wide", 64, 2048, 8192, dict(bias=True, residual=torch.float32, out=torch.float32)),
    ("gemm_skinny_wide", 24, 10240, 2560, dict(bias=True, act=GB.ACT_GELU_TANH)),
]


@pytest.mark.parametrize("kernel,M,N,K,epi", SKINNY_GAUSS, ids=[f"{c[0]}-{c[1]}x{c[2]}x{c[3]}" for c in SKINNY_GAUSS])
def test_skinny_gaussian_model_shapes(cuda, kernel, M, N, K, epi):
    from ymp import ops
    g = torch.Generator(device=cuda).manual_seed(M * N + K)
    x = torch.randn(M, K, device=cuda, generator=g).to(bf16)
    w = (torch.randn(N, K, device=cuda, generator=g) * 2.0 * K ** -0.5).to(bf16)
    kw, rk = {}, {}
    if epi.get("bias"):
        rk["bias"] = kw["bias"] = torch.randn(N, device=cuda, generator=g).to(bf16)
    if epi.get("act"):
        rk["act"] = kw["act"] = epi["act"]
    if epi.get("residual") is not None:
        rk["residual"] = kw["residual"] = torch.randn(M, N, device=cuda, generator=g).to(epi["residual"])
    out_dtype = epi.get("out", bf16)
    y = getattr(ops, kernel)(x, w, out_dtype=out_dtype, **kw)
    ref = GB.reference(x, w, **rk)
    e_out, _ = GB.bounds(ref, K, split=GB.skinny_slices(N, K), out_bf16=out_dtype == bf16)
    epi_name = "+".join(k for k in epi if k != "out") or "plain"
    _check(f"{kernel}.{M}x{N}x{K}({epi_name}).y", y, ref["out"], e_out)
