"""ymp_gemm's 192-row tiles against its 128-row tiles, bit for bit.

Every output element runs the same k-step sequence and the same epilogue statements whichever tile height it sits in,
so a non-accumulating launch must give bit-identical outputs (D and aux_out) with tile_m = 128 and tile_m = 192:
every epilogue kind, all four operand layouts, ragged M and N, and the full shapes of the training step's
non-accumulating launches on Gaussian operands.  Split-K accumulation reorders fp32 atomic adds, so it is compared on
exact-integer operands, where every order gives the same sum.
"""
import pytest
import torch

from ymp import ops
from ymp.lib import YmpError

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16


def _gauss(g, *shape, scale=1.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).to(bf16)


def _both(a, b, **kw):
    """Run one launch with 128- and 192-row tiles into fresh (NaN-filled) outputs; return both sets of outputs."""
    outs = []
    for tm in (128, 192):
        k = dict(kw)
        for name in ("out", "aux_out"):
            if name in k:
                k[name] = torch.full_like(k[name], float("nan"))
        ops.gemm(a, b, tile_m=tm, tile_n=256, **k)
        outs.append([k[n] for n in ("out", "aux_out") if n in k])
    torch.cuda.synchronize()
    return outs


def _assert_bits(outs, what):
    for x, y in zip(*outs):
        assert torch.equal(x.view(torch.int16 if x.element_size() == 2 else torch.int32),
                           y.view(torch.int16 if y.element_size() == 2 else torch.int32)), what


EPILOGUES = ["plain", "bias", "res32", "gelu_erf_aux", "gelu_tanh_aux", "gelu_erf", "mul", "dropout", "res16",
             "res_row_mod", "d_row_block", "alpha", "aux_value", "f32_out"]


def _epilogue(g, epi, M, N, K):
    kw = dict(out=torch.empty(M, N, device="cuda", dtype=bf16))
    if epi == "bias":
        kw["bias"] = _gauss(g, N)
    elif epi == "res32":
        kw.update(bias=_gauss(g, N), residual=torch.randn(M, N, device="cuda", generator=g),
                  out=torch.empty(M, N, device="cuda"))
    elif epi in ("gelu_erf_aux", "gelu_tanh_aux"):
        kw.update(bias=_gauss(g, N), act=ops.ACT_GELU_ERF if epi == "gelu_erf_aux" else ops.ACT_GELU_TANH,
                  aux_out=torch.empty(M, N, device="cuda", dtype=bf16))
    elif epi == "gelu_erf":
        kw["act"] = ops.ACT_GELU_ERF
    elif epi == "mul":
        kw.update(act=ops.ACT_GELU_ERF, aux_in=_gauss(g, M, N))
    elif epi == "dropout":
        rng = torch.tensor([1234, 7], dtype=torch.int64, device="cuda")
        kw.update(bias=_gauss(g, N), residual=torch.randn(M, N, device="cuda", generator=g),
                  out=torch.empty(M, N, device="cuda"), drop=ops.Drop(rng, 3, 0.1))
    elif epi == "res16":
        kw["residual"] = _gauss(g, M, N)
    elif epi == "res_row_mod":
        kw.update(residual=torch.randn(40, N, device="cuda", generator=g), res_row_mod=40,
                  out=torch.empty(M, N, device="cuda"))
    elif epi == "d_row_block":
        blk = M // 4
        kw.update(out=torch.empty(3 * 2 * blk + blk, N, device="cuda", dtype=bf16), d_row_block=blk, d_row_stride=2 * blk)
    elif epi == "alpha":
        kw["alpha"] = 0.37
    elif epi == "aux_value":
        kw["aux_out"] = torch.empty(M, N, device="cuda", dtype=bf16)
    elif epi == "f32_out":
        kw["out"] = torch.empty(M, N, device="cuda")
    return kw


@pytest.mark.parametrize("epi", EPILOGUES)
def test_tile_m_epilogues_bit_equal(cuda, epi):
    g = torch.Generator(device="cuda").manual_seed(11)
    M, N, K = 772, 520, 320    # ragged in M for both heights, a ragged N tile
    a, b = _gauss(g, M, K, scale=K ** -0.25), _gauss(g, N, K, scale=K ** -0.25)
    _assert_bits(_both(a, b, **_epilogue(g, epi, M, N, K)), epi)


@pytest.mark.parametrize("a_t,b_t", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("m_mod", [0, 1, 64, 65, 128, 191])
def test_tile_m_layouts_ragged_bit_equal(cuda, a_t, b_t, m_mod):
    g = torch.Generator(device="cuda").manual_seed(100 + m_mod + 2 * a_t + b_t)
    M = 3 * 192 + m_mod
    for N, K in ((256, 128), (328, 200)):
        a = _gauss(g, K, (M + 7) // 8 * 8)[:, :M] if a_t else _gauss(g, M, K)   # MN-major A: ld a multiple of 8
        b = _gauss(g, K, N) if b_t else _gauss(g, N, K)
        kw = dict(a_t=a_t, b_t=b_t, out=torch.empty(M, N, device="cuda", dtype=bf16), bias=_gauss(g, N),
                  act=ops.ACT_GELU_TANH, aux_out=torch.empty(M, N, device="cuda", dtype=bf16))
        _assert_bits(_both(a, b, **kw), f"M={M} N={N} K={K} a_t={a_t} b_t={b_t}")


# (M, N, K, a_t, b_t, epilogue) of the non-accumulating launches of the pre-training step (ViT-B/16 at 8 frames and
# B = 32, GPT-3 1.3B), DESIGN.md §5
STEP_LAUNCHES = [
    (50208, 3072, 768, False, False, "gelu_erf_aux"),
    (50208, 3072, 768, False, True, "mul"),
    (50208, 2304, 768, False, False, "plain"),
    (50208, 768, 768, False, False, "res32"),
    (50208, 768, 3072, False, False, "res32"),
    (50208, 768, 3072, False, True, "plain"),
    (8192, 8192, 2048, False, False, "gelu_tanh_aux"),
    (8192, 2048, 8192, False, False, "res32"),
    (8192, 2048, 8192, False, True, "plain"),
    (8192, 6144, 2048, False, False, "plain"),
    (4096, 51200, 2048, False, False, "plain"),
    (4096, 2048, 51200, False, True, "plain"),
]


@pytest.mark.parametrize("M,N,K,a_t,b_t,epi", STEP_LAUNCHES)
def test_tile_m_step_shapes_bit_equal(cuda, M, N, K, a_t, b_t, epi):
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    a = _gauss(g, K, M, scale=K ** -0.25) if a_t else _gauss(g, M, K, scale=K ** -0.25)
    b = _gauss(g, K, N, scale=K ** -0.25) if b_t else _gauss(g, N, K, scale=K ** -0.25)
    kw = _epilogue(g, epi, M, N, K)
    kw.update(a_t=a_t, b_t=b_t)
    _assert_bits(_both(a, b, **kw), f"{M}x{N}x{K} {epi}")
    del a, b, kw
    torch.cuda.empty_cache()


@pytest.mark.parametrize("split_k", [1, 3, 0])
def test_tile_m_split_k_exact(cuda, split_k):
    g = torch.Generator(device="cuda").manual_seed(7 + split_k)
    M, N, K = 2304 + 64, 768 + 40, 4096   # ragged for both tile heights; MN-major A needs M % 8 == 0
    a = torch.randint(-2, 3, (K, M), device="cuda", generator=g).to(bf16)
    b = torch.randint(-2, 3, (K, N), device="cuda", generator=g).to(bf16)
    d0 = torch.randint(-100, 100, (M, N), device="cuda", generator=g).float()
    want = d0.double() + a.double().t() @ b.double()
    for tm in (128, 192):
        out = d0.clone()
        ops.gemm(a, b, a_t=True, b_t=True, out=out, accumulate=True, split_k=split_k, tile_m=tm, tile_n=256)
        assert torch.equal(out.double(), want), f"tile_m={tm} split_k={split_k}"


def test_tile_m_192_rejects_narrow_tile_and_im2col(cuda):
    g = torch.Generator(device="cuda").manual_seed(3)
    a, b = _gauss(g, 256, 128), _gauss(g, 256, 128)
    with pytest.raises(YmpError, match="tile_m = 192"):
        ops.gemm(a, b, tile_m=192, tile_n=128)
    with pytest.raises(YmpError, match="tile_m must be"):
        ops.gemm(a, b, tile_m=64)
    B, T, H, W, D = 2, 8, 32, 32, 256
    video = _gauss(g, B, 3, T, H, W)
    w = _gauss(g, D, 3 * 16 * 16)
    with pytest.raises(YmpError, match="tile_m = 192"):
        ops.patch_embed_gemm(video, w, 16, tile_m=192)
    # auto keeps the fused im2col operand on 128-row tiles
    want = ops.patch_embed_gemm(video, w, 16, tile_n=256, tile_m=128)
    got = ops.patch_embed_gemm(video, w, 16, tile_n=256, tile_m=0)
    assert torch.equal(got, want)
