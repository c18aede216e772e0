"""Every dropout keep bit the kernels draw, read back exactly and compared with the oracle (oracle/philox.py).

A. Attention.  The readouts of dropout_bits.py make the bits of the forward, the dQ and the dK / dV kernel visible as
   zero versus non-zero outputs, window by window over every (query, key) pair of every sequence and head, at the shapes
   of dropout_bits.CASES: the wgmma kernels, the mma.sync kernels with the quad exchange and with one Philox call per
   element, and the mma.sync forward with the wgmma backward.  Inputs sit in buffers with poison outside the view,
   outputs in buffers holding a NaN pattern (test_attention_bounds_gpu.py), and the served family is asserted.
B. The GEMM's bias-dropout-add.  Integer operands in [-2, 2], K <= 256 and bias 0.5 make x = a b^T + bias exact in
   fp32 and never 0, so every output is an exact function of its keep bit: fl32(x * k) or 0, plus the residual in
   fp32, rounded once to the output type.
C. The fp32 threshold: the element-wise dropout drops the one element of its row whose Philox word lies between the
   double p's threshold and the fp32 p's.
"""
import numpy as np
import pytest
import torch

import attn_bounds as AB
import dropout_bits as DB
import gemm_bounds as GB
from oracle import philox
from test_attention_bounds_gpu import Lse, Operand, _family_name, bwd_family, fwd_family
from test_gemm_bounds_gpu import Out, _in, _in_vec, _ints

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16
SITE = 4 * 5 + 1


def _rng(cuda):
    return torch.tensor([DB.SEED, DB.OFFSET], dtype=torch.int64, device=cuda)


# ---------------------------------------------------------------------------------- A. attention
@pytest.mark.parametrize("c", DB.CASES, ids=[c["name"] for c in DB.CASES])
def test_attention_keep_bits(cuda, c):
    from ymp import lib, ops
    n, H, sq, skv, hd = c["n"], c["H"], c["s_q"], c["s_kv"], c["hd"]
    fwd_path = fwd_family(hd, sq, skv, c["mask"], c["mask_block"], c["total_rows"], drop=True)
    bwd_path = bwd_family(hd, c["mask"], c["mask_block"], drop=True)
    gen = torch.Generator().manual_seed(hd + sq + skv)
    mq, mkv = AB.dense(sq), AB.dense(skv)
    lq, lkv = AB.lengths(n, sq, skv, c["total_rows"])
    vis = DB.visible(c)
    keep = DB.oracle_keep(c, SITE)
    kw = dict(n_seq=n, n_heads=H, head_dim=hd, s_q=sq, s_kv=skv, causal=c["mask"], scale=hd ** -0.5,
              mask_block=c["mask_block"], total_rows=c["total_rows"], drop=ops.Drop(_rng(cuda), SITE, c["p"]))
    for kind in DB.KINDS:
        bits = DB.Bits(c)
        for base in DB.windows(kind, c):
            x = DB.inputs(kind, base, c, vis, gen)
            Q, dO = (Operand(cuda, mq, n, sq, H, hd, lq, False, gen) for _ in range(2))
            K, V = (Operand(cuda, mkv, n, skv, H, hd, lkv, False, gen) for _ in range(2))
            for t, w in ((Q, "q"), (K, "k"), (V, "v"), (dO, "do")):
                t.set(x[w].to(cuda))
            if kind == "fwd":
                O, lse = Operand(cuda, mq, n, sq, H, hd, lq, True), Lse(cuda, n, H, sq, lq)
                ops.attn_fwd(Q.view, K.view, V.view, O.view, lse=lse.t, **kw)
                path = fwd_path
            else:
                Oi = Operand(cuda, mq, n, sq, H, hd, lq, False, gen)
                Oi.set(x["o"].to(cuda))
                Li = Lse(cuda, n, H, sq, lq, values=x["lse"].to(cuda))
                dQ = Operand(cuda, mq, n, sq, H, hd, lq, True)
                dK, dV = (Operand(cuda, mkv, n, skv, H, hd, lkv, True) for _ in range(2))
                ops.attn_bwd(Q.view, K.view, V.view, Oi.view, Li.t, dO.view, dQ.view, dK.view, dV.view, **kw)
                path = bwd_path
            fam = lib.attn_last_path()
            assert fam == path, f"{kind}: served by {_family_name(fam)}, expected {_family_name(path)}"
            torch.cuda.synchronize()
            if kind == "fwd":
                O.check_untouched(f"{kind} O")
                lse.check_untouched()
                bits.add(kind, base, O.gather())
            else:
                for t, w in ((dQ, "dQ"), (dK, "dK"), (dV, "dV")):
                    t.check_untouched(f"{kind} {w}")
                bits.add(kind, base, (dQ if kind == "dq" else dV).gather())
        bits.check(f"{_family_name(fwd_path if kind == 'fwd' else bwd_path)} {kind}", keep, vis)


# ---------------------------------------------------------------------------------- B. GEMM bias-dropout-add
# (tile_m, tile_n, M, N, K, residual dtype, res_row_mod, out dtype, d_row_block, d_row_stride)
GEMM_CASES = [
    (128, 128, 300, 262, 72, None, 0, torch.float32, 0, 0),
    (128, 128, 129, 131, 256, bf16, 0, bf16, 0, 0),
    (128, 256, 200, 510, 256, torch.float32, 0, bf16, 0, 0),
    (128, 256, 257, 300, 64, None, 0, bf16, 0, 0),
    (192, 256, 400, 262, 136, torch.float32, 0, torch.float32, 0, 0),
    (192, 256, 250, 301, 72, bf16, 7, torch.float32, 0, 0),
    (128, 128, 200, 131, 72, torch.float32, 7, bf16, 50, 64),
    (192, 256, 384, 258, 200, bf16, 0, bf16, 96, 100),
]


@pytest.mark.parametrize("p", DB.P_DROP)
@pytest.mark.parametrize("tm,tn,M,N,K,res_dtype,mod,out_dtype,blk,stride", GEMM_CASES)
def test_gemm_bias_dropout_add_exact(cuda, tm, tn, M, N, K, res_dtype, mod, out_dtype, blk, stride, p):
    """out = residual + dropout(a b^T + bias), bit for bit, on the vector epilogue and the ragged-N scalar tail; the
    keep bits follow the logical row m, also when d_row_block stores it elsewhere."""
    from ymp import ops
    g = torch.Generator(device=cuda).manual_seed(M + N + K)
    a, b = _ints(g, M, K), _ints(g, N, K)
    bias = torch.full((N,), 0.5, dtype=bf16, device=cuda)
    x = (a.double() @ b.double().t() + 0.5).float().cpu()                       # exact, never 0
    keep = torch.from_numpy(philox.keep_mask(DB.SEED, DB.OFFSET, SITE, np.arange(M), N, p))
    want = torch.where(keep, x * torch.tensor(philox.scale(p), dtype=torch.float32), torch.zeros_like(x))
    kw = {}
    if res_dtype is not None:
        res = (torch.randn(mod or M, N, generator=g, device=cuda) * 100).to(res_dtype)
        kw.update(residual=_in(res), res_row_mod=mod)
        want = want + res.float().cpu()[GB.res_rows(M, mod)]
    want = want.to(out_dtype)
    rows = GB.store_rows(M, blk, stride)
    out = Out(cuda, int(rows[-1]) + 1, N, out_dtype)
    ops.gemm(_in(a), _in(b), bias=_in_vec(bias), out=out.view, out_dtype=out_dtype, tile_m=tm, tile_n=tn,
             d_row_block=blk, d_row_stride=stride, drop=ops.Drop(_rng(cuda), SITE, p), **kw)
    got = out.check("bias-dropout-add", rows).cpu()
    itype = torch.int32 if out_dtype == torch.float32 else torch.int16
    bad = got.view(itype) != want.view(itype)
    if bool(bad.any()):
        m, c = (int(i) for i in bad.nonzero()[0])
        raise AssertionError(f"{int(bad.sum())} outputs differ, first at row {m} column {c}: got {got[m, c].item()}, "
                             f"want {want[m, c].item()} (oracle {'keeps' if keep[m, c] else 'drops'} it)")


# ---------------------------------------------------------------------------------- C. the fp32 threshold
def test_elementwise_dropout_uses_the_fp32_threshold(cuda):
    """Row 6350 of site 9 at p = 0.1: the word of column 9906 (429496732) lies between floor(0.1 * 2^32) and
    floor(fl32(0.1) * 2^32); the kernel drops it, like the oracle."""
    from ymp import ops
    x = torch.ones(1, 9912, device=cuda)
    y = ops.dropout(x, ops.Drop(_rng(cuda), 9, 0.1), row0=6350)
    keep = torch.from_numpy(philox.keep_mask(DB.SEED, DB.OFFSET, 9, [6350], 9912, 0.1))
    assert float(y[0, 9906]) == 0.0
    assert torch.equal((y != 0).cpu(), keep)
