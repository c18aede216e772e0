"""GPU parity for the non-GEMM kernels: each op vs a plain fp32 torch restatement of the same math
(the checker runs in fp32 on the same bf16-rounded inputs; tolerances are bf16 output rounding)."""
import math

import pytest
import torch

from oracle import port

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16


def _rel(a, b):
    return ((a.float() - b.float()).abs().max() / (b.float().abs().max() + 1e-6)).item()


@pytest.mark.parametrize("rows,D", [(100, 768), (37, 2048), (16, 2560), (9, 1408), (64, 192), (5, 128)])
def test_layernorm_fwd_bwd(cuda, rows, D):
    from ymp import ops
    torch.manual_seed(0)
    x = (torch.randn(rows, D, device=cuda) * 2 + 0.5).to(bf16)
    g = (1 + 0.1 * torch.randn(D, device=cuda)).to(bf16)
    b = (0.1 * torch.randn(D, device=cuda)).to(bf16)
    dy = torch.randn(rows, D, device=cuda).to(bf16)
    add = torch.randn(rows, D, device=cuda).to(bf16)
    y, mean, rstd = ops.layernorm_fwd(x, g, b, 1e-6)
    xf, gf, bf_ = x.float().requires_grad_(), g.float().requires_grad_(), b.float().requires_grad_()
    ref = torch.nn.functional.layer_norm(xf, (D,), gf, bf_, 1e-6)
    assert _rel(y, ref) < 1e-2
    ref.backward(dy.float())
    dgam = torch.zeros(D, device=cuda)
    dbet = torch.zeros(D, device=cuda)
    dx = ops.layernorm_bwd(dy, x, g, mean, rstd, add=add, dgamma=dgam, dbeta=dbet)
    assert _rel(dx, xf.grad + add.float()) < 1e-2
    assert _rel(dgam, gf.grad) < 5e-3
    assert _rel(dbet, bf_.grad) < 5e-3
    dx2 = ops.layernorm_bwd(dy, x, g, mean, rstd)  # frozen affine, no add
    assert _rel(dx2, xf.grad) < 1e-2


@pytest.mark.parametrize("D", [768, 2048])
def test_layernorm_fp32_stream(cuda, D):
    """fp32 residual-stream input (and optionally fp32 output), bf16 gradients."""
    from ymp import ops
    torch.manual_seed(11)
    rows = 77
    x = torch.randn(rows, D, device=cuda) * 3 + 1
    g = (1 + 0.1 * torch.randn(D, device=cuda)).to(bf16)
    b = (0.1 * torch.randn(D, device=cuda)).to(bf16)
    y, mean, rstd = ops.layernorm_fwd(x, g, b, 1e-5)
    assert y.dtype == bf16
    xf = x.clone().requires_grad_()
    ref = torch.nn.functional.layer_norm(xf, (D,), g.float(), b.float(), 1e-5)
    assert _rel(y, ref) < 5e-3
    y32, _, _ = ops.layernorm_fwd(x, g, b, 1e-5, out_dtype=torch.float32)
    assert y32.dtype == torch.float32 and _rel(y32, ref) < 1e-5
    dy = torch.randn(rows, D, device=cuda).to(bf16)
    ref.backward(dy.float())
    dg, db = torch.zeros(D, device=cuda), torch.zeros(D, device=cuda)
    dx = ops.layernorm_bwd(dy, x, g, mean, rstd, dgamma=dg, dbeta=db)
    assert dx.dtype == bf16 and _rel(dx, xf.grad) < 1e-2
    xh = (x - x.mean(-1, keepdim=True)) * torch.rsqrt(x.var(-1, unbiased=False, keepdim=True) + 1e-5)
    assert _rel(dg, (dy.float() * xh).sum(0)) < 5e-3 and _rel(db, dy.float().sum(0)) < 5e-3


def test_layernorm_row_gather(cuda):
    from ymp import ops
    torch.manual_seed(1)
    rows, D = 50, 768
    x = torch.randn(rows, D, device=cuda).to(bf16)
    g = torch.ones(D, device=cuda, dtype=bf16)
    b = torch.zeros(D, device=cuda, dtype=bf16)
    perm = torch.randperm(rows, device=cuda).int()
    y, mean, rstd = ops.layernorm_fwd(x, g, b, 1e-6, in_rows=perm)
    ref = torch.nn.functional.layer_norm(x.float()[perm.long()], (D,))
    assert _rel(y, ref) < 1e-2
    dy = torch.randn(rows, D, device=cuda).to(bf16)
    dx = ops.layernorm_bwd(dy, x, g, mean, rstd, in_rows=perm)
    xf = x.float().requires_grad_()
    torch.nn.functional.layer_norm(xf[perm.long()], (D,)).backward(dy.float())
    assert _rel(dx, xf.grad) < 1e-2


def _attn_ref(q, k, v, scale, causal):
    """q [n,h,sq,d] etc. fp32 -> out, with autograd."""
    s = (q @ k.transpose(-1, -2)) * scale
    if causal:
        m = torch.ones(s.shape[-2:], dtype=torch.bool, device=s.device).triu(1)
        s = s.masked_fill(m, -10000.0)
    return s.softmax(-1) @ v


@pytest.mark.parametrize("hd,heads,S,causal,layout", [
    (64, 4, 256, True, "gpt"), (64, 2, 100, True, "gpt"), (80, 2, 130, True, "gpt"),
    (96, 2, 197, False, "vit"), (96, 8, 64, False, "vit"), (64, 2, 300, False, "vit"),
    # tensor-core tiles at block boundaries: one / two key blocks, partial second query block, tiny sequences
    (64, 2, 129, True, "gpt"), (96, 1, 33, True, "vit"), (96, 2, 128, False, "vit"), (96, 2, 256, False, "gpt"),
    (64, 3, 160, False, "gpt"), (64, 1, 8, True, "gpt"),
    # key ranges > 256 (KV loop + online softmax, dQ partial parked across > 2 key blocks) and head_dim 80 / 88
    # zero-padded to 96: the 2.7B decoder (hd 80, S = 384), EVA-g (hd 88, 257 tokens)
    (80, 2, 384, True, "gpt"), (88, 2, 257, False, "vit"), (96, 2, 600, False, "vit"), (64, 2, 700, True, "gpt"),
    (80, 1, 257, True, "gpt"), (88, 3, 40, False, "gpt")])
def test_attn_dense_fwd_bwd(cuda, hd, heads, S, causal, layout):
    from ymp import lib, ops
    torch.manual_seed(2)
    n = 3
    C = heads * hd
    qkv = (torch.randn(n * S, 3 * C, device=cuda) * 0.7).to(bf16)
    if layout == "gpt":  # per head [q|k|v]
        hs, offs = 3 * hd, (0, hd, 2 * hd)
        qkv5 = qkv.float().view(n, S, heads, 3, hd)
        q, k, v = (qkv5[:, :, :, i].permute(0, 2, 1, 3) for i in range(3))
    else:                # [3, heads, hd]
        hs, offs = hd, (0, C, 2 * C)
        qkv5 = qkv.float().view(n, S, 3, heads, hd)
        q, k, v = (qkv5[:, :, i].permute(0, 2, 1, 3) for i in range(3))
    q, k, v = (t.contiguous().requires_grad_() for t in (q, k, v))
    scale = hd ** -0.5
    m = ops.dense_map(S)
    out = torch.zeros(n * S, C, device=cuda, dtype=bf16)
    tq, tk, tv = (ops.TView(qkv, o, hs, m) for o in offs)
    to = ops.TView(out, 0, hd, m)
    kw = dict(n_seq=n, n_heads=heads, head_dim=hd, s_q=S, s_kv=S, causal=causal, scale=scale)
    lse = ops.attn_fwd(tq, tk, tv, to, **kw)
    assert lib.attn_last_path() == lib.ATTN_PATH_WGMMA    # no dense shape of the model falls back to mma.sync
    ref = _attn_ref(q, k, v, scale, causal)
    assert _rel(out.view(n, S, heads, hd).permute(0, 2, 1, 3), ref) < 2e-2
    dout = torch.randn(n * S, C, device=cuda).to(bf16)
    ref.backward(dout.float().view(n, S, heads, hd).permute(0, 2, 1, 3))
    dqkv = torch.zeros_like(qkv)
    tdo = ops.TView(dout, 0, hd, m)
    tdq, tdk, tdv = (ops.TView(dqkv, o, hs, m) for o in offs)
    ops.attn_bwd(tq, tk, tv, to, lse, tdo, tdq, tdk, tdv, **kw)
    assert lib.attn_last_path() == lib.ATTN_PATH_WGMMA
    if layout == "gpt":
        d5 = dqkv.float().view(n, S, heads, 3, hd)
        dq, dk, dv = (d5[:, :, :, i].permute(0, 2, 1, 3) for i in range(3))
    else:
        d5 = dqkv.float().view(n, S, 3, heads, hd)
        dq, dk, dv = (d5[:, :, i].permute(0, 2, 1, 3) for i in range(3))
    assert _rel(dq, q.grad) < 3e-2
    assert _rel(dk, k.grad) < 3e-2
    assert _rel(dv, v.grad) < 3e-2


@pytest.mark.parametrize("hd,S,total,causal", [(64, 100, 250, True), (96, 197, 300, False), (64, 256, 700, True)])
def test_attn_dense_ragged_total_rows(cuda, hd, S, total, causal):
    """Dense packed sequences whose last sequence is cut short by total_rows (forward + backward)."""
    from ymp import ops
    torch.manual_seed(12)
    heads = 2
    C = heads * hd
    n = (total + S - 1) // S
    qkv = (torch.randn(total, 3 * C, device=cuda) * 0.7).to(bf16)
    out = torch.zeros(total, C, device=cuda, dtype=bf16)
    m = ops.dense_map(S)
    tq, tk, tv = (ops.TView(qkv, i * C, hd, m) for i in range(3))
    kw = dict(n_seq=n, n_heads=heads, head_dim=hd, s_q=S, s_kv=S, causal=causal, scale=hd ** -0.5, total_rows=total)
    lse = ops.attn_fwd(tq, tk, tv, ops.TView(out, 0, hd, m), **kw)
    dout = torch.randn(total, C, device=cuda).to(bf16)
    dqkv = torch.zeros_like(qkv)
    ops.attn_bwd(tq, tk, tv, ops.TView(out, 0, hd, m), lse, ops.TView(dout, 0, hd, m),
                 *(ops.TView(dqkv, i * C, hd, m) for i in range(3)), **kw)
    for s in range(n):
        r0, r1 = s * S, min(total, (s + 1) * S)
        x = qkv[r0:r1].float().view(r1 - r0, 3, heads, hd)
        q, k, v = (x[:, i].permute(1, 0, 2)[None].contiguous().requires_grad_() for i in range(3))
        ref = _attn_ref(q, k, v, hd ** -0.5, causal)
        assert _rel(out[r0:r1].view(r1 - r0, heads, hd).permute(1, 0, 2)[None], ref) < 2e-2
        ref.backward(dout[r0:r1].float().view(r1 - r0, heads, hd).permute(1, 0, 2)[None])
        d = dqkv[r0:r1].float().view(r1 - r0, 3, heads, hd)
        for i, g in enumerate((q.grad, k.grad, v.grad)):
            assert _rel(d[:, i].permute(1, 0, 2)[None], g) < 3e-2, (s, i)


@pytest.mark.parametrize("hd,sq,skv", [(64, 70, 200), (96, 256, 33), (96, 129, 256), (64, 128, 128),
                                       (96, 128, 1570), (64, 300, 520), (80, 130, 300), (96, 16, 1000)])
def test_attn_cross_short_kv(cuda, hd, sq, skv):
    """Non-causal cross attention with s_q != s_kv on the tensor-core kernels: short key ranges and the long ones
    of the abstractor (128 queries x 1570 keys, models/vision_transformer.py:368-374)."""
    from ymp import lib, ops
    torch.manual_seed(21)
    n, heads = 3, 2
    C = heads * hd
    qb = (torch.randn(n * sq, C, device=cuda) * 0.7).to(bf16)
    kvb = (torch.randn(n * skv, 2 * C, device=cuda) * 0.7).to(bf16)
    out = torch.zeros(n * sq, C, device=cuda, dtype=bf16)
    mq, mkv = ops.dense_map(sq), ops.dense_map(skv)
    tq, tk, tv, to = ops.TView(qb, 0, hd, mq), ops.TView(kvb, 0, hd, mkv), ops.TView(kvb, C, hd, mkv), ops.TView(out, 0, hd, mq)
    kw = dict(n_seq=n, n_heads=heads, head_dim=hd, s_q=sq, s_kv=skv, causal=False, scale=hd ** -0.5)
    lse = ops.attn_fwd(tq, tk, tv, to, **kw)
    assert lib.attn_last_path() == lib.ATTN_PATH_WGMMA
    q = qb.float().view(n, sq, heads, hd).permute(0, 2, 1, 3).contiguous().requires_grad_()
    kv = kvb.float().view(n, skv, 2, heads, hd)
    k, v = (kv[:, :, i].permute(0, 2, 1, 3).contiguous().requires_grad_() for i in range(2))
    ref = _attn_ref(q, k, v, hd ** -0.5, False)
    assert _rel(out.view(n, sq, heads, hd).permute(0, 2, 1, 3), ref) < 2e-2
    dout = torch.randn(n * sq, C, device=cuda).to(bf16)
    ref.backward(dout.float().view(n, sq, heads, hd).permute(0, 2, 1, 3))
    dqb, dkvb = torch.zeros_like(qb), torch.zeros_like(kvb)
    ops.attn_bwd(tq, tk, tv, to, lse, ops.TView(dout, 0, hd, mq), ops.TView(dqb, 0, hd, mq), ops.TView(dkvb, 0, hd, mkv),
                 ops.TView(dkvb, C, hd, mkv), **kw)
    assert _rel(dqb.view(n, sq, heads, hd).permute(0, 2, 1, 3), q.grad) < 3e-2
    d = dkvb.float().view(n, skv, 2, heads, hd)
    assert _rel(d[:, :, 0].permute(0, 2, 1, 3), k.grad) < 3e-2
    assert _rel(d[:, :, 1].permute(0, 2, 1, 3), v.grad) < 3e-2


@pytest.mark.parametrize("hd", [64, 80, 96, 128])
def test_attn_device_side_key_count(cuda, hd):
    """ymp_attn_args.s_kv_dev (the captured decoding step): one query row per sequence over a cache of max_len rows of
    which only *s_kv_dev exist - identical to passing that count as s_kv, for every count, without re-building args."""
    from ymp import lib, ops
    torch.manual_seed(5)
    n, heads, ML = 5, 3, 200
    C = heads * hd
    qb = (torch.randn(n, C, device=cuda) * 0.7).to(bf16)
    kvb = (torch.randn(n * ML, 2 * C, device=cuda) * 0.7).to(bf16)
    mq, mkv = ops.dense_map(1), ops.dense_map(ML)
    tq, tk, tv = ops.TView(qb, 0, hd, mq), ops.TView(kvb, 0, hd, mkv), ops.TView(kvb, C, hd, mkv)
    cnt = torch.zeros(1, device=cuda, dtype=torch.int32)
    for L in (1, 31, 33, 127, 128, 129, 200):
        out_a, out_b = torch.zeros(n, C, device=cuda, dtype=bf16), torch.zeros(n, C, device=cuda, dtype=bf16)
        kw = dict(n_seq=n, n_heads=heads, head_dim=hd, s_q=1, causal=False, scale=hd ** -0.5)
        cnt.fill_(L)
        ops.attn_fwd(tq, tk, tv, ops.TView(out_a, 0, hd, mq), s_kv=ML, s_kv_dev=cnt, **kw)
        assert lib.attn_last_path() == (lib.ATTN_PATH_DECODE if hd != 128 else lib.ATTN_PATH_MMA_SYNC)
        ops.attn_fwd(tq, tk, tv, ops.TView(out_b, 0, hd, mq), s_kv=L, **kw)
        k = kvb.float().view(n, ML, 2, heads, hd)[:, :L]
        ref = _attn_ref(qb.float().view(n, 1, heads, hd).permute(0, 2, 1, 3), k[:, :, 0].permute(0, 2, 1, 3), k[:, :, 1].permute(0, 2, 1, 3),
                        hd ** -0.5, False)
        assert _rel(out_a.view(n, 1, heads, hd).permute(0, 2, 1, 3), ref) < 2e-2, L
        assert _rel(out_a, out_b.float()) < 1e-2, L   # (hd 128: the count-less call may run on another kernel family)
        if hd != 128:
            assert torch.equal(out_a, out_b), L


def test_attn_cross_shared_q(cuda):
    """Abstractor pattern: one shared query block for every sample, long KV with a ragged tail."""
    from ymp import ops
    torch.manual_seed(3)
    B, Q, S, heads, hd = 2, 128, 330, 8, 96
    C = heads * hd
    qp = (torch.randn(Q, C, device=cuda) * 0.5).to(bf16)
    kv = (torch.randn(B * S, 2 * C, device=cuda) * 0.5).to(bf16)
    out = torch.zeros(B * Q, C, device=cuda, dtype=bf16)
    mq = ops.seqmap(seq_div=1, outer_stride=0, pos_stride=1)  # every sequence reads the same rows
    mkv, mo = ops.dense_map(S), ops.dense_map(Q)
    tq, tk, tv, to = ops.TView(qp, 0, hd, mq), ops.TView(kv, 0, hd, mkv), ops.TView(kv, C, hd, mkv), ops.TView(out, 0, hd, mo)
    kw = dict(n_seq=B, n_heads=heads, head_dim=hd, s_q=Q, s_kv=S, causal=False, scale=hd ** -0.5)
    lse = ops.attn_fwd(tq, tk, tv, to, **kw)
    q = qp.float().view(1, Q, heads, hd).permute(0, 2, 1, 3).expand(B, -1, -1, -1).contiguous().requires_grad_()
    k = kv.float()[:, :C].reshape(B, S, heads, hd).permute(0, 2, 1, 3).contiguous().requires_grad_()
    v = kv.float()[:, C:].reshape(B, S, heads, hd).permute(0, 2, 1, 3).contiguous().requires_grad_()
    ref = _attn_ref(q, k, v, hd ** -0.5, False)
    assert _rel(out.view(B, Q, heads, hd).permute(0, 2, 1, 3), ref) < 2e-2
    dout = torch.randn(B * Q, C, device=cuda).to(bf16)
    ref.backward(dout.float().view(B, Q, heads, hd).permute(0, 2, 1, 3))
    dq = torch.zeros(B * Q, C, device=cuda, dtype=bf16)   # per-sample dq, summed by the caller
    dkv = torch.zeros_like(kv)
    ops.attn_bwd(tq, tk, tv, to, lse, ops.TView(dout, 0, hd, mo), ops.TView(dq, 0, hd, mo),
                 ops.TView(dkv, 0, hd, mkv), ops.TView(dkv, C, hd, mkv), **kw)
    assert _rel(dq.view(B, Q, heads, hd).permute(0, 2, 1, 3), q.grad) < 3e-2
    assert _rel(dkv[:, :C].reshape(B, S, heads, hd).permute(0, 2, 1, 3), k.grad) < 3e-2
    assert _rel(dkv[:, C:].reshape(B, S, heads, hd).permute(0, 2, 1, 3), v.grad) < 3e-2


def test_attn_timesformer_spatial_map(cuda):
    """Per-frame sequences [cls_b ; x[b, :, t]] read in place from the (b n t)+cls row layout."""
    from ymp import ops
    torch.manual_seed(4)
    B, N, T, heads, hd = 2, 9, 3, 2, 96
    C = heads * hd
    R = B * N * T
    qkv = (torch.randn(R + B, 3 * C, device=cuda) * 0.6).to(bf16)
    out = torch.zeros(R, C, device=cuda, dtype=bf16)
    cls_out = torch.zeros(B * T, C, device=cuda, dtype=bf16)
    m_in = ops.seqmap(seq_div=T, outer_stride=N * T, inner_stride=1, pos_stride=T, n_prefix=1,
                      prefix_base=R, prefix_stride=1, prefix_per_seq=0)
    # outputs: tokens back in (b n t) rows of `out`; the per-frame cls outputs go to cls_out[(b t)]
    big = torch.cat([out, cls_out], 0)  # one buffer: token rows then B*T cls rows
    m_out = ops.seqmap(seq_div=T, outer_stride=N * T, inner_stride=1, pos_stride=T, n_prefix=1,
                       prefix_base=R, prefix_stride=1, prefix_per_seq=1)
    kw = dict(n_seq=B * T, n_heads=heads, head_dim=hd, s_q=N + 1, s_kv=N + 1, causal=False, scale=hd ** -0.5)
    tq, tk, tv = (ops.TView(qkv, i * C, hd, m_in) for i in range(3))
    to = ops.TView(big, 0, hd, m_out)
    lse = ops.attn_fwd(tq, tk, tv, to, **kw)
    # reference: build the explicit sequences
    f = qkv.float()
    tok = f[:R].view(B, N, T, 3, heads, hd)
    cls = f[R:].view(B, 1, 1, 3, heads, hd).expand(B, 1, T, 3, heads, hd)
    seq = torch.cat([cls, tok], dim=1).permute(0, 2, 3, 4, 1, 5).reshape(B * T, 3, heads, N + 1, hd)
    q, k, v = (seq[:, i].contiguous().requires_grad_() for i in range(3))
    ref = _attn_ref(q, k, v, hd ** -0.5, False)          # [B*T, heads, N+1, hd]
    got_tok = big[:R].float().view(B, N, T, heads, hd).permute(0, 2, 3, 1, 4).reshape(B * T, heads, N, hd)
    got_cls = big[R:].float().view(B * T, heads, 1, hd)
    assert _rel(got_tok, ref[:, :, 1:]) < 2e-2
    assert _rel(got_cls, ref[:, :, :1]) < 2e-2
    # backward: token grads in place, cls-row grads per frame (caller sums over T)
    dbig = torch.randn_like(big.float()).to(bf16)
    dref = torch.cat([dbig[R:].float().view(B * T, heads, 1, hd),
                      dbig[:R].float().view(B, N, T, heads, hd).permute(0, 2, 3, 1, 4).reshape(B * T, heads, N, hd)], 2)
    ref.backward(dref)
    dqkv = torch.zeros(R + B * T, 3 * C, device=cuda, dtype=bf16)
    tdq, tdk, tdv = (ops.TView(dqkv, i * C, hd, m_out) for i in range(3))
    ops.attn_bwd(tq, tk, tv, to, lse, ops.TView(dbig, 0, hd, m_out), tdq, tdk, tdv, **kw)
    for i, gr in enumerate((q.grad, k.grad, v.grad)):
        d = dqkv.float()[:, i * C:(i + 1) * C]
        d_tok = d[:R].view(B, N, T, heads, hd).permute(0, 2, 3, 1, 4).reshape(B * T, heads, N, hd)
        d_cls = d[R:].view(B * T, heads, 1, hd)
        assert _rel(d_tok, gr[:, :, 1:]) < 3e-2, i
        assert _rel(d_cls, gr[:, :, :1]) < 3e-2, i


@pytest.mark.parametrize("S,heads,hd,n", [(8, 8, 96, 37), (4, 2, 96, 16), (2, 2, 64, 5), (16, 4, 80, 9), (12, 2, 64, 7)])
def test_attn_temporal_packed(cuda, S, heads, hd, n):
    """Short sequences packed into 64-row tiles with a block-diagonal mask (ragged last tile)."""
    from ymp import ops
    torch.manual_seed(5)
    C = heads * hd
    R = n * S
    qkv = (torch.randn(R, 3 * C, device=cuda) * 0.6).to(bf16)
    out = torch.zeros(R, C, device=cuda, dtype=bf16)
    scale = hd ** -0.5
    lse = ops.attn_temporal_fwd(qkv, out, R=R, n_heads=heads, T=S, D=hd, scale=scale)
    q5 = qkv.float().view(n, S, 3, heads, hd)
    q, k, v = (q5[:, :, i].permute(0, 2, 1, 3).contiguous().requires_grad_() for i in range(3))
    ref = _attn_ref(q, k, v, scale, False)
    assert _rel(out.view(n, S, heads, hd).permute(0, 2, 1, 3), ref) < 2e-2
    dout = torch.randn(R, C, device=cuda).to(bf16)
    ref.backward(dout.float().view(n, S, heads, hd).permute(0, 2, 1, 3))
    dqkv = torch.zeros_like(qkv)
    ops.attn_temporal_bwd(qkv, out, lse, dout, dqkv, R=R, n_heads=heads, T=S, D=hd, scale=scale)
    d5 = dqkv.float().view(n, S, 3, heads, hd)
    for i, gr in enumerate((q.grad, k.grad, v.grad)):
        assert _rel(d5[:, :, i].permute(0, 2, 1, 3), gr) < 3e-2, i


def test_im2col_matches_conv(cuda):
    from ymp import ops
    torch.manual_seed(6)
    B, T, H, P, D = 2, 3, 64, 16, 128
    video = torch.randn(B, 3, T, H, H, device=cuda).to(bf16)
    w = (torch.randn(D, 3, P, P, device=cuda) * 0.05).to(bf16)
    patches = ops.im2col(video, P)
    y = ops.gemm(patches, w.view(D, -1))
    N = (H // P) ** 2
    ref = torch.nn.functional.conv2d(video.float().permute(0, 2, 1, 3, 4).reshape(B * T, 3, H, H), w.float(), stride=P)
    ref = ref.flatten(2).transpose(1, 2).reshape(B, T, N, D).permute(0, 2, 1, 3).reshape(B * N * T, D)
    assert _rel(y, ref) < 1e-2
    # bit-exact gather
    ref_p = video.view(B, 3, T, H // P, P, H // P, P).permute(0, 3, 5, 2, 1, 4, 6).reshape(B * N * T, 3 * P * P)
    assert torch.equal(patches, ref_p)


def test_embed_gather_bit_exact(cuda):
    from ymp import ops
    torch.manual_seed(7)
    B, Ln, Q, Hd, V = 3, 10, 6, 256, 1000
    S = Q + Ln
    table = torch.randn(V, Hd, device=cuda).to(bf16)
    pos = torch.randn(64, Hd, device=cuda).to(bf16)
    ids = torch.randint(0, V, (B, Ln), device=cuda)
    out = torch.zeros(B * S, Hd, device=cuda, dtype=bf16)
    ops.embed_gather(ids, table, pos, out, S, Q)
    ref = (table[ids].float() + pos[Q:Q + Ln].float()[None]).to(bf16)
    assert torch.equal(out.view(B, S, Hd)[:, Q:], ref)
    assert out.view(B, S, Hd)[:, :Q].abs().sum() == 0
    out2 = torch.zeros(B * S, Hd, device=cuda, dtype=bf16)
    ops.embed_gather(ids, table, None, out2, S, Q)
    assert torch.equal(out2.view(B, S, Hd)[:, Q:], table[ids])


@pytest.mark.parametrize("V", [512, 51200, 1000])
def test_cross_entropy(cuda, V):
    from ymp import ops
    torch.manual_seed(8)
    rows = 33
    logits = (torch.randn(rows, V, device=cuda) * 3).to(bf16)
    labels = torch.randint(0, V, (rows,), device=cuda)
    loss, lse = ops.ce_fwd(logits, labels)
    lf = logits.float().requires_grad_()
    ref = torch.nn.functional.cross_entropy(lf, labels, reduction="none")
    assert _rel(loss, ref) < 1e-4
    g = torch.rand(rows, device=cuda)
    g[::5] = 0
    ref.backward(g)
    d = ops.ce_bwd(logits, labels, lse, g, dlogits=torch.empty_like(logits))
    assert _rel(d, lf.grad) < 1e-2
    d2 = ops.ce_bwd(logits.clone(), labels, lse, g)  # in place
    assert torch.equal(d2, d)


def test_fp32_stream_epilogues(cuda):
    """fp32 residual in / fp32 out of the GEMM epilogue and fp32 rows from the embedding gather."""
    from ymp import ops
    torch.manual_seed(12)
    M, N, K = 300, 256, 128
    a = torch.randn(M, K, device=cuda).to(bf16)
    w = (torch.randn(N, K, device=cuda) * 0.1).to(bf16)
    res = torch.randn(M, N, device=cuda)
    out = ops.gemm(a, w, residual=res, out_dtype=torch.float32)
    assert out.dtype == torch.float32
    assert _rel(out, a.float() @ w.float().t() + res) < 1e-5
    out_bf = ops.gemm(a, w, residual=res)
    assert out_bf.dtype == bf16 and _rel(out_bf, a.float() @ w.float().t() + res) < 1e-2
    table = torch.randn(100, 256, device=cuda).to(bf16)
    pos = torch.randn(32, 256, device=cuda).to(bf16)
    ids = torch.randint(0, 100, (2, 5), device=cuda)
    o = torch.zeros(2 * 9, 256, device=cuda)
    ops.embed_gather(ids, table, pos, o, 9, 4)
    assert torch.equal(o.view(2, 9, 256)[:, 4:], table[ids].float() + pos[4:9].float()[None])


def test_colsum_and_group(cuda):
    from ymp import ops
    torch.manual_seed(9)
    x = torch.randn(1000, 768, device=cuda).to(bf16)
    out = torch.ones(768, device=cuda)
    ops.colsum(x, out)
    assert _rel(out, x.float().sum(0) + 1) < 1e-4
    xs = torch.randn(500, 2304, device=cuda).to(bf16)[:, 768:1536]  # strided slice
    o2 = torch.zeros(768, device=cuda)
    ops.colsum(xs, o2)
    assert _rel(o2, xs.float().sum(0)) < 1e-4
    G, T, C = 6, 8, 768
    y = torch.randn(G * T, C, device=cuda).to(bf16)
    o = torch.empty(G, C, device=cuda, dtype=bf16)
    ops.group_reduce(y, G, T, o, scale=1.0 / T)
    assert _rel(o, y.float().view(G, T, C).mean(1)) < 1e-2
    bb = torch.empty(G * T, C, device=cuda, dtype=bf16)
    ops.group_reduce(o, G, T, bb, scale=0.5, broadcast=True)
    assert _rel(bb.view(G, T, C), (o.float() * 0.5)[:, None].expand(G, T, C)) < 1e-2


def test_gemm_row_remap_and_broadcast_residual(cuda):
    from ymp import ops
    torch.manual_seed(10)
    B, Q, S, K, N = 3, 8, 20, 64, 128
    a = torch.randn(B * Q, K, device=cuda).to(bf16)
    w = (torch.randn(N, K, device=cuda) * 0.1).to(bf16)
    pos = torch.randn(32, N, device=cuda).to(bf16)
    out = torch.zeros(B * S, N, device=cuda, dtype=bf16)
    ops.gemm(a, w, residual=pos, res_row_mod=Q, out=out, d_row_block=Q, d_row_stride=S)
    ref = (a.float() @ w.float().t()).view(B, Q, N) + pos[:Q].float()[None]
    assert _rel(out.view(B, S, N)[:, :Q], ref) < 1e-2
    assert out.view(B, S, N)[:, Q:].abs().sum() == 0


@pytest.mark.parametrize("B,T,H,W,C", [(2, 3, 32, 24, 3), (1, 8, 224, 224, 3), (3, 2, 16, 8, 1), (2, 2, 8, 16, 4)])
def test_clip_normalize_bit_exact(cuda, B, T, H, W, C):
    """uint8 clips -> normalised bf16 model input: bit-exact against the reference's ClipToTensor + Normalize."""
    from ymp import ops
    g = torch.Generator().manual_seed(9)
    frames = torch.randint(0, 256, (B, T, H, W, C), generator=g, dtype=torch.uint8)
    mean, std = (port.CLIP_MEAN + [0.5])[:C], (port.CLIP_STD + [0.25])[:C]
    ref = port.clip_to_model_input(frames, mean, std)
    out = ops.clip_normalize(frames.to(cuda), mean, std)
    assert out.shape == ref.shape and out.dtype == torch.bfloat16
    assert torch.equal(out.cpu().view(torch.int16), ref.view(torch.int16))


def test_device_prefetcher_orders_copies(cuda):
    from ymp.data import DevicePrefetcher
    pf = DevicePrefetcher(cuda)
    hosts = [torch.full((1 << 20,), float(i)).pin_memory() for i in range(4)]
    pf.submit(hosts[0], hosts[1])
    pf.submit(hosts[2], hosts[3])
    with pytest.raises(RuntimeError):
        pf.submit(hosts[0])
    a, b = pf.take()
    c, d = pf.take()
    assert len(pf) == 0
    for t, v in ((a, 0.0), (b, 1.0), (c, 2.0), (d, 3.0)):
        assert t.is_cuda and float(t.sum()) == v * (1 << 20)


@pytest.mark.parametrize("B,T,H,W,D,tile_n", [(3, 8, 64, 48, 128, 0), (2, 16, 32, 64, 256, 0), (5, 8, 224, 224, 768, 512), (2, 8, 48, 32, 768, 128)])
def test_patch_embed_fused_im2col(cuda, B, T, H, W, D, tile_n):
    """The patch embedding as ONE GEMM whose operand tiles are gathered from the video by 5-D TMA boxes (forward: A
    operand; weight gradient: MN-major B operand) against the explicit im2col matrix (models/vision_transformer.py:392-398)."""
    from ymp import ops
    torch.manual_seed(31)
    P, C = 16, 3
    video = torch.randn(B, C, T, H, W, device=cuda).to(bf16)
    w = (torch.randn(D, C * P * P, device=cuda) * 0.05).to(bf16)
    bias = torch.randn(D, device=cuda).to(bf16)
    N = (H // P) * (W // P)
    table = torch.randn(N * T, D, device=cuda).to(bf16)
    patches = ops.im2col(video, P)
    want = ops.gemm(patches, w, bias=bias, residual=table, res_row_mod=N * T, out_dtype=torch.float32, tile_n=tile_n)
    got = ops.patch_embed_gemm(video, w, P, bias=bias, residual=table, res_row_mod=N * T, out_dtype=torch.float32, tile_n=tile_n)
    assert torch.equal(got, want)                       # same tiles, same accumulation order: bit-identical
    ref = patches.float() @ w.float().t() + bias.float() + table.float().repeat(B, 1)
    assert _rel(got, ref) < 1e-2
    # K-range tail tiles and row tails: another weight width / more samples than one tile
    got2 = ops.patch_embed_gemm(video, w[: D // 2].contiguous(), P, out_dtype=torch.bfloat16, tile_n=tile_n)
    assert _rel(got2, patches.float() @ w[: D // 2].float().t()) < 1e-2
