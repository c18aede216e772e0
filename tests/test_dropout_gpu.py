"""GPU parity of the decoder's dropout (SURVEY 8a rows a10/a11/a13, the ★ row of the round-1 review): every
kernel that applies or back-propagates a dropout mask against the CPU oracle's Philox restatement
(oracle/philox.py, pinned by Random123 known-answer vectors) - masks bit-exact, values within bf16 tolerance -
and the whole model in train() mode against the UNMODIFIED reference run with the same masks
(tests/golden/tiny_pretrain_dropout.pt)."""
import os

import numpy as np
import pytest
import torch

from oracle import philox, port
from oracle.make_golden import make_inputs
from helpers import build_pretrain

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
bf16 = torch.bfloat16
SEED, OFFSET = 0x1234567812345, 7


def _rng(dev, seed=SEED, offset=OFFSET):
    return torch.tensor([seed, offset], dtype=torch.int64, device=dev)


def _rel(a, b):
    return ((a.float().cpu() - b.float().cpu()).abs().max() / (b.float().abs().max() + 1e-12)).item()


@pytest.mark.parametrize("dtype", [torch.float32, bf16])
def test_elementwise_dropout_mask_bit_exact(cuda, dtype):
    from ymp import ops
    R, C, p, site = 77, 2048, 0.1, 9
    x = torch.ones(R, C, device=cuda, dtype=dtype)
    y = ops.dropout(x.clone(), ops.Drop(_rng(cuda), site, p), row0=1000)
    keep = philox.keep_mask(SEED, OFFSET, site, np.arange(1000, 1000 + R), C, p)
    assert torch.equal((y != 0).cpu(), torch.from_numpy(keep))
    kept = y[y != 0].float()
    assert torch.allclose(kept, torch.full_like(kept, 1.0 / (1.0 - p)), rtol=4e-3 if dtype == bf16 else 1e-6)


@pytest.mark.parametrize("M,N,K,tile_n", [(300, 320, 256, 0), (512, 768, 768, 512), (1000, 2048, 2048, 512), (130, 264, 72, 128)])
def test_gemm_bias_dropout_add(cuda, M, N, K, tile_n):
    """out = residual + dropout(a b^T + bias)  (bias_dropout_add, modeling_distributed_gpt3.py:953-957) on every
    epilogue flavour: 1-CTA tiles, ragged N tail, CTA pairs with the TMA epilogue (K <= 1024) and the register one."""
    from ymp import ops
    torch.manual_seed(0)
    a = torch.randn(M, K, device=cuda).to(bf16)
    b = (torch.randn(N, K, device=cuda) * 0.05).to(bf16)
    bias = torch.randn(N, device=cuda).to(bf16)
    res = torch.randn(M, N, device=cuda)
    p, site = 0.1, 4 * 3 + 2
    out = ops.gemm(a, b, bias=bias, residual=res, out_dtype=torch.float32, tile_n=tile_n, drop=ops.Drop(_rng(cuda), site, p))
    pre = a.float() @ b.float().t() + bias.float()
    ref = res + philox.dropout(pre.cpu(), SEED, OFFSET, site, p).to(cuda)
    assert _rel(out, ref) < 1e-2
    dropped = torch.from_numpy(~philox.keep_mask(SEED, OFFSET, site, np.arange(M), N, p)).to(cuda)
    assert torch.equal(out[dropped], res[dropped])               # dropped positions pass the residual through exactly


def test_layernorm_bwd_second_output_is_dropout_backward(cuda):
    from ymp import ops
    torch.manual_seed(1)
    R, D, p, site = 200, 2048, 0.1, 4 * 2 + 3
    x = torch.randn(R, D, device=cuda)
    g = (1 + 0.1 * torch.randn(D, device=cuda)).to(bf16)
    b = torch.zeros(D, device=cuda, dtype=bf16)
    y, mean, rstd = ops.layernorm_fwd(x, g, b, 1e-5)
    dy = torch.randn(R, D, device=cuda).to(bf16)
    add = torch.randn(R, D, device=cuda).to(bf16)
    dx_plain = ops.layernorm_bwd(dy, x, g, mean, rstd, add=add)
    dx, dxd = ops.layernorm_bwd(dy, x, g, mean, rstd, add=add, drop=ops.Drop(_rng(cuda), site, p))
    assert torch.equal(dx, dx_plain)
    keep = torch.from_numpy(philox.keep_mask(SEED, OFFSET, site, np.arange(R), D, p)).to(cuda)
    assert torch.equal(dxd != 0, keep & (dx != 0))
    want = dx.float() * keep / (1 - p)
    assert _rel(dxd, want) < 1e-2
    # gathered rows (final LayerNorm over the text rows only): untouched rows stay zero in both outputs
    rows = torch.tensor([5, 17, 3, 150], dtype=torch.int32, device=cuda)
    y2, m2, r2 = ops.layernorm_fwd(x, g, b, 1e-5, in_rows=rows)
    dx0 = torch.zeros(R, D, device=cuda, dtype=bf16)
    dxg, dxgd = ops.layernorm_bwd(dy[:4].contiguous(), x, g, m2, r2, in_rows=rows, dx=dx0, drop=ops.Drop(_rng(cuda), site, p))
    sel = torch.zeros(R, dtype=torch.bool, device=cuda)
    sel[rows.long()] = True
    assert float(dxgd[~sel].abs().max()) == 0.0
    assert torch.equal(dxgd[sel] != 0, (keep & (dxg != 0))[sel])


def _attn_ref(q, k, v, scale, causal, keep, p):
    s = (q @ k.transpose(-1, -2)) * scale
    if causal:
        m = torch.ones(s.shape[-2:], dtype=torch.bool, device=s.device).triu(1)
        s = s.masked_fill(m, -10000.0)
    pr = s.softmax(-1)
    return (pr * keep / (1 - p)) @ v


@pytest.mark.parametrize("hd,heads,S,causal", [(64, 4, 256, True), (64, 2, 100, True), (80, 2, 384, True), (96, 2, 197, False),
                                               (64, 2, 520, False)])
def test_attention_dropout_fwd_bwd(cuda, hd, heads, S, causal):
    """O = dropout(P) V forward and backward on the wgmma kernels (GPT3CoreAttention, :768-782), masks regenerated in
    the backward from (seed, offset, site, row, key)."""
    from ymp import lib, ops
    torch.manual_seed(3)
    n, p, site = 2, 0.1, 4 * 5 + 1
    qkv = (torch.randn(n * S, 3 * heads * hd, device=cuda) * 0.7).to(bf16)
    qkv5 = qkv.float().view(n, S, heads, 3, hd)
    q, k, v = (qkv5[:, :, :, i].permute(0, 2, 1, 3).contiguous().requires_grad_() for i in range(3))
    m = ops.dense_map(S)
    out = torch.zeros(n * S, heads * hd, device=cuda, dtype=bf16)
    tq, tk, tv = (ops.TView(qkv, i * hd, 3 * hd, m) for i in range(3))
    to = ops.TView(out, 0, hd, m)
    drop = ops.Drop(_rng(cuda), site, p)
    kw = dict(n_seq=n, n_heads=heads, head_dim=hd, s_q=S, s_kv=S, causal=causal, scale=hd ** -0.5, drop=drop)
    lse = ops.attn_fwd(tq, tk, tv, to, **kw)
    assert lib.attn_last_path() == lib.ATTN_PATH_WGMMA
    keep = torch.from_numpy(philox.keep_mask(SEED, OFFSET, site, np.arange(n * heads * S), S, p)).to(cuda).view(n, heads, S, S).float()
    ref = _attn_ref(q, k, v, hd ** -0.5, causal, keep, p)
    assert _rel(out.view(n, S, heads, hd).permute(0, 2, 1, 3), ref) < 2e-2
    # lse is that of the undropped probabilities
    lse_plain = ops.attn_fwd(tq, tk, tv, ops.TView(torch.zeros_like(out), 0, hd, m), **dict(kw, drop=None))
    assert torch.allclose(lse, lse_plain, rtol=1e-5, atol=1e-5)
    dout = torch.randn(n * S, heads * hd, device=cuda).to(bf16)
    ref.backward(dout.float().view(n, S, heads, hd).permute(0, 2, 1, 3))
    dqkv = torch.zeros_like(qkv)
    tdq, tdk, tdv = (ops.TView(dqkv, i * hd, 3 * hd, m) for i in range(3))
    ops.attn_bwd(tq, tk, tv, to, lse, ops.TView(dout, 0, hd, m), tdq, tdk, tdv, **kw)
    d5 = dqkv.float().view(n, S, heads, 3, hd)
    dq, dk, dv = (d5[:, :, :, i].permute(0, 2, 1, 3) for i in range(3))
    assert _rel(dq, q.grad) < 3e-2 and _rel(dk, k.grad) < 3e-2 and _rel(dv, v.grad) < 3e-2


def _text(ids, att, dev):
    import models.modeling_distributed_gpt3 as G
    return G.BatchEncoding(dict(input_ids=ids.to(dev), attention_mask=att.to(dev)))


def test_pretrain_train_mode_matches_reference_with_dropout(cuda):
    """DistributedGPT3_Pretrain in train() mode, hidden / attention dropout 0.1: loss, per-token losses and all
    gradients against the unmodified reference run with the same Philox masks."""
    from ymp import functional as YF
    fx = torch.load(os.path.join(GOLD, "tiny_pretrain_dropout.pt"), weights_only=False)
    d = fx["drop"]
    sd = port.init_state_dict(fx["vcfg"], fx["gcfg"], fx["Q"], seed=fx["wseed"], randomize=True)
    model = build_pretrain(fx["vcfg"], fx["gcfg"], fx["Q"], sd=sd, device=cuda, dtype=bf16, dropout=(d["p_hidden"], d["p_attn"]))
    video, ids, att = make_inputs(fx["B"], fx["vcfg"], fx["L"], fx["gcfg"]["vocab_size"], fx["iseed"])
    v = video.to(cuda).bfloat16()
    model.train()
    YF.set_dropout_seed(d["seed"])           # first decoder pass after seeding: offset 0 == the fixture's
    loss, _ = model(v, _text(ids, att, cuda))
    loss.backward()
    assert abs(loss.item() - fx["loss"].item()) < 1e-2 * abs(fx["loss"].item())
    Q = fx["Q"]
    assert _rel(model.last_losses[:, Q:-1], fx["losses"][:, Q:]) < 3e-2
    # the oracle on bf16-rounded weights with the same masks isolates kernel error from weight rounding
    train = set(port.trainable_keys(sd))
    psd = {k: t.bfloat16().float().requires_grad_(k in train) for k, t in sd.items()}
    res = port.pretrain_forward(video.bfloat16().float(), ids, att, psd, fx["vcfg"], fx["gcfg"], return_all=True, drop=d)
    res["loss"].backward()
    assert abs(loss.item() - res["loss"].item()) < 5e-3 * abs(res["loss"].item())
    worst = 0.0
    for k, prm in model.named_parameters():
        if k.startswith("text_decoder."):
            continue
        g_ref = psd[k].grad
        if g_ref.abs().max().item() < 1e-7:
            continue
        err = _rel(prm.grad, g_ref)
        worst = max(worst, err)
        assert err < 8e-2, (k, err)
    print("dropout model parity: worst grad rel err vs oracle", worst)
    # a second pass advances the offset: different masks, different loss; eval() switches dropout off
    loss2, _ = model(v, _text(ids, att, cuda))
    assert abs(loss2.item() - loss.item()) > 1e-4
    model.eval()
    with torch.no_grad():
        le, _ = model(v, _text(ids, att, cuda))
    assert abs(le.item() - fx["loss_eval"].item()) < 1e-2 * abs(fx["loss_eval"].item())


def test_graph_replay_draws_fresh_masks(cuda):
    """The captured training step reads {seed, offset} from device memory: consecutive replays on the SAME batch
    see different masks (losses differ), and re-seeding reproduces the sequence."""
    from ymp import functional as YF
    from ymp.train import TrainEngine
    sd = port.init_state_dict(port.VCFG_TINY, port.GCFG_TINY, 8, seed=3, randomize=True)
    video, ids, att = make_inputs(2, port.VCFG_TINY, 8, port.GCFG_TINY["vocab_size"], 100)
    v, t = video.to(cuda).bfloat16(), _text(ids, att, cuda)

    def run():
        YF.set_dropout_seed(99)
        eng = TrainEngine(build_pretrain(port.VCFG_TINY, port.GCFG_TINY, 8, sd=sd, device=cuda, dtype=bf16, dropout=(0.1, 0.1)), lr=0.0,
                          weight_decay=0.0)
        return [eng.train_step(v, t, use_graph=True, graph_warmup=1).item() for _ in range(4)], eng

    a, eng = run()
    assert any("graph" in st for st in eng._graphs.values())
    assert len({round(x, 5) for x in a}) == 4, a          # lr = 0: only the masks change from step to step
    b, _ = run()
    assert all(abs(x - y) < 1e-3 * abs(x) for x, y in zip(a, b)), (a, b)
