"""GPU: scoring many texts against one visual prefix.

Offset-causal attention (s_q < s_kv, bottom-right aligned) through a shared-prefix key map, the shared-prefix decoder
pass against gpt_fwd on the repeated layout, and the Cls / Retrieval_Cls eval branches that use it.  Every comparison
with the repeated computation is exact (torch.equal): each kernel computes a row on its own, so sharing the prefix
rows changes no bit of a text row."""
import pytest
import torch

from oracle import port
from helpers import build_pretrain

pytestmark = pytest.mark.gpu
VC, GC = port.VCFG_TINY, port.GCFG_TINY


# ------------------------------------------------------------------------------------------ kernel
def _offset_causal(cuda, hd, V, t, Q, L, heads=2, seed=0):
    """q/k/v rows [N*L text | V*Q prefix]; returns (O, lse) of the offset call, of the square call on the materialised
    [prefix | text] sequences (text rows only), and the fp32 reference of the text rows."""
    from ymp import engine, lib, ops
    g = torch.Generator(device=cuda).manual_seed(seed)
    N, S, C = V * t, Q + L, heads * hd
    T = N * L
    q, k, v = (torch.randn(T + V * Q, C, device=cuda, generator=g).bfloat16() for _ in range(3))
    scale = hd ** -0.5
    m_txt, m_keys, _ = engine.shared_prefix_maps(V, t, Q, L)
    o = torch.empty(T, C, device=cuda, dtype=torch.bfloat16)
    lse = ops.attn_fwd(ops.TView(q, 0, hd, m_txt), ops.TView(k, 0, hd, m_keys), ops.TView(v, 0, hd, m_keys),
                       ops.TView(o, 0, hd, m_txt), n_seq=N, n_heads=heads, head_dim=hd, s_q=L, s_kv=S, causal=True,
                       scale=scale)
    assert lib.attn_last_path() == lib.ATTN_PATH_WGMMA
    # materialised sequences n = [prefix n // t | text n]
    pre = torch.arange(N, device=cuda) // t
    idx = torch.cat([T + pre[:, None] * Q + torch.arange(Q, device=cuda)[None, :],
                     torch.arange(N, device=cuda)[:, None] * L + torch.arange(L, device=cuda)[None, :]], 1).reshape(-1)
    qm, km, vm = (x.index_select(0, idx).contiguous() for x in (q, k, v))
    om = torch.empty(N * S, C, device=cuda, dtype=torch.bfloat16)
    dm = ops.dense_map(S)
    lsem = ops.attn_fwd(ops.TView(qm, 0, hd, dm), ops.TView(km, 0, hd, dm), ops.TView(vm, 0, hd, dm), ops.TView(om, 0, hd, dm),
                        n_seq=N, n_heads=heads, head_dim=hd, s_q=S, s_kv=S, causal=True, scale=scale)
    o_sq = om.view(N, S, C)[:, Q:].reshape(T, C)
    lse_sq = lsem[:, :, Q:]
    # fp32 reference: query i of the text sees keys j <= i + Q of [prefix | text]
    qf = qm.view(N, S, heads, hd)[:, Q:].float().transpose(1, 2)
    kf, vf = (x.view(N, S, heads, hd).float().transpose(1, 2) for x in (km, vm))
    s = qf @ kf.transpose(-1, -2) * scale
    mask = torch.arange(S, device=cuda)[None, :] > (torch.arange(L, device=cuda)[:, None] + Q)
    s = s.masked_fill(mask, float("-inf"))
    ref = (s.softmax(-1) @ vf).transpose(1, 2).reshape(T, C)
    return (o, lse), (o_sq, lse_sq), (ref, torch.logsumexp(s, -1))


@pytest.mark.parametrize("hd", [64, 80])
@pytest.mark.parametrize("V,t,Q,L", [(2, 3, 128, 80), (3, 2, 8, 8), (1, 5, 100, 37), (2, 1, 64, 130), (2, 4, 128, 1)])
def test_offset_causal_attention_matches_square_call_and_reference(cuda, hd, V, t, Q, L):
    (o, lse), (o_sq, lse_sq), (ref, ref_lse) = _offset_causal(cuda, hd, V, t, Q, L)
    assert torch.equal(o, o_sq)
    assert torch.equal(lse, lse_sq)
    err = (o.float() - ref).abs().max().item()
    assert err <= 2e-2 * ref.abs().max().item(), err
    assert (lse - ref_lse).abs().max().item() < 2e-2


def test_offset_causal_rejections(cuda):
    from ymp import engine, lib, ops
    V, t, Q, L, heads = 2, 2, 16, 8, 2
    m_txt, m_keys, _ = engine.shared_prefix_maps(V, t, Q, L)
    rows = V * t * L + V * Q

    def views(hd):
        q, k, v = (torch.randn(rows, heads * hd, device=cuda).bfloat16() for _ in range(3))
        o = torch.empty(V * t * L, heads * hd, device=cuda, dtype=torch.bfloat16)
        return (ops.TView(q, 0, hd, m_txt), ops.TView(k, 0, hd, m_keys), ops.TView(v, 0, hd, m_keys), ops.TView(o, 0, hd, m_txt))

    kw = dict(n_seq=V * t, n_heads=heads, s_q=L, s_kv=Q + L, causal=True, scale=0.125)
    with pytest.raises(lib.YmpError, match="head_dim"):
        ops.attn_fwd(*views(128), head_dim=128, **kw)
    rng = torch.tensor([7, 0], dtype=torch.int64, device=cuda)
    with pytest.raises(lib.YmpError, match="dropout"):
        ops.attn_fwd(*views(64), head_dim=64, drop=ops.Drop(rng, ops.site_attn(0), 0.1), **kw)
    q, k, v, o = views(64)
    lse = ops.attn_fwd(q, k, v, o, head_dim=64, **kw)
    with pytest.raises(lib.YmpError, match="forward only"):
        ops.attn_bwd(q, k, v, o, lse, o, q, k, v, head_dim=64, **kw)


# ------------------------------------------------------------------------------------------ engine
def _decoder_weights(cuda, gcfg, seed):
    from ymp import engine
    H, F, Vv = gcfg["hidden_size"], gcfg["ffn_hidden_size"], gcfg["vocab_size"]
    g = torch.Generator(device=cuda).manual_seed(seed)
    W = {}
    for i in range(gcfg["num_hidden_layers"]):
        pre = f"{engine.GPT}encoder.layers.{i}."
        for nm in ("input_layernorm", "post_attention_layernorm"):
            W[pre + nm + ".weight"] = (1 + 0.1 * torch.randn(H, device=cuda, generator=g)).bfloat16()
            W[pre + nm + ".bias"] = (0.1 * torch.randn(H, device=cuda, generator=g)).bfloat16()
        for nm, (n, k) in (("self_attention.query_key_value", (3 * H, H)), ("self_attention.dense", (H, H)),
                           ("mlp.dense_h_to_4h", (F, H)), ("mlp.dense_4h_to_h", (H, F))):
            W[pre + nm + ".weight"] = (torch.randn(n, k, device=cuda, generator=g) * k ** -0.5).bfloat16()
            W[pre + nm + ".bias"] = (0.02 * torch.randn(n, device=cuda, generator=g)).bfloat16()
    W[engine.GPT + "encoder.final_layernorm.weight"] = (1 + 0.1 * torch.randn(H, device=cuda, generator=g)).bfloat16()
    W[engine.GPT + "encoder.final_layernorm.bias"] = (0.1 * torch.randn(H, device=cuda, generator=g)).bfloat16()
    W[engine.GPT + "embedding.word_embeddings.weight"] = (0.05 * torch.randn(Vv, H, device=cuda, generator=g)).bfloat16()
    W[engine.GPT + "embedding.position_embeddings.weight"] = (0.05 * torch.randn(gcfg["max_position_embeddings"], H, device=cuda,
                                                                               generator=g)).bfloat16()
    return W


@pytest.mark.parametrize("gcfg,V,t,Q,L,Le", [
    (GC, 2, 3, 8, 8, 8),
    (GC, 3, 2, 8, 12, 5),
    (dict(port.GCFG_1_3B, num_hidden_layers=2, vocab_size=4096), 2, 3, 128, 80, 80),
    (dict(port.GCFG_1_3B, num_hidden_layers=2, vocab_size=4096), 3, 2, 128, 80, 37),
    (dict(port.GCFG_2_7B, num_hidden_layers=2, vocab_size=4096), 2, 2, 128, 80, 80),
    (dict(port.GCFG_2_7B, num_hidden_layers=2, vocab_size=4096), 2, 3, 100, 64, 29),
], ids=["tiny", "tiny_trimmed", "1.3B_width", "1.3B_width_trimmed", "2.7B_width", "2.7B_width_q100_trimmed"])
def test_shared_prefix_pass_is_bit_identical_to_repeated(cuda, gcfg, V, t, Q, L, Le):
    """Text rows of the shared pass (over the first Le text columns) against gpt_fwd + LM head + CE on the repeated
    [N, Q + L] layout: final hidden states and per-token losses are equal bit for bit."""
    from ymp import engine, functional as YF
    W = _decoder_weights(cuda, gcfg, seed=Q + L)
    H, N, S = gcfg["hidden_size"], V * t, Q + L
    g = torch.Generator(device=cuda).manual_seed(3)
    qf = torch.randn(V, Q, H, device=cuda, generator=g).bfloat16()
    emb = (0.5 * torch.randn(N, L, H, device=cuda, generator=g)).bfloat16()
    labels = torch.randint(0, gcfg["vocab_size"], (N, S), device=cuda, generator=g)
    # repeated: GptFn's input chain on cat([prefix n // t, text n])
    pos = W[engine.GPT + "embedding.position_embeddings.weight"]
    x = (torch.cat([qf.repeat_interleave(t, 0), emb], 1).float() + pos[:S][None].float()).reshape(N * S, H).contiguous()
    hid, _ = engine.gpt_fwd(W, x, gcfg, N, S, save=False)
    _, losses, _ = engine.lm_head_fwd(W, hid, labels)
    hid_rep = hid.view(N, S, H)[:, Q:Q + Le]
    loss_rep = losses.view(N, S)[:, Q:Q + Le]
    keys, params = list(W), list(W.values())
    l_sh, h_none = YF.gpt_shared_prefix(qf, emb[:, :Le], labels[:, Q:Q + Le], None, gcfg, keys, params)
    assert h_none is None and l_sh.shape == (N, Le)
    assert torch.equal(l_sh, loss_rep)
    _, h_sh = YF.gpt_shared_prefix(qf, emb[:, :Le], None, None, gcfg, keys, params)
    assert torch.equal(h_sh.view(N, Le, H), hid_rep)
    rows = torch.arange(N, device=cuda) * Le + torch.randint(0, Le, (N,), device=cuda, generator=g)
    _, h_rows = YF.gpt_shared_prefix(qf, emb[:, :Le], None, rows, gcfg, keys, params)
    assert torch.equal(h_rows, hid_rep.reshape(N * Le, H)[rows])


# ------------------------------------------------------------------------------------------ models
def _enc(dev, **kw):
    import models.modeling_distributed_gpt3 as G
    return G.BatchEncoding({k: v.to(dev) for k, v in kw.items()})


def _texts(n, L, vocab, seed, lo, prompt):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(3, vocab, (n, L), generator=g)
    lens = torch.randint(lo, L + 1, (n,), generator=g)
    att = (torch.arange(L)[None, :] < lens[:, None]).long()
    d = dict(input_ids=torch.where(att.bool(), ids, torch.zeros_like(ids)), attention_mask=att)
    if prompt:
        d["prompt_lengths"] = torch.minimum(torch.randint(1, 4, (n,), generator=g), lens - 1)
    return d


def _model(cuda, cls_name, gcfg, Q, ncls, dropout=(0.0, 0.0)):
    torch.manual_seed(17)
    return build_pretrain(VC, gcfg, Q, device=cuda, dtype=torch.bfloat16, cls_name=cls_name, num_frames=VC["num_frames"],
                          use_cls=True, num_classes=ncls, dropout=dropout)


def _repeated(m, video, text, prompt):
    """The eval branch composed as before the shared pass: prefixes copied per text, then _gen_pass / _cls_pass."""
    _, _, _, qf = m.visual_prefix(video)
    V = qf.shape[0]
    t = text.input_ids.shape[0] // V
    qr = qf.repeat_interleave(t, 0)
    out, lm = m._gen_pass(qr, text)
    gen = (-(out.losses * lm).sum(-1)).view(V, t)
    if type(m).__name__ == "DistributedGPT3_Cls":
        return gen.softmax(-1), m._cls_pass(qf, prompt, False)
    return gen, m._cls_pass(qr, prompt, False).float().softmax(-1)[:, 1].view(V, t)


def _count_shared(monkeypatch):
    from ymp import engine
    calls = []
    real = engine.gpt_fwd_shared_prefix

    def counted(*a, **k):
        calls.append(1)
        return real(*a, **k)
    monkeypatch.setattr(engine, "gpt_fwd_shared_prefix", counted)
    return calls


@pytest.mark.parametrize("cls_name", ["DistributedGPT3_Cls", "DistributedGPT3_Retrieval_Cls"])
@pytest.mark.parametrize("width", ["tiny", "1.3B_width"])
def test_eval_outputs_equal_repeated_composition(cuda, monkeypatch, cls_name, width):
    gcfg, Q, L = (GC, 8, 8) if width == "tiny" else (dict(port.GCFG_1_3B, num_hidden_layers=2), 128, 40)
    V, t = (2, 5) if cls_name == "DistributedGPT3_Cls" else (3, 4)
    m = _model(cuda, cls_name, gcfg, Q, t if cls_name == "DistributedGPT3_Cls" else 2)
    video = torch.randn(V, 3, VC["num_frames"], VC["img_size"], VC["img_size"], generator=torch.Generator().manual_seed(4))
    video = video.to(cuda).bfloat16()
    n_prompt = V if cls_name == "DistributedGPT3_Cls" else V * t
    calls = _count_shared(monkeypatch)
    for lo in (L, 2):   # all texts at full length, then varying lengths (trailing columns trimmed)
        text = _enc(cuda, **_texts(V * t, L, gcfg["vocab_size"], 5 + lo, lo, True))
        prompt = _enc(cuda, **_texts(n_prompt, L, gcfg["vocab_size"], 6 + lo, lo, False))
        with torch.no_grad():
            n0 = len(calls)
            gen, cls = m(video, text, prompt, train=False)
            assert len(calls) - n0 == 2   # generation pass + cls pass
            gen_r, cls_r = _repeated(m, video, text, prompt)
        assert gen.shape == gen_r.shape and cls.shape == cls_r.shape
        assert torch.equal(gen, gen_r) and torch.equal(cls, cls_r)


@pytest.mark.parametrize("cls_name", ["DistributedGPT3_Cls", "DistributedGPT3_Retrieval_Cls"])
def test_eval_routing_keeps_repeated_path_when_needed(cuda, monkeypatch, cls_name):
    V, t, Q, L = 2, 3, 8, 8
    n_prompt = V if cls_name == "DistributedGPT3_Cls" else V * t
    video = torch.randn(V, 3, VC["num_frames"], VC["img_size"], VC["img_size"], generator=torch.Generator().manual_seed(8))
    video = video.to(cuda).bfloat16()
    text = _enc(cuda, **_texts(V * t, L, GC["vocab_size"], 9, 3, True))
    prompt = _enc(cuda, **_texts(n_prompt, L, GC["vocab_size"], 10, 3, False))
    calls = _count_shared(monkeypatch)
    # grad mode with trainable query features: the outputs keep their autograd history
    m = _model(cuda, cls_name, GC, Q, t)
    assert m.learnable_queries.requires_grad
    with torch.enable_grad():
        gen, cls = m(video, text, prompt, train=False)
    assert not calls and gen.grad_fn is not None
    # decoder dropout active (train mode, p = 0.1): repeated path even without grad
    m = _model(cuda, cls_name, GC, Q, t, dropout=(0.1, 0.1))
    assert m.text_decoder.training and m.text_decoder.dropout_active()
    with torch.no_grad():
        m(video, text, prompt, train=False)
    assert not calls
    with pytest.raises(ValueError, match="dropout"):
        m.text_decoder.forward_shared_prefix(torch.zeros(1, Q, GC["hidden_size"], device=cuda).bfloat16(),
                                             torch.zeros(1, L, GC["hidden_size"], device=cuda).bfloat16())
    # the same model in eval mode shares the prefixes
    m.eval()
    with torch.no_grad():
        m(video, text, prompt, train=False)
    assert len(calls) == 2
