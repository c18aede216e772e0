"""GPU: scoring a video's texts against one copy of their common title columns.

The prefix-table attention call (a key prefix per video in one launch) against the square causal call on materialised
sequences and an fp32 reference, the shared pass with shared title columns against gpt_fwd on the repeated layout, and
the Cls / Retrieval_Cls eval branches on title-structured texts.  Every comparison with the repeated computation is
exact (torch.equal): each kernel computes a row on its own, so sharing the title rows changes no bit of a scored
value."""
import pytest
import torch

from oracle import port
from helpers import build_pretrain

pytestmark = pytest.mark.gpu
VC, GC = port.VCFG_TINY, port.GCFG_TINY


# ------------------------------------------------------------------------------------------ kernel
def _table_call(cuda, hd, V, t, Q, P, Ls, heads=2, seed=0):
    """q/k/v rows [N*Ls suffix | V*(Q + Pmax) blocks]; text n attends to the first Q + P_v rows of block n // t, then
    its own Ls rows.  Returns (O, lse) of the table call and, per video, (O, lse) of the square causal call on the
    materialised [block rows | suffix rows] sequences (suffix rows only) and the fp32 reference of the suffix rows."""
    from ymp import engine, lib, ops
    g = torch.Generator(device=cuda).manual_seed(seed)
    N, C, B = V * t, heads * hd, Q + max(P)
    T = N * Ls
    q, k, v = (torch.randn(T + V * B, C, device=cuda, generator=g).bfloat16() for _ in range(3))
    scale = hd ** -0.5
    m_txt, m_keys, _ = engine.shared_title_maps(V, t, Q, Ls, B - Q)
    table = torch.tensor([Q + p for p in P], device=cuda, dtype=torch.int32)
    o = torch.empty(T, C, device=cuda, dtype=torch.bfloat16)
    lse = ops.attn_fwd(ops.TView(q, 0, hd, m_txt), ops.TView(k, 0, hd, m_keys), ops.TView(v, 0, hd, m_keys),
                       ops.TView(o, 0, hd, m_txt), n_seq=N, n_heads=heads, head_dim=hd, s_q=Ls, s_kv=B + Ls, causal=True,
                       scale=scale, n_prefix=table)
    assert lib.attn_last_path() == lib.ATTN_PATH_WGMMA
    per_video = []
    for vi in range(V):
        S = Q + P[vi] + Ls
        ns = torch.arange(vi * t, (vi + 1) * t, device=cuda)
        idx = torch.cat([(T + vi * B + torch.arange(Q + P[vi], device=cuda))[None, :].expand(t, -1),
                         ns[:, None] * Ls + torch.arange(Ls, device=cuda)[None, :]], 1).reshape(-1)
        qm, km, vm = (x.index_select(0, idx).contiguous() for x in (q, k, v))
        om = torch.empty(t * S, C, device=cuda, dtype=torch.bfloat16)
        dm = ops.dense_map(S)
        lsem = ops.attn_fwd(ops.TView(qm, 0, hd, dm), ops.TView(km, 0, hd, dm), ops.TView(vm, 0, hd, dm),
                            ops.TView(om, 0, hd, dm), n_seq=t, n_heads=heads, head_dim=hd, s_q=S, s_kv=S, causal=True,
                            scale=scale)
        a = Q + P[vi]
        qf = qm.view(t, S, heads, hd)[:, a:].float().transpose(1, 2)
        kf, vf = (x.view(t, S, heads, hd).float().transpose(1, 2) for x in (km, vm))
        s = (qf @ kf.transpose(-1, -2) * scale).masked_fill(
            torch.arange(S, device=cuda)[None, :] > (torch.arange(Ls, device=cuda)[:, None] + a), float("-inf"))
        ref = (s.softmax(-1) @ vf).transpose(1, 2).reshape(t * Ls, C)
        per_video.append(((om.view(t, S, C)[:, a:].reshape(t * Ls, C), lsem[:, :, a:]), (ref, torch.logsumexp(s, -1))))
    return (o, lse), per_video


# Q + P_v mod 64: 0, 1, 63, 1, 0 (Q = 128), and a prefix shorter than one tile (Q = 8)
@pytest.mark.parametrize("hd", [64, 80, 88, 96])
@pytest.mark.parametrize("s_q", [1, 5, 64, 70])
@pytest.mark.parametrize("Q,P", [(128, [0, 1, 63, 65, 64]), (8, [0, 55, 56])])
def test_prefix_table_matches_square_call_and_reference(cuda, hd, s_q, Q, P):
    V, t = len(P), 3
    (o, lse), per_video = _table_call(cuda, hd, V, t, Q, P, s_q)
    for vi, ((o_sq, lse_sq), (ref, ref_lse)) in enumerate(per_video):
        rows = slice(vi * t * s_q, (vi + 1) * t * s_q)
        assert torch.equal(o[rows], o_sq), vi
        assert torch.equal(lse[vi * t:(vi + 1) * t], lse_sq), vi
        err = (o[rows].float() - ref).abs().max().item()
        assert err <= 2e-2 * ref.abs().max().item(), (vi, err)
        assert (lse[vi * t:(vi + 1) * t] - ref_lse).abs().max().item() < 2e-2


def test_prefix_table_rejections(cuda):
    from ymp import engine, lib, ops
    V, t, Q, P, Ls, heads = 2, 2, 16, [3, 0], 8, 2
    B = Q + max(P)
    m_txt, m_keys, _ = engine.shared_title_maps(V, t, Q, Ls, B - Q)
    rows = V * t * Ls + V * B
    table = torch.tensor([Q + p for p in P], device=cuda, dtype=torch.int32)

    def views(hd):
        q, k, v = (torch.randn(rows, heads * hd, device=cuda).bfloat16() for _ in range(3))
        o = torch.empty(V * t * Ls, heads * hd, device=cuda, dtype=torch.bfloat16)
        return (ops.TView(q, 0, hd, m_txt), ops.TView(k, 0, hd, m_keys), ops.TView(v, 0, hd, m_keys), ops.TView(o, 0, hd, m_txt))

    kw = dict(n_seq=V * t, n_heads=heads, s_q=Ls, s_kv=B + Ls, causal=True, scale=0.125)
    with pytest.raises(lib.YmpError, match="head_dim"):
        ops.attn_fwd(*views(128), head_dim=128, n_prefix=table, **kw)
    rng = torch.tensor([7, 0], dtype=torch.int64, device=cuda)
    with pytest.raises(lib.YmpError, match="dropout"):
        ops.attn_fwd(*views(64), head_dim=64, drop=ops.Drop(rng, ops.site_attn(0), 0.1), n_prefix=table, **kw)
    q, k, v, o = views(64)
    args = ops._attn_args(q, k, v, o, None, head_dim=64, **kw)
    ta = lib.AttnPrefixTableArgs()
    ta.attn, ta.n_prefix = args, None
    with pytest.raises(lib.YmpError, match="null n_prefix"):
        lib.call(lib._attn_fwd_prefix_table, ta, "ymp_attn_fwd_prefix_table")
    ta.attn, ta.n_prefix = ops._attn_args(q, k, v, o, None, head_dim=64, **dict(kw, s_q=0)), table.data_ptr()
    with pytest.raises(lib.YmpError, match="bad sizes"):
        lib.call(lib._attn_fwd_prefix_table, ta, "ymp_attn_fwd_prefix_table")
    # forward only: the backward rejects the offset geometry the table call serves
    lse = ops.attn_fwd(q, k, v, o, head_dim=64, n_prefix=table, **kw)
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


W13 = dict(port.GCFG_1_3B, num_hidden_layers=2, vocab_size=4096)
W27 = dict(port.GCFG_2_7B, num_hidden_layers=2, vocab_size=4096)


@pytest.mark.parametrize("gcfg,t,Q,L,P,Le", [
    (GC, 3, 8, 24, [5, 0], [9, 24]),
    (GC, 2, 8, 24, [0, 0, 0], [24, 10, 3]),
    (W13, 4, 128, 80, [20, 0, 63], [26, 5, 68]),
    (W13, 3, 100, 66, [12, 60], [17, 66]),
    (W27, 3, 128, 80, [1, 40, 64], [80, 45, 69]),
    (W27, 2, 100, 40, [0, 31], [40, 35]),
], ids=["tiny", "tiny_unshared", "1.3B_width", "1.3B_width_q100", "2.7B_width", "2.7B_width_q100"])
def test_shared_title_pass_is_bit_identical_to_repeated(cuda, gcfg, t, Q, L, P, Le):
    """Text columns of the shared pass (video v's texts share their first P_v columns and use Le_v) against gpt_fwd +
    LM head + CE on the repeated [N, Q + L] layout: final hidden states and per-token losses are equal bit for bit;
    columns not computed read +0."""
    from ymp import engine, functional as YF
    V = len(P)
    W = _decoder_weights(cuda, gcfg, seed=Q + L)
    H, N, S = gcfg["hidden_size"], V * t, Q + L
    g = torch.Generator(device=cuda).manual_seed(3)
    qf = torch.randn(V, Q, H, device=cuda, generator=g).bfloat16()
    emb = (0.5 * torch.randn(N, L, H, device=cuda, generator=g)).bfloat16()
    for v, p in enumerate(P):   # the texts of video v agree on their first P_v columns
        emb[v * t:(v + 1) * t, :p] = emb[v * t, :p]
    labels = torch.randint(0, gcfg["vocab_size"], (N, S), device=cuda, generator=g)
    pos = W[engine.GPT + "embedding.position_embeddings.weight"]
    x = (torch.cat([qf.repeat_interleave(t, 0), emb], 1).float() + pos[:S][None].float()).reshape(N * S, H).contiguous()
    hid, _ = engine.gpt_fwd(W, x, gcfg, N, S, save=False)
    _, losses, _ = engine.lm_head_fwd(W, hid, labels)
    hid_rep = hid.view(N, S, H)[:, Q:]
    loss_rep = losses.view(N, S)[:, Q:]
    _, Ls, _ = YF.shared_title_layout(V, L, P, Le)
    j = torch.arange(L, device=cuda)[None, :]
    p_n = torch.tensor(P, device=cuda).repeat_interleave(t)[:, None]
    le_n = torch.tensor(Le, device=cuda).repeat_interleave(t)[:, None]
    computed = (j < p_n + Ls).expand(N, L)   # every text column that has a row in the shared pass
    scored = (j >= p_n) & computed           # ... and a loss (the LM head runs on the suffix rows only)
    assert bool((j < le_n).le(computed).all())

    keys, params = list(W), list(W.values())
    l_sh, h_none = YF.gpt_shared_prefix(qf, emb, labels[:, Q:], None, gcfg, keys, params, shared=P, used=Le)
    assert h_none is None and l_sh.shape == (N, L)
    assert torch.equal(l_sh[scored], loss_rep[scored])
    assert bool((l_sh[~scored] == 0).all()) and not torch.signbit(l_sh[~scored]).any()
    _, h_sh = YF.gpt_shared_prefix(qf, emb, None, None, gcfg, keys, params, shared=P, used=Le)
    h_sh = h_sh.view(N, L, H)
    assert torch.equal(h_sh[computed], hid_rep[computed])
    assert bool((h_sh[~computed] == 0).all())
    # requested rows anywhere in each text's used columns, some of them in its shared columns
    cols = (torch.rand(N, device=cuda, generator=g) * le_n[:, 0]).long()
    rows = torch.arange(N, device=cuda) * L + cols
    l_r, h_rows = YF.gpt_shared_prefix(qf, emb, labels[:, Q:], rows, gcfg, keys, params, shared=P, used=Le)
    assert torch.equal(h_rows, hid_rep.reshape(N * L, H)[rows])
    assert torch.equal(l_r, l_sh)


# ------------------------------------------------------------------------------------------ models
BOS, EOS = 1, 2


def _titles(V, t, L, vocab, lo, hi, seed, cls_name):
    """Cls-style texts: per video a title prompt of lo..hi tokens, its t class labels of 1-4 tokens (the same class
    list for every video; some share a first token), laid out as DistributedGPT3Tokenizer._fit_prompt does, padded to
    L; and the prompt_text rows of the cls pass ([bos | prompt | eos]: one per video for Cls, one per pair for ITM)."""
    g = torch.Generator().manual_seed(seed)
    labels = [torch.randint(3, vocab, (int(torch.randint(1, 5, (1,), generator=g)),), generator=g).tolist() for _ in range(t)]
    labels[1][0] = labels[0][0]
    ids, att, plen, pids, patt = [], [], [], [], []
    for _ in range(V):
        prompt = torch.randint(3, vocab, (int(torch.randint(lo, hi + 1, (1,), generator=g)),), generator=g).tolist()
        for lab in labels:
            room = L - len(lab) - 2
            pr = prompt[:room] if 2 + len(prompt) + len(lab) > L else prompt
            row = [BOS] + pr + lab + [EOS]
            ids.append(row + [0] * (L - len(row)))
            att.append([1] * len(row) + [0] * (L - len(row)))
            plen.append(len(pr))
        for _ in range(1 if cls_name == "DistributedGPT3_Cls" else t):
            row = ([BOS] + prompt + [EOS])[:L]
            pids.append(row + [0] * (L - len(row)))
            patt.append([1] * len(row) + [0] * (L - len(row)))
    text = dict(input_ids=torch.tensor(ids), attention_mask=torch.tensor(att), prompt_lengths=torch.tensor(plen))
    return text, dict(input_ids=torch.tensor(pids), attention_mask=torch.tensor(patt))


def _enc(dev, d):
    import models.modeling_distributed_gpt3 as G
    return G.BatchEncoding({k: v.to(dev) for k, v in d.items()})


def _repeated(m, video, text, prompt):
    """The eval branch composed with every video's prefix copied per text, then _gen_pass / _cls_pass."""
    _, _, _, qf = m.visual_prefix(video)
    V = qf.shape[0]
    t = text.input_ids.shape[0] // V
    qr = qf.repeat_interleave(t, 0)
    out, lm = m._gen_pass(qr, text)
    gen = (-(out.losses * lm).sum(-1)).view(V, t)
    if type(m).__name__ == "DistributedGPT3_Cls":
        return gen.softmax(-1), m._cls_pass(qf, prompt, False)
    return gen, m._cls_pass(qr, prompt, False).float().softmax(-1)[:, 1].view(V, t)


@pytest.mark.parametrize("cls_name", ["DistributedGPT3_Cls", "DistributedGPT3_Retrieval_Cls"])
@pytest.mark.parametrize("width", ["tiny", "1.3B_width"])
def test_eval_on_titles_equals_repeated_composition(cuda, monkeypatch, cls_name, width):
    from ymp import engine
    gcfg, Q, L, lo, hi = (GC, 8, 24, 4, 16) if width == "tiny" else (dict(port.GCFG_1_3B, num_hidden_layers=2), 128, 80, 12, 60)
    V, t = (3, 5) if cls_name == "DistributedGPT3_Cls" else (3, 4)
    torch.manual_seed(17)
    m = build_pretrain(VC, gcfg, Q, device=cuda, dtype=torch.bfloat16, cls_name=cls_name, num_frames=VC["num_frames"],
                       use_cls=True, num_classes=t if cls_name == "DistributedGPT3_Cls" else 2)
    video = torch.randn(V, 3, VC["num_frames"], VC["img_size"], VC["img_size"], generator=torch.Generator().manual_seed(4))
    video = video.to(cuda).bfloat16()
    text_d, prompt_d = _titles(V, t, L, gcfg["vocab_size"], lo, hi, 5, cls_name)
    text, prompt = _enc(cuda, text_d), _enc(cuda, prompt_d)
    calls = []
    real = engine.gpt_fwd_shared_prefix

    def recorded(*a, **k):
        calls.append(list(k.get("shared") or []))
        return real(*a, **k)
    monkeypatch.setattr(engine, "gpt_fwd_shared_prefix", recorded)
    with torch.no_grad():
        gen, cls = m(video, text, prompt, train=False)
        assert len(calls) == 2   # generation pass + cls pass
        gen_r, cls_r = _repeated(m, video, text, prompt)
    # the generation pass shared each video's bos + title: P_v = its prompt length
    plen = text_d["prompt_lengths"].view(V, t)
    assert calls[0] == plen.min(1).values.tolist() and min(calls[0]) > 0
    assert gen.shape == gen_r.shape and cls.shape == cls_r.shape
    assert torch.equal(gen, gen_r) and torch.equal(cls, cls_r)
