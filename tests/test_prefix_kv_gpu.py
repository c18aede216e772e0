"""GPU: the evaluation's prefix cache - each video's decoder prefix keys and values computed once and read by every
scoring pass and text chunk against that video.

The prefix-cache attention call against the prefix-table call on one buffer with the cached rows copied in front of
the block rows, and against the float64 reference within the derived bounds; the shared pass with a PrefixKV against
the same pass without one and against gpt_fwd on the repeated layout; and the Cls / Retrieval_Cls eval calls, whose
outputs must not change by a bit while the visual encoder runs once per clip tensor.  Every comparison with the
uncached computation is exact (torch.equal): each kernel computes a row on its own."""
import pytest
import torch

import attn_bounds as AB
from oracle import port
from helpers import build_pretrain
from test_shared_title_gpu import W13, W27, _decoder_weights, _enc, _repeated, _titles

pytestmark = pytest.mark.gpu
VC, GC = port.VCFG_TINY, port.GCFG_TINY


# ------------------------------------------------------------------------------------------ kernel
def _cache_of(k, v, rows, heads, hd):
    """The PrefixKV layout of one layer: rows `rows` of k and v, each head's [k | v] side by side."""
    kv = torch.empty(rows.numel(), heads, 2, hd, device=k.device, dtype=torch.bfloat16)
    kv[:, :, 0] = k[rows].view(-1, heads, hd)
    kv[:, :, 1] = v[rows].view(-1, heads, hd)
    return kv.view(rows.numel(), 2 * heads * hd)


def _cache_views(kv, hd):
    from ymp import ops
    return ops.TView(kv, 0, 2 * hd, None), ops.TView(kv, hd, 2 * hd, None)


@pytest.mark.parametrize("hd", [64, 80, 88, 96])
@pytest.mark.parametrize("Q", [1, 63, 64, 128])
@pytest.mark.parametrize("s_q", [1, 70])
def test_prefix_kv_call_matches_table_call_and_reference(cuda, hd, Q, s_q):
    """Text rows (n0 = Q cached keys, then P_v title rows, then their own rows) and title rows (n0 = n_prefix = Q)
    against the single-buffer calls they replace: equal O and lse; and against the float64 reference."""
    from ymp import engine, lib, ops
    P, t, heads = [0, 5, 0, 64, 63], 2, 2
    V, N, C, Pmax = len(P), len(P) * t, heads * hd, max(P)
    B, T = Q + Pmax, len(P) * t * s_q
    g = torch.Generator(device=cuda).manual_seed(Q * 7 + s_q)
    q, k, v = (torch.randn(T + V * B, C, device=cuda, generator=g).bfloat16() for _ in range(3))
    scale = hd ** -0.5
    kw = dict(n_heads=heads, head_dim=hd, causal=True, scale=scale)
    # the single-buffer layout: [suffix rows | blocks of Q prefix rows + Pmax title rows]
    m_txt, m_keys, m_blk = engine.shared_title_maps(V, t, Q, s_q, Pmax)
    table = torch.tensor([Q + p for p in P], device=cuda, dtype=torch.int32)
    o_ref = torch.empty(T, C, device=cuda, dtype=torch.bfloat16)
    lse_ref = ops.attn_fwd(ops.TView(q, 0, hd, m_txt), ops.TView(k, 0, hd, m_keys), ops.TView(v, 0, hd, m_keys),
                           ops.TView(o_ref, 0, hd, m_txt), n_seq=N, s_q=s_q, s_kv=B + s_q, n_prefix=table, **kw)
    ob_ref = torch.empty(V * B, C, device=cuda, dtype=torch.bfloat16)
    lseb_ref = ops.attn_fwd(*(ops.TView(x[T:], 0, hd, m_blk) for x in (q, k, v)), ops.TView(ob_ref, 0, hd, m_blk),
                            n_seq=V, s_q=B, s_kv=B, **kw)
    # the cached layout: the blocks' prefix rows in a PrefixKV, the buffer holds [suffix rows | title rows]
    blk = torch.arange(V * B, device=cuda).view(V, B)
    kv = _cache_of(k, v, T + blk[:, :Q].reshape(-1), heads, hd)
    title = T + blk[:, Q:].reshape(-1)
    q2, k2, v2 = (torch.cat([x[:T], x[title]]) for x in (q, k, v))
    c_txt, c_keys, c_title = engine.cached_title_maps(V, t, s_q, Pmax)
    cache = (*_cache_views(kv, hd), Q)
    o = torch.empty(T, C, device=cuda, dtype=torch.bfloat16)
    lse = ops.attn_fwd(ops.TView(q2, 0, hd, c_txt), ops.TView(k2, 0, hd, c_keys), ops.TView(v2, 0, hd, c_keys),
                       ops.TView(o, 0, hd, c_txt), n_seq=N, s_q=s_q, s_kv=B + s_q, n_prefix=table, cache=cache, **kw)
    assert lib.attn_last_path() == lib.ATTN_PATH_WGMMA
    assert torch.equal(o, o_ref) and torch.equal(lse, lse_ref)
    ot = torch.empty(V * Pmax, C, device=cuda, dtype=torch.bfloat16)
    n_title = torch.full((V,), Q, device=cuda, dtype=torch.int32)
    lset = ops.attn_fwd(*(ops.TView(x[T:], 0, hd, c_title) for x in (q2, k2, v2)), ops.TView(ot, 0, hd, c_title),
                        n_seq=V, s_q=Pmax, s_kv=B, n_prefix=n_title, cache=cache, **kw)
    assert lib.attn_last_path() == lib.ATTN_PATH_WGMMA
    assert torch.equal(ot.view(V, Pmax, C), ob_ref.view(V, B, C)[:, Q:])
    assert torch.equal(lset, lseb_ref[:, :, Q:])
    # float64 reference of the text rows, one video at a time: keys [cached Q | title P_v | own rows]
    for vi in range(V):
        S = Q + P[vi] + s_q
        ns = torch.arange(vi * t, (vi + 1) * t, device=cuda)
        idx = torch.cat([(T + vi * B + torch.arange(Q + P[vi], device=cuda))[None, :].expand(t, -1),
                         ns[:, None] * s_q + torch.arange(s_q, device=cuda)[None, :]], 1)
        qs, ks, vs = (x[idx].view(t, S, heads, hd).transpose(1, 2) for x in (q, k, v))
        qs = qs[:, :, Q + P[vi]:]
        vis = AB.visible(t, s_q, S, AB.MASK_CAUSAL)
        ref = AB.reference(qs, ks, vs, vis, scale)
        e_o, e_lse = AB.fwd_bounds(qs, ks, vs, scale, ref)
        rows = slice(vi * t * s_q, (vi + 1) * t * s_q)
        got = o[rows].view(t, s_q, heads, hd).transpose(1, 2)
        assert AB.worst_ratio(got, ref["O"], e_o) <= 1.0, vi
        assert AB.worst_ratio(lse[vi * t:(vi + 1) * t], ref["lse"], e_lse) <= 1.0, vi


def test_prefix_kv_call_rejections(cuda):
    from ymp import engine, lib, ops
    V, t, Q, P, Ls, heads, hd = 2, 2, 16, [3, 0], 8, 2, 64
    m_txt, m_keys, _ = engine.cached_title_maps(V, t, Ls, max(P))
    rows = V * t * Ls + V * max(P)
    q, k, v = (torch.randn(rows, heads * hd, device=cuda).bfloat16() for _ in range(3))
    o = torch.empty(V * t * Ls, heads * hd, device=cuda, dtype=torch.bfloat16)
    views = (ops.TView(q, 0, hd, m_txt), ops.TView(k, 0, hd, m_keys), ops.TView(v, 0, hd, m_keys), ops.TView(o, 0, hd, m_txt))
    table = torch.tensor([Q + p for p in P], device=cuda, dtype=torch.int32)
    kv = torch.randn(V * Q, 2 * heads * hd, device=cuda).bfloat16()
    kw = dict(n_seq=V * t, n_heads=heads, head_dim=hd, s_q=Ls, s_kv=Q + max(P) + Ls, causal=True, scale=0.125)
    rng = torch.tensor([7, 0], dtype=torch.int64, device=cuda)
    with pytest.raises(lib.YmpError, match="dropout"):
        ops.attn_fwd(*views, drop=ops.Drop(rng, ops.site_attn(0), 0.1), n_prefix=table, cache=(*_cache_views(kv, hd), Q), **kw)
    odd = torch.randn(V * Q, 2 * heads * hd + 4, device=cuda).bfloat16()
    with pytest.raises(lib.YmpError, match="ld_cache"):
        ops.attn_fwd(*views, n_prefix=table, cache=(*_cache_views(odd, hd), Q), **kw)
    c = lib.AttnPrefixKvArgs()
    t_args = lib.AttnPrefixTableArgs()
    t_args.attn, t_args.n_prefix = ops._attn_args(*views, None, **kw), table.data_ptr()
    c.table, c.k_cache, c.v_cache, c.ld_cache, c.cache_head_stride, c.n0 = t_args, None, kv.data_ptr(), kv.stride(0), 2 * hd, Q
    with pytest.raises(lib.YmpError, match="k_cache"):
        lib.call(lib._attn_fwd_prefix_kv, c, "ymp_attn_fwd_prefix_kv")
    c.k_cache, c.n0 = kv.data_ptr(), -1
    with pytest.raises(lib.YmpError, match="n0"):
        lib.call(lib._attn_fwd_prefix_kv, c, "ymp_attn_fwd_prefix_kv")
    c.n0 = Q
    lib.call(lib._attn_fwd_prefix_kv, c, "ymp_attn_fwd_prefix_kv")
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------ engine
@pytest.mark.parametrize("gcfg,t,Q,L,P,Le", [
    (GC, 3, 8, 24, [5, 0], [9, 24]),
    (GC, 2, 8, 24, [0, 0, 0], [24, 10, 3]),
    (W13, 4, 128, 80, [20, 0, 63], [26, 5, 68]),
    (W13, 2, 128, 80, [0, 0], [80, 80]),
    (W27, 3, 128, 80, [1, 40, 64], [80, 45, 69]),
    (W27, 2, 100, 40, [0, 0], [40, 35]),
], ids=["tiny", "tiny_unshared", "1.3B_width", "1.3B_width_unshared", "2.7B_width", "2.7B_width_unshared"])
def test_shared_pass_with_prefix_kv_is_bit_identical(cuda, gcfg, t, Q, L, P, Le):
    """gpt_shared_prefix with a PrefixKV against the same call without one and against gpt_fwd + LM head + CE on the
    repeated [N, Q + L] layout: per-token losses and final hidden states equal bit for bit."""
    from ymp import engine, functional as YF
    V = len(P)
    W = _decoder_weights(cuda, gcfg, seed=Q + L + 1)
    H, N, S = gcfg["hidden_size"], V * t, Q + L
    g = torch.Generator(device=cuda).manual_seed(5)
    qf = torch.randn(V, Q, H, device=cuda, generator=g).bfloat16()
    emb = (0.5 * torch.randn(N, L, H, device=cuda, generator=g)).bfloat16()
    for v, p in enumerate(P):
        emb[v * t:(v + 1) * t, :p] = emb[v * t, :p]
    labels = torch.randint(0, gcfg["vocab_size"], (N, S), device=cuda, generator=g)
    keys, params = list(W), list(W.values())
    kv = YF.gpt_prefix_kv(qf, gcfg, keys, params)
    assert kv.kv.shape == (gcfg["num_hidden_layers"], V * Q, 2 * H) and kv.kv.dtype == torch.bfloat16
    cols = (torch.rand(N, device=cuda, generator=g) * torch.tensor(Le, device=cuda).repeat_interleave(t)).long()
    rows = torch.arange(N, device=cuda) * L + cols
    base = YF.gpt_shared_prefix(qf, emb, labels[:, Q:], rows, gcfg, keys, params, shared=P, used=Le)
    got = YF.gpt_shared_prefix(qf, emb, labels[:, Q:], rows, gcfg, keys, params, shared=P, used=Le, prefix_kv=kv)
    assert torch.equal(got[0], base[0]) and torch.equal(got[1], base[1])
    lazy = engine.PrefixKV.empty(gcfg, V, Q, cuda)   # filled by the first pass that receives it
    first = YF.gpt_shared_prefix(qf, emb, labels[:, Q:], rows, gcfg, keys, params, shared=P, used=Le, prefix_kv=lazy)
    assert lazy.filled and torch.equal(lazy.kv, kv.kv)
    assert torch.equal(first[0], base[0]) and torch.equal(first[1], base[1])
    h_all = YF.gpt_shared_prefix(qf, emb, None, None, gcfg, keys, params, shared=P, used=Le, prefix_kv=kv)[1]
    assert torch.equal(h_all, YF.gpt_shared_prefix(qf, emb, None, None, gcfg, keys, params, shared=P, used=Le)[1])
    # against the repeated layout
    pos = W[engine.GPT + "embedding.position_embeddings.weight"]
    x = (torch.cat([qf.repeat_interleave(t, 0), emb], 1).float() + pos[:S][None].float()).reshape(N * S, H).contiguous()
    hid, _ = engine.gpt_fwd(W, x, gcfg, N, S, save=False)
    _, losses, _ = engine.lm_head_fwd(W, hid, labels)
    assert torch.equal(got[1], hid.view(N, S, H)[:, Q:].reshape(N * L, H)[rows])
    _, Ls, _ = YF.shared_title_layout(V, L, P, Le)
    j = torch.arange(L, device=cuda)[None, :]
    p_n = torch.tensor(P, device=cuda).repeat_interleave(t)[:, None]
    scored = (j >= p_n) & (j < p_n + Ls)
    assert torch.equal(got[0][scored], losses.view(N, S)[:, Q:][scored])


def test_prefix_kv_handle_must_match_the_call(cuda):
    from ymp import functional as YF
    W = _decoder_weights(cuda, GC, seed=1)
    keys, params = list(W), list(W.values())
    H = GC["hidden_size"]
    qf = torch.randn(2, 8, H, device=cuda).bfloat16()
    emb = torch.randn(4, 10, H, device=cuda).bfloat16()
    kv3 = YF.gpt_prefix_kv(torch.randn(3, 8, H, device=cuda).bfloat16(), GC, keys, params)
    kvq = YF.gpt_prefix_kv(torch.randn(2, 6, H, device=cuda).bfloat16(), GC, keys, params)
    for bad in (kv3, kvq):
        with pytest.raises(ValueError, match="PrefixKV"):
            YF.gpt_shared_prefix(qf, emb, None, None, GC, keys, params, prefix_kv=bad)
    with pytest.raises(ValueError, match="PrefixKV"):   # another layer count
        YF.gpt_shared_prefix(qf, emb, None, None, dict(GC, num_hidden_layers=GC["num_hidden_layers"] + 1), keys, params,
                             prefix_kv=YF.gpt_prefix_kv(qf, GC, keys, params))


# ------------------------------------------------------------------------------------------ models
def _model(cuda, cls_name, t, dropout=(0.0, 0.0)):
    torch.manual_seed(17)
    return build_pretrain(VC, GC, 8, device=cuda, dtype=torch.bfloat16, cls_name=cls_name, num_frames=VC["num_frames"],
                          use_cls=True, num_classes=t if cls_name == "DistributedGPT3_Cls" else 2, dropout=dropout)


def _video(cuda, V, seed=4):
    v = torch.randn(V, 3, VC["num_frames"], VC["img_size"], VC["img_size"], generator=torch.Generator().manual_seed(seed))
    return v.to(cuda).bfloat16()


def _chunks(cuda, V, t, n):
    return [tuple(_enc(cuda, d) for d in _titles(V, t, 24, GC["vocab_size"], 4, 16, 30 + c, "DistributedGPT3_Retrieval_Cls"))
            for c in range(n)]


def _count_encoder(m):
    n = [0]
    m.visual_encoder.register_forward_hook(lambda *_: n.__setitem__(0, n[0] + 1))
    return n


def test_itm_chunk_loop_reuses_the_clip_and_stays_bit_identical(cuda):
    """The reference's ITM loop: one clip tensor, several text chunks.  Outputs equal those of calls whose cache is
    never reused (and the repeated composition); the encoder runs once per clip tensor, again after an in-place edit,
    for a clone, after an optimizer step and after train() / eval()."""
    from ymp import train
    V, t = 3, 4
    m = _model(cuda, "DistributedGPT3_Retrieval_Cls", t).eval()
    video = _video(cuda, V)
    chunks = _chunks(cuda, V, t, 3)
    enc = _count_encoder(m)
    with torch.no_grad():
        cached = [m(video, text, prompt, train=False) for text, prompt in chunks]
        assert enc[0] == 1 and m._prefix_cache is not None and m._prefix_cache[0] is video
        fresh = []
        for text, prompt in chunks:
            m._prefix_cache = None
            fresh.append(m(video, text, prompt, train=False))
        for (g, c), (gf, cf), (text, prompt) in zip(cached, fresh, chunks):
            assert torch.equal(g, gf) and torch.equal(c, cf)
            gr, cr = _repeated(m, video, text, prompt)
            assert torch.equal(g, gr) and torch.equal(c, cr)
        text, prompt = chunks[0]
        enc[0] = 0
        m(video, text, prompt, train=False)
        assert enc[0] == 0
        video[0, 0, 0, 0, 0] += 1                     # edited in place
        m(video, text, prompt, train=False)
        assert enc[0] == 1
        clone = video.clone()
        m(clone, text, prompt, train=False)
        m(clone, text, prompt, train=False)
        assert enc[0] == 2 and m._prefix_cache[0] is clone
        m.train()
        assert m._prefix_cache is None
        m.eval()
        m(clone, text, prompt, train=False)
        assert enc[0] == 3
    eng = train.TrainEngine(m, lr=1e-3)
    with torch.no_grad():
        m(clone, text, prompt, train=False)
        assert enc[0] == 4                           # the engine took the parameters over
        m(clone, text, prompt, train=False)
        assert enc[0] == 4
        eng.step()                                   # AdamW writes the weights through raw pointers
        after = m(clone, text, prompt, train=False)
        assert enc[0] == 5
        m._prefix_cache = None
        fresh = m(clone, text, prompt, train=False)
        assert torch.equal(after[0], fresh[0]) and torch.equal(after[1], fresh[1])


def test_no_cache_under_grad_or_dropout(cuda):
    V, t = 2, 3
    text, prompt = _chunks(cuda, V, t, 1)[0]
    video = _video(cuda, V)
    m = _model(cuda, "DistributedGPT3_Retrieval_Cls", t).eval()
    assert any(p.requires_grad for p in m.visual_encoder.parameters())
    enc = _count_encoder(m)
    with torch.enable_grad():                         # trainable prefixes under grad: no cache read or created
        m(video, text, prompt, train=False)
        m(video, text, prompt, train=False)
    assert enc[0] == 2 and m._prefix_cache is None
    md = _model(cuda, "DistributedGPT3_Retrieval_Cls", t, dropout=(0.1, 0.1)).train()
    enc = _count_encoder(md)
    with torch.no_grad():                             # train mode, dropout active
        md(video, text, prompt, train=False)
        md(video, text, prompt, train=False)
    assert enc[0] == 2 and md._prefix_cache is None


@pytest.mark.parametrize("cls_name", ["DistributedGPT3_Cls", "DistributedGPT3_Retrieval_Cls"])
def test_eval_passes_share_one_handle(cuda, monkeypatch, cls_name):
    from ymp import engine
    V, t = 3, 5
    m = _model(cuda, cls_name, t).eval()
    video = _video(cuda, V)
    text, prompt = (_enc(cuda, d) for d in _titles(V, t, 24, GC["vocab_size"], 4, 16, 5, cls_name))
    handles, built = [], []
    real_fwd, real_kv = engine.gpt_fwd_shared_prefix, engine.gpt_prefix_kv

    def rec_fwd(*a, **k):
        handles.append(k.get("prefix_kv"))
        return real_fwd(*a, **k)

    def rec_kv(*a, **k):
        built.append(real_kv(*a, **k))
        return built[-1]
    monkeypatch.setattr(engine, "gpt_fwd_shared_prefix", rec_fwd)
    monkeypatch.setattr(engine, "gpt_prefix_kv", rec_kv)
    with torch.no_grad():
        gen, cls = m(video, text, prompt, train=False)
        # the generation pass fills the handle, the cls pass reads it: no pass of its own
        assert not built and len(handles) == 2 and handles[0] is not None and handles[1] is handles[0]
        assert handles[0].filled
        gen_r, cls_r = _repeated(m, video, text, prompt)
    assert torch.equal(gen, gen_r) and torch.equal(cls, cls_r)
