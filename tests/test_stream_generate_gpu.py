"""GPU: the streaming beam search's per-sequence decoding step.  Decode attention with a key count per sequence
(ymp_attn_fwd_seq_lens) against one scalar-count call per sequence; the skinny GEMM's per-row KV-cache copy
(ymp_gemm_skinny_rows / _wide_rows) against the scalar-offset call; the per-row TokenStep captured against eager, across
a mid-decode group prefill whose cache rows equal a fresh prefill; DistributedGPT3_Caption.generate on the streaming
path against the per-clip loop (sequences and scores bit for bit)."""
import ctypes
import json
import os

import pytest
import torch

from oracle import port
from oracle.make_golden import make_inputs
from helpers import build_pretrain

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
CFGS = os.path.join(ROOT, "youku-mplug_b200", "configs", "models")
HEADS = 3


def _gcfg(name, layers=None):
    with open(os.path.join(CFGS, f"config_gpt3_{name}.json")) as f:
        g = json.load(f)
    if layers is not None:
        g["num_hidden_layers"] = layers
    return g


def _tiny(dev):
    fx = torch.load(os.path.join(GOLD, "tiny_generate.pt"), weights_only=False)
    sd = port.generation_state_dict(fx["vcfg"], fx["gcfg"], fx["Q"], fx["wseed"], fx["pos_gain"], fx["ln_gain"])
    model = build_pretrain(fx["vcfg"], fx["gcfg"], fx["Q"], sd=sd, device=dev, dtype=torch.bfloat16,
                           cls_name="DistributedGPT3_Caption", num_frames=fx["vcfg"]["num_frames"]).eval()
    model.text_decoder.config.tokens_to_generate = fx["n_new"]
    return fx, model


# ------------------------------------------------------------------------------------------ decode attention
def _attn(q, buf, hd, n_seq, s_kv, m_kv, kv_rows=None, kv_lens=None):
    from ymp import ops
    o = torch.full((n_seq, HEADS * hd), float("nan"), device=q.device, dtype=torch.bfloat16)
    k, v = ops.TView(buf, hd, 3 * hd, m_kv), ops.TView(buf, 2 * hd, 3 * hd, m_kv)
    lse = ops.attn_fwd(ops.TView(q, 0, 3 * hd, ops.dense_map(1)), k, v, ops.TView(o, 0, hd, ops.dense_map(1)), n_seq=n_seq,
                       n_heads=HEADS, head_dim=hd, s_q=1, s_kv=s_kv, causal=False, scale=hd ** -0.5, kv_rows=kv_rows,
                       kv_lens=kv_lens)
    return o, lse


@pytest.mark.parametrize("table", [False, True])
@pytest.mark.parametrize("hd", [64, 80, 96])
def test_seq_lens_decode_equals_scalar_calls(cuda, hd, table):
    """Key counts 1 .. s_kv (around the 128-key prefetch): each sequence's O and lse equal a call over that sequence
    alone with s_kv = its count, bit for bit.  Keys past a sequence's count are NaN and must not reach O."""
    from ymp import ops
    s_kv, lens = 301, [1, 2, 127, 128, 129, 200, 256, 257, 300, 301]
    n = len(lens)
    g = torch.Generator(device=cuda).manual_seed(hd + table)
    buf = torch.randn(n * s_kv, 3 * HEADS * hd, device=cuda, generator=g).bfloat16()
    q = torch.randn(n, 3 * HEADS * hd, device=cuda, generator=g).bfloat16()
    rows = None
    if table:   # sequence s reads scrambled rows; rows past its count are named by no entry below it
        rows = torch.stack([torch.randperm(n * s_kv, device=cuda, generator=g)[:s_kv] for _ in range(n)]).int()
        used = torch.zeros(n * s_kv, dtype=torch.bool, device=cuda)
        for s, L in enumerate(lens):
            used[rows[s, :L].long()] = True
        buf[~used] = float("nan")
    else:
        for s, L in enumerate(lens):
            buf[s * s_kv + L:(s + 1) * s_kv] = float("nan")
    kv_lens = torch.tensor(lens, dtype=torch.int32, device=cuda)
    o, lse = _attn(q, buf, hd, n, s_kv, ops.dense_map(s_kv), kv_rows=rows, kv_lens=kv_lens)
    for s, L in enumerate(lens):
        if table:
            o1, l1 = _attn(q[s:s + 1], buf, hd, 1, L, ops.dense_map(s_kv), kv_rows=rows[s:s + 1].contiguous())
        else:
            o1, l1 = _attn(q[s:s + 1], buf[s * s_kv:], hd, 1, L, ops.dense_map(s_kv))
        assert not o1.isnan().any()
        assert torch.equal(o[s:s + 1], o1), (s, L)
        assert torch.equal(lse[s:s + 1], l1), (s, L)


def test_seq_lens_rejected_combinations(cuda):
    """Every combination the per-sequence count does not serve returns an error and launches nothing."""
    from ymp import lib, ops
    hd, n, s_kv = 64, 4, 64
    buf = torch.randn(n * s_kv, 3 * HEADS * hd, device=cuda).bfloat16()
    q = torch.randn(n * 2, 3 * HEADS * hd, device=cuda).bfloat16()
    o = torch.empty(n * 2, HEADS * hd, device=cuda, dtype=torch.bfloat16)
    lens = torch.full((n,), 10, dtype=torch.int32, device=cuda)
    dev1 = torch.tensor([10], dtype=torch.int32, device=cuda)
    rng = torch.zeros(2, dtype=torch.int64, device=cuda)

    def args(head_dim=hd, s_q=1, causal=False, total_rows=0, drop=None, s_kv_dev=None):
        m = ops.dense_map(s_kv)
        return ops._attn_args(ops.TView(q, 0, 3 * hd, ops.dense_map(s_q)), ops.TView(buf, hd, 3 * hd, m),
                              ops.TView(buf, 2 * hd, 3 * hd, m), ops.TView(o, 0, hd, ops.dense_map(s_q)), None, n, HEADS,
                              head_dim, s_q, s_kv if not total_rows else s_q, causal, hd ** -0.5, 0, total_rows, drop,
                              s_kv_dev)
    bad = [args(s_q=2), args(causal=True), args(drop=ops.Drop(rng, 0, 0.1)), args(total_rows=n, s_q=1),
           args(head_dim=88), args(head_dim=128), args(s_kv_dev=dev1)]
    torch.cuda.synchronize()
    n0 = lib.launch_count()
    for a in bad:
        assert lib._attn_fwd_seq_lens(ctypes.byref(a), lens.data_ptr(), lib.cur_stream()) != 0
    assert lib._attn_fwd_seq_lens(ctypes.byref(args()), None, lib.cur_stream()) != 0
    assert lib.launch_count() == n0
    assert lib._attn_fwd_seq_lens(ctypes.byref(args()), lens.data_ptr(), lib.cur_stream()) == 0


# ------------------------------------------------------------------------------------------ skinny GEMM
@pytest.mark.parametrize("M", [1, 5, 8, 9, 17, 40, 64])
def test_skinny_row_offsets_equal_scalar_offset(cuda, M):
    """Row m's second copy lands at out2 row m * stride + off[m], equal to the scalar-offset call's row m; every other
    row of the sentinel-filled buffer is untouched; the first copy is the scalar call's."""
    from ymp import ops
    g = torch.Generator(device=cuda).manual_seed(M)
    N, K, stride = 3 * 2048, 2048, 7
    x = torch.randn(M, K, device=cuda, generator=g).bfloat16()
    w = (torch.randn(N, K, device=cuda, generator=g) * 0.02).bfloat16()
    bias = torch.randn(N, device=cuda, generator=g).bfloat16()
    offs = torch.randint(0, stride, (M,), device=cuda, generator=g)
    fn = ops.gemm_skinny if M <= 8 else ops.gemm_skinny_wide
    sentinel = torch.tensor(-3.25, dtype=torch.bfloat16)
    buf = torch.full((M * stride, N), float(sentinel), device=cuda, dtype=torch.bfloat16)
    y = fn(x, w, bias=bias, out2=buf, out2_row_stride=stride, out2_row_off=offs)
    ref_buf = torch.zeros((M * stride, N), device=cuda, dtype=torch.bfloat16)
    y0 = fn(x, w, bias=bias, out2=ref_buf, out2_row_stride=stride, out2_off=torch.zeros(1, dtype=torch.int64, device=cuda))
    assert torch.equal(y, y0)
    view = buf.view(M, stride, N)
    written = torch.zeros(M, stride, dtype=torch.bool, device=cuda)
    written[torch.arange(M, device=cuda), offs] = True
    assert torch.equal(view[written], y0)
    assert bool((view[~written] == sentinel.to(cuda)).all())
    if M <= 8:   # the wide entry point's M <= 8 launch is the same kernel
        buf2 = torch.full_like(buf, float(sentinel))
        ops.gemm_skinny_wide(x, w, bias=bias, out2=buf2, out2_row_stride=stride, out2_row_off=offs)
        assert torch.equal(buf, buf2)


def test_skinny_row_offsets_rejected(cuda):
    from ymp import lib
    x = torch.randn(4, 256, device=cuda).bfloat16()
    w = torch.randn(64, 256, device=cuda).bfloat16()
    y = torch.empty(4, 64, device=cuda, dtype=torch.bfloat16)
    buf = torch.empty(16, 64, device=cuda, dtype=torch.bfloat16)
    off = torch.zeros(4, dtype=torch.int64, device=cuda)

    def args(y2=True, scalar=False, f32=False):
        a = lib.GemmSkinnyArgs()
        a.x, a.w, a.y = x.data_ptr(), w.data_ptr(), y.data_ptr()
        a.M, a.N, a.K, a.ldx, a.ldw, a.ldy = 4, 64, 256, 256, 256, 64
        a.out_dtype = lib.DT_F32 if f32 else lib.DT_BF16
        if y2:
            a.y2, a.ldy2, a.y2_off_stride = buf.data_ptr(), 4 * 64, 64
        if scalar:
            a.y2_off_dev = off.data_ptr()
        return a
    torch.cuda.synchronize()
    n0 = lib.launch_count()
    for fn in (lib._gemm_skinny_rows, lib._gemm_skinny_wide_rows):
        for a, p in ((args(y2=False), off), (args(scalar=True), off), (args(f32=True), off), (args(), None)):
            assert fn(ctypes.byref(a), None if p is None else p.data_ptr(), lib.cur_stream()) != 0
    assert lib.launch_count() == n0


# ------------------------------------------------------------------------------------------ engine
def _per_row_run(dec, qf, ids, beam, G, ML, graph, n_steps, refill_at, refill_clip, monkeypatch):
    """A per-row cache of G groups: clips 0 .. G-1 prefilled (prompt lengths 3 + g % 3), then n_steps per-row steps
    (fixed tokens, random in-group permutations); at step refill_at group 1 takes clip refill_clip (prompt length 5)
    and the last group is frozen.  Returns (stacked logits, cache, the refill's logits)."""
    from ymp import engine, ops
    from ymp import functional as YF
    monkeypatch.setenv("YMP_DECODE_GRAPH", "1" if graph else "0")
    rows, Q = G * beam, qf.shape[1]
    W = {k: YF.as_bf16(p) for k, p in zip(*dec._param_list())}
    emb = dec.dist_model.language_model.embedding.word_embeddings
    pos = W[engine.GPT + "embedding.position_embeddings.weight"]
    cache = engine.KVCache(dec.config.engine_cfg(), rows, ML, ids.device)
    cache.reset_rows()
    ts = engine.TokenStep(cache, W, emb.weight.dtype, None, True, per_row=True)

    def prefill(g, c, n):
        x = torch.cat([qf[c:c + 1], emb(ids[c:c + 1, :n])], 1)
        x = (x.float() + pos[:n + Q][None].float()).reshape(n + Q, -1).contiguous()
        return ops.gemm(cache.prefill_groups(W, x, n + Q, g, 1, beam), W[engine.GPT + "embedding.word_embeddings.weight"]).float()

    gen = torch.Generator().manual_seed(9)
    outs = [torch.cat([prefill(g, g, 3 + g % 3) for g in range(G)])]
    refill_logits = None
    with torch.no_grad():
        for t in range(n_steps):
            if t == refill_at:
                refill_logits = prefill(1, refill_clip, 5)
                cache.set_live([g != G - 1 for g in range(G) for _ in range(beam)])
            tok = torch.randint(0, dec.config.vocab_size, (rows, 1), generator=gen).to(ids.device)
            _, logits = ts.run(emb(tok).reshape(rows, -1))
            outs.append(logits.clone())
            idx = torch.cat([g * beam + torch.randperm(beam, generator=gen) for g in range(G)]).to(ids.device)
            cache.reindex_rows(idx)
    assert (ts.graph is not None) == graph
    return torch.cat(outs), cache, refill_logits


@pytest.mark.parametrize("width", ["tiny", "1.3B"])
def test_per_row_token_step_graph_equals_eager_and_refill_equals_fresh_prefill(cuda, monkeypatch, width):
    """The captured per-row step equals the eager one bit for bit, across a mid-decode group prefill and a frozen group;
    the refilled group's cache rows (prefix + prompt) and first logits equal a fresh prefill of that clip alone."""
    import models.modeling_distributed_gpt3 as M
    if width == "tiny":
        fx, model = _tiny(cuda)
        vcfg, Q, L = fx["vcfg"], fx["Q"], fx["L"]
    else:
        vcfg, Q, L = port.VCFG_TINY, 128, 20
        model = build_pretrain(vcfg, _gcfg(width, layers=2), Q, device=cuda, dtype=torch.bfloat16,
                               cls_name="DistributedGPT3_Caption", num_frames=vcfg["num_frames"]).eval()
    dec = model.text_decoder
    beam, G = 5, 12
    video, ids, _ = make_inputs(G + 1, vcfg, L, dec.config.vocab_size, 31)
    with torch.no_grad():
        qf = model.visual_prefix(video.to(cuda).bfloat16())[3]
    ids = ids.to(cuda)
    ML = Q + 5 + 12
    eager, _, _ = _per_row_run(dec, qf, ids, beam, G, ML, False, 10, 4, G, monkeypatch)
    graphed, cache, refill_logits = _per_row_run(dec, qf, ids, beam, G, ML, True, 10, 4, G, monkeypatch)
    assert torch.equal(eager, graphed)
    assert max(cache.lens_host) < ML and cache.lens.tolist() == cache.lens_host
    # the refilled group (1): its first slot's rows up to the refill's length equal a fresh prefill of clip G alone
    with torch.no_grad():
        dec.inference_params = ip = M.InferenceParams(1, Q + 5 + 1)
        out = dec(tokens=ids[G:G + 1, :5], query_embeds=qf[G:G + 1])
    fresh = ip.cache.store.view(ip.cache.g.layers, 1, Q + 5 + 1, -1)[:, 0, :Q + 5]
    st = cache.store.view(cache.g.layers, G * beam, ML, -1)
    assert torch.equal(st[:, beam, :Q + 5], fresh)
    assert torch.equal(refill_logits[0], out.logits[0, -1])


# ------------------------------------------------------------------------------------------ model level
def _generate_both(model, video, text, beam):
    """(model.generate's list on the streaming path, its AttrDicts, the per-clip beam searches' AttrDicts)."""
    import models.modeling_distributed_gpt3 as M
    dec = model.text_decoder
    orig, calls, got = M.DistributedGPT3._per_row_decoder, [], []

    def counted(self, *a, **k):
        calls.append(a)
        return orig(self, *a, **k)
    M.DistributedGPT3._per_row_decoder = counted
    bs = dec.beam_search

    def beam_search(*a, **k):
        got.append(bs(*a, **dict(k, beam_size=beam)))
        return got[-1]
    dec.beam_search = beam_search
    try:
        res = model.generate(video, text)
        stream = got[0]
        eos = dec.config.eod_id
        per = []
        with torch.no_grad():
            qf = model.visual_prefix(video)[3]
            for i in range(text.input_ids.shape[0]):
                per.append(dec.generate(text.input_ids[i:i + 1], query_embeds=qf[i:i + 1], termination_id=eos,
                                        do_sample=False, prompt_length=text.attention_mask.sum(-1)[i] - 1))
    finally:
        M.DistributedGPT3._per_row_decoder = orig
        del dec.beam_search
    assert len(calls) == 1
    return res, stream, per


def _check(res, stream, per, B):
    assert len(res) == len(stream) == len(per) == B
    for i in range(B):
        assert torch.equal(stream[i].sequences, per[i].sequences), i
        assert torch.equal(stream[i].scores, per[i].scores), i
        assert torch.equal(res[i], per[i].sequences.cpu())


def _mixed_text(M, ids, dev, plens):
    att = torch.zeros_like(ids)
    for i, p in enumerate(plens):
        att[i, :p + 1] = 1
    return M.BatchEncoding(dict(input_ids=ids.to(dev), attention_mask=att.to(dev)))


def test_caption_generate_per_row_state_equals_per_clip_tiny(cuda):
    """30 clips at beam 5 on the tiny fixture (its weights make beams finish early), prompt lengths 3 .. 6."""
    import models.modeling_distributed_gpt3 as M
    fx, model = _tiny(cuda)
    B = 30
    video, ids, _ = make_inputs(B, fx["vcfg"], fx["L"], fx["gcfg"]["vocab_size"], 17)
    ids[:2] = fx["ids"]
    text = _mixed_text(M, ids, cuda, [3 + i % 4 for i in range(B)])
    res, stream, per = _generate_both(model, video.to(cuda).bfloat16(), text, 5)
    _check(res, stream, per, B)
    assert any((s.sequences == fx["eod"]).any() for s in per)


@pytest.mark.parametrize("width", ["1.3B", "2.7B"])
def test_caption_generate_per_row_state_equals_per_clip_wide(cuda, width):
    """2-layer decoders at the 1.3B / 2.7B widths, 30 clips at beam 5 (12 groups: 18 refills), mixed prompt lengths,
    the stop token's embedding row scaled so that captions end at varying steps."""
    import models.modeling_distributed_gpt3 as M
    vcfg, Q, L, B = port.VCFG_TINY, 128, 20, 30
    model = build_pretrain(vcfg, _gcfg(width, layers=2), Q, device=cuda, dtype=torch.bfloat16,
                           cls_name="DistributedGPT3_Caption", num_frames=vcfg["num_frames"]).eval()
    dec = model.text_decoder
    dec.config.tokens_to_generate = 12
    with torch.no_grad():
        dec.dist_model.language_model.embedding.word_embeddings.weight[dec.config.eod_id] *= 4
    video, ids, _ = make_inputs(B, vcfg, L, dec.config.vocab_size, 19)
    text = _mixed_text(M, ids, cuda, [12 + (7 * i) % 8 for i in range(B)])
    res, stream, per = _generate_both(model, video.to(cuda).bfloat16(), text, 5)
    _check(res, stream, per, B)
