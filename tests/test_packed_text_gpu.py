"""GPU: retrieval text features from texts packed back to back.

The packed causal attention (ymp_attn_fwd_packed) against the square causal call on the same sequences padded to a
common length (bit-equal O and lse, canary rows untouched) and against the float64 reference with its derived error
bound; DistributedGPT3_Retrieval.extract_text_feature's packed pass against the padded training-step pass (bit-equal,
no LM-head GEMM launched); the reference fixture through the packed pass; and the cases that keep the padded pass."""
import os

import pytest
import torch
import torch.nn.functional as F

import attn_bounds as AB
from helpers import build_pretrain
from oracle import port
from oracle.make_golden import make_inputs

pytestmark = pytest.mark.gpu
VC, GC, Q = port.VCFG_TINY, port.GCFG_TINY, 8
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CANARY = -7.0


# ------------------------------------------------------------------------------------------ kernel
LENS = [0, 1, 63, 64, 65, 80, 200]
CASES = {"one_long": [200], "one_row": [1], "one_tile": [64],
         "mixed_33": LENS * 4 + [17, 0, 129, 192, 31]}


def _packed_vs_padded(cuda, hd, lens, heads=2, seed=0, margin=5):
    """Sequences of the given lengths padded to P = max(lens) rows (square causal ymp_attn_fwd) and packed back to back
    from row `margin` of canary-filled buffers (ymp_attn_fwd_packed).  Returns what the tests compare."""
    from ymp import lib, ops
    g = torch.Generator(device=cuda).manual_seed(seed)
    n, P, C = len(lens), max(max(lens), 1), heads * hd
    scale = hd ** -0.5
    q, k, v = (torch.randn(n * P, C, device=cuda, generator=g).bfloat16() for _ in range(3))
    o_pad = torch.empty(n * P, C, device=cuda, dtype=torch.bfloat16)
    dm = ops.dense_map(P)
    lse_pad = ops.attn_fwd(*(ops.TView(x, 0, hd, dm) for x in (q, k, v, o_pad)), n_seq=n, n_heads=heads, head_dim=hd,
                           s_q=P, s_kv=P, causal=True, scale=scale)
    lens_t = torch.tensor(lens, device=cuda)
    starts = torch.zeros(n + 1, dtype=torch.int64, device=cuda)
    starts[1:] = lens_t.cumsum(0)
    starts += margin
    T = int(lens_t.sum())
    seq = torch.repeat_interleave(torch.arange(n, device=cuda), lens_t)
    col = torch.arange(T, device=cuda) + margin - starts[:-1][seq]
    idx = seq * P + col                                   # padded row of each packed row
    rows = margin + T + margin
    qp, kp, vp = (torch.randn(rows, C, device=cuda, generator=g).bfloat16() * 50 for _ in range(3))   # rows never read
    for dst, src in ((qp, q), (kp, k), (vp, v)):
        dst[margin:margin + T] = src[idx]
    op = torch.full((rows, C), CANARY, device=cuda, dtype=torch.bfloat16)
    lsep = torch.full((rows, heads), CANARY, device=cuda, dtype=torch.float32)
    ops.attn_fwd_packed(*(ops.TView(x, 0, hd, None) for x in (qp, kp, vp, op)), starts=starts.to(torch.int32),
                        max_len=max(lens), n_heads=heads, head_dim=hd, scale=scale, lse=lsep)
    assert lib.attn_last_path() == lib.ATTN_PATH_WGMMA
    return dict(q=q, k=k, v=v, o_pad=o_pad, lse_pad=lse_pad, op=op, lsep=lsep, idx=idx, seq=seq, col=col, T=T,
                margin=margin, P=P, n=n, scale=scale, heads=heads, hd=hd)


@pytest.mark.parametrize("hd", [64, 80, 88, 96])
@pytest.mark.parametrize("case", list(CASES))
def test_packed_attention_equals_padded_call_and_reference(cuda, hd, case):
    lens = CASES[case]
    r = _packed_vs_padded(cuda, hd, lens)
    m, T, H = r["margin"], r["T"], r["heads"]
    # every valid row: bit-equal O and lse
    assert torch.equal(r["op"][m:m + T], r["o_pad"][r["idx"]])
    assert torch.equal(r["lsep"][m:m + T], r["lse_pad"][r["seq"], :, r["col"]])
    # nothing outside [starts[0], starts[n_seq]) is written
    assert (r["op"][:m] == CANARY).all() and (r["op"][m + T:] == CANARY).all()
    assert (r["lsep"][:m] == CANARY).all() and (r["lsep"][m + T:] == CANARY).all()
    # float64 reference of the padded sequences, valid rows only
    n, P, hd_ = r["n"], r["P"], r["hd"]
    q4, k4, v4 = (x.view(n, P, H, hd_).transpose(1, 2) for x in (r["q"], r["k"], r["v"]))
    vis = AB.visible(n, P, P, AB.MASK_CAUSAL).to(cuda)
    valid = torch.arange(P, device=cuda)[None, :] < torch.tensor(lens, device=cuda)[:, None]   # [n, P]
    vis = vis & valid[:, :, None]
    ref = AB.reference(q4, k4, v4, vis, r["scale"])
    e_o, e_lse = AB.fwd_bounds(q4, k4, v4, r["scale"], ref)
    got_o = torch.zeros(n * P, H * hd_, device=cuda, dtype=torch.bfloat16)
    got_o[r["idx"]] = r["op"][m:m + T]
    got_o = got_o.view(n, P, H, hd_).transpose(1, 2)
    got_lse = torch.zeros(n, P, H, device=cuda)
    got_lse.view(n * P, H)[r["idx"]] = r["lsep"][m:m + T]
    where = valid[:, None, :]
    assert AB.worst_ratio(got_o, ref["O"], e_o, where[..., None]) <= 1.0
    assert AB.worst_ratio(got_lse.transpose(1, 2), ref["lse"], e_lse, where) <= 1.0


def test_packed_attention_rejections(cuda):
    from ymp import lib, ops
    hd, heads = 64, 2
    starts = torch.tensor([0, 3, 8], device=cuda, dtype=torch.int32)
    q, k, v, o = (torch.randn(8, heads * hd, device=cuda).bfloat16() for _ in range(4))
    views = [ops.TView(x, 0, hd, ops.seqmap()) for x in (q, k, v, o)]

    def call(**over):
        a = lib.AttnPackedArgs()
        a.attn = ops._attn_args(*views, None, 2, heads, over.pop("head_dim", hd), 5, 5, over.pop("causal", 1), 0.125,
                                **over)
        a.starts, a.max_len = starts.data_ptr(), 5
        lib.call(lib._attn_fwd_packed, a, "ymp_attn_fwd_packed")

    call()
    rng = torch.tensor([7, 0], dtype=torch.int64, device=cuda)
    with pytest.raises(lib.YmpError, match="dropout"):
        call(drop=ops.Drop(rng, ops.site_attn(0), 0.1))
    with pytest.raises(lib.YmpError, match="s_kv_dev"):
        call(s_kv_dev=torch.ones(1, device=cuda, dtype=torch.int32))
    with pytest.raises(lib.YmpError, match="kv_rows"):
        call(kv_rows=torch.zeros(2, 5, device=cuda, dtype=torch.int32))
    with pytest.raises(lib.YmpError, match="total_rows"):
        call(total_rows=8)
    with pytest.raises(lib.YmpError, match="causal"):
        call(causal=0)
    with pytest.raises(lib.YmpError, match="head_dim"):
        call(head_dim=128)
    a = lib.AttnPackedArgs()
    a.attn, a.starts, a.max_len = ops._attn_args(*views, None, 2, heads, hd, 5, 5, 1, 0.125), None, 5
    with pytest.raises(lib.YmpError, match="null starts"):
        lib.call(lib._attn_fwd_packed, a, "ymp_attn_fwd_packed")


# ------------------------------------------------------------------------------------------ model
def _retrieval(cuda, gcfg, dropout=(0.0, 0.0), seed=21):
    sd = port.init_state_dict(VC, gcfg, Q, seed=seed, randomize=True) if gcfg is GC else None
    m = build_pretrain(VC, gcfg, Q, sd=sd, device=cuda, dtype=torch.bfloat16, cls_name="DistributedGPT3_Retrieval",
                       num_frames=VC["num_frames"], contrastive_embed_dim=32, dropout=dropout)
    return m


def _texts(cuda, B, L, vocab, seed):
    import models.modeling_distributed_gpt3 as G
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(1, L + 1, (B,), generator=g)
    lens[0], lens[1] = L, 1
    att = (torch.arange(L)[None, :] < lens[:, None]).long()
    ids = torch.where(att.bool(), torch.randint(3, vocab, (B, L), generator=g), torch.zeros((), dtype=torch.long))
    return G.BatchEncoding(dict(input_ids=ids.to(cuda), attention_mask=att.to(cuda)))


def _padded_feature(m, text):
    return F.normalize(m.text_proj(m._pooled_text_padded(text)).float(), dim=-1)


def _gpt(name, layers=2):
    import json
    with open(os.path.join(ROOT, "youku-mplug_b200", "configs", "models", name)) as f:
        return dict(json.load(f), num_hidden_layers=layers)


@pytest.mark.parametrize("which", ["tiny", "1.3B", "2.7B"])
def test_packed_text_features_equal_padded_pass(cuda, which, monkeypatch):
    from ymp import engine, ops
    gcfg = GC if which == "tiny" else _gpt(f"config_gpt3_{which}.json")
    L = 24 if which == "tiny" else 80
    m = _retrieval(cuda, gcfg).eval()
    vocab = gcfg["vocab_size"]
    word = m.text_decoder.dist_model.language_model.embedding.word_embeddings.weight
    for all80 in (False, True):
        text = _texts(cuda, 32, L, vocab, 7 + all80)
        if all80:
            text.attention_mask.fill_(1)
        with torch.no_grad():
            want = _padded_feature(m, text)
            gemm_b, ce = [], []
            real_gemm, real_ce = ops.gemm, ops.ce_fwd
            monkeypatch.setattr(ops, "gemm", lambda a, b, **kw: (gemm_b.append(b.data_ptr()), real_gemm(a, b, **kw))[1])
            monkeypatch.setattr(ops, "ce_fwd", lambda *a, **kw: (ce.append(1), real_ce(*a, **kw))[1])
            calls = []
            real_packed = engine.gpt_fwd_packed
            monkeypatch.setattr(engine, "gpt_fwd_packed", lambda *a, **kw: (calls.append(1), real_packed(*a, **kw))[1])
            got = m.extract_text_feature(text)
            monkeypatch.undo()
        assert calls == [1]
        assert gemm_b and word.data_ptr() not in gemm_b and not ce   # the tied LM head never runs
        assert torch.equal(got, want), (which, all80)
        with torch.no_grad():
            assert torch.equal(m.text_decoder.text_features(text.input_ids, text.attention_mask),
                               m._pooled_text_padded(text))


def test_fixture_retrieval_features_through_the_packed_pass(cuda, monkeypatch):
    from ymp import engine
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "tiny_downstream.pt"), weights_only=False)
    assert fx["Q"] == Q and fx["vcfg"] == VC and fx["gcfg"] == GC
    r = fx["retrieval"]
    sd = port.init_state_dict(VC, GC, Q, seed=fx["wseed"], randomize=True)
    sd.update(dict(r["proj"], temp=torch.tensor(0.07)))
    m = build_pretrain(VC, GC, Q, sd=sd, device=cuda, dtype=torch.bfloat16, cls_name="DistributedGPT3_Retrieval",
                       num_frames=VC["num_frames"], contrastive_embed_dim=32)
    _, ids, att = make_inputs(3, VC, 8, GC["vocab_size"], r["seed"])
    import models.modeling_distributed_gpt3 as G
    text = G.BatchEncoding(dict(input_ids=ids.to(cuda), attention_mask=att.to(cuda)))
    calls = []
    real = engine.gpt_fwd_packed
    monkeypatch.setattr(engine, "gpt_fwd_packed", lambda *a, **kw: (calls.append(1), real(*a, **kw))[1])
    with torch.no_grad():
        t = m.extract_text_feature(text)
    assert calls == [1]
    want = r["text_feats"].float()
    assert ((t.float().cpu() - want).abs().max() <= 2e-2 * want.abs().max()).item()


def test_dropout_or_trainable_decoder_keeps_the_padded_pass(cuda, monkeypatch):
    from ymp import engine, functional as YF

    def refuse(*a, **kw):
        raise AssertionError("the packed pass ran")

    text = _texts(cuda, 8, 24, GC["vocab_size"], 3)
    # dropout active (train() mode, p > 0): the padded pass with its own masks
    m = _retrieval(cuda, GC, dropout=(0.1, 0.1)).train()
    monkeypatch.setattr(engine, "gpt_fwd_packed", refuse)
    with torch.no_grad():
        YF.set_dropout_seed(11)
        got = m.extract_text_feature(text)
        YF.set_dropout_seed(11)
        want = _padded_feature(m, text)
    assert torch.equal(got, want)
    monkeypatch.undo()
    # no dropout, but a trainable decoder parameter under grad mode: the padded pass, whose value the packed pass equals
    m = _retrieval(cuda, GC).train()
    with torch.no_grad():
        packed = m.extract_text_feature(text)
    dict(m.text_decoder.named_parameters())["dist_model.language_model.encoder.layers.0.mlp.dense_h_to_4h.weight"].requires_grad_(True)
    monkeypatch.setattr(engine, "gpt_fwd_packed", refuse)
    got = m.extract_text_feature(text)
    assert got.requires_grad
    assert torch.equal(got.detach(), _padded_feature(m, text).detach())
    assert torch.equal(got.detach(), packed)


def test_captured_pass_keeps_the_padded_pass(cuda, monkeypatch):
    """Under CUDA-graph capture (TrainEngine.train_step) the padded pass runs: the packed layout is read on the host."""
    from ymp import engine
    m = _retrieval(cuda, GC).eval()
    text = _texts(cuda, 8, 24, GC["vocab_size"], 5)
    with torch.no_grad():
        want = m.extract_text_feature(text)
        _padded_feature(m, text)   # (every kernel of the padded pass launched once before the capture)
        torch.cuda.synchronize()
        monkeypatch.setattr(engine, "gpt_fwd_packed", lambda *a, **kw: (_ for _ in ()).throw(AssertionError("packed")))
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            got = m.extract_text_feature(text)
        g.replay()
        torch.cuda.synchronize()
    assert torch.equal(got, want)
