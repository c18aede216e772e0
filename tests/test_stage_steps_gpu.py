"""Record the hand-scheduled stages kernel call by kernel call on the H100 and walk each trace against the float64
step programs of tests/stage_steps.py: schedule, dataflow (every operand bit for bit the quantity its step names) and
value (every output element within its kernel's bound of the float64 value of the recorded operands).  The gradient
buffers start non-zero, so a wgrad that overwrites fails.  YMP_STAGE_BOUNDS_REPORT=<file> writes the largest err/bound
per stage and step as JSON."""
import pytest
import torch

import stage_steps as SS
from oracle import port
from oracle.make_golden import make_inputs

pytestmark = pytest.mark.gpu

F64, BF16 = torch.float64, torch.bfloat16
SEED = 20261017

VIT_B = dict(img_size=64, patch_size=16, embed_dim=768, depth=2, num_heads=8, mlp_ratio=4, num_frames=8, clip_model=True)
GPT_1P3B = dict(port.GCFG_1_3B, num_hidden_layers=2)
GPT_2P7B = dict(port.GCFG_2_7B, num_hidden_layers=2)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _seeded_g(sd, keys, dev):
    g = torch.Generator().manual_seed(11)
    return {k: (0.01 * torch.randn(sd[k].numel(), generator=g)).float().to(dev) for k in keys}


def _walk(stage, trace, G0, run, G_final, dev):
    X = SS.Exec("walk", G0=G0, trace=trace, sms=_sms(), dev=dev)
    try:
        out = run(X)
        X.finish(G_final)
    finally:
        SS.write_report(X, stage)
    return X, out


@pytest.mark.parametrize("case", ["tiny_p0.1", "vitb_1p3b_p0.1", "vitb_1p3b_p0"])
def test_pretrain_step_walks(cuda, monkeypatch, case):
    """One PretrainFn forward and backward (TimeSformer, AttentionPool, visual_fc, the frozen decoder, LM head, CE):
    the tiny configs (T = 2: explicit im2col, warp-per-sequence temporal attention) and the ViT-B/16 + GPT-3 1.3B
    widths at 2 + 2 layers (T = 8: fused-im2col patch GEMM; 32 x 64 heads: wgmma attention), 128 queries, L = 37 text
    rows (S = 165, not a multiple of 64), V = 51200."""
    from ymp import functional, ops
    p = 0.0 if case.endswith("p0") else 0.1
    if case.startswith("tiny"):
        vcfg, gcfg, Q, L = port.VCFG_TINY, port.GCFG_TINY, 8, 5
    else:
        vcfg, gcfg, Q, L = VIT_B, GPT_1P3B, 128, 37
    gcfg = dict(gcfg, training=True, hidden_dropout=p, attention_dropout=p)
    sd = port.init_state_dict(vcfg, gcfg, Q, seed=3, randomize=True)
    keys = sorted(sd)
    T = set(port.trainable_keys(sd))
    params = [sd[k].to(cuda, BF16).requires_grad_(k in T) for k in keys]
    G = _seeded_g(sd, sorted(T), cuda)
    G0 = {k: v.clone() for k, v in G.items()}
    sink = {id(pp): G[k] for k, pp in zip(keys, params) if k in T}
    video, ids, att = make_inputs(2, vcfg, L, gcfg["vocab_size"], 5)
    video, ids, att = video.to(cuda, BF16), ids.to(cuda), att.to(cuda)
    targets, loss_mask = port.build_targets(ids, att, Q)
    functional.set_dropout_seed(SEED, cuda)
    seed, offset = functional._RNG[cuda]["state"].tolist()
    rec = SS.Recorder(ops, G)
    rec.install(monkeypatch)
    with functional.grad_sink(sink):
        loss, losses = functional.PretrainFn.apply(video, ids, targets, loss_mask, vcfg, gcfg, keys, *params)
        loss.backward()
    torch.cuda.synchronize()
    monkeypatch.undo()
    assert all(pp.grad is None for pp in params)
    W = {k: pp.detach().to(F64) for k, pp in zip(keys, params)}
    drop = SS.Drop(seed, offset, p, p) if p > 0 else None
    fused = ops.fused_im2col_ok(vcfg["num_frames"], vcfg["patch_size"])

    def run(X):
        l64, lbs, c = SS.pretrain_fwd(X, W, video.to(F64), ids, targets, loss_mask, vcfg, gcfg, Q, drop=drop, fused=fused)
        X.returned("losses", losses, lbs.to(torch.float32))
        terms = (lbs[:, :-1].reshape(-1) * loss_mask.reshape(-1).to(F64)).abs()
        bound = SS.C * (terms.numel() + 2) * SS.U32 * float(terms.sum()) / float(loss_mask.sum()) + SS.TINY
        assert abs(float(loss.detach()) - float(l64)) <= bound, (float(loss.detach()), float(l64), bound)
        SS.pretrain_bwd(X, W, T, c, loss_mask)

    X, _ = _walk(f"pretrain.{case}", rec.trace, G0, run, G, cuda)
    assert max(X.report.values()) <= 1.0


@pytest.mark.parametrize("case", ["1p3b_train_w_p0.1", "1p3b_frozen_p0.1", "1p3b_train_w_p0", "2p7b_frozen_p0.1"])
def test_decoder_walks(cuda, monkeypatch, case):
    """gpt_fwd / gpt_bwd at the 1.3B (32 x 64) and 2.7B (32 x 80) widths, 2 layers, B = 2, S = 165: with every layer
    trained (train_w: the wgrad GEMMs and bias colsums) or frozen (dgrad only), dropout 0.1 or off; the final
    LayerNorm over all rows."""
    from ymp import engine, ops
    p = 0.0 if case.endswith("p0") else 0.1
    gcfg = GPT_2P7B if case.startswith("2p7b") else GPT_1P3B
    train_w = "train_w" in case
    B, S, H = 2, 165, gcfg["hidden_size"]
    g = torch.Generator().manual_seed(4)
    W = {}
    for i in range(gcfg["num_hidden_layers"]):
        pre = f"{SS.GPT}encoder.layers.{i}."
        F4 = gcfg["ffn_hidden_size"]
        for nm in ("input_layernorm", "post_attention_layernorm"):
            W[pre + nm + ".weight"] = 1.0 + 0.1 * torch.randn(H, generator=g)
            W[pre + nm + ".bias"] = 0.02 * torch.randn(H, generator=g)
        for nm, shp in (("self_attention.query_key_value", (3 * H, H)), ("self_attention.dense", (H, H)),
                        ("mlp.dense_h_to_4h", (F4, H)), ("mlp.dense_4h_to_h", (H, F4))):
            W[pre + nm + ".weight"] = 0.02 * torch.randn(*shp, generator=g)
            W[pre + nm + ".bias"] = 0.02 * torch.randn(shp[0], generator=g)
    W[SS.GPT + "encoder.final_layernorm.weight"] = 1.0 + 0.1 * torch.randn(H, generator=g)
    W[SS.GPT + "encoder.final_layernorm.bias"] = 0.02 * torch.randn(H, generator=g)
    Wb = {k: v.to(cuda, BF16) for k, v in W.items()}
    T = {k for k in W if k.startswith(SS.GPT + "encoder.layers.")} if train_w else set()
    G = _seeded_g(W, sorted(T), cuda)
    G0 = {k: v.clone() for k, v in G.items()}
    x = (0.5 * torch.randn(B * S, H, generator=g)).float().to(cuda)
    dh = torch.randn(B * S, H, generator=g).to(cuda, BF16)
    rng = torch.tensor([SEED, 3], dtype=torch.int64, device=cuda)
    gdrop = engine.GptDrop(rng, p, p)
    x64 = x.to(F64)
    rec = SS.Recorder(ops, G)
    rec.install(monkeypatch)
    hid, c = engine.gpt_fwd(Wb, x, gcfg, B, S, train_w=train_w, drop=gdrop)
    dx = engine.gpt_bwd(Wb, G, c, dh)
    torch.cuda.synchronize()
    monkeypatch.undo()
    W64 = {k: v.to(F64) for k, v in Wb.items()}
    drop = SS.Drop(SEED, 3, p, p) if p > 0 else None

    def run(X):
        h64, cc = SS.gpt_fwd(X, W64, x64, gcfg, B, S, drop=drop)
        X.returned("hidden", hid, h64.to(BF16))
        d64 = SS.gpt_bwd(X, W64, T, cc, dh.to(F64), train_w=train_w)
        X.returned("dx", dx, d64.to(BF16))

    X, _ = _walk(f"decoder.{case}", rec.trace, G0, run, G, cuda)
    assert max(X.report.values()) <= 1.0


EVA_G = dict(img_size=56, patch_size=14, embed_dim=1408, depth=2, num_heads=16, mlp_ratio=4.3637)


def test_eva_walks(cuda, monkeypatch):
    """EvaFn forward and backward at the EVA-g width (1408, 16 x 88 heads, 6144 MLP), depth 2, 56 x 56 images
    (16 patches of 14 x 14: K = 588 zero-padded to 592), B = 2, every encoder parameter trained."""
    from ymp import functional, ops
    sd = {k: v for k, v in port.eva_state_dict(EVA_G, port.GCFG_TINY, 8, seed=6).items() if k.startswith(SS.VE)}
    keys = sorted(sd)
    params = [sd[k].to(cuda, BF16).requires_grad_(True) for k in keys]
    G = _seeded_g(sd, keys, cuda)
    G0 = {k: v.clone() for k, v in G.items()}
    sink = {id(pp): G[k] for k, pp in zip(keys, params)}
    g = torch.Generator().manual_seed(9)
    image = torch.randn(2, 3, 56, 56, generator=g).to(cuda, BF16)
    dout = torch.randn(2, 17, 1408, generator=g).to(cuda, BF16)
    rec = SS.Recorder(ops, G)
    rec.install(monkeypatch)
    with functional.grad_sink(sink):
        out = functional.EvaFn.apply(image, EVA_G, True, keys, *params)
        out.backward(dout)
    torch.cuda.synchronize()
    monkeypatch.undo()
    assert all(pp.grad is None for pp in params)
    W = {k: pp.detach().to(F64) for k, pp in zip(keys, params)}

    def run(X):
        o64, c = SS.eva_fwd(X, W, image.to(F64), EVA_G)
        X.returned("tokens", out.reshape(o64.shape), o64.to(BF16))
        SS.eva_bwd(X, W, set(keys), c, dout.reshape(-1, 1408).to(F64))

    X, _ = _walk("eva.evag_width", rec.trace, G0, run, G, cuda)
    assert max(X.report.values()) <= 1.0


def test_component_path_walks(cuda, monkeypatch):
    """The component path VitFn -> AttnPoolFn -> LinearFn(visual_fc) -> GptFn at the ViT-B/16 + GPT-3 1.3B widths
    (2 + 2 layers, 128 queries, L = 37, V = 51200, dropout 0.1), loss = masked_mean_loss of GptFn's losses: the
    functional.py glue (bf16 casts, padded columns, gradient store, the decoder input concatenation) between the
    same kernels."""
    from ymp import functional, ops
    vcfg, Q, L, p = VIT_B, 128, 37, 0.1
    gcfg = dict(GPT_1P3B, training=True, hidden_dropout=p, attention_dropout=p)
    sd = port.init_state_dict(vcfg, gcfg, Q, seed=3, randomize=True)
    keys = sorted(sd)
    T = set(port.trainable_keys(sd))
    P = {k: sd[k].to(cuda, BF16).requires_grad_(k in T) for k in keys}
    G = _seeded_g(sd, sorted(T), cuda)
    G0 = {k: v.clone() for k, v in G.items()}
    sink = {id(P[k]): G[k] for k in T}
    video, ids, att = make_inputs(2, vcfg, L, gcfg["vocab_size"], 5)
    video, ids, att = video.to(cuda, BF16), ids.to(cuda), att.to(cuda)
    targets, loss_mask = port.build_targets(ids, att, Q)
    functional.set_dropout_seed(SEED, cuda)
    seed, offset = functional._RNG[cuda]["state"].tolist()
    vkeys = [k for k in keys if k.startswith(SS.VE)]
    akeys = [k for k in keys if k.startswith(SS.AP) or k == "learnable_queries"]
    gkeys = [k for k in keys if k.startswith("text_decoder.")]
    rec = SS.Recorder(ops, G)
    rec.install(monkeypatch)
    with functional.grad_sink(sink):
        img = functional.VitFn.apply(video, vcfg, True, vkeys, *[P[k] for k in vkeys])
        q = functional.AttnPoolFn.apply(img, vcfg["num_heads"], True, akeys, *[P[k] for k in akeys])
        qf = functional.LinearFn.apply(q, P["visual_fc.weight"], P["visual_fc.bias"])
        emb = torch.nn.functional.embedding(ids, P[SS.GPT + "embedding.word_embeddings.weight"])
        inp = torch.cat([qf, emb.to(qf.dtype)], 1)
        _, losses, _ = functional.GptFn.apply(inp, targets, gcfg, False, gkeys, *[P[k] for k in gkeys])
        loss = functional.masked_mean_loss(losses, loss_mask)
        loss.backward()
    torch.cuda.synchronize()
    monkeypatch.undo()
    assert all(pp.grad is None for pp in P.values())
    W = {k: pp.detach().to(F64) for k, pp in P.items()}
    fused = ops.fused_im2col_ok(vcfg["num_frames"], vcfg["patch_size"])

    def run(X):
        l64, c = SS.component_fwd(X, W, video.to(F64), ids, targets, vcfg, gcfg, Q, drop=SS.Drop(seed, offset, p, p),
                                  fused=fused)
        X.returned("losses", losses, l64.to(torch.float32))
        SS.component_bwd(X, W, T, c, loss_mask)

    X, _ = _walk("component.vitb_1p3b_p0.1", rec.trace, G0, run, G, cuda)
    assert max(X.report.values()) <= 1.0


# ---------------------------------------------------------------------------------- decoding
GPT_HD128 = dict(port.GCFG_TINY, hidden_size=256, ffn_hidden_size=1024, num_attention_heads=2, max_position_embeddings=256)
# case: (decoder config, clips, beam (0: sample), step program kind)
DECODE_CASES = {
    "1p3b_beam5": (GPT_1P3B, 1, 5, "skinny"),
    "2p7b_12clips_beam5": (GPT_2P7B, 12, 5, "skinny"),
    "1p3b_sample12": (GPT_1P3B, 12, 0, "gemm"),
    "hd128_2clips_beam3": (GPT_HD128, 2, 3, "skinny"),
}


def _decoder(cuda, gcfg, Q, n_new):
    """A 2-layer DistributedGPT3 in eval mode with random LayerNorm parameters and biases (the defaults are 1 and 0)."""
    from helpers import build_pretrain
    vcfg = port.VCFG_TINY
    dec = build_pretrain(vcfg, gcfg, Q, device=cuda, dtype=BF16, cls_name="DistributedGPT3_Caption",
                         num_frames=vcfg["num_frames"]).eval().text_decoder
    dec.config.tokens_to_generate, dec.config.top_k, dec.config.top_p = n_new, 1, 0.0
    g = torch.Generator().manual_seed(4)
    with torch.no_grad():
        for k, p in dec.named_parameters():
            if k.endswith("layernorm.weight"):
                p.copy_(1.0 + 0.1 * torch.randn(p.shape, generator=g))
            elif k.endswith("bias"):
                p.copy_(0.02 * torch.randn(p.shape, generator=g))
    return dec


@pytest.mark.parametrize("case", sorted(DECODE_CASES))
def test_decode_walks(cuda, monkeypatch, case):
    """Caption decoding through the public entry points (beam_search of one clip, the batched beam search, sample()),
    recorded eagerly (YMP_DECODE_GRAPH=0: the recorder synchronises inside every call) with every new cache store
    poisoned, and walked against decode_session: the prefill into the KV cache, 7 single-token steps (TokenStep's
    skinny GEMMs, 60 rows on the wide entry point, or gpt_decode's n = 1 step for 12 sampled rows of two prompt
    lengths), the row table under reindex and share_prefill, and the logits every decode returned.  2-layer decoders
    at the 1.3B (32 x 64) and 2.7B (32 x 80) widths and at head_dim 128, Q = 128 prefix rows."""
    import models.modeling_distributed_gpt3 as M
    from ymp import engine, ops
    gcfg, C, beam, kind = DECODE_CASES[case]
    Q, L, n_new = 128, 8, 7
    H, V = gcfg["hidden_size"], gcfg["vocab_size"]
    dec = _decoder(cuda, gcfg, Q, n_new)
    g = torch.Generator().manual_seed(7)
    qf = (0.5 * torch.randn(C, Q, H, generator=g)).to(cuda, BF16)
    ids = torch.randint(0, V, (C, L), generator=g).to(cuda)
    monkeypatch.setenv("YMP_DECODE_GRAPH", "0")
    init = engine.KVCache.__init__

    def poisoned(cache, *a, **k):
        init(cache, *a, **k)
        SS.poison_(cache.store)
    monkeypatch.setattr(engine.KVCache, "__init__", poisoned)
    rec = SS.Recorder(ops)
    rec.install(monkeypatch)
    rec.install_decode(monkeypatch, engine.KVCache, M.DistributedGPT3)
    with torch.no_grad():
        if beam == 0:
            dec.sample(ids, query_embeds=qf, prompt_length=torch.tensor([5, 8] * (C // 2)))
        else:
            dec.beam_search(ids, query_embeds=qf, beam_size=beam, stop_token=dec.config.eod_id)
    torch.cuda.synchronize()
    monkeypatch.undo()
    keys, params = dec._param_list()
    W = {k: pp.detach().to(F64) for k, pp in zip(keys, params)}
    rows, stride = (C, 1) if beam == 0 else (C * beam, beam if C > 1 else 1)
    qf_rows = qf if beam == 0 or C > 1 else qf.repeat(beam, 1, 1)

    def run(X):
        return SS.decode_session(X, W, gcfg, qf_rows.to(F64), B=rows, max_len=L + n_new + Q, stride=stride, kind=kind)

    X, logits = _walk(f"decode.{case}", rec.trace, {}, run, None, cuda)
    assert len(logits) >= 7 and max(X.report.values()) <= 1.0
    ops_seen = {r.op for r in rec.trace}
    assert ("gemm_skinny_wide" if rows > 8 and kind != "gemm" else "gemm_skinny") in ops_seen or kind == "gemm"
    if beam:
        reidx = [r.ins["idx"].tolist() for r in rec.trace if r.op == "event" and r.kw["kind"] == "reindex"]
        assert len(reidx) >= 6
        # after the first step (every beam continues its clip's first) some step takes two beams from one ancestor
        assert any(len(set(ix[c * beam:(c + 1) * beam])) < beam for ix in reidx[1:] for c in range(C)), reidx
