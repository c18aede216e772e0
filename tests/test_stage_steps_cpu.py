"""The step programs of tests/stage_steps.py without a GPU: their float64 composition is the reference layer
(autograd through oracle/port.py), a trace synthesised from them passes the walker, and a trace with one wiring
defect fails at the step that carries it."""
import pytest
import torch

import stage_steps as SS
from oracle import port
from oracle.make_golden import make_inputs

F64 = torch.float64
VC, GC, Q = port.VCFG_TINY, port.GCFG_TINY, 8
SEED, OFFSET = 1234, 7
GPT = SS.GPT


def _weights(seed=3):
    sd = port.init_state_dict(VC, GC, Q, seed=seed, randomize=True)
    return {k: v.bfloat16().to(F64) for k, v in sd.items()}


def _inputs():
    video, ids, att = make_inputs(2, VC, 5, GC["vocab_size"], 5)
    targets, loss_mask = port.build_targets(ids, att, Q)
    return video.bfloat16().to(F64), ids, att, targets, loss_mask


def _close(got, want, what, tol=1e-5):
    scale = float(want.abs().max())
    err = float((got.reshape(want.shape) - want).abs().max())
    assert err <= tol * scale + 1e-300, f"{what}: max err {err:.3e} vs max |ref| {scale:.3e}"


def _drop(p):
    return SS.Drop(SEED, OFFSET, p, p) if p > 0 else None


def _port_drop(p):
    return dict(seed=SEED, offset=OFFSET, p_hidden=p, p_attn=p) if p > 0 else None


def _pretrain(X, W, drop, trainable, fused=False):
    video, ids, att, targets, loss_mask = _inputs()
    loss, lbs, c = SS.pretrain_fwd(X, W, video, ids, targets, loss_mask, VC, GC, Q, drop=drop, fused=fused)
    SS.pretrain_bwd(X, W, trainable, c, loss_mask)
    return loss, lbs


# ---------------------------------------------------------------------------------- composition
@pytest.mark.parametrize("p,fused", [(0.0, False), (0.1, False), (0.1, True)])
def test_pretrain_steps_compose_to_reference(p, fused):
    """TimeSformer, AttentionPool, visual_fc, the frozen decoder (dgrad only), LM head and CE: loss, per-token losses
    and every trainable parameter's gradient of the float64 step programs against autograd through
    port.pretrain_forward on the same weights and dropout masks.  fused: the patch GEMM reading the video directly,
    with the im2col in the backward only."""
    W = _weights()
    T = set(port.trainable_keys(W))
    X = SS.Exec("exact")
    loss, lbs = _pretrain(X, W, _drop(p), T, fused)
    video, ids, att, targets, loss_mask = _inputs()
    sd = {k: v.clone().requires_grad_(k in T) for k, v in W.items()}
    out = port.pretrain_forward(video, ids, att, sd, VC, GC, return_all=True, drop=_port_drop(p))
    out["loss"].backward()
    _close(loss, out["loss"].detach(), "loss")
    _close(lbs[:, Q:], out["losses"].detach()[:, Q:], "losses")
    assert set(X.G) == T
    for k in sorted(T):
        _close(X.G[k], sd[k].grad, f"grad {k}")


@pytest.mark.parametrize("p", [0.0, 0.1])
def test_decoder_steps_compose_to_reference_train_w(p):
    """gpt3_decoder with every decoder weight trainable (the wgrad steps of each layer), dropout at p: final hidden
    states, the input-embedding gradient and every decoder parameter gradient against autograd."""
    W = _weights()
    g = torch.Generator().manual_seed(5)
    B, S, H = 2, 11, GC["hidden_size"]
    emb = (0.5 * torch.randn(B, S, H, generator=g)).to(F64)
    dh = torch.randn(B, S, H, generator=g).to(F64)
    T = {k for k in W if k.startswith(GPT + "encoder.")}
    X = SS.Exec("exact")
    pos = W[GPT + "embedding.position_embeddings.weight"][:S]
    hid, c = SS.gpt_fwd(X, W, (emb + pos[None]).reshape(B * S, H), GC, B, S, drop=_drop(p))
    dx = SS.gpt_bwd(X, W, T, c, dh.reshape(B * S, H), train_w=True)
    sd = {k: v.clone().requires_grad_(k in T) for k, v in W.items()}
    e = emb.clone().requires_grad_(True)
    ref = port.gpt3_decoder(e, sd, GC, drop=_port_drop(p))
    (ref * dh).sum().backward()
    _close(hid, ref.detach().reshape(B * S, H), "hidden")
    _close(dx, e.grad.reshape(B * S, H), "d input_embeds")
    assert set(X.G) == T
    for k in sorted(T):
        _close(X.G[k], sd[k].grad, f"grad {k}")


# ---------------------------------------------------------------------------------- walker on synthetic traces
def _seed_g(W, T):
    g = torch.Generator().manual_seed(11)
    return {k: (0.01 * torch.randn(W[k].numel(), generator=g)).float().to(F64) for k in sorted(T)}


def _synth_pretrain(tamper=None, p=0.1):
    W = _weights()
    T = set(port.trainable_keys(W))
    G0 = _seed_g(W, T)
    X = SS.Exec("synth", G0=G0, tamper=tamper)
    _pretrain(X, W, _drop(p), T)
    return W, T, G0, X


def _walk_pretrain(W, T, G0, Xs, p=0.1):
    Xw = SS.Exec("walk", G0=G0, trace=Xs.out_trace)
    _pretrain(Xw, W, _drop(p), T)
    Xw.finish({k: v.to(torch.float32) for k, v in Xs.G.items()})
    return Xw


def _synth_decoder(tamper=None, p=0.1):
    W = _weights()
    T = {k for k in W if k.startswith(GPT + "encoder.layers.")}
    G0 = _seed_g(W, T)
    g = torch.Generator().manual_seed(5)
    B, S, H = 2, 11, GC["hidden_size"]
    x = (0.5 * torch.randn(B * S, H, generator=g)).float().to(F64)
    dh = torch.randn(B * S, H, generator=g).bfloat16().to(F64)

    def run(X):
        hid, c = SS.gpt_fwd(X, W, x, GC, B, S, drop=_drop(p))
        return SS.gpt_bwd(X, W, T, c, dh, train_w=True)

    Xs = SS.Exec("synth", G0=G0, tamper=tamper)
    run(Xs)
    return run, G0, Xs


def test_clean_synthetic_trace_passes():
    W, T, G0, Xs = _synth_pretrain()
    Xw = _walk_pretrain(W, T, G0, Xs)
    assert Xw.report and max(Xw.report.values()) <= 1.0
    run, G0, Xs = _synth_decoder()
    Xw = SS.Exec("walk", G0=G0, trace=Xs.out_trace)
    run(Xw)
    Xw.finish({k: v.to(torch.float32) for k, v in Xs.G.items()})


VB0 = SS.VE + "blocks.0."
L0, L1 = GPT + "encoder.layers.0.", GPT + "encoder.layers.1."


def _set_kw(**upd):
    def f(ins, kw, vals):
        kw.update(upd)
        return ins, kw
    return f


def _no_dres(ins, kw, vals):
    ins["dy"] = vals["ap.q_proj.dgrad"]["D"].to(torch.bfloat16).to(F64)
    return ins, kw


def _bias_row_kept(ins, kw, vals):
    r = vals["ap.attn.bwd"]
    ins["x"] = torch.cat([SS.unheads(r["dk"]), SS.unheads(r["dv"])], 1)
    return ins, kw


def _grow_over_b(ins, kw, vals):
    _, _, att, _, loss_mask = _inputs()
    ins["g"] = ins["g"] * float(loss_mask.sum()) / loss_mask.shape[0]
    return ins, kw


def _overwrite(ins, kw, vals):
    kw["accumulate"] = False
    ins["d0"] = torch.zeros(ins["A"].shape[0], ins["B"].shape[0], dtype=F64)   # the buffer is overwritten
    return ins, kw


PRETRAIN_DEFECTS = {
    "a_cls_mean_scale_1": ({VB0 + "cls_mean": _set_kw(scale=1.0)}, VB0 + "cls_mean"),
    "b_cls_dqkv_scale_1_over_T": ({VB0 + "attn.cls_sum": _set_kw(scale=1.0 / VC["num_frames"])}, VB0 + "attn.cls_sum"),
    "c_attn_pool_without_dres": ({"ap.norm1.bwd": _no_dres}, "ap.norm1.bwd"),
    "d_bias_kv_row_not_zeroed": ({"ap.kv_proj.bgrad": _bias_row_kept}, "ap.kv_proj.bgrad"),
    "h_pos_embed0_without_cls": ({"vit.pos_embed0.grad": lambda t, _, v: None}, "G[visual_encoder.pos_embed]"),
    "j_grow_over_batch": ({"ce.bwd": _grow_over_b}, "ce.bwd"),
    "k_wgrad_overwrites": ({VB0 + "mlp.fc2.wgrad": _overwrite}, VB0 + "mlp.fc2.wgrad"),
}


@pytest.mark.parametrize("defect", sorted(PRETRAIN_DEFECTS))
def test_pretrain_wiring_defect_fails_at_its_step(defect):
    tamper, step = PRETRAIN_DEFECTS[defect]
    W, T, G0, Xs = _synth_pretrain(tamper)
    with pytest.raises(SS.StepFailure) as e:
        _walk_pretrain(W, T, G0, Xs)
    assert e.value.step == step, str(e.value)


def _dout_d(ins, kw, vals):
    ins["add"] = vals[L1 + "input_layernorm.bwd"]["dx_drop"]
    return ins, kw


def _dense_undropped(ins, kw, vals):
    ins["A"] = vals[L0 + "post_attention_layernorm.bwd"]["dx"].T
    return ins, kw


def _wrong_site(ins, kw, vals):
    s, o, site, p = kw["drop"]
    kw["drop"] = (s, o, 4 * 1 + 3, p)        # this layer's own MLP site instead of layer 0's
    return ins, kw


DECODER_DEFECTS = {
    "e_post_ln_add_dropped": ({L0 + "post_attention_layernorm.bwd": _dout_d}, L0 + "post_attention_layernorm.bwd"),
    "f_dense_wgrad_undropped": ({L0 + "dense.wgrad": _dense_undropped}, L0 + "dense.wgrad"),
    "g_ln_bwd_wrong_dropout_site": ({L1 + "input_layernorm.bwd": _wrong_site}, L1 + "input_layernorm.bwd"),
    "k_decoder_wgrad_overwrites": ({L1 + "qkv.wgrad": _overwrite}, L1 + "qkv.wgrad"),
}


@pytest.mark.parametrize("defect", sorted(DECODER_DEFECTS))
def test_decoder_wiring_defect_fails_at_its_step(defect):
    tamper, step = DECODER_DEFECTS[defect]
    run, G0, Xs = _synth_decoder(tamper)
    Xw = SS.Exec("walk", G0=G0, trace=Xs.out_trace)
    with pytest.raises(SS.StepFailure) as e:
        run(Xw)
        Xw.finish({k: v.to(torch.float32) for k, v in Xs.G.items()})
    assert e.value.step == step, str(e.value)


# ---------------------------------------------------------------------------------- EVA and the component path
EC = port.ECFG_TINY


def _eva_case(seed=3):
    sd = port.eva_state_dict(EC, GC, Q, seed=seed)
    W = {k: v.bfloat16().to(F64) for k, v in sd.items() if k.startswith(SS.VE)}
    g = torch.Generator().manual_seed(9)
    image = torch.randn(2, 3, EC["img_size"], EC["img_size"], generator=g).bfloat16().to(F64)
    N = (EC["img_size"] // EC["patch_size"]) ** 2
    dout = torch.randn(2 * (N + 1), EC["embed_dim"], generator=g).bfloat16().to(F64)
    return W, image, dout


def test_eva_steps_compose_to_reference():
    """EVA encoder (zero-padded patch K, row-blocked patch store, pre-LN blocks, final norm): tokens, the image
    gradient's effect on every encoder parameter against autograd through port.eva_vit."""
    W, image, dout = _eva_case()
    T = set(W)
    X = SS.Exec("exact")
    out, c = SS.eva_fwd(X, W, image, EC)
    SS.eva_bwd(X, W, T, c, dout)
    sd = {k: v.clone().requires_grad_(True) for k, v in W.items()}
    ref = port.eva_vit(image, sd, EC)
    (ref * dout.view(ref.shape)).sum().backward()
    _close(out, ref.detach().reshape(out.shape), "tokens")
    assert set(X.G) == T
    for k in sorted(T):
        _close(X.G[k], sd[k].grad, f"grad {k}")


def _synth_eva(tamper=None):
    W, image, dout = _eva_case()
    T = set(W)
    G0 = _seed_g(W, T)

    def run(X):
        out, c = SS.eva_fwd(X, W, image, EC)
        SS.eva_bwd(X, W, T, c, dout)

    Xs = SS.Exec("synth", G0=G0, tamper=tamper)
    run(Xs)
    return run, G0, Xs


def test_eva_clean_trace_and_defect_i():
    """A clean EVA trace passes; (i) the pos_embed gradient summed over the patch rows only fails at G[pos_embed]."""
    run, G0, Xs = _synth_eva()
    Xw = SS.Exec("walk", G0=G0, trace=Xs.out_trace)
    run(Xw)
    Xw.finish({k: v.to(torch.float32) for k, v in Xs.G.items()})

    def patch_rows_only(terms, _, vals):
        terms = terms.clone()
        terms[:, 0] = 0.0
        return terms

    run, G0, Xs = _synth_eva({"eva.pos_embed.grad": patch_rows_only})
    Xw = SS.Exec("walk", G0=G0, trace=Xs.out_trace)
    with pytest.raises(SS.StepFailure) as e:
        run(Xw)
        Xw.finish({k: v.to(torch.float32) for k, v in Xs.G.items()})
    assert e.value.step == "G[visual_encoder.pos_embed]", str(e.value)


def _component(X, W, T, p):
    video, ids, att, targets, loss_mask = _inputs()
    losses, c = SS.component_fwd(X, W, video, ids, targets, VC, GC, Q, drop=_drop(p))
    SS.component_bwd(X, W, T, c, loss_mask)
    lm = loss_mask.reshape(-1).to(F64)
    return (losses[:, :-1].reshape(-1) * lm).sum() / lm.sum()


def test_component_path_steps_compose_to_reference():
    """VitFn -> AttnPoolFn -> LinearFn -> GptFn with the CE over every row: the masked-mean loss and every trainable
    gradient against autograd through port.pretrain_forward; a synthesised trace of it passes the walker."""
    W = _weights()
    T = set(port.trainable_keys(W))
    X = SS.Exec("exact")
    loss = _component(X, W, T, 0.1)
    video, ids, att, targets, loss_mask = _inputs()
    sd = {k: v.clone().requires_grad_(k in T) for k, v in W.items()}
    ref = port.pretrain_forward(video, ids, att, sd, VC, GC, drop=_port_drop(0.1))
    ref.backward()
    _close(loss, ref.detach(), "loss")
    for k in sorted(T):
        _close(X.G[k], sd[k].grad, f"grad {k}")
    G0 = _seed_g(W, T)
    Xs = SS.Exec("synth", G0=G0)
    _component(Xs, W, T, 0.1)
    Xw = SS.Exec("walk", G0=G0, trace=Xs.out_trace)
    _component(Xw, W, T, 0.1)
    Xw.finish({k: v.to(torch.float32) for k, v in Xs.G.items()})


# ---------------------------------------------------------------------------------- one stage at a time
def _rand(*shape, seed, scale=1.0):
    return (scale * torch.randn(*shape, generator=torch.Generator().manual_seed(seed))).bfloat16().to(F64)


def _grads_close(X, sd, T):
    assert set(X.G) == T
    for k in sorted(T):
        _close(X.G[k], sd[k].grad, f"grad {k}")


def test_timesformer_block_steps_compose_to_reference():
    """One TimeSformer block on the engine's row layout (token row (b N + n) T + t, then the cls rows) against
    port.timesformer_block: outputs, the input gradient and the block's parameter gradients."""
    W = _weights()
    d = SS.dims_vit(VC, 2)
    B, T_, N, D, R = d["B"], d["T"], d["N"], d["D"], d["R"]
    pre = SS.VE + "blocks.1."
    T = {k for k in W if k.startswith(pre)}
    x4, cls = _rand(B, T_, N, D, seed=1), _rand(B, D, seed=2)
    dx4, dcls = _rand(B, T_, N, D, seed=3), _rand(B, D, seed=4)
    rows = lambda t4, c: torch.cat([t4.permute(0, 2, 1, 3).reshape(R, D), c])  # noqa: E731
    X = SS.Exec("exact")
    out, c = SS.vit_block_fwd(X, W, pre, rows(x4, cls), d)
    dx = SS.vit_block_bwd(X, W, T, pre, c, rows(dx4, dcls), d)
    sd = {k: v.clone().requires_grad_(k in T) for k, v in W.items()}
    xa, ca = x4.clone().requires_grad_(), cls.clone().requires_grad_()
    yo, co = port.timesformer_block(xa, ca, sd, pre, VC["num_heads"])
    ((yo * dx4).sum() + (co * dcls).sum()).backward()
    _close(out, rows(yo.detach(), co.detach()), "block output")
    _close(dx, rows(xa.grad, ca.grad), "d block input")
    _grads_close(X, sd, T)


@pytest.mark.parametrize("fused", [False, True])
def test_timesformer_steps_compose_to_reference(fused):
    """Embedding, blocks and the (t n)-ordered final LayerNorm against port.timesformer for a random output gradient."""
    W = _weights()
    T = {k for k in W if k.startswith(SS.VE)}
    video = _inputs()[0]
    d = SS.dims_vit(VC, 2)
    dout = _rand(2 * (1 + d["T"] * d["N"]), d["D"], seed=5)
    X = SS.Exec("exact")
    out, c = SS.vit_fwd(X, W, video, VC, fused)
    SS.vit_bwd(X, W, T, c, dout)
    sd = {k: v.clone().requires_grad_(k in T) for k, v in W.items()}
    ref = port.timesformer(video, sd, VC)
    (ref * dout.view(ref.shape)).sum().backward()
    _close(out, ref.detach().reshape(out.shape), "image_embeds")
    _grads_close(X, sd, T)


def test_attention_pool_steps_compose_to_reference():
    """AttentionPool on learnable_queries.repeat(B) against port.attention_pool: output, image gradient, and the
    abstractor, bias_k / bias_v and learnable_queries gradients."""
    W = _weights()
    T = {k for k in W if k.startswith(SS.AP) or k == "learnable_queries"}
    B, K1, D = 2, 9, VC["embed_dim"]
    img, dout = _rand(B * K1, D, seed=6), _rand(B * Q, D, seed=7)
    X = SS.Exec("exact")
    out, c = SS.attn_pool_fwd(X, W, img, B, VC["num_heads"])
    d_img = SS.attn_pool_bwd(X, W, T, c, dout)
    sd = {k: v.clone().requires_grad_(k in T) for k, v in W.items()}
    ia = img.view(B, K1, D).clone().requires_grad_()
    ref = port.attention_pool(sd["learnable_queries"].expand(B, -1, -1), ia, sd, VC["num_heads"])
    (ref * dout.view(ref.shape)).sum().backward()
    _close(out, ref.detach().reshape(out.shape), "queries")
    _close(d_img, ia.grad.reshape(d_img.shape), "d image_embeds")
    _grads_close(X, sd, T)


@pytest.mark.parametrize("p", [0.0, 0.1])
def test_gpt3_layer_steps_compose_to_reference(p):
    """One decoder layer (layer 0, train_w) against port.gpt3_layer with its dropout sites: output, input gradient,
    every parameter gradient."""
    W = _weights()
    g = SS.dims_gpt(GC)
    B, S, H = 2, 11, g["H"]
    pre = GPT + "encoder.layers.0."
    T = {k for k in W if k.startswith(pre)}
    x, dout = _rand(B * S, H, seed=8, scale=0.5), _rand(B * S, H, seed=9)
    drop = _drop(p)
    X = SS.Exec("exact")
    out, c = SS.gpt_layer_fwd(X, W, pre, x, g, B, S, drop, 0)
    dout_d = dout if drop is None else dout * SS.drop_mult(drop.bda_mlp(0), range(B * S), H, "cpu")
    dx, _ = SS.gpt_layer_bwd(X, W, T, pre, c, dout, dout_d, g, B, S, drop, 0, True)
    sd = {k: v.clone().requires_grad_(k in T) for k, v in W.items()}
    xa = x.view(B, S, H).clone().requires_grad_()
    ref = port.gpt3_layer(xa, sd, pre, g["nh"], 1, g["eps"], _port_drop(p))
    (ref * dout.view(ref.shape)).sum().backward()
    _close(out, ref.detach().reshape(out.shape), "layer output")
    _close(dx, xa.grad.reshape(dx.shape), "d layer input")
    _grads_close(X, sd, T)


def test_lm_head_steps_compose_to_reference():
    """Tied LM head and CE against port.lm_head_losses: per-token losses, the hidden-state gradient and the word
    embedding gradient (trained) for per-row loss weights."""
    W = _weights()
    emb = GPT + "embedding.word_embeddings.weight"
    T = {emb}
    rows, H, V = 14, GC["hidden_size"], GC["vocab_size"]
    hid = _rand(rows, H, seed=10)
    labels = torch.randint(0, V, (rows,), generator=torch.Generator().manual_seed(11))
    grow = torch.rand(rows, generator=torch.Generator().manual_seed(12)).to(F64)
    X = SS.Exec("exact")
    logits, losses, lse = SS.lm_head_fwd(X, W, hid, labels)
    dhid = SS.lm_head_bwd(X, W, T, hid, logits, labels, lse, grow)
    sd = {k: v.clone().requires_grad_(k in T) for k, v in W.items()}
    ha = hid.view(1, rows, H).clone().requires_grad_()
    _, ref = port.lm_head_losses(ha, sd[emb], labels.view(1, rows))
    (ref.reshape(-1) * grow).sum().backward()
    _close(losses, ref.detach().reshape(-1), "losses")
    _close(dhid, ha.grad.reshape(dhid.shape), "d hidden")
    _grads_close(X, sd, T)


# ---------------------------------------------------------------------------------- decoding
DQ, DPLEN, DSTEPS = 4, 3, 4
GC_HD80 = dict(GC, hidden_size=160, ffn_hidden_size=640, num_attention_heads=2)
GC_HD128 = dict(GC, hidden_size=256, ffn_hidden_size=1024, num_attention_heads=2)
# the beam permutations before each token step of a batched beam search of 2 clips x 2 beams (rows c * 2 + b): each
# keeps a row within its clip; the later ones take two beams from one ancestor after the beams' histories differ
REINDEX = ([1, 0, 3, 2], [1, 0, 2, 3], [1, 1, 2, 2], [0, 1, 3, 3])


def _dec_weights(gcfg, seed=3):
    sd = port.init_state_dict(VC, gcfg, DQ, seed=seed, randomize=True)
    return {k: v.bfloat16().to(F64) for k, v in sd.items() if k.startswith(GPT)}


def _beam_case(gcfg, C=2, beam=2, seed=21):
    """A batched beam search's host events: the prefill of C clips [qf | prompt], then DSTEPS x (reindex, one token per
    row).  Returns (qf [C, Q, H], script, the token history of every row the logits of each decode belong to)."""
    g = torch.Generator().manual_seed(seed)
    V, H = gcfg["vocab_size"], gcfg["hidden_size"]
    qf = (0.5 * torch.randn(C, DQ, H, generator=g)).bfloat16().to(F64)
    prompts = torch.randint(0, V, (C, DPLEN), generator=g)
    script = [("decode", dict(tokens=prompts, query=True))]
    hist = [prompts[b // beam].tolist() for b in range(C * beam)]
    hists = [[prompts[c].tolist() for c in range(C)]]
    for t in range(DSTEPS):
        idx = torch.tensor(REINDEX[t])
        tok = torch.randint(0, V, (C * beam, 1), generator=g)
        script += [("reindex", dict(idx=idx)), ("decode", dict(tokens=tok, query=False))]
        hist = [hist[j] + [int(tok[b])] for b, j in enumerate(idx.tolist())]
        hists.append([list(h) for h in hist])
    return qf, script, hists


def _session(X, W, gcfg, qf, script, kind="skinny", beam=2):
    B = qf.shape[0] * beam
    return SS.decode_session(X, W, gcfg, qf, script, B=B, max_len=DQ + DPLEN + DSTEPS, stride=beam, kind=kind)


def _port_f64(monkeypatch):
    """port computes its LayerNorm statistics and attention scores in fp32 (.float()): keep float64 tensors float64,
    so that port.next_token_logits is the float64 reference."""
    orig = torch.Tensor.float
    monkeypatch.setattr(torch.Tensor, "float", lambda t, *a, **k: t if t.dtype == F64 else orig(t, *a, **k))


@pytest.mark.parametrize("cfg", ["tiny", "hd80", "hd128"])
@pytest.mark.parametrize("kind", ["skinny", "gemm"])
def test_decode_steps_compose_to_reference(monkeypatch, cfg, kind):
    """The prefill and single-token step programs, in exact mode over a batched beam history (shared prefill,
    permutations with repeated ancestors): every decode's logits are port.next_token_logits in float64 of that row's
    [prefix | token history] within 1e-9 of their maximum."""
    _port_f64(monkeypatch)
    gcfg = dict(tiny=GC, hd80=GC_HD80, hd128=GC_HD128)[cfg]
    W = _dec_weights(gcfg)
    qf, script, hists = _beam_case(gcfg)
    logits = _session(SS.Exec("exact"), W, gcfg, qf, script, kind)
    assert len(logits) == len(hists) == DSTEPS + 1
    for t, (got, hs) in enumerate(zip(logits, hists)):
        rows = qf if t == 0 else qf.repeat_interleave(2, 0)
        want = port.next_token_logits(rows, torch.tensor(hs), W, gcfg)
        _close(got, want, f"decode {t} logits", tol=1e-9)


@pytest.mark.parametrize("kind", ["skinny", "gemm"])
def test_clean_decode_trace_passes(kind):
    W = _dec_weights(GC)
    qf, script, _ = _beam_case(GC)
    Xs = SS.Exec("synth")
    want = _session(Xs, W, GC, qf, script, kind)
    Xw = SS.Exec("walk", trace=Xs.out_trace)
    got = _session(Xw, W, GC, qf, None, kind)
    Xw.finish()
    assert len(got) == DSTEPS + 1 and all(torch.equal(a, b) for a, b in zip(got, want))
    assert Xw.report and max(Xw.report.values()) <= 1.0


def _decode_defects(W, qf, script):
    """(tamper, step that must fail) of each wiring defect of the decoding path, on _beam_case's tiny trace."""
    pos = W[GPT + "embedding.position_embeddings.weight"]
    n = DQ + DPLEN
    prompts, tok2 = script[0][1]["tokens"], script[4][1]["tokens"]

    def x_of(emb):
        return emb.to(torch.float32).to(F64).reshape(-1, GC["hidden_size"])

    def token_pos_minus_1(ins, kw, vals):            # decode 2 runs at position n + 1
        ins["x"] = x_of(SS._emb_pos(W, tok2, n, 1))
        return ins, kw

    def prefill_pos_plus_1(ins, kw, vals):
        ins["x"] = x_of(SS._emb_pos(W, prompts, 0, n, qf) - pos[:n] + pos[1:n + 1])
        return ins, kw

    def keys_len(ins, kw, vals):
        ins["k"], ins["v"], kw["keys"] = ins["k"][:, :, :-1], ins["v"][:, :, :-1], kw["keys"] - 1
        return ins, kw

    def rows(f):
        def t(ins, kw, vals):
            kw["out2_rows"] = f(kw["out2_rows"])
            return ins, kw
        return t

    def residual_x(ins, kw, vals):
        ins["residual"] = vals["decode.2.L0.4h_to_h"]["D"]
        return ins, kw

    def wrong_ln(ins, kw, vals):
        pre = GPT + "encoder.layers.1.input_layernorm"
        ins["gamma"], ins["beta"] = W[pre + ".weight"], W[pre + ".bias"]
        return ins, kw

    def first_row(ins, kw, vals):
        r = torch.arange(qf.shape[0], dtype=torch.int32) * n
        ins["x"], kw["in_rows"] = vals["decode.0.L1.4h_to_h"]["D"][r.long()], r
        return ins, kw

    def wrong_clip(ins, kw, vals):
        ins["x"] = ins["x"].roll(n, 0)
        return ins, kw

    return {
        "a_token_position_len_minus_1": ({"decode.2.L0.input_layernorm": token_pos_minus_1}, "decode.2.L0.input_layernorm"),
        "b_prefill_positions_shifted": ({"decode.0.L0.input_layernorm": prefill_pos_plus_1}, "decode.0.L0.input_layernorm"),
        "c_attention_count_len": ({"decode.2.L0.attn": keys_len}, "decode.2.L0.attn"),
        "d_kv_row_at_len_plus_1": ({"decode.2.L0.qkv": rows(lambda r: r + 1)}, "decode.2.L0.qkv"),
        "d_kv_row_other_sequence": ({"decode.2.L0.qkv": rows(lambda r: r.roll(1))}, "decode.2.L0.qkv"),
        "e_reindex_not_applied": ({"decode.3.reindex": lambda p, _, v: None}, "decode.3.L0.attn"),
        "f_share_prefill_not_applied": ({"decode.0.share_prefill": lambda p, _, v: None}, "decode.1.L0.attn"),
        "g_mlp_residual_from_x": ({"decode.2.L1.4h_to_h": residual_x}, "decode.2.L1.4h_to_h"),
        "h_final_layernorm_params": ({"decode.2.final_layernorm": wrong_ln}, "decode.2.final_layernorm"),
        "i_prefill_final_ln_first_row": ({"decode.0.final_layernorm": first_row}, "decode.0.final_layernorm"),
        "j_prefill_wrong_clip": ({"decode.0.L0.input_layernorm": wrong_clip}, "decode.0.L0.input_layernorm"),
    }


DECODE_DEFECTS = ("a_token_position_len_minus_1", "b_prefill_positions_shifted", "c_attention_count_len",
                  "d_kv_row_at_len_plus_1", "d_kv_row_other_sequence", "e_reindex_not_applied",
                  "f_share_prefill_not_applied", "g_mlp_residual_from_x", "h_final_layernorm_params",
                  "i_prefill_final_ln_first_row", "j_prefill_wrong_clip")


@pytest.mark.parametrize("defect", DECODE_DEFECTS)
def test_decode_wiring_defect_fails_at_its_step(defect):
    W = _dec_weights(GC)
    qf, script, _ = _beam_case(GC)
    defects = _decode_defects(W, qf, script)
    assert set(defects) == set(DECODE_DEFECTS)
    tamper, step = defects[defect]
    Xs = SS.Exec("synth", tamper=tamper)
    _session(Xs, W, GC, qf, script)
    Xw = SS.Exec("walk", trace=Xs.out_trace)
    with pytest.raises(SS.StepFailure) as e:
        _session(Xw, W, GC, qf, None)
        Xw.finish()
    assert e.value.step == step, str(e.value)
