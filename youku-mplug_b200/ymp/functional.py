"""torch.autograd bridges over ymp.engine.

Each Function takes the module's parameters as explicit inputs (so autograd / DDP / DeepSpeed see
ordinary nn.Parameters and ordinary .grad tensors) and runs the hand-scheduled forward/backward of
ymp.engine.  `ctx.needs_input_grad` decides which weight gradients are computed at all: frozen
parameters (the GPT-3 decoder, models/distributed_gpt3.py:91-93) cost no wgrad GEMM.
"""
import contextlib

import torch

from . import engine, ops
from .ops import bf16

def as_bf16(p):
    """Kernels consume bf16.  bf16 params are used in place.  fp32 params (module not cast by the caller):
    trainable ones are converted on every call (an optimizer that writes through `p.data` does not bump
    `_version`, so no cache can be trusted for them; 130 M parameters cost ~0.1 ms), frozen ones are converted
    once and the copy is kept ON the parameter object (it dies with it - no id() reuse, no leak) and
    re-validated against version / storage / shape / device."""
    if p.dtype == bf16:
        return p.detach()
    if p.requires_grad:
        return p.detach().to(bf16)
    key = (p._version, p.data_ptr(), tuple(p.shape), p.device)
    ent = getattr(p, "_ymp_bf16", None)
    if ent is None or ent[0] != key:
        ent = (key, p.detach().to(bf16))
        p._ymp_bf16 = ent
    return ent[1]


def _require_cuda(t, what):
    if not t.is_cuda:
        raise RuntimeError(f"{what}: the H100 kernels need CUDA tensors (got {t.device}); there is no CPU fallback")


_SINK = None
_READY = None


@contextlib.contextmanager
def grad_sink(sink, on_ready=None):
    """While active, weight gradients of parameters found in `sink` ({id(param): fp32 flat view}) are
    accumulated straight into those views and autograd receives None for them (ymp.train.TrainEngine).
    `on_ready(prefix)` is called from inside the backward as soon as every weight gradient under a
    state-dict prefix (one TimeSformer block) is final, so that its all-reduce can start while the
    remaining backward still runs."""
    global _SINK, _READY
    prev, _SINK = _SINK, sink
    prev_r, _READY = _READY, on_ready
    try:
        yield
    finally:
        _SINK, _READY = prev, prev_r


class GradDict(dict):
    """key -> fp32 accumulator, plus the `ready(prefix)` notification of the active grad sink."""

    def ready(self, prefix):
        if _READY is not None:
            _READY(prefix)


class _GradStore:
    """fp32 accumulators for the parameters that need grads: views of the active grad sink when there
    is one, otherwise carved from one freshly zeroed flat buffer."""

    def __init__(self, keys, params, needs, dev):
        self.G, self.sunk = GradDict(), set()
        local = []
        for k, p, n in zip(keys, params, needs):
            if not n:
                continue
            if _SINK is not None and id(p) in _SINK:
                self.G[k] = _SINK[id(p)]
                self.sunk.add(k)
            else:
                local.append((k, p))
        total = sum((p.numel() + 3) // 4 * 4 for _, p in local)
        self.flat = torch.zeros(max(total, 4), device=dev, dtype=torch.float32)
        off = 0
        for k, p in local:
            self.G[k] = self.flat[off:off + p.numel()]
            off += (p.numel() + 3) // 4 * 4

    def grads(self, keys, params):
        return tuple(self.G[k].view(p.shape).to(p.dtype) if (k in self.G and k not in self.sunk) else None
                     for k, p in zip(keys, params))


# ------------------------------------------------------------------------------------------ dropout RNG
# One {seed, offset} pair per device, kept in DEVICE memory: every decoder pass takes a private copy (saved for
# its backward, which regenerates the same masks) and advances the offset with an in-stream add, so a captured
# CUDA graph draws fresh masks on every replay without host involvement.
_RNG = {}


def set_dropout_seed(seed, device=None):
    """(Re)seed the decoder's dropout stream (default seed: torch.initial_seed() at first use)."""
    if device is None:
        _RNG.clear()
        _RNG["seed"] = int(seed)
    else:
        dev = torch.device(device)
        _RNG[dev] = dict(state=torch.tensor([int(seed) & 0x7FFFFFFFFFFFFFFF, 0], dtype=torch.int64, device=dev),
                         inc=torch.tensor([0, 1], dtype=torch.int64, device=dev))


def _pass_rng(dev):
    st = _RNG.get(dev)
    if st is None:
        set_dropout_seed(_RNG.get("seed", torch.initial_seed()), dev)
        st = _RNG[dev]
    rng = st["state"].clone()
    st["state"].add_(st["inc"])
    return rng


def gpt_drop(gcfg, dev):
    """engine.GptDrop for one decoder pass, or None (eval mode / both probabilities zero)."""
    if not gcfg.get("training", False):
        return None
    ph, pa = float(gcfg.get("hidden_dropout", 0.0) or 0.0), float(gcfg.get("attention_dropout", 0.0) or 0.0)
    if ph <= 0.0 and pa <= 0.0:
        return None
    return engine.GptDrop(_pass_rng(dev), ph, pa)


# Writes to the model weights that the parameters' autograd version counters do not see: the fused AdamW writes the
# bf16 parameters through raw pointers.  TrainEngine bumps this count on every optimizer step and checkpoint load, and
# state derived from the weights (the evaluation's prefix cache) keys on it.
_weight_writes = 0


def note_weight_write():
    global _weight_writes
    _weight_writes += 1


def weight_writes():
    return _weight_writes


def gpt_dropout_active(gcfg):
    """Would gpt_drop draw masks for a pass with this config (without drawing them)?"""
    return bool(gcfg.get("training", False)) and (float(gcfg.get("hidden_dropout", 0.0) or 0.0) > 0.0
                                                  or float(gcfg.get("attention_dropout", 0.0) or 0.0) > 0.0)


def _vit_recompute(vcfg):
    """TimeSformer grad_ckpt: recompute every block's activations in the backward instead of keeping them."""
    return bool(vcfg.get("grad_ckpt", False))


def _gpt_recompute(gcfg):
    """megatron_cfg.checkpoint_activations: recompute every decoder layer's activations in the backward."""
    return bool(gcfg.get("checkpoint_activations", False))


_TEXT_ROWS = {}


def _text_rows(B, S, Q, dev):
    """int32 row indices b*S + s for s >= Q (cached: the tensor must outlive CUDA-graph replays)."""
    key = (B, S, Q, str(dev))
    if key not in _TEXT_ROWS:
        r = torch.arange(B, device=dev, dtype=torch.int32)[:, None] * S + torch.arange(Q, S, device=dev, dtype=torch.int32)[None, :]
        _TEXT_ROWS[key] = r.reshape(-1).contiguous()
    return _TEXT_ROWS[key]


def masked_mean_loss(losses_bs, loss_mask):
    """models/modeling_distributed_gpt3.py:1612-1617."""
    lm = loss_mask.reshape(-1).float()
    return torch.sum(losses_bs[:, :-1].reshape(-1).float() * lm) / lm.sum()


class PretrainFn(torch.autograd.Function):
    """DistributedGPT3_Pretrain.forward (use_contrastive=False) - models/distributed_gpt3.py:130-166
    end to end: returns (loss, losses [B,S] fp32)."""

    @staticmethod
    def forward(ctx, video, input_ids, targets, loss_mask, vcfg, gcfg, keys, *params):
        _require_cuda(video, "PretrainFn")
        W = {k: as_bf16(p) for k, p in zip(keys, params)}
        B = video.shape[0]
        need_bwd = any(ctx.needs_input_grad[7:])
        img, cv = engine.vit_fwd(W, video.to(bf16), vcfg, save=need_bwd, recompute=need_bwd and _vit_recompute(vcfg))
        q, ca = engine.attn_pool_fwd(W, img, B, vcfg["num_heads"], save=need_bwd)
        Q, L = ca.Q, input_ids.shape[1]
        S = Q + L
        H = gcfg["hidden_size"]
        pos = W[engine.GPT + "embedding.position_embeddings.weight"]
        x_in = torch.empty((B * S, H), device=video.device, dtype=torch.float32)  # fp32 residual stream
        # visual_fc (+ optional visual_norm is Identity without connect_ln) written straight into the
        # decoder input rows [b*S, b*S+Q) with the learned positions added (:136,:155-156; GPT3Embedding :646-650)
        ops.gemm(q, W["visual_fc.weight"], bias=W["visual_fc.bias"], residual=pos, res_row_mod=Q, out=x_in,
                 d_row_block=Q, d_row_stride=S)
        ops.embed_gather(input_ids.contiguous(), W[engine.GPT + "embedding.word_embeddings.weight"], pos, x_in, S, Q)
        train_gpt = any(n for k, n in zip(keys, ctx.needs_input_grad[7:]) if k.startswith(engine.GPT + "encoder.layers"))
        # The visual-prefix positions never reach the loss (loss_mask = cat(0*Q, ...), distributed_gpt3.py:
        # 142-159), so the final LayerNorm, the LM head and the CE run on the B*L text rows only; their
        # per-token losses are reported as 0.
        text_rows = _text_rows(B, S, Q, video.device)
        targets_t = targets[:, Q:].contiguous()
        hid, cg = engine.gpt_fwd(W, x_in, gcfg, B, S, train_w=train_gpt, save=need_bwd, out_rows=text_rows,
                                 drop=gpt_drop(gcfg, video.device), recompute=need_bwd and _gpt_recompute(gcfg))
        logits, losses, lse = engine.lm_head_fwd(W, hid, targets_t)
        losses_bs = torch.zeros((B, S), device=video.device, dtype=torch.float32)
        losses_bs[:, Q:] = losses.view(B, L)
        loss = masked_mean_loss(losses_bs, loss_mask)
        if need_bwd:
            ctx.W, ctx.keys, ctx.cv, ctx.ca, ctx.cg = W, keys, cv, ca, cg
            ctx.q, ctx.hid, ctx.logits, ctx.lse, ctx.targets, ctx.loss_mask = q, hid, logits, lse, targets_t, loss_mask
            ctx.dims = (B, S, Q, H)
            ctx.params = params
        ctx.mark_non_differentiable(losses_bs)
        return loss, losses_bs

    @staticmethod
    def backward(ctx, dloss, _dlosses):
        W, keys, params = ctx.W, ctx.keys, ctx.params
        B, S, Q, H = ctx.dims
        dev = dloss.device
        store = _GradStore(keys, params, ctx.needs_input_grad[7:], dev)
        G = store.G
        for k in (engine.GPT + "embedding.word_embeddings.weight", engine.GPT + "embedding.position_embeddings.weight"):
            if k in G:
                raise NotImplementedError("training the GPT-3 embeddings is not supported (the reference freezes the decoder)")
        lm = ctx.loss_mask.float()
        grow = torch.zeros((B, S), device=dev, dtype=torch.float32)
        grow[:, :-1] = lm * (dloss.float() / lm.sum())
        dhid = engine.lm_head_bwd(W, G, ctx.hid, ctx.logits, ctx.targets, ctx.lse, grow[:, Q:].reshape(-1))
        ctx.logits = None
        dx_in = engine.gpt_bwd(W, G, ctx.cg, dhid)
        dqf = dx_in.view(B, S, H)[:, :Q].reshape(B * Q, H)
        engine.linear_wgrad(dqf, ctx.q, "visual_fc.weight", "visual_fc.bias", G)
        dq = engine.linear_dgrad(dqf, W["visual_fc.weight"])
        d_img = engine.attn_pool_bwd(W, G, ctx.ca, dq)
        engine.vit_bwd(W, G, ctx.cv, d_img)
        ctx.cv = ctx.ca = ctx.cg = None
        return (None,) * 7 + store.grads(keys, params)


class VitFn(torch.autograd.Function):
    """TimeSformer.forward_features: video -> image_embeds [B, 1+T*N, D].  grad: the caller's grad mode
    (torch.is_grad_enabled() where the module is called; inside forward it is always off): without it no block
    activations are kept."""

    @staticmethod
    def forward(ctx, video, vcfg, grad, keys, *params):
        _require_cuda(video, "VitFn")
        W = {k: as_bf16(p) for k, p in zip(keys, params)}
        need_bwd = grad and any(ctx.needs_input_grad[4:])
        out, c = engine.vit_fwd(W, video.to(bf16), vcfg, save=need_bwd, recompute=need_bwd and _vit_recompute(vcfg))
        if need_bwd:
            ctx.W, ctx.keys, ctx.c, ctx.params = W, keys, c, params
        return out.view(video.shape[0], -1, out.shape[1])

    @staticmethod
    def backward(ctx, dout):
        store = _GradStore(ctx.keys, ctx.params, ctx.needs_input_grad[4:], dout.device)
        engine.vit_bwd(ctx.W, store.G, ctx.c, dout.reshape(-1, dout.shape[-1]).to(bf16).contiguous())
        ctx.c = None
        return (None, None, None, None) + store.grads(ctx.keys, ctx.params)


class EvaFn(torch.autograd.Function):
    """EVA image encoder (models/eva_vit.py VisionTransformer.forward_features): image [B,3,H,W] -> tokens [B, 1+N, D].
    grad: the caller's grad mode, as for VitFn."""

    @staticmethod
    def forward(ctx, image, ecfg, grad, keys, *params):
        _require_cuda(image, "EvaFn")
        W = {k: as_bf16(p) for k, p in zip(keys, params)}
        need_bwd = grad and any(ctx.needs_input_grad[4:])
        out, c = engine.eva_fwd(W, image.to(bf16), ecfg, save=need_bwd)
        if need_bwd:
            ctx.W, ctx.keys, ctx.c, ctx.params = W, keys, c, params
        return out.view(image.shape[0], -1, out.shape[1])

    @staticmethod
    def backward(ctx, dout):
        store = _GradStore(ctx.keys, ctx.params, ctx.needs_input_grad[4:], dout.device)
        engine.eva_bwd(ctx.W, store.G, ctx.c, dout.reshape(-1, dout.shape[-1]).to(bf16).contiguous())
        ctx.c = None
        return (None, None, None, None) + store.grads(ctx.keys, ctx.params)


class AttnPoolFn(torch.autograd.Function):
    """AttentionPool on learnable_queries.repeat(B): image_embeds [B,K1,D] -> [B,Q,D].  grad: the caller's grad mode,
    as for VitFn."""

    @staticmethod
    def forward(ctx, image_embeds, heads, grad, keys, *params):
        _require_cuda(image_embeds, "AttnPoolFn")
        W = {k: as_bf16(p) for k, p in zip(keys, params)}
        B, K1, D = image_embeds.shape
        need_bwd = grad and any(ctx.needs_input_grad)
        out, c = engine.attn_pool_fwd(W, image_embeds.reshape(B * K1, D).to(bf16).contiguous(), B, heads, save=need_bwd)
        if need_bwd:
            ctx.W, ctx.keys, ctx.c, ctx.params, ctx.shape = W, keys, c, params, (B, K1, D)
        return out.view(B, -1, D)

    @staticmethod
    def backward(ctx, dout):
        store = _GradStore(ctx.keys, ctx.params, ctx.needs_input_grad[4:], dout.device)
        d_img = engine.attn_pool_bwd(ctx.W, store.G, ctx.c, dout.reshape(-1, dout.shape[-1]).to(bf16).contiguous())
        ctx.c = None
        return (d_img.view(ctx.shape), None, None, None) + store.grads(ctx.keys, ctx.params)


def _pad8(n):
    return (n + 7) // 8 * 8


def _padded_cols(t, dtype=bf16):
    """[M, N] -> a [M, N] view (row stride rounded up to 8 elements) holding t in `dtype`: the GEMM's TMA
    maps need 16-byte aligned rows; columns beyond N are never read (the tensor map's extent is N)."""
    M, N = t.shape
    if N % 8 == 0 and t.dtype == dtype and t.is_contiguous():
        return t
    buf = torch.empty((M, _pad8(N)), device=t.device, dtype=dtype)
    view = buf[:, :N]
    view.copy_(t)
    return view


class LinearFn(torch.autograd.Function):
    """y = x W^T + b on the wgmma GEMM (visual_fc, projection heads, cls_head layers).  Any out_features:
    outputs narrower than / not a multiple of 8 columns (the 2 / 5 / 45-way classifier heads) are written
    into a row-padded buffer and returned as a view."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        _require_cuda(x, "LinearFn")
        x2 = x.reshape(-1, x.shape[-1]).to(bf16).contiguous()
        w = as_bf16(weight)
        N = w.shape[0]
        if x2.shape[1] % 8:
            raise ValueError(f"LinearFn: in_features must be a multiple of 8 (got {x2.shape[1]})")
        b = None
        if bias is not None:
            b = as_bf16(bias)
            if b.data_ptr() % 16:
                b = b.clone()
        out = torch.empty((x2.shape[0], _pad8(N)), device=x2.device, dtype=bf16)[:, :N]
        y = ops.gemm(x2, w, bias=b, out=out)
        ctx.save_for_backward(x2, w)
        ctx.meta = (x.shape, x.dtype, weight.dtype, None if bias is None else bias.dtype)
        ctx.ids = (id(weight), None if bias is None else id(bias))
        return y.reshape(*x.shape[:-1], N) if N % 8 == 0 else y.unflatten(0, x.shape[:-1])

    @staticmethod
    def backward(ctx, dy):
        x2, w = ctx.saved_tensors
        xshape, xdt, wdt, bdt = ctx.meta
        dy2 = _padded_cols(dy.reshape(-1, dy.shape[-1]))
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = ops.gemm(dy2, w, b_t=True).view(xshape).to(xdt)
        wid, bid = ctx.ids
        if ctx.needs_input_grad[1]:
            if _SINK is not None and wid in _SINK:
                ops.gemm(dy2, x2, a_t=True, b_t=True, out=_SINK[wid].view(w.shape), accumulate=True)
            else:
                dw = torch.zeros(w.shape, device=dy.device, dtype=torch.float32)
                ops.gemm(dy2, x2, a_t=True, b_t=True, out=dw, accumulate=True)
                dw = dw.to(wdt)
        if bdt is not None and ctx.needs_input_grad[2]:
            if _SINK is not None and bid in _SINK:
                ops.colsum(dy2, _SINK[bid])
            else:
                db = torch.zeros(w.shape[0], device=dy.device, dtype=torch.float32)
                ops.colsum(dy2, db)
                db = db.to(bdt)
        return dx, dw, db


class MatmulNTFn(torch.autograd.Function):
    """s = x @ y^T in fp32 from bf16 operands on the wgmma GEMM, with both gradients: the similarity
    contractions of the contrastive branches (models/distributed_gpt3.py:186-202, :957-958)."""

    @staticmethod
    def forward(ctx, x, y):
        _require_cuda(x, "MatmulNTFn")
        x2, y2 = x.to(bf16).contiguous(), y.to(bf16).contiguous()
        M, K = x2.shape
        N = y2.shape[0]
        if K % 8:
            raise ValueError(f"MatmulNTFn: the contraction dim must be a multiple of 8 (got {K})")
        out = torch.empty((M, _pad8(N)), device=x2.device, dtype=torch.float32)[:, :N]
        ops.gemm(x2, y2, out=out)
        ctx.save_for_backward(x2, y2)
        ctx.dts = (x.dtype, y.dtype)
        return out

    @staticmethod
    def backward(ctx, ds):
        x2, y2 = ctx.saved_tensors
        dsp = _padded_cols(ds)
        dx = dy = None
        if ctx.needs_input_grad[0]:
            dx = ops.gemm(dsp, y2, b_t=True, out_dtype=torch.float32).to(ctx.dts[0])
        if ctx.needs_input_grad[1]:
            dy = ops.gemm(dsp, x2, a_t=True, b_t=True, out_dtype=torch.float32).to(ctx.dts[1])
        return dx, dy


def matmul_nt(x, y):
    return MatmulNTFn.apply(x, y)


class LayerNormFn(torch.autograd.Function):
    """LayerNormWithForceFP32 (models/vision_transformer.py:69-71) on the LayerNorm kernels; used for the
    optional visual_norm of `connect_ln` configs (models/distributed_gpt3.py:112-116)."""

    @staticmethod
    def forward(ctx, x, weight, bias, eps):
        _require_cuda(x, "LayerNormFn")
        x2 = x.reshape(-1, x.shape[-1]).to(bf16).contiguous()
        w, b = as_bf16(weight), as_bf16(bias)
        y, mean, rstd = ops.layernorm_fwd(x2, w, b, eps)
        ctx.save_for_backward(x2, w, mean, rstd)
        ctx.meta = (x.shape, x.dtype, weight.dtype, id(weight), id(bias))
        return y.view(x.shape)

    @staticmethod
    def backward(ctx, dy):
        x2, w, mean, rstd = ctx.saved_tensors
        xshape, xdt, wdt, wid, bid = ctx.meta
        D = x2.shape[1]
        sunk = _SINK is not None and wid in _SINK
        dg = _SINK[wid] if sunk else torch.zeros(D, device=dy.device, dtype=torch.float32)
        db = _SINK[bid] if sunk else torch.zeros(D, device=dy.device, dtype=torch.float32)
        dx = ops.layernorm_bwd(dy.reshape(-1, D).to(bf16).contiguous(), x2, w, mean, rstd, dgamma=dg, dbeta=db)
        return dx.view(xshape).to(xdt), (None if sunk else dg.to(wdt)), (None if sunk else db.to(wdt)), None


class GptFn(torch.autograd.Function):
    """GPT3Model.forward (models/modeling_distributed_gpt3.py:1309-1366) on input embeddings
    [B,S,H] (positions NOT yet added): returns (logits [B,S,V] bf16, losses [B,S] fp32 or None-like
    zeros when labels is None, hidden [B,S,H])."""

    @staticmethod
    def forward(ctx, input_embeds, labels, gcfg, want_logits, keys, *params):
        _require_cuda(input_embeds, "GptFn")
        W = {k: as_bf16(p) for k, p in zip(keys, params)}
        B, S, H = input_embeds.shape
        pos = W[engine.GPT + "embedding.position_embeddings.weight"]
        x_in = (input_embeds.float() + pos[:S][None].float()).reshape(B * S, H).contiguous()  # fp32 stream
        need_bwd = any(ctx.needs_input_grad)
        train_gpt = any(n for k, n in zip(keys, ctx.needs_input_grad[5:]) if k.startswith(engine.GPT + "encoder.layers"))
        hid, cg = engine.gpt_fwd(W, x_in, gcfg, B, S, train_w=train_gpt, save=need_bwd,
                                 drop=gpt_drop(gcfg, input_embeds.device), recompute=need_bwd and _gpt_recompute(gcfg))
        logits = losses = lse = None
        if labels is not None or want_logits:
            lab = labels if labels is not None else torch.zeros((B, S), dtype=torch.long, device=input_embeds.device)
            logits, losses, lse = engine.lm_head_fwd(W, hid, lab)
        if need_bwd:
            ctx.W, ctx.keys, ctx.cg, ctx.params = W, keys, cg, params
            ctx.hid, ctx.logits, ctx.lse, ctx.labels, ctx.dims = hid, logits, lse, labels, (B, S, H)
            ctx.in_dtype = input_embeds.dtype
        V = gcfg["vocab_size"]
        out_logits = logits.view(B, S, V) if logits is not None else torch.empty(0, device=input_embeds.device)
        out_losses = losses.view(B, S) if (losses is not None and labels is not None) else torch.empty(0, device=input_embeds.device)
        ctx.mark_non_differentiable(out_logits)
        return out_logits, out_losses, hid.view(B, S, H)

    @staticmethod
    def backward(ctx, _dlogits, dlosses, dhid_out):
        W, keys, params = ctx.W, ctx.keys, ctx.params
        B, S, H = ctx.dims
        store = _GradStore(keys, params, ctx.needs_input_grad[5:], dhid_out.device)
        G = store.G
        dhid = dhid_out.reshape(B * S, H).to(bf16).contiguous() if dhid_out is not None else None
        if ctx.labels is not None and dlosses is not None and dlosses.numel() > 0:
            d2 = engine.lm_head_bwd(W, G, ctx.hid, ctx.logits, ctx.labels, ctx.lse,
                                    dlosses.reshape(-1).float().contiguous(), keep_logits=True)
            dhid = d2 if dhid is None else (dhid + d2)
        dx = engine.gpt_bwd(W, G, ctx.cg, dhid)
        ctx.cg = None
        pk = engine.GPT + "embedding.position_embeddings.weight"
        if pk in G:
            G[pk].view(-1, H)[:S].add_(dx.view(B, S, H).float().sum(0))
        return (dx.view(B, S, H).to(ctx.in_dtype), None, None, None, None) + store.grads(keys, params)


def shared_title_layout(V, L, shared=None, used=None):
    """Host-side sizes of gpt_shared_prefix's rows: (P list, Ls, Pmax).  shared: P_v per video (None: all 0), used:
    Le_v per video, the text columns video v's texts use (None: all L).  Ls = max_v (Le_v - P_v) suffix columns per
    text."""
    P = [0] * V if shared is None else [int(p) for p in shared]
    Le = [L] * V if used is None else [int(u) for u in used]
    if len(P) != V or len(Le) != V or any(not (0 <= p < u <= L) for p, u in zip(P, Le)):
        raise ValueError(f"gpt_shared_prefix: need 0 <= shared[v] < used[v] <= {L} for each of {V} videos, "
                         f"got shared={P} used={Le}")
    return P, max(u - p for p, u in zip(P, Le)), max(P)


def shared_title_rows(p_n, t, Q, L, Ls, Pmax, want):
    """Rows of engine.gpt_fwd_shared_prefix's x that hold the caller's text rows want = n*L + j (int64 tensor), and
    whether column j of text n is computed at all (j < P_v + Ls).  p_n: P_v of each text [N]."""
    n, j = want // L, want % L
    p = p_n[n]
    rows = torch.where(j >= p, n * Ls + j - p, p_n.numel() * Ls + (n // t) * (Q + Pmax) + Q + j)
    return rows, j < p + Ls


def cached_title_rows(p_n, t, L, Ls, Pmax, want):
    """shared_title_rows for the layout of a pass with a PrefixKV, [N*Ls suffix rows | V*Pmax title rows]: the rows of
    x that hold the caller's text rows want = n*L + j, and whether column j of text n is computed at all."""
    n, j = want // L, want % L
    p = p_n[n]
    rows = torch.where(j >= p, n * Ls + j - p, p_n.numel() * Ls + (n // t) * Pmax + j)
    return rows, j < p + Ls


def gpt_prefix_kv(query_embeds, gcfg, keys, params):
    """engine.gpt_prefix_kv on the decoder parameters: the keys and values of the V prefixes query_embeds [V,Q,H] at
    every layer, for later gpt_shared_prefix(prefix_kv=...) calls on the same prefixes.  Forward only, no dropout."""
    _require_cuda(query_embeds, "gpt_prefix_kv")
    if gpt_dropout_active(gcfg):
        raise ValueError("gpt_prefix_kv: the decoder's dropout is active; the prefix cache is for evaluation")
    W = {k: as_bf16(p) for k, p in zip(keys, params)}
    with torch.no_grad():
        return engine.gpt_prefix_kv(W, query_embeds, gcfg)


def packed_text_rows(attention_mask):
    """Host-side layout of gpt_text_features' packed rows, from one host read of the mask [B, L]: (starts, lengths,
    pooled), int64 CPU tensors [B + 1], [B], [B].  The pooled column of text b is attention_mask[b].sum() - 1, the
    reference's pooling index (read as Python indexes it: -1 is column L - 1).  Text b keeps its columns 0 ..
    lengths[b] - 1 with lengths[b] = 1 + max(last attended column, pooled column), which holds for a mask with holes
    too; under the causal mask no kept column sees a dropped one.  starts[b] is its first packed row and pooled[b] =
    starts[b] + pooled column its pooled row."""
    att = attention_mask.detach().to("cpu", torch.int64)
    B, L = att.shape
    col = att.sum(-1) - 1
    if bool(((col < -L) | (col >= L)).any()):
        raise ValueError(f"packed_text_rows: pooled columns {col.tolist()} outside a mask of {L} columns")
    col = torch.where(col < 0, col + L, col)
    last = torch.where(att.ne(0), torch.arange(L), -1).amax(-1) if L else torch.full((B,), -1)
    lengths = 1 + torch.maximum(last, col)
    starts = torch.zeros(B + 1, dtype=torch.int64)
    starts[1:] = lengths.cumsum(0)
    return starts, lengths, starts[:-1] + col


def gpt_text_features(tokens, attention_mask, gcfg, keys, params):
    """Final hidden state of each text's pooled column (attention_mask.sum(-1) - 1) for tokens [B, L], from one
    forward-only decoder pass over the texts packed back to back (engine.gpt_fwd_packed; packed_text_rows gives the
    rows): no padding rows, no LM head, no dropout.  The input rows use GptFn's dtype chain (the word embedding in its
    parameter's dtype, then + the position of the column within its text, in fp32), so the result [B, H] bf16 is
    bit-identical to the same rows of GptFn's hidden states on the padded tokens."""
    _require_cuda(tokens, "gpt_text_features")
    if gpt_dropout_active(gcfg):
        raise ValueError("gpt_text_features: the decoder's dropout is active; the packed pass is forward only")
    W = {k: as_bf16(p) for k, p in zip(keys, params)}
    word = dict(zip(keys, params))[engine.GPT + "embedding.word_embeddings.weight"]
    dev = tokens.device
    starts, lengths, pooled = packed_text_rows(attention_mask)
    text = torch.repeat_interleave(torch.arange(len(lengths)), lengths)
    col = torch.arange(int(starts[-1])) - starts[:-1][text]
    text, col = text.to(dev), col.to(dev)
    pos = W[engine.GPT + "embedding.position_embeddings.weight"]
    with torch.no_grad():
        x = (torch.nn.functional.embedding(tokens[text, col], word).float() + pos[col].float()).contiguous()
        return engine.gpt_fwd_packed(W, x, gcfg, starts.to(device=dev, dtype=torch.int32), int(lengths.max()),
                                     pooled.to(device=dev, dtype=torch.int32))


def gpt_shared_prefix(query_embeds, input_embeds, labels, hidden_rows, gcfg, keys, params, shared=None, used=None,
                      prefix_kv=None):
    """Forward-only decoder pass over [prefix v | text n] for N = V*t texts, text n after prefix v = n // t, with each
    prefix computed once (engine.gpt_fwd_shared_prefix).  query_embeds [V,Q,H], input_embeds [N,L,H] (positions NOT
    yet added, the same dtype chain as GptFn on the concatenation), labels [N,L] of the text positions or None,
    hidden_rows: int tensor of text rows n*L + j whose final hidden states are wanted, or None.
    shared: per-video count P_v of leading text columns that all t texts of video v have in common (the title prompt of
    the Cls evaluation), or None.  Those columns are computed once per video, from its first text, after the prefix;
    each text then computes its columns P_v .. P_v + Ls - 1 (used: per-video count Le_v of columns its texts use,
    default L; Ls = max_v (Le_v - P_v)).  A text column that is not computed has loss +0 and hidden state +0: those
    before P_v have no loss (hidden rows there are read from the shared block), those from P_v + Ls on have neither.
    Returns (losses [N,L] fp32 or None, hidden [len(hidden_rows), H] bf16 or None); text position j of sequence n is
    bit-identical to position Q + j of GptFn on the repeated [N, Q+L] layout.
    prefix_kv: the PrefixKV of these query_embeds (gpt_prefix_kv), or None.  With it, no prefix row is computed and the
    values stay bit-identical; query_embeds then only give V, Q and H.  An unfilled one (PrefixKV.empty) is filled by
    this pass, which computes the prefix rows as without it."""
    _require_cuda(input_embeds, "gpt_shared_prefix")
    if gpt_dropout_active(gcfg):
        raise ValueError("gpt_shared_prefix: the decoder's dropout is active; the shared-prefix pass is for evaluation")
    W = {k: as_bf16(p) for k, p in zip(keys, params)}
    V, Q, H = query_embeds.shape
    N, L, _ = input_embeds.shape
    if V == 0 or N % V:
        raise ValueError(f"gpt_shared_prefix: {N} texts do not split evenly over {V} prefixes")
    if prefix_kv is not None:
        got, want_ = (prefix_kv.V, prefix_kv.Q, prefix_kv.H, prefix_kv.layers), (V, Q, H, gcfg["num_hidden_layers"])
        if got != want_:
            raise ValueError(f"gpt_shared_prefix: the PrefixKV holds (V, Q, H, layers) = {got}, the call needs {want_}")
    t, dev = N // V, input_embeds.device
    P, Ls, Pmax = shared_title_layout(V, L, shared, used)
    T = N * Ls
    cached = prefix_kv is not None and prefix_kv.filled
    B = Pmax if cached else Q + Pmax   # block rows per video: [prefix | title] or [title]
    pos = W[engine.GPT + "embedding.position_embeddings.weight"]
    p_n = torch.tensor(P, device=dev).repeat_interleave(t)                   # P_v of each text
    col = p_n[:, None] + torch.arange(Ls, device=dev)[None, :]                # [N, Ls] text column of each suffix row
    cc = col.clamp(max=L - 1)             # (columns past the text's end: any finite row, computed and never read)
    n_ix = torch.arange(N, device=dev)[:, None]
    x = torch.empty((T + V * B, H), device=dev, dtype=torch.float32)  # [suffix rows | blocks (prefix, shared columns)]
    x[:T] = (input_embeds[n_ix, cc].float() + pos[Q + cc].float()).reshape(T, H)
    xb = x[T:].view(V, B, H)
    if not cached:
        xb[:, :Q] = query_embeds.float() + pos[:Q][None].float()
    xb[:, B - Pmax:] = input_embeds[::t, :Pmax].float() + pos[Q:Q + Pmax][None].float()   # video v's first text (rows past P_v: padding)
    complete = all(p + Ls >= L for p in P)   # every text column is computed somewhere
    rows = keep = None
    if hidden_rows is not None or labels is None:
        want = (torch.arange(N * L, device=dev) if hidden_rows is None
                else hidden_rows.to(device=dev, dtype=torch.long))
        rows, keep = (cached_title_rows(p_n, t, L, Ls, Pmax, want) if cached
                      else shared_title_rows(p_n, t, Q, L, Ls, Pmax, want))
        if complete:
            keep = None
        else:
            rows = torch.where(keep, rows, 0)
        rows = rows.to(torch.int32).contiguous()
    with torch.no_grad():
        if labels is None:
            out_rows = rows
        elif rows is None:
            out_rows = None
        else:   # the LM head's suffix rows, then the wanted hidden rows
            out_rows = torch.cat([torch.arange(T, device=dev, dtype=torch.int32), rows])
        hid = engine.gpt_fwd_shared_prefix(W, x, gcfg, V, t, Q, Ls, out_rows=out_rows, shared=P, prefix_kv=prefix_kv)
        losses = hidden = None
        if labels is not None:
            _, sl, _ = engine.lm_head_fwd(W, hid[:T], labels[n_ix, cc].contiguous())
            if Pmax == 0 and Ls == L:
                losses = sl.view(N, L)
            else:
                losses = torch.zeros((N, L), device=dev, dtype=torch.float32)
                ok = col < L
                losses[n_ix.expand(N, Ls)[ok], col[ok]] = sl.view(N, Ls)[ok]
            if rows is not None:
                hidden = hid[T:]
        else:
            hidden = hid
        if hidden is not None and keep is not None:
            hidden = torch.where(keep[:, None], hidden, torch.zeros((), device=dev, dtype=hidden.dtype))
    return losses, hidden
