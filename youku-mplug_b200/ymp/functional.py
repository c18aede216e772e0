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
        img, cv = engine.vit_fwd(W, video.to(bf16), vcfg, save=need_bwd)
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
                                 drop=gpt_drop(gcfg, video.device))
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
    """TimeSformer.forward_features: video -> image_embeds [B, 1+T*N, D]."""

    @staticmethod
    def forward(ctx, video, vcfg, keys, *params):
        _require_cuda(video, "VitFn")
        W = {k: as_bf16(p) for k, p in zip(keys, params)}
        need_bwd = any(ctx.needs_input_grad[3:])
        out, c = engine.vit_fwd(W, video.to(bf16), vcfg, save=need_bwd)
        if need_bwd:
            ctx.W, ctx.keys, ctx.c, ctx.params = W, keys, c, params
        return out.view(video.shape[0], -1, out.shape[1])

    @staticmethod
    def backward(ctx, dout):
        store = _GradStore(ctx.keys, ctx.params, ctx.needs_input_grad[3:], dout.device)
        engine.vit_bwd(ctx.W, store.G, ctx.c, dout.reshape(-1, dout.shape[-1]).to(bf16).contiguous())
        ctx.c = None
        return (None, None, None) + store.grads(ctx.keys, ctx.params)


class EvaFn(torch.autograd.Function):
    """EVA image encoder (models/eva_vit.py VisionTransformer.forward_features): image [B,3,H,W] -> tokens [B, 1+N, D]."""

    @staticmethod
    def forward(ctx, image, ecfg, keys, *params):
        _require_cuda(image, "EvaFn")
        W = {k: as_bf16(p) for k, p in zip(keys, params)}
        need_bwd = any(ctx.needs_input_grad[3:])
        out, c = engine.eva_fwd(W, image.to(bf16), ecfg, save=need_bwd)
        if need_bwd:
            ctx.W, ctx.keys, ctx.c, ctx.params = W, keys, c, params
        return out.view(image.shape[0], -1, out.shape[1])

    @staticmethod
    def backward(ctx, dout):
        store = _GradStore(ctx.keys, ctx.params, ctx.needs_input_grad[3:], dout.device)
        engine.eva_bwd(ctx.W, store.G, ctx.c, dout.reshape(-1, dout.shape[-1]).to(bf16).contiguous())
        ctx.c = None
        return (None, None, None) + store.grads(ctx.keys, ctx.params)


class AttnPoolFn(torch.autograd.Function):
    """AttentionPool on learnable_queries.repeat(B): image_embeds [B,K1,D] -> [B,Q,D]."""

    @staticmethod
    def forward(ctx, image_embeds, heads, keys, *params):
        _require_cuda(image_embeds, "AttnPoolFn")
        W = {k: as_bf16(p) for k, p in zip(keys, params)}
        B, K1, D = image_embeds.shape
        need_bwd = any(ctx.needs_input_grad)
        out, c = engine.attn_pool_fwd(W, image_embeds.reshape(B * K1, D).to(bf16).contiguous(), B, heads, save=need_bwd)
        if need_bwd:
            ctx.W, ctx.keys, ctx.c, ctx.params, ctx.shape = W, keys, c, params, (B, K1, D)
        return out.view(B, -1, D)

    @staticmethod
    def backward(ctx, dout):
        store = _GradStore(ctx.keys, ctx.params, ctx.needs_input_grad[3:], dout.device)
        d_img = engine.attn_pool_bwd(ctx.W, store.G, ctx.c, dout.reshape(-1, dout.shape[-1]).to(bf16).contiguous())
        ctx.c = None
        return (d_img.view(ctx.shape), None, None) + store.grads(ctx.keys, ctx.params)


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
                                 drop=gpt_drop(gcfg, input_embeds.device))
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
