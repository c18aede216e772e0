"""Hand-scheduled forward/backward of the mPLUG-Video pre-training hot path on the C-ABI kernels.

No autograd inside: every stage saves exactly what its backward needs, weight gradients are
accumulated in fp32 (split-K atomics in the GEMM epilogue), and the frozen GPT-3 decoder runs
dgrad only (SURVEY.md section 2.2: no wgrad GEMMs, no saved GEMM inputs).

Weights are addressed by the reference's own state_dict keys.  `W` maps key -> bf16 CUDA tensor,
`G` maps key -> fp32 gradient accumulator for the *trainable* keys (absent key == frozen).

The residual streams (ViT x / xt / y, decoder x / x1) are kept in fp32: they are only ever read by
LayerNorm and by the GEMM epilogue's residual add, never by a tensor-core operand, and rounding them
to bf16 84 times along the depth is the dominant error term against the fp32 reference (measured on
the 1.3B config: 1.3 % -> 0.66 % relative L2 error of the logits).  Everything a GEMM consumes is bf16.

Row layouts (all activations are 2-D [rows, features]; bf16 unless noted):
  ViT tokens : row = (b*N + n)*T + t  (patch-major, as inside the reference Block,
               models/vision_transformer.py:247-274), followed by B cls rows  -> RB = B*N*T + B rows
  decoder    : row = b*S + s  (the reference uses [s,b,h]; per-(b,head) arithmetic is identical)
"""
import math

import torch

from . import ops
from .ops import ACT_GELU_ERF, ACT_GELU_TANH, TView, bf16

GPT = "text_decoder.dist_model.language_model."
VE = "visual_encoder."
AP = "attn_pool."


def _zeros_f32(n, dev):
    return torch.zeros(n, device=dev, dtype=torch.float32)


class Ctx(dict):
    """Saved activations of one forward (attribute access for brevity)."""
    __getattr__ = dict.__getitem__
    __setattr__ = dict.__setitem__


# ------------------------------------------------------------------------------------------
# linear helpers
# ------------------------------------------------------------------------------------------
def linear_wgrad(dy, x, wkey, bkey, G):
    """G[wkey] += dy^T x ; G[bkey] += colsum(dy)   (both optional / skipped when frozen)."""
    if wkey in G:
        g = G[wkey]
        ops.gemm(dy, x, a_t=True, b_t=True, out=g.view(dy.shape[1], x.shape[1]), accumulate=True)
    if bkey is not None and bkey in G:
        ops.colsum(dy, G[bkey])


def linear_dgrad(dy, w, **kw):
    """dx = dy @ w   (w is the forward [out, in] weight, consumed MN-major: no transpose copy)."""
    return ops.gemm(dy, w, b_t=True, **kw)


# ------------------------------------------------------------------------------------------
# TimeSformer encoder
# ------------------------------------------------------------------------------------------
class VitDims:
    def __init__(self, vcfg, B):
        self.P, self.D, self.depth = vcfg["patch_size"], vcfg["embed_dim"], vcfg["depth"]
        self.heads, self.T = vcfg["num_heads"], vcfg["num_frames"]
        self.hd = self.D // self.heads
        self.N = (vcfg["img_size"] // self.P) ** 2
        self.hid = int(self.D * vcfg["mlp_ratio"])
        self.B = B
        self.R = B * self.N * self.T
        self.RB = self.R + B
        self.eps = 1e-6
        self.scale = self.hd ** -0.5


_gather_cache = {}


def _final_gather_rows(d, dev):
    """Output row (b, 0)=cls, (b, 1 + t*N + n) <- internal token row (b*N + n)*T + t
    (models/vision_transformer.py:582-585 emits (t n) order after the cls token)."""
    key = (d.B, d.N, d.T, str(dev))
    if key not in _gather_cache:
        b = torch.arange(d.B).view(d.B, 1, 1)
        t = torch.arange(d.T).view(1, d.T, 1)
        n = torch.arange(d.N).view(1, 1, d.N)
        tok = ((b * d.N + n) * d.T + t).reshape(d.B, d.T * d.N)
        cls = (d.R + torch.arange(d.B)).view(d.B, 1)
        _gather_cache[key] = torch.cat([cls, tok], 1).reshape(-1).int().to(dev)
    return _gather_cache[key]


def _qkv_bias(W, pre):
    """cat(q_bias, 0, v_bias) - models/vision_transformer.py:171-175 (K has no bias)."""
    qb, vb = W[pre + "q_bias"], W[pre + "v_bias"]
    return torch.cat([qb, torch.zeros_like(vb), vb])


def _spatial_maps(d, prefix_base_in, prefix_base_out):
    m_in = ops.seqmap(seq_div=d.T, outer_stride=d.N * d.T, inner_stride=1, pos_stride=d.T, n_prefix=1,
                      prefix_base=prefix_base_in, prefix_stride=1, prefix_per_seq=0)
    m_out = ops.seqmap(seq_div=d.T, outer_stride=d.N * d.T, inner_stride=1, pos_stride=d.T, n_prefix=1,
                       prefix_base=prefix_base_out, prefix_stride=1, prefix_per_seq=1)
    return m_in, m_out


def vit_block_fwd(W, pre, x, d, save=True, compute_out=True):
    """Block.forward - models/vision_transformer.py:243-275.  x [RB, D] -> [RB, D].
    compute_out=False skips the mlp.fc2 GEMM and returns None as the output: the recompute in vit_bwd needs only
    the saved activations (the block output is the next block's input, which the forward kept)."""
    R, RB, D, B, T = d.R, d.RB, d.D, d.B, d.T
    c = Ctx()
    # ---- temporal attention over the T frames of each patch
    ln_t, c.m_t, c.r_t = ops.layernorm_fwd(x[:R], W[pre + "temporal_ln.weight"], W[pre + "temporal_ln.bias"], d.eps)
    qkv_t = ops.gemm(ln_t, W[pre + "temporal_attn.qkv.weight"], bias=_qkv_bias(W, pre + "temporal_attn."))
    att_t = torch.empty((R, D), device=x.device, dtype=bf16)
    c.lse_t = ops.attn_temporal_fwd(qkv_t, att_t, R=R, n_heads=d.heads, T=T, D=d.hd, scale=d.scale)
    proj_t = ops.gemm(att_t, W[pre + "temporal_attn.proj.weight"], bias=W[pre + "temporal_attn.proj.bias"])
    xt = torch.empty((RB, D), device=x.device, dtype=torch.float32)
    ops.gemm(proj_t, W[pre + "temporal_fc.weight"], bias=W[pre + "temporal_fc.bias"], residual=x[:R], out=xt[:R])
    xt[R:].copy_(x[R:])
    # ---- spatial attention per frame, cls token shared by the T frames of a sample
    ln_s, c.m_s, c.r_s = ops.layernorm_fwd(xt, W[pre + "norm1.weight"], W[pre + "norm1.bias"], d.eps)
    qkv_s = ops.gemm(ln_s, W[pre + "attn.qkv.weight"], bias=_qkv_bias(W, pre + "attn."))
    att_s = torch.empty((RB + B * T, D), device=x.device, dtype=bf16)  # tokens | cls mean | per-frame cls
    m_in, m_out = _spatial_maps(d, R, RB)
    q, k, v = (TView(qkv_s, i * D, d.hd, m_in) for i in range(3))
    c.lse_s = ops.attn_fwd(q, k, v, TView(att_s, 0, d.hd, m_out), n_seq=B * T, n_heads=d.heads, head_dim=d.hd,
                           s_q=d.N + 1, s_kv=d.N + 1, causal=False, scale=d.scale)
    ops.group_reduce(att_s[RB:], B, T, att_s[R:RB], scale=1.0 / T)  # cls averaged over frames (:262)
    y = ops.gemm(att_s[:RB], W[pre + "attn.proj.weight"], bias=W[pre + "attn.proj.bias"], residual=xt,
                 out_dtype=torch.float32)
    # ---- MLP
    ln_m, c.m_m, c.r_m = ops.layernorm_fwd(y, W[pre + "norm2.weight"], W[pre + "norm2.bias"], d.eps)
    dact = torch.empty((RB, d.hid), device=x.device, dtype=bf16)
    h = ops.gemm(ln_m, W[pre + "mlp.fc1.weight"], bias=W[pre + "mlp.fc1.bias"], act=ACT_GELU_ERF, aux_out=dact)
    out = None
    if compute_out:
        out = ops.gemm(h, W[pre + "mlp.fc2.weight"], bias=W[pre + "mlp.fc2.bias"], residual=y, out_dtype=torch.float32)
    if save:
        c.update(x=x, ln_t=ln_t, qkv_t=qkv_t, att_t=att_t, proj_t=proj_t, xt=xt, ln_s=ln_s, qkv_s=qkv_s,
                 att_s=att_s, y=y, ln_m=ln_m, dact=dact, h=h)
    return out, c


def vit_block_bwd(W, G, pre, c, dout, d):
    """Backward of vit_block_fwd: dout [RB, D] -> dx [RB, D]; accumulates the block's weight grads."""
    R, RB, D, B, T = d.R, d.RB, d.D, d.B, d.T
    dev = dout.device
    # ---- MLP
    linear_wgrad(dout, c.h, pre + "mlp.fc2.weight", pre + "mlp.fc2.bias", G)
    dpre = linear_dgrad(dout, W[pre + "mlp.fc2.weight"], act=ACT_GELU_ERF, aux_in=c.dact)
    linear_wgrad(dpre, c.ln_m, pre + "mlp.fc1.weight", pre + "mlp.fc1.bias", G)
    dln_m = linear_dgrad(dpre, W[pre + "mlp.fc1.weight"])
    dy = ops.layernorm_bwd(dln_m, c.y, W[pre + "norm2.weight"], c.m_m, c.r_m, add=dout,
                           dgamma=G.get(pre + "norm2.weight"), dbeta=G.get(pre + "norm2.bias"))
    # ---- spatial attention
    linear_wgrad(dy, c.att_s[:RB], pre + "attn.proj.weight", pre + "attn.proj.bias", G)
    datt = torch.empty((RB + B * T, D), device=dev, dtype=bf16)
    linear_dgrad(dy, W[pre + "attn.proj.weight"], out=datt[:RB])
    ops.group_reduce(datt[R:RB], B, T, datt[RB:], scale=1.0 / T, broadcast=True)
    dqkv = torch.empty((RB + B * T, 3 * D), device=dev, dtype=bf16)
    m_in, m_out = _spatial_maps(d, R, RB)
    q, k, v = (TView(c.qkv_s, i * D, d.hd, m_in) for i in range(3))
    dq, dk, dv = (TView(dqkv, i * D, d.hd, m_out) for i in range(3))
    ops.attn_bwd(q, k, v, TView(c.att_s, 0, d.hd, m_out), c.lse_s, TView(datt, 0, d.hd, m_out), dq, dk, dv,
                 n_seq=B * T, n_heads=d.heads, head_dim=d.hd, s_q=d.N + 1, s_kv=d.N + 1, causal=False, scale=d.scale)
    ops.group_reduce(dqkv[RB:], B, T, dqkv[R:RB], scale=1.0)  # the shared cls row collects all T frames
    _qkv_wgrad(G, pre + "attn.", dqkv[:RB], c.ln_s, D, dev)
    dln_s = linear_dgrad(dqkv[:RB], W[pre + "attn.qkv.weight"])
    dxt = ops.layernorm_bwd(dln_s, c.xt, W[pre + "norm1.weight"], c.m_s, c.r_s, add=dy,
                            dgamma=G.get(pre + "norm1.weight"), dbeta=G.get(pre + "norm1.bias"))
    # ---- temporal attention
    linear_wgrad(dxt[:R], c.proj_t, pre + "temporal_fc.weight", pre + "temporal_fc.bias", G)
    dproj = linear_dgrad(dxt[:R], W[pre + "temporal_fc.weight"])
    linear_wgrad(dproj, c.att_t, pre + "temporal_attn.proj.weight", pre + "temporal_attn.proj.bias", G)
    datt_t = linear_dgrad(dproj, W[pre + "temporal_attn.proj.weight"])
    dqkv_t = torch.empty((R, 3 * D), device=dev, dtype=bf16)
    ops.attn_temporal_bwd(c.qkv_t, c.att_t, c.lse_t, datt_t, dqkv_t, R=R, n_heads=d.heads, T=T, D=d.hd, scale=d.scale)
    _qkv_wgrad(G, pre + "temporal_attn.", dqkv_t, c.ln_t, D, dev)
    dln_t = linear_dgrad(dqkv_t, W[pre + "temporal_attn.qkv.weight"])
    dx = torch.empty((RB, D), device=dev, dtype=bf16)
    ops.layernorm_bwd(dln_t, c.x[:R], W[pre + "temporal_ln.weight"], c.m_t, c.r_t, add=dxt[:R],
                      dgamma=G.get(pre + "temporal_ln.weight"), dbeta=G.get(pre + "temporal_ln.bias"), dx=dx[:R])
    dx[R:].copy_(dxt[R:])
    return dx


def _qkv_wgrad(G, apre, dqkv, x, D, dev):
    linear_wgrad(dqkv, x, apre + "qkv.weight", None, G)
    # the qkv bias is cat(q_bias, 0, v_bias) (models/vision_transformer.py:171-175): only the q and the v column blocks
    # have a bias gradient, and their column sums accumulate straight into the flat gradient buffer
    if apre + "q_bias" in G:
        ops.colsum(dqkv[:, :D], G[apre + "q_bias"].view(-1))
    if apre + "v_bias" in G:
        ops.colsum(dqkv[:, 2 * D:], G[apre + "v_bias"].view(-1))


def vit_fwd(W, video, vcfg, save=True, recompute=False):
    """TimeSformer.forward_features - models/vision_transformer.py:544-587.
    video [B,3,T,H,W] bf16 -> image_embeds [B*(1+T*N), D] in the reference's (t n) order.
    recompute (with save): activation checkpointing per block (the reference's grad_ckpt, :575-577).  Only each
    block's fp32 input [RB, D] is kept; vit_bwd re-runs the block's forward from it just before its backward."""
    B = video.shape[0]
    d = VitDims(vcfg, B)
    assert video.shape[2] == d.T, f"video has {video.shape[2]} frames, model expects {d.T}"
    dev = video.device
    recompute = bool(save and recompute)
    c = Ctx(d=d, blocks=[], recompute=recompute)
    video = video.contiguous()
    pos, temb = W[VE + "pos_embed"], W[VE + "temporal_embed"]
    table = (pos[0, 1:, None, :] + temb[0, None, :, :]).reshape(d.N * d.T, d.D).contiguous()
    x0 = torch.empty((d.RB, d.D), device=dev, dtype=torch.float32)
    wp = W[VE + "patch_embed.proj.weight"].reshape(d.D, -1)
    # PatchEmbed (:392-398) + position / temporal embedding add (:552-566) in ONE GEMM: the TMA producer gathers the
    # 16x16 patches straight from the video (fused im2col), the epilogue adds bias and the (pos + temporal) table
    fused = ops.fused_im2col_ok(d.T, d.P) and video.shape[1] * d.P * d.P % 64 == 0
    patches = None
    if fused:
        ops.patch_embed_gemm(video, wp, d.P, bias=W.get(VE + "patch_embed.proj.bias"), residual=table, res_row_mod=d.N * d.T,
                             out=x0[:d.R])
    else:   # frame counts below 8 (tiny test configs): explicit patch matrix
        patches = ops.im2col(video, d.P)
        ops.gemm(patches, wp, bias=W.get(VE + "patch_embed.proj.bias"), residual=table, res_row_mod=d.N * d.T, out=x0[:d.R])
    x0[d.R:] = (W[VE + "cls_token"][0, 0].float() + pos[0, 0].float())
    if VE + "norm_pre.weight" in W:
        x, c.m0, c.r0 = ops.layernorm_fwd(x0, W[VE + "norm_pre.weight"], W[VE + "norm_pre.bias"], d.eps,
                                          out_dtype=torch.float32)
    else:
        x = x0
    for i in range(d.depth):
        out, bc = vit_block_fwd(W, f"{VE}blocks.{i}.", x, d, save and not recompute)
        c.blocks.append(x if recompute else bc)   # recompute: blocks[i] is the block's input
        x, bc = out, None
    rows = _final_gather_rows(d, dev)
    out, c.mf, c.rf = ops.layernorm_fwd(x, W[VE + "norm.weight"], W[VE + "norm.bias"], d.eps, in_rows=rows)
    if save:
        c.update(patches=patches, video=video if fused else None, x0=x0, xL=x, rows=rows)
    return out, c


def vit_block_saved(W, c, i):
    """What block i's backward reads: the activations kept by vit_fwd, or in recompute mode the same tensors rebuilt
    from the block's saved input by the same kernels (the forward is deterministic: bit-identical to the kept ones)."""
    if not c.recompute:
        return c.blocks[i]
    return vit_block_fwd(W, f"{VE}blocks.{i}.", c.blocks[i], c.d, compute_out=False)[1]


def vit_bwd(W, G, c, d_out):
    """d_out [B*(1+T*N), D] (grad of image_embeds) -> accumulates all encoder weight grads."""
    d = c.d
    dev = d_out.device
    dx = ops.layernorm_bwd(d_out, c.xL, W[VE + "norm.weight"], c.mf, c.rf, in_rows=c.rows,
                           dgamma=G.get(VE + "norm.weight"), dbeta=G.get(VE + "norm.bias"))
    for i in reversed(range(d.depth)):
        bc = vit_block_saved(W, c, i)
        dx = vit_block_bwd(W, G, f"{VE}blocks.{i}.", bc, dx, d)
        c.blocks[i] = bc = None  # release activations as we go
        if hasattr(G, "ready"):
            G.ready(f"{VE}blocks.{i}.")  # this block's weight gradients are final: their all-reduce may start
    if VE + "norm_pre.weight" in W:
        dx0 = ops.layernorm_bwd(dx, c.x0, W[VE + "norm_pre.weight"], c.m0, c.r0,
                                dgamma=G.get(VE + "norm_pre.weight"), dbeta=G.get(VE + "norm_pre.bias"))
    else:
        dx0 = dx
    # cls_token + pos[0]
    if VE + "cls_token" in G or VE + "pos_embed" in G:
        dcls = _zeros_f32(d.D, dev)
        ops.colsum(dx0[d.R:], dcls)
        if VE + "cls_token" in G:
            G[VE + "cls_token"].view(-1).add_(dcls)
        if VE + "pos_embed" in G:
            G[VE + "pos_embed"].view(d.N + 1, d.D)[0].add_(dcls)
    # pos[1+n] + temporal[t] table: sum over the batch, then over t / n
    if VE + "pos_embed" in G or VE + "temporal_embed" in G:
        dtab = _zeros_f32(d.N * d.T * d.D, dev)
        ops.colsum(dx0[:d.R].view(d.B, d.N * d.T * d.D), dtab)
        dtab = dtab.view(d.N, d.T, d.D)
        if VE + "pos_embed" in G:
            G[VE + "pos_embed"].view(d.N + 1, d.D)[1:].add_(dtab.sum(1))
        if VE + "temporal_embed" in G:
            G[VE + "temporal_embed"].view(d.T, d.D).add_(dtab.sum(0))
    patches = c.patches
    if patches is None and VE + "patch_embed.proj.weight" in G:
        # the forward gathered its operand tiles from the video; the weight gradient (an MN-major B operand: four pixel
        # rows per 128-byte shared-memory row, which TMA boxes cannot produce from [B,C,T,H,W]) materialises the patch
        # matrix here, in the backward only
        patches = ops.im2col(c.video, d.P)
    if patches is not None:
        linear_wgrad(dx0[:d.R], patches, VE + "patch_embed.proj.weight", VE + "patch_embed.proj.bias", G)
    elif VE + "patch_embed.proj.bias" in G:
        ops.colsum(dx0[:d.R], G[VE + "patch_embed.proj.bias"])


# ------------------------------------------------------------------------------------------
# EVA image encoder (SURVEY 8f N3): plain pre-LN ViT over [cls | 16 x 16 patches of 14 x 14 pixels]
# ------------------------------------------------------------------------------------------
class EvaDims:
    def __init__(self, ecfg, B):
        self.P, self.D, self.depth, self.heads = ecfg["patch_size"], ecfg["embed_dim"], ecfg["depth"], ecfg["num_heads"]
        self.hd = self.D // self.heads
        self.N = (ecfg["img_size"] // self.P) ** 2
        self.S = self.N + 1
        self.hid = int(self.D * ecfg["mlp_ratio"])
        self.B, self.R = B, B * (self.N + 1)
        self.eps = ecfg.get("eps", 1e-6)
        self.scale = self.hd ** -0.5


def eva_fwd(W, image, ecfg, save=True):
    """EVA VisionTransformer.forward_features - models/eva_vit.py:334-350 (Block :174-181, Attention :117-145, PatchEmbed
    :200-207 with bias, final norm).  image [B,3,H,W] bf16 -> tokens [B*(1+N), D], row b*(N+1) + i, cls first."""
    B = image.shape[0]
    d = EvaDims(ecfg, B)
    dev = image.device
    c = Ctx(d=d, blocks=[])
    patches = ops.im2col(image.contiguous().unsqueeze(2), d.P)               # [B*N, Kp] (588 -> 592 zero-padded)
    Kp = patches.shape[1]
    wp = W[VE + "patch_embed.proj.weight"].reshape(d.D, -1)
    if wp.shape[1] != Kp:
        wpad = torch.zeros((d.D, Kp), device=dev, dtype=bf16)
        wpad[:, :wp.shape[1]] = wp
        wp = wpad
    pos = W[VE + "pos_embed"][0]
    x = torch.empty((d.R, d.D), device=dev, dtype=torch.float32)
    # patch rows land at b*(N+1) + 1 + n (row re-blocking), position embeddings added by the epilogue
    ops.gemm(patches, wp, bias=W[VE + "patch_embed.proj.bias"], residual=pos[1:], res_row_mod=d.N, out=x[1:], d_row_block=d.N,
             d_row_stride=d.S)
    x.view(B, d.S, d.D)[:, 0] = W[VE + "cls_token"][0, 0].float() + pos[0].float()
    m = ops.dense_map(d.S)
    for i in range(d.depth):
        pre = f"{VE}blocks.{i}."
        bc = Ctx()
        ln1, bc.m1, bc.r1 = ops.layernorm_fwd(x, W[pre + "norm1.weight"], W[pre + "norm1.bias"], d.eps)
        qkv = ops.gemm(ln1, W[pre + "attn.qkv.weight"], bias=_qkv_bias(W, pre + "attn."))
        att = torch.empty((d.R, d.D), device=dev, dtype=bf16)
        q, k, v = (TView(qkv, j * d.D, d.hd, m) for j in range(3))
        bc.lse = ops.attn_fwd(q, k, v, TView(att, 0, d.hd, m), n_seq=B, n_heads=d.heads, head_dim=d.hd, s_q=d.S, s_kv=d.S,
                              causal=False, scale=d.scale)
        x1 = ops.gemm(att, W[pre + "attn.proj.weight"], bias=W[pre + "attn.proj.bias"], residual=x, out_dtype=torch.float32)
        ln2, bc.m2, bc.r2 = ops.layernorm_fwd(x1, W[pre + "norm2.weight"], W[pre + "norm2.bias"], d.eps)
        dact = torch.empty((d.R, d.hid), device=dev, dtype=bf16)
        h = ops.gemm(ln2, W[pre + "mlp.fc1.weight"], bias=W[pre + "mlp.fc1.bias"], act=ACT_GELU_ERF, aux_out=dact)
        xn = ops.gemm(h, W[pre + "mlp.fc2.weight"], bias=W[pre + "mlp.fc2.bias"], residual=x1, out_dtype=torch.float32)
        if save:
            bc.update(x=x, ln1=ln1, qkv=qkv, att=att, x1=x1, ln2=ln2, dact=dact, h=h)
        c.blocks.append(bc)
        x = xn
    out, c.mf, c.rf = ops.layernorm_fwd(x, W[VE + "norm.weight"], W[VE + "norm.bias"], d.eps)
    if save:
        c.update(patches=patches, xL=x, Kp=Kp)
    return out, c


def eva_bwd(W, G, c, d_out):
    """d_out [B*(1+N), D] -> accumulates every encoder weight gradient."""
    d = c.d
    dev = d_out.device
    B = d.B
    m = ops.dense_map(d.S)
    dx = ops.layernorm_bwd(d_out, c.xL, W[VE + "norm.weight"], c.mf, c.rf, dgamma=G.get(VE + "norm.weight"), dbeta=G.get(VE + "norm.bias"))
    for i in reversed(range(d.depth)):
        pre, bc = f"{VE}blocks.{i}.", c.blocks[i]
        linear_wgrad(dx, bc.h, pre + "mlp.fc2.weight", pre + "mlp.fc2.bias", G)
        dpre = linear_dgrad(dx, W[pre + "mlp.fc2.weight"], act=ACT_GELU_ERF, aux_in=bc.dact)
        linear_wgrad(dpre, bc.ln2, pre + "mlp.fc1.weight", pre + "mlp.fc1.bias", G)
        dln2 = linear_dgrad(dpre, W[pre + "mlp.fc1.weight"])
        dx1 = ops.layernorm_bwd(dln2, bc.x1, W[pre + "norm2.weight"], bc.m2, bc.r2, add=dx,
                                dgamma=G.get(pre + "norm2.weight"), dbeta=G.get(pre + "norm2.bias"))
        linear_wgrad(dx1, bc.att, pre + "attn.proj.weight", pre + "attn.proj.bias", G)
        datt = linear_dgrad(dx1, W[pre + "attn.proj.weight"])
        dqkv = torch.empty_like(bc.qkv)
        q, k, v = (TView(bc.qkv, j * d.D, d.hd, m) for j in range(3))
        dq, dk, dv = (TView(dqkv, j * d.D, d.hd, m) for j in range(3))
        ops.attn_bwd(q, k, v, TView(bc.att, 0, d.hd, m), bc.lse, TView(datt, 0, d.hd, m), dq, dk, dv, n_seq=B, n_heads=d.heads,
                     head_dim=d.hd, s_q=d.S, s_kv=d.S, causal=False, scale=d.scale)
        _qkv_wgrad(G, pre + "attn.", dqkv, bc.ln1, d.D, dev)
        dln1 = linear_dgrad(dqkv, W[pre + "attn.qkv.weight"])
        dx = ops.layernorm_bwd(dln1, bc.x, W[pre + "norm1.weight"], bc.m1, bc.r1, add=dx1,
                               dgamma=G.get(pre + "norm1.weight"), dbeta=G.get(pre + "norm1.bias"))
        c.blocks[i] = None
    dx3 = dx.view(B, d.S, d.D)
    if VE + "cls_token" in G:
        G[VE + "cls_token"].view(-1).add_(dx3[:, 0].float().sum(0))
    if VE + "pos_embed" in G:
        G[VE + "pos_embed"].view(d.S, d.D).add_(dx3.float().sum(0))
    dpatch = dx3[:, 1:].reshape(B * d.N, d.D).contiguous()
    pk = VE + "patch_embed.proj.weight"
    if pk in G:
        K = G[pk].numel() // d.D
        if c.Kp == K:
            ops.gemm(dpatch, c.patches, a_t=True, b_t=True, out=G[pk].view(d.D, K), accumulate=True)
        else:   # padded patch rows: accumulate into a padded buffer, fold the real columns back
            tmp = torch.zeros((d.D, c.Kp), device=dev, dtype=torch.float32)
            ops.gemm(dpatch, c.patches, a_t=True, b_t=True, out=tmp, accumulate=True)
            G[pk].view(d.D, K).add_(tmp[:, :K])
    if VE + "patch_embed.proj.bias" in G:
        ops.colsum(dpatch, G[VE + "patch_embed.proj.bias"])


# ------------------------------------------------------------------------------------------
# visual abstractor (AttentionPool) + visual_fc
# ------------------------------------------------------------------------------------------
_pad_cache = {}


def _kv_pad_rows(B, K1, dev):
    """in_rows for the key LayerNorm: each sample gets K1 real rows plus one slot (-1) that the
    learned bias_k / bias_v row (nn.MultiheadAttention add_bias_kv) is written into."""
    key = (B, K1, str(dev))
    if key not in _pad_cache:
        r = torch.arange(B * K1).view(B, K1)
        _pad_cache[key] = torch.cat([r, torch.full((B, 1), -1)], 1).reshape(-1).int().to(dev)
    return _pad_cache[key]


def attn_pool_fwd(W, image_embeds, B, heads, save=True):
    """AttentionPool.forward - models/vision_transformer.py:368-374 on
    learnable_queries.repeat(B) (models/distributed_gpt3.py:134).  image_embeds [B*K1, D] -> [B*Q, D]."""
    dev = image_embeds.device
    D = image_embeds.shape[1]
    K1 = image_embeds.shape[0] // B
    KP = K1 + 1
    hd = D // heads
    lq = W["learnable_queries"][0]
    Q = lq.shape[0]
    c = Ctx(B=B, Q=Q, K1=K1, D=D, heads=heads, hd=hd)
    eps = 1e-6
    # the query block is identical for every sample: normalise / project it once
    xq, c.mq, c.rq = ops.layernorm_fwd(lq, W[AP + "norm1.weight"], W[AP + "norm1.bias"], eps)
    rows = _kv_pad_rows(B, K1, dev)
    kvn, c.mk, c.rk = ops.layernorm_fwd(image_embeds, W[AP + "normk.weight"], W[AP + "normk.bias"], eps, in_rows=rows)
    w_in, b_in = W[AP + "attn.in_proj_weight"], W[AP + "attn.in_proj_bias"]
    qp = ops.gemm(xq, w_in[:D], bias=b_in[:D])
    kvp = ops.gemm(kvn, w_in[D:], bias=b_in[D:])                      # [B*KP, 2D]: k | v
    kvp.view(B, KP, 2 * D)[:, K1] = torch.cat([W[AP + "attn.bias_k"].view(-1), W[AP + "attn.bias_v"].view(-1)])
    att = torch.empty((B * Q, D), device=dev, dtype=bf16)
    mq = ops.seqmap(seq_div=1, outer_stride=0, pos_stride=1)
    mkv, mo = ops.dense_map(KP), ops.dense_map(Q)
    c.lse = ops.attn_fwd(TView(qp, 0, hd, mq), TView(kvp, 0, hd, mkv), TView(kvp, D, hd, mkv), TView(att, 0, hd, mo),
                         n_seq=B, n_heads=heads, head_dim=hd, s_q=Q, s_kv=KP, causal=False, scale=hd ** -0.5)
    # residual from the *normalised* queries (:369-371)
    x1 = ops.gemm(att, W[AP + "attn.out_proj.weight"], bias=W[AP + "attn.out_proj.bias"], residual=xq, res_row_mod=Q,
                  out_dtype=torch.float32)
    ln2, c.m2, c.r2 = ops.layernorm_fwd(x1, W[AP + "norm2.weight"], W[AP + "norm2.bias"], eps)
    dact = torch.empty((B * Q, W[AP + "mlp.fc1.weight"].shape[0]), device=dev, dtype=bf16)
    h = ops.gemm(ln2, W[AP + "mlp.fc1.weight"], bias=W[AP + "mlp.fc1.bias"], act=ACT_GELU_ERF, aux_out=dact)
    out = ops.gemm(h, W[AP + "mlp.fc2.weight"], bias=W[AP + "mlp.fc2.bias"], residual=x1)
    if save:
        c.update(lq=lq, xq=xq, kvn=kvn, qp=qp, kvp=kvp, att=att, x1=x1, ln2=ln2, dact=dact, h=h,
                 image_embeds=image_embeds, rows=rows)
    return out, c


def attn_pool_bwd(W, G, c, dout):
    """dout [B*Q, D] -> d_image_embeds [B*K1, D]; accumulates abstractor + learnable_queries grads."""
    B, Q, K1, D, hd, heads = c.B, c.Q, c.K1, c.D, c.hd, c.heads
    KP = K1 + 1
    dev = dout.device
    linear_wgrad(dout, c.h, AP + "mlp.fc2.weight", AP + "mlp.fc2.bias", G)
    dpre = linear_dgrad(dout, W[AP + "mlp.fc2.weight"], act=ACT_GELU_ERF, aux_in=c.dact)
    linear_wgrad(dpre, c.ln2, AP + "mlp.fc1.weight", AP + "mlp.fc1.bias", G)
    dln2 = linear_dgrad(dpre, W[AP + "mlp.fc1.weight"])
    dx1 = ops.layernorm_bwd(dln2, c.x1, W[AP + "norm2.weight"], c.m2, c.r2, add=dout,
                            dgamma=G.get(AP + "norm2.weight"), dbeta=G.get(AP + "norm2.bias"))
    linear_wgrad(dx1, c.att, AP + "attn.out_proj.weight", AP + "attn.out_proj.bias", G)
    datt = linear_dgrad(dx1, W[AP + "attn.out_proj.weight"])
    dqp_b = torch.empty((B * Q, D), device=dev, dtype=bf16)
    dkvp = torch.empty((B * KP, 2 * D), device=dev, dtype=bf16)
    mq = ops.seqmap(seq_div=1, outer_stride=0, pos_stride=1)
    mkv, mo = ops.dense_map(KP), ops.dense_map(Q)
    ops.attn_bwd(TView(c.qp, 0, hd, mq), TView(c.kvp, 0, hd, mkv), TView(c.kvp, D, hd, mkv), TView(c.att, 0, hd, mo),
                 c.lse, TView(datt, 0, hd, mo), TView(dqp_b, 0, hd, mo), TView(dkvp, 0, hd, mkv), TView(dkvp, D, hd, mkv),
                 n_seq=B, n_heads=heads, head_dim=hd, s_q=Q, s_kv=KP, causal=False, scale=hd ** -0.5)
    # learned bias_k / bias_v row, then zero it so it does not leak into the projection grads
    dkv3 = dkvp.view(B, KP, 2 * D)
    dbias = dkv3[:, K1].float().sum(0)
    if AP + "attn.bias_k" in G:
        G[AP + "attn.bias_k"].view(-1).add_(dbias[:D])
    if AP + "attn.bias_v" in G:
        G[AP + "attn.bias_v"].view(-1).add_(dbias[D:])
    dkv3[:, K1].zero_()
    # shared query block: sum the per-sample grads (query path + residual path)
    dq_sum = _zeros_f32(Q * D, dev)
    ops.colsum(dqp_b.view(B, Q * D), dq_sum)
    dqp = dq_sum.view(Q, D).to(bf16)
    dres = _zeros_f32(Q * D, dev)
    ops.colsum(dx1.view(B, Q * D), dres)
    w_in = W[AP + "attn.in_proj_weight"]
    if AP + "attn.in_proj_weight" in G:
        gw = G[AP + "attn.in_proj_weight"].view(3 * D, D)
        ops.gemm(dqp, c.xq, a_t=True, b_t=True, out=gw[:D], accumulate=True)
        ops.gemm(dkvp, c.kvn, a_t=True, b_t=True, out=gw[D:], accumulate=True)
    if AP + "attn.in_proj_bias" in G:
        gb = G[AP + "attn.in_proj_bias"]
        ops.colsum(dqp, gb[:D])
        ops.colsum(dkvp, gb[D:])
    dxq = linear_dgrad(dqp, w_in[:D], out_dtype=torch.float32)
    dxq = (dxq + dres.view(Q, D)).to(bf16)
    dlq = ops.layernorm_bwd(dxq, c.lq, W[AP + "norm1.weight"], c.mq, c.rq,
                            dgamma=G.get(AP + "norm1.weight"), dbeta=G.get(AP + "norm1.bias"))
    if "learnable_queries" in G:
        G["learnable_queries"].view(Q, D).add_(dlq.float())
    dkvn = linear_dgrad(dkvp, w_in[D:])
    d_img = torch.empty_like(c.image_embeds)
    ops.layernorm_bwd(dkvn, c.image_embeds, W[AP + "normk.weight"], c.mk, c.rk, in_rows=c.rows,
                      dgamma=G.get(AP + "normk.weight"), dbeta=G.get(AP + "normk.bias"), dx=d_img)
    return d_img


# ------------------------------------------------------------------------------------------
# GPT-3 decoder
# ------------------------------------------------------------------------------------------
class GptDrop:
    """Dropout of one decoder pass (the reference runs the frozen decoder in train() mode: hidden_dropout on the
    embeddings and the two bias-dropout-adds, attention_dropout on the probabilities - modeling_distributed_gpt3.py:
    631,732,1056-1078).  `rng` is the pass's {seed, offset} device tensor; the backward regenerates the same masks."""

    def __init__(self, rng, p_hidden, p_attn):
        self.rng, self.p_hidden, self.p_attn = rng, float(p_hidden), float(p_attn)

    def embed(self):
        return ops.Drop(self.rng, ops.site_embed(), self.p_hidden) if self.p_hidden > 0 else None

    def attn(self, i):
        return ops.Drop(self.rng, ops.site_attn(i), self.p_attn) if self.p_attn > 0 else None

    def bda_attn(self, i):
        return ops.Drop(self.rng, ops.site_bda_attn(i), self.p_hidden) if self.p_hidden > 0 else None

    def bda_mlp(self, i):
        return ops.Drop(self.rng, ops.site_bda_mlp(i), self.p_hidden) if self.p_hidden > 0 else None


class GptDims:
    def __init__(self, gcfg):
        self.H = gcfg["hidden_size"]
        self.heads = gcfg["num_attention_heads"]
        self.hd = self.H // self.heads
        self.layers = gcfg["num_hidden_layers"]
        self.F = gcfg.get("ffn_hidden_size") or 4 * self.H
        self.V = gcfg["vocab_size"]
        self.eps = gcfg.get("layernorm_epsilon", 1e-12)
        # q.k / (sqrt(hn)*layer) * layer == q.k / sqrt(hn)  (modeling_distributed_gpt3.py:718-762)
        self.scale = 1.0 / math.sqrt(self.hd)


def gpt_layer_fwd(W, pre, x, g, B, S, train_w=False, drop=None, li=0, compute_out=True, attend=None):
    """GPT3ParallelTransformerLayer.forward - models/modeling_distributed_gpt3.py:1034-1089
    (causal mask over the whole [prefix|text] sequence, :1329-1332; `drop`: GptDrop or None, li: layer index).
    compute_out=False skips the dense_4h_to_h GEMM and returns None as the output (the recompute in gpt_bwd).
    attend(qkv, att): a forward-only attention step over the packed [q|k|v] rows of x in place of the causal one over
    B dense sequences of S rows (gpt_fwd_shared_prefix); such a layer has no backward, so act' is not stored."""
    H, hd = g.H, g.hd
    c = Ctx()
    d_at = drop.attn(li) if drop else None
    d_b1 = drop.bda_attn(li) if drop else None
    d_b2 = drop.bda_mlp(li) if drop else None
    ln1, c.m1, c.r1 = ops.layernorm_fwd(x, W[pre + "input_layernorm.weight"], W[pre + "input_layernorm.bias"], g.eps)
    qkv = ops.gemm(ln1, W[pre + "self_attention.query_key_value.weight"], bias=W[pre + "self_attention.query_key_value.bias"])
    att = torch.empty((x.shape[0], H), device=x.device, dtype=bf16)
    if attend is None:
        m = ops.dense_map(S)
        q, k, v = (TView(qkv, i * hd, 3 * hd, m) for i in range(3))  # rows grouped per head as [q|k|v] (:894-902)
        c.lse = ops.attn_fwd(q, k, v, TView(att, 0, hd, m), n_seq=B, n_heads=g.heads, head_dim=hd, s_q=S, s_kv=S,
                             causal=True, scale=g.scale, drop=d_at)
    else:
        attend(qkv, att)
    x1 = ops.gemm(att, W[pre + "self_attention.dense.weight"], bias=W[pre + "self_attention.dense.bias"], residual=x,
                  out_dtype=torch.float32, drop=d_b1)
    ln2, c.m2, c.r2 = ops.layernorm_fwd(x1, W[pre + "post_attention_layernorm.weight"], W[pre + "post_attention_layernorm.bias"], g.eps)
    dact = torch.empty((x.shape[0], g.F), device=x.device, dtype=bf16) if attend is None else None
    h = ops.gemm(ln2, W[pre + "mlp.dense_h_to_4h.weight"], bias=W[pre + "mlp.dense_h_to_4h.bias"], act=ACT_GELU_TANH, aux_out=dact)
    out = None
    if compute_out:
        out = ops.gemm(h, W[pre + "mlp.dense_4h_to_h.weight"], bias=W[pre + "mlp.dense_4h_to_h.bias"], residual=x1,
                       out_dtype=torch.float32, drop=d_b2)
    c.update(x=x, qkv=qkv, att=att, x1=x1, dact=dact)
    if train_w:
        c.update(ln1=ln1, ln2=ln2, h=h)
    return out, c


def gpt_layer_bwd(W, G, pre, c, dout, g, B, S, drop=None, li=0, dout_d=None):
    """dout: gradient of the layer output (residual stream).  With dropout, dout_d = dropout_backward(dout) for this
    layer's MLP bias-dropout-add (the gradient of the branch output); returns (dx, dx_d) where dx_d is masked for the
    dropout site that produced this layer's input (previous layer's MLP bias-dropout-add, or the embedding)."""
    hd = g.hd
    dev = dout.device
    if dout_d is None:
        dout_d = dout
    if "h" in c:
        linear_wgrad(dout_d, c.h, pre + "mlp.dense_4h_to_h.weight", pre + "mlp.dense_4h_to_h.bias", G)
    dpre = linear_dgrad(dout_d, W[pre + "mlp.dense_4h_to_h.weight"], act=ACT_GELU_TANH, aux_in=c.dact)
    if "ln2" in c:
        linear_wgrad(dpre, c.ln2, pre + "mlp.dense_h_to_4h.weight", pre + "mlp.dense_h_to_4h.bias", G)
    dln2 = linear_dgrad(dpre, W[pre + "mlp.dense_h_to_4h.weight"])
    del dpre   # temporaries go back to the allocator at their last use: the layer's backward peak is what recompute pays
    d_b1 = drop.bda_attn(li) if drop else None
    r = ops.layernorm_bwd(dln2, c.x1, W[pre + "post_attention_layernorm.weight"], c.m2, c.r2, add=dout,
                          dgamma=G.get(pre + "post_attention_layernorm.weight"), dbeta=G.get(pre + "post_attention_layernorm.bias"),
                          drop=d_b1)
    del dln2
    dx1, dx1_d = r if d_b1 is not None else (r, r)
    linear_wgrad(dx1_d, c.att, pre + "self_attention.dense.weight", pre + "self_attention.dense.bias", G)
    datt = linear_dgrad(dx1_d, W[pre + "self_attention.dense.weight"])
    dqkv = torch.empty_like(c.qkv)
    m = ops.dense_map(S)
    q, k, v = (TView(c.qkv, i * hd, 3 * hd, m) for i in range(3))
    dq, dk, dv = (TView(dqkv, i * hd, 3 * hd, m) for i in range(3))
    ops.attn_bwd(q, k, v, TView(c.att, 0, hd, m), c.lse, TView(datt, 0, hd, m), dq, dk, dv, n_seq=B, n_heads=g.heads,
                 head_dim=hd, s_q=S, s_kv=S, causal=True, scale=g.scale, drop=drop.attn(li) if drop else None)
    if "ln1" in c:
        linear_wgrad(dqkv, c.ln1, pre + "self_attention.query_key_value.weight", pre + "self_attention.query_key_value.bias", G)
    dln1 = linear_dgrad(dqkv, W[pre + "self_attention.query_key_value.weight"])
    del dqkv, dq, dk, dv, datt
    d_in = (drop.bda_mlp(li - 1) if li > 0 else drop.embed()) if drop else None
    r = ops.layernorm_bwd(dln1, c.x, W[pre + "input_layernorm.weight"], c.m1, c.r1, add=dx1,
                          dgamma=G.get(pre + "input_layernorm.weight"), dbeta=G.get(pre + "input_layernorm.bias"), drop=d_in)
    return r if d_in is not None else (r, r)


def gpt_fwd(W, x, gcfg, B, S, train_w=False, save=True, out_rows=None, drop=None, recompute=False):
    """x [B*S, H] fp32: input embeddings with the learned position embeddings already added
    (GPT3Embedding.forward, :640-666); with `drop` (GptDrop) the embedding dropout (:631) is applied to x IN PLACE
    first.  Returns final-LN hidden states [B*S, H], or only the rows listed in out_rows (int32 row indices,
    compact [len(out_rows), H]) when the caller needs no others.
    recompute (with save): activation checkpointing per layer (Megatron-LM's checkpoint_activations).  Only each
    layer's fp32 input [B*S, H] is kept; gpt_bwd re-runs the layer's forward from it, with the pass's own dropout
    state, just before its backward."""
    g = GptDims(gcfg)
    if drop is not None and drop.p_hidden <= 0 and drop.p_attn <= 0:
        drop = None
    recompute = bool(save and recompute)
    c = Ctx(g=g, B=B, S=S, layers=[], out_rows=out_rows, drop=drop, train_w=train_w, recompute=recompute)
    if drop is not None and drop.embed() is not None:
        ops.dropout(x, drop.embed())
    for i in range(g.layers):
        out, lc = gpt_layer_fwd(W, f"{GPT}encoder.layers.{i}.", x, g, B, S, train_w, drop, i)
        c.layers.append((x if recompute else lc) if save else None)   # recompute: layers[i] is the layer's input
        x, lc = out, None
    hid, c.mf, c.rf = ops.layernorm_fwd(x, W[GPT + "encoder.final_layernorm.weight"], W[GPT + "encoder.final_layernorm.bias"], g.eps,
                                        in_rows=out_rows)
    if save:
        c.xL = x
    return hid, c


def shared_prefix_maps(V, t, Q, L):
    """Sequence maps of gpt_fwd_shared_prefix's attention over rows [N*L text rows | V*Q prefix rows] (N = V*t,
    sequence n uses prefix n // t): (text rows, keys of a text sequence = its video's prefix then its own text rows,
    prefix rows)."""
    N = V * t
    keys = ops.seqmap(seq_div=t, outer_stride=t * L, inner_stride=L, pos_stride=1, n_prefix=Q, prefix_base=N * L,
                      prefix_stride=Q, prefix_per_seq=0)
    return ops.dense_map(L), keys, ops.dense_map(Q)


def shared_title_maps(V, t, Q, Ls, Pmax):
    """Sequence maps of gpt_fwd_shared_prefix's attention with shared text columns, over rows [N*Ls suffix rows |
    V*(Q + Pmax) block rows] (N = V*t, text n in video n // t): (suffix rows of a text, keys of a text = the first
    Q + P_v rows of its video's block then its own suffix rows, block rows).  The key map's prefix length is not used:
    the attention call reads it per video from its n_prefix table (Q + P_v)."""
    N = V * t
    keys = ops.seqmap(seq_div=t, outer_stride=t * Ls, inner_stride=Ls, pos_stride=1, prefix_base=N * Ls,
                      prefix_stride=Q + Pmax, prefix_per_seq=0)
    return ops.dense_map(Ls), keys, ops.dense_map(Q + Pmax)


def cached_title_maps(V, t, Ls, Pmax):
    """Sequence maps of gpt_fwd_shared_prefix's attention with a PrefixKV, over rows [N*Ls suffix rows | V*Pmax title
    rows] (N = V*t, text n in video n // t): (suffix rows of a text, keys of a text after the cached ones = the first
    P_v title rows of its video then its own suffix rows, title rows).  The key map's prefix length is not used: the
    attention call reads it per video from its n_prefix table (Q + P_v, of which Q come from the cache)."""
    N = V * t
    keys = ops.seqmap(seq_div=t, outer_stride=t * Ls, inner_stride=Ls, pos_stride=1, prefix_base=N * Ls,
                      prefix_stride=Pmax, prefix_per_seq=0)
    return ops.dense_map(Ls), keys, ops.dense_map(Pmax)


class PrefixKV:
    """Keys and values of V visual prefixes of Q rows at every decoder layer (gpt_prefix_kv): kv [layers, V*Q, 2H] bf16,
    row v*Q + i of layer l holds prefix row i of video v, each head's [k | v] columns side by side (head stride 2*hd).
    A later gpt_fwd_shared_prefix reads them instead of computing the prefix rows again.  filled=False (empty()): the
    first gpt_fwd_shared_prefix that receives the handle computes the prefix rows as without one and fills it, so the
    passes of one call share the prefixes without a pass of their own."""

    def __init__(self, kv, V, Q, filled=True):
        self.kv, self.V, self.Q, self.filled = kv, V, Q, filled
        self.layers, self.H = kv.shape[0], kv.shape[2] // 2

    @staticmethod
    def empty(gcfg, V, Q, device):
        g = GptDims(gcfg)
        return PrefixKV(torch.empty((g.layers, V * Q, 2 * g.H), device=device, dtype=bf16), V, Q, filled=False)

    def views(self, li, hd):
        """(kc, vc) TViews of layer li's cache for ops.attn_fwd(cache=...)."""
        return ops.TView(self.kv[li], 0, 2 * hd, None), ops.TView(self.kv[li], hd, 2 * hd, None)


def gpt_prefix_kv(W, query_embeds, gcfg):
    """Run V visual prefixes (query_embeds [V, Q, H], positions 0 .. Q-1) through the decoder layers and keep every
    layer's keys and values: a PrefixKV.  Square causal attention per prefix; no final LayerNorm and no LM head.  Each
    kernel computes a row on its own, so the cached rows are bit-identical to the prefix rows of gpt_fwd_shared_prefix
    and of gpt_fwd on [prefix | text] sequences."""
    g = GptDims(gcfg)
    V, Q, H = query_embeds.shape
    pos = W[GPT + "embedding.position_embeddings.weight"]
    x = (query_embeds.float() + pos[:Q][None].float()).reshape(V * Q, H)
    kv = torch.empty((g.layers, V * Q, 2 * H), device=x.device, dtype=bf16)
    m = ops.dense_map(Q)

    def attend(qkv, att, li):
        kv[li].view(V * Q, g.heads, 2, g.hd).copy_(qkv.view(V * Q, g.heads, 3, g.hd)[:, :, 1:])
        ops.attn_fwd(*(TView(qkv, j * g.hd, 3 * g.hd, m) for j in range(3)), TView(att, 0, g.hd, m), n_seq=V,
                     n_heads=g.heads, head_dim=g.hd, s_q=Q, s_kv=Q, causal=True, scale=g.scale)

    for i in range(g.layers):   # (the last layer's output is not needed, only its keys and values)
        x, _ = gpt_layer_fwd(W, f"{GPT}encoder.layers.{i}.", x, g, None, None, compute_out=i + 1 < g.layers,
                             attend=lambda qkv, att, i=i: attend(qkv, att, i))
    return PrefixKV(kv, V, Q)


def gpt_fwd_shared_prefix(W, x, gcfg, V, t, Q, L, out_rows=None, shared=None, prefix_kv=None):
    """Forward-only decoder pass over V prefixes of Q rows, each followed by t texts of L rows (the scoring evaluations:
    N = V*t sequences [prefix v | text n], v = n // t), without repeating the prefixes.
    x [N*L + V*Q, H] fp32: rows n*L + j are the text embeddings + positions Q + j, rows N*L + v*Q + i the prefix
    embeddings + positions i.  Causal attention lets no prefix row see a text row, so each layer runs its LayerNorms
    and GEMMs once over all rows and attends twice over its packed QKV: square causal over the prefixes, then the text
    rows causally after their video's prefix (s_q = L, per-video key prefix Q).  Every kernel computes each row on its
    own, so the text rows are bit-identical to the same rows of gpt_fwd on the repeated [N, Q + L] layout.
    shared: per-video counts P_v of leading text columns that all t texts of video v have in common (the title prompt
    of the Cls evaluation; None: all 0).  Those columns are computed once per video as part of its block, and L is the
    number of suffix columns per text (Ls).  x [N*L + V*(Q + Pmax), H], Pmax = max P_v:
      row n*L + j:                    text column P_v + j of text n (position Q + P_v + j);
      row N*L + v*(Q + Pmax) + i:     prefix row i (i < Q), text column i - Q of video v's texts (position i) up to
                                      Q + P_v; the Pmax - P_v rows after them are padding that no kept row attends to.
    The text rows attend to Q + P_v block rows of their video through the per-video prefix table.
    prefix_kv: a PrefixKV of the same V prefixes (gpt_prefix_kv).  No prefix row is computed then, and x holds only
    [N*L suffix rows | V*Pmax title rows]: row N*L + v*Pmax + i is text column i of video v's texts (position Q + i);
    the title rows attend to their video's Q cached keys, then causally to each other, and the text rows to the Q
    cached keys, their video's P_v title rows, then their own rows.  Every row stays bit-identical.  An unfilled
    prefix_kv (PrefixKV.empty) takes the layout without one; the pass fills it with its prefix rows' keys and values.
    Returns the final-LayerNorm hidden states of out_rows (int32 indices into x's rows; default: all text rows)."""
    g = GptDims(gcfg)
    N, hd = V * t, g.hd
    T = N * L
    shared = [0] * V if shared is None else [int(p) for p in shared]
    assert len(shared) == V and min(shared) >= 0, shared
    Pmax = max(shared)
    if prefix_kv is not None:
        assert (prefix_kv.V, prefix_kv.Q, prefix_kv.H, prefix_kv.layers) == (V, Q, g.H, g.layers), "PrefixKV shape"
    cached = prefix_kv is not None and prefix_kv.filled
    fill = prefix_kv is not None and not cached
    B = Pmax if cached else Q + Pmax   # rows of a video's block
    assert x.shape == (T + V * B, g.H) and x.dtype == torch.float32
    n_prefix = torch.tensor([Q + p for p in shared], dtype=torch.int32, device=x.device)
    if not cached:
        m_txt, m_keys, m_blk = shared_title_maps(V, t, Q, L, Pmax)
    else:
        m_txt, m_keys, m_blk = cached_title_maps(V, t, L, Pmax)
        n_title = torch.full((V,), Q, dtype=torch.int32, device=x.device)

    def attend(qkv, att, li):
        pq, pa = qkv[T:], att[T:]
        cache = None
        if not cached:
            ops.attn_fwd(*(TView(pq, i * hd, 3 * hd, m_blk) for i in range(3)), TView(pa, 0, hd, m_blk), n_seq=V,
                         n_heads=g.heads, head_dim=hd, s_q=B, s_kv=B, causal=True, scale=g.scale)
            if fill:
                prefix_kv.kv[li].view(V, Q, g.heads, 2, hd).copy_(pq.view(V, B, g.heads, 3, hd)[:, :Q, :, 1:])
        else:
            cache = (*prefix_kv.views(li, hd), Q)
            if Pmax:
                ops.attn_fwd(*(TView(pq, i * hd, 3 * hd, m_blk) for i in range(3)), TView(pa, 0, hd, m_blk), n_seq=V,
                             n_heads=g.heads, head_dim=hd, s_q=Pmax, s_kv=Q + Pmax, causal=True, scale=g.scale,
                             n_prefix=n_title, cache=cache)
        ops.attn_fwd(TView(qkv, 0, 3 * hd, m_txt), TView(qkv, hd, 3 * hd, m_keys), TView(qkv, 2 * hd, 3 * hd, m_keys),
                     TView(att, 0, hd, m_txt), n_seq=N, n_heads=g.heads, head_dim=hd, s_q=L, s_kv=Q + Pmax + L,
                     causal=True, scale=g.scale, n_prefix=n_prefix, cache=cache)

    for i in range(g.layers):
        x, _ = gpt_layer_fwd(W, f"{GPT}encoder.layers.{i}.", x, g, None, None,
                             attend=lambda qkv, att, i=i: attend(qkv, att, i))
    if fill:
        prefix_kv.filled = True
    if out_rows is None:
        out_rows = torch.arange(T, device=x.device, dtype=torch.int32)
    hid, _, _ = ops.layernorm_fwd(x, W[GPT + "encoder.final_layernorm.weight"], W[GPT + "encoder.final_layernorm.bias"], g.eps,
                                  in_rows=out_rows)
    return hid


def gpt_fwd_packed(W, x, gcfg, starts, max_len, out_rows):
    """Forward-only decoder pass over sequences stored back to back without padding rows (the retrieval text features).
    x [T, H] fp32: sequence s is rows starts[s] .. starts[s+1]-1 (starts: int32 CUDA tensor [n_seq + 1]), row starts[s]
    + j holding its embedding + position j; max_len bounds every length.  Each layer runs its LayerNorms and GEMMs over
    the T rows and causal attention within each sequence (ops.attn_fwd_packed).  Every kernel computes each row on its
    own, so each row is bit-identical to the same row of gpt_fwd on the sequences padded to a common length.  No dropout,
    no LM head, nothing kept for a backward.  Returns the final-LayerNorm hidden states of out_rows (int32 indices into
    x's rows), [len(out_rows), H] bf16."""
    g = GptDims(gcfg)
    assert x.dim() == 2 and x.shape[1] == g.H and x.dtype == torch.float32

    def attend(qkv, att):
        ops.attn_fwd_packed(*(TView(qkv, j * g.hd, 3 * g.hd, None) for j in range(3)), TView(att, 0, g.hd, None),
                            starts=starts, max_len=max_len, n_heads=g.heads, head_dim=g.hd, scale=g.scale)

    for i in range(g.layers):
        x, _ = gpt_layer_fwd(W, f"{GPT}encoder.layers.{i}.", x, g, None, None, attend=attend)
    hid, _, _ = ops.layernorm_fwd(x, W[GPT + "encoder.final_layernorm.weight"], W[GPT + "encoder.final_layernorm.bias"], g.eps,
                                  in_rows=out_rows)
    return hid


def gpt_layer_saved(W, c, i):
    """What layer i's backward reads: the activations kept by gpt_fwd, or in recompute mode the same tensors rebuilt
    from the layer's saved input (deterministic kernels, counter-based dropout masks: bit-identical to the kept ones)."""
    if not c.recompute:
        return c.layers[i]
    return gpt_layer_fwd(W, f"{GPT}encoder.layers.{i}.", c.layers[i], c.g, c.B, c.S, c.train_w, c.drop, i,
                         compute_out=False)[1]


def gpt_bwd(W, G, c, dhid):
    """Returns the gradient w.r.t. the decoder input embeddings (before the embedding dropout when active)."""
    g, B, S, drop = c.g, c.B, c.S, c.drop
    dx = dx_d = None
    if c.out_rows is not None:  # rows without a consumer get no gradient from the final LayerNorm
        dx = torch.zeros((c.xL.shape[0], c.xL.shape[1]), device=dhid.device, dtype=torch.bfloat16)
    d_last = drop.bda_mlp(g.layers - 1) if drop else None
    r = ops.layernorm_bwd(dhid, c.xL, W[GPT + "encoder.final_layernorm.weight"], c.mf, c.rf,
                          dgamma=G.get(GPT + "encoder.final_layernorm.weight"), dbeta=G.get(GPT + "encoder.final_layernorm.bias"),
                          in_rows=c.out_rows, dx=dx, drop=d_last)
    c.xL = None   # the last layer's output is not read again
    dx, dx_d = r if d_last is not None else (r, r)
    for i in reversed(range(g.layers)):
        lc = gpt_layer_saved(W, c, i)
        dx, dx_d = gpt_layer_bwd(W, G, f"{GPT}encoder.layers.{i}.", lc, dx, g, B, S, drop, i, dx_d)
        c.layers[i] = lc = None
    return dx_d


class KVCache:
    """Incremental-decoding state (SURVEY.md 8f N2; the reference's InferenceParams.key_value_memory_dict,
    models/modeling_distributed_gpt3.py:874-923).  One packed QKV buffer [B*max_len, 3H] per layer in the
    per-head [q|k|v] column layout of the QKV GEMM, so new rows are written by the GEMM epilogue itself
    (row re-blocking) and the attention kernels read K/V of all cached positions in place.  All layers live in
    one allocation that never moves (the captured single-token step holds its pointers), and the number of
    cached positions is mirrored on the device (`len_idx`, `len1`) for that graph.

    `rows` [B, max_len] int32 (also allocated once) is the row table the single-token steps read keys through: position p
    of sequence b lives in cache row rows[b, p].  Each position's K/V row is written once, by sequence b at step p into
    its own slot b * max_len + p, and never changes; so a beam search permutes its beams with `reindex`, which gathers
    the table's cached columns and moves no K/V byte.  Columns >= len are never gathered and stay the identity
    b * max_len + p, so every entry always names a valid row (the decode kernel requests keys before it reads the
    device-side count).

    Per-sequence lengths (`lens` int64 [B]: position / cache row of each sequence's next token; `lens1` int32 [B]: keys
    it attends to; host mirror `lens_host`) serve a decoding step whose sequences sit at different positions: a beam
    search that starts a new clip in the beam slots of a finished one (prefill_groups, reindex_rows, set_live).  There
    the table invariant holds per row: column p of row b is the identity b * max_len + p for every p >= lens[b]."""

    def __init__(self, gcfg, batch, max_len, device):
        g = GptDims(gcfg)
        self.g, self.B, self.max_len, self.len = g, batch, max_len, 0
        self.store = torch.zeros((g.layers, batch * max_len, 3 * g.H), device=device, dtype=bf16)
        self.qkv = [self.store[i] for i in range(g.layers)]
        self.len_idx = torch.zeros(1, device=device, dtype=torch.int64)   # = len: position / cache row of the next token
        self.len1 = torch.ones(1, device=device, dtype=torch.int32)       # = len + 1: keys the next token attends to
        self._identity = torch.arange(batch * max_len, device=device, dtype=torch.int32).view(batch, max_len)
        self.rows = self._identity.clone()
        self._indexed = False   # rows differs from the identity
        self.token = None   # TokenStep of the single-token steps (built by the caller that owns the weights)
        self.lens = torch.zeros(batch, device=device, dtype=torch.int64)
        self.lens1 = torch.ones(batch, device=device, dtype=torch.int32)
        self.lens_host = [0] * batch
        self.adv = torch.ones(batch, device=device, dtype=torch.int64)   # 1: the per-row step advances the row, 0: frozen
        self.adv_host = [1] * batch
        self._cols = torch.arange(max_len, device=device, dtype=torch.int64).view(1, max_len)

    def reset(self):
        """Forget the cached positions (the rows are overwritten by the next prefill; stale rows past `len` are never read)."""
        self.len = 0
        self.len_idx.zero_()
        self.len1.fill_(1)
        self._reset_rows()

    def _reset_rows(self):
        if self._indexed:
            self.rows.copy_(self._identity)
            self._indexed = False

    def _set_len(self, n):
        self.len = n
        self.len_idx.fill_(n)
        self.len1.fill_(n + 1)

    def share_prefill(self, stride):
        """After a prefill that wrote only slots b * stride (gpt_decode's seq_stride): every sequence of a group of
        `stride` reads the cached positions from its group's first slot."""
        if stride == 1 or self.len == 0:
            return
        self.rows[:, :self.len] = self._identity[::stride, :self.len].repeat_interleave(stride, 0)
        self._indexed = True

    def reindex(self, idx):
        """Sequence b becomes old sequence idx[b] (beam search) by gathering the row table's cached columns: no K/V byte
        moves.  Single-token steps read through the table; sequence b's next rows still go into its own slots."""
        assert idx.numel() == self.B
        if self.len == 0:
            return
        self.rows[:, :self.len] = self.rows[:, :self.len].index_select(0, idx)
        self._indexed = True

    def _materialize(self):
        """Move the cached rows so that slot b * max_len + p holds position p of sequence b, and reset the table."""
        if not self._indexed:
            return
        if self.len > 0:
            v = self.store.view(self.g.layers, self.B, self.max_len, -1)
            src = self.store.index_select(1, self.rows[:, :self.len].reshape(-1).to(torch.long))
            v[:, :, :self.len].copy_(src.view(self.g.layers, self.B, self.len, -1))
        self._reset_rows()

    def reset_rows(self):
        """Per-row mode: forget every sequence's cached positions; every row is live."""
        self.reset()
        self.lens.zero_()
        self.lens1.fill_(1)
        self.lens_host = [0] * self.B
        self.set_live([True] * self.B)

    def set_live(self, live):
        """Per-row mode: which rows the next single-token steps advance.  A frozen row keeps its length, so its step
        writes its K/V row again at the same position of its own slot and never moves past max_len."""
        live = [1 if x else 0 for x in live]
        assert len(live) == self.B
        if live != self.adv_host:
            self.adv_host = live
            self.adv.copy_(torch.tensor(live, dtype=torch.int64), non_blocking=False)

    def reindex_rows(self, idx):
        """Per-row mode reindex: row b takes old row idx[b]'s table columns p < lens[b] (idx[b] holds at least as many
        positions: a beam search permutes rows within a group of equal lengths) and keeps the identity past them, so no
        row ever reads another row's identity entries."""
        assert idx.numel() == self.B
        self.rows.copy_(torch.where(self._cols < self.lens.view(-1, 1), self.rows.index_select(0, idx), self._identity))
        self._indexed = True

    def prefill_groups(self, W, x, n, group0, group_stride, stride):
        """Per-row mode: run k sequences of n positions (x [k*n, H] fp32, rows i*n + j at positions 0 .. n-1) into
        the first slots of groups group0 + i * group_stride (group g = rows g*stride .. g*stride + stride - 1) while the
        other groups keep their cached positions.  Each group's other rows read the new positions from its first slot
        through the row table (reset to the identity first); the group's lengths become n.  Same kernels as gpt_decode's
        first call, so the rows equal a fresh prefill of the sequence.  Returns the final hidden state of each
        sequence's last position [k, H]."""
        k = x.shape[0] // n
        first = group0 * stride
        assert x.shape[0] == k * n and 0 < n <= self.max_len and first + ((k - 1) * group_stride + 1) * stride <= self.B
        x = _decode_layers(W, x, self, n, 0, k, self.max_len * stride * group_stride, first * self.max_len)
        for i in range(k):
            g0 = first + i * group_stride * stride
            rows = self.rows[g0:g0 + stride]
            rows.copy_(self._identity[g0:g0 + stride])
            rows[:, :n] = self._identity[g0, :n]
            self.lens_host[g0:g0 + stride] = [n] * stride
        sel = torch.tensor([first + i * group_stride * stride + j for i in range(k) for j in range(stride)],
                           dtype=torch.long)
        self.lens.index_fill_(0, sel.to(self.lens.device), n)
        self.lens1.index_fill_(0, sel.to(self.lens.device), n + 1)
        self._indexed = True
        return _last_hidden(W, x, self.g, k, n)

    def reorder(self, idx):
        """Row b of the cache becomes old row idx[b] (beam search, swap_key_value_dict :1460-1473), in place and for
        the cached positions only: two launches for all layers.  A table left by reindex / share_prefill is first
        materialised, so the physical rows always end up as the all-moving history would have left them."""
        assert idx.numel() == self.B
        self._materialize()
        if self.len == 0:
            return
        v = self.store.view(self.g.layers, self.B, self.max_len, -1)[:, :, :self.len]
        v.copy_(v.index_select(1, idx))


class TokenStep:
    """The single-token decoding step (n == 1, cache not empty) for at most ops.SKINNY_WIDE_MAX_ROWS sequences, as ONE
    CUDA graph: every linear is a skinny GEMM (one pass over its weights, csrc/gemv.cu), the new K/V row goes into the cache
    at the device-side position `len_idx`, attention reads `len1` keys (ymp_attn_args.s_kv_dev), and the graph ends by
    advancing both counters - so one captured graph serves every position of every generate() call that reuses this
    cache.  ~8 kernels per layer; the latency floor is the weight stream (2.6 GB at 1.3B).
    per_row: every sequence at its own position (the cache's `lens` / `lens1`): position embeddings gathered per row,
    the new K/V rows written at per-row offsets (ymp_gemm_skinny_rows), attention over per-sequence key counts
    (ymp_attn_fwd_seq_lens), and the graph advances the rows the cache marks live (`adv`)."""

    def __init__(self, cache, W, emb_dtype, sig=None, static=True, per_row=False):
        """sig: anything that changes when the weight tensors behind W move; static: W may be captured (raw pointers)."""
        g, dev = cache.g, cache.store.device
        self.cache, self.W, self.sig, self.static, self.per_row = cache, W, sig, static, per_row
        self.emb_in = torch.zeros((cache.B, g.H), device=dev, dtype=emb_dtype)
        self.stage = torch.zeros((cache.B, 3 * g.H), device=dev, dtype=bf16)   # the new token's [q|k|v] row per sequence
        self.graph = None
        self.out = None
        self.warm = False

    def body(self):
        """Enqueue the step on the current stream (eagerly or under capture): reads emb_in, returns (hid, logits)."""
        c, W = self.cache, self.W
        g, B, ML = c.g, c.B, c.max_len
        H, hd = g.H, g.hd
        pos = W[GPT + "embedding.position_embeddings.weight"]
        x = self.emb_in.float() + pos.index_select(0, c.lens if self.per_row else c.len_idx).float()
        # K/V row of the new token: at the shared device-side length, or at each row's own length
        kv_out = dict(out2_row_off=c.lens) if self.per_row else dict(out2_off=c.len_idx)
        kv_len = dict(kv_lens=c.lens1) if self.per_row else dict(s_kv_dev=c.len1)
        mkv = ops.dense_map(ML)
        # more rows than ymp_gemm_skinny takes (a batched beam search): the wide entry point, same per-row results
        skinny = ops.gemm_skinny if B <= ops.SKINNY_MAX_ROWS else ops.gemm_skinny_wide

        def gemm_ln(a, wname, residual, ln_prefix):
            """fp32 residual-stream GEMM followed by the LayerNorm of its complete result: (y, LN(y))."""
            y = skinny(a, W[wname + ".weight"], bias=W[wname + ".bias"], residual=residual, out_dtype=torch.float32)
            return y, ops.layernorm_fwd(y, W[ln_prefix + ".weight"], W[ln_prefix + ".bias"], g.eps, stats=False)[0]

        ln1, _, _ = ops.layernorm_fwd(x, W[f"{GPT}encoder.layers.0.input_layernorm.weight"], W[f"{GPT}encoder.layers.0.input_layernorm.bias"],
                                      g.eps, stats=False)
        for i in range(g.layers):
            pre = f"{GPT}encoder.layers.{i}."
            st = self.stage
            buf = c.qkv[i]
            # [q|k|v] of the new token: into the staging rows (q for this step) and into cache row b*ML + len (k, v)
            skinny(ln1, W[pre + "self_attention.query_key_value.weight"], bias=W[pre + "self_attention.query_key_value.bias"],
                   out=st, out2=buf, out2_row_stride=ML, **kv_out)
            att = torch.empty((B, H), device=x.device, dtype=bf16)
            q = TView(st, 0, 3 * hd, ops.dense_map(1))
            k, v = TView(buf, hd, 3 * hd, mkv), TView(buf, 2 * hd, 3 * hd, mkv)
            ops.attn_fwd(q, k, v, TView(att, 0, hd, ops.dense_map(1)), n_seq=B, n_heads=g.heads, head_dim=hd, s_q=1, s_kv=ML,
                         causal=False, scale=g.scale, kv_rows=c.rows, **kv_len)
            x1, ln2 = gemm_ln(att, pre + "self_attention.dense", x, pre + "post_attention_layernorm")
            h = skinny(ln2, W[pre + "mlp.dense_h_to_4h.weight"], bias=W[pre + "mlp.dense_h_to_4h.bias"], act=ACT_GELU_TANH)
            nxt = f"{GPT}encoder.layers.{i + 1}.input_layernorm" if i + 1 < g.layers else GPT + "encoder.final_layernorm"
            x, ln1 = gemm_ln(h, pre + "mlp.dense_4h_to_h", x1, nxt)
        hid = ln1
        logits = skinny(hid, W[GPT + "embedding.word_embeddings.weight"], out_dtype=torch.float32)
        if self.per_row:
            c.lens += c.adv
            c.lens1.copy_(c.lens)
            c.lens1 += 1
        else:
            c.len_idx += 1
            c.len1 += 1
        return hid, logits

    def run(self, emb):
        c = self.cache
        use_graph = self.static and decode_graph_enabled()
        n = max(l for l, a in zip(c.lens_host, c.adv_host) if a) if self.per_row and any(c.adv_host) else c.len
        if n + 1 > c.max_len:
            raise ValueError(f"KV cache overflow: {n} + 1 > {c.max_len}")
        self.emb_in.copy_(emb)
        if not use_graph or not self.warm:
            # the first step runs eagerly: it is also the warm-up the capture needs (lazy kernel attributes)
            hid, logits = self.body()
            self.warm = True
        else:
            if self.graph is None:
                torch.cuda.synchronize()
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph):
                    self.out = self.body()
                self.graph = graph
            self.graph.replay()
            hid, logits = self.out[0].clone(), self.out[1].clone()
        if self.per_row:
            c.lens_host = [l + a for l, a in zip(c.lens_host, c.adv_host)]
        else:
            c.len += 1
        return hid, logits


def decode_graph_enabled():
    import os
    return os.environ.get("YMP_DECODE_GRAPH", "1") != "0"


def gpt_decode(W, x, cache, n, seq_stride=1):
    """n new positions per sequence through all layers with the KV cache.  x [B*n, H] fp32 = embeddings +
    learned positions of positions cache.len .. cache.len+n-1 (rows b*n + i).  Either the first call
    (cache empty: causal attention inside the block) or single-token steps (n == 1: the query sees every
    cached key).  Returns the final-LayerNorm hidden state of the LAST new position of every sequence [B, H].
    seq_stride > 1 (first call only): x holds B = cache.B / seq_stride sequences and sequence b goes into cache slot
    b * seq_stride (a batched beam search fills each clip's first beam slot); the row table then points the other
    slots of the group at it, so no cached row is copied.  The single-token steps read keys through the row table."""
    ML, off = cache.max_len, cache.len
    assert cache.B % seq_stride == 0 and (seq_stride == 1 or off == 0)
    B = cache.B // seq_stride
    assert x.shape[0] == B * n
    SL = ML * seq_stride   # cache rows from one sequence to the next
    if off + n > ML:
        raise ValueError(f"KV cache overflow: {off} + {n} > {ML}")
    if off > 0 and n != 1:
        raise NotImplementedError("multi-token continuation after the first block is not supported")
    x = _decode_layers(W, x, cache, n, off, B, SL)
    cache._set_len(off + n)
    cache.share_prefill(seq_stride)
    return _last_hidden(W, x, cache.g, B, n)


def _decode_layers(W, x, cache, n, off, B, SL, row0=0):
    """gpt_decode's layers: B sequences of n new positions from position off, position p of sequence b in cache row
    row0 + b * SL + p.  Returns the last layer's output [B*n, H] fp32."""
    g = cache.g
    H, hd = g.H, g.hd
    for i in range(g.layers):
        pre = f"{GPT}encoder.layers.{i}."
        ln1, _, _ = ops.layernorm_fwd(x, W[pre + "input_layernorm.weight"], W[pre + "input_layernorm.bias"], g.eps, stats=False)
        buf = cache.qkv[i][row0:]
        new_rows = buf[off:]  # GEMM row (b, i) -> buffer row b*SL + off + i
        ops.gemm(ln1, W[pre + "self_attention.query_key_value.weight"], bias=W[pre + "self_attention.query_key_value.bias"],
                 out=new_rows, d_row_block=n, d_row_stride=SL)
        att = torch.empty((B * n, H), device=x.device, dtype=bf16)
        mq = ops.seqmap(seq_div=1, outer_stride=SL, pos_stride=1)
        mkv = ops.dense_map(SL)
        q = TView(new_rows, 0, 3 * hd, mq)
        k, v = TView(buf, hd, 3 * hd, mkv), TView(buf, 2 * hd, 3 * hd, mkv)
        ops.attn_fwd(q, k, v, TView(att, 0, hd, ops.dense_map(n)), n_seq=B, n_heads=g.heads, head_dim=hd, s_q=n, s_kv=off + n,
                     causal=(off == 0 and n > 1), scale=g.scale, kv_rows=cache.rows if n == 1 and off > 0 else None)
        x1 = ops.gemm(att, W[pre + "self_attention.dense.weight"], bias=W[pre + "self_attention.dense.bias"], residual=x,
                      out_dtype=torch.float32)
        ln2, _, _ = ops.layernorm_fwd(x1, W[pre + "post_attention_layernorm.weight"], W[pre + "post_attention_layernorm.bias"], g.eps,
                                      stats=False)
        h = ops.gemm(ln2, W[pre + "mlp.dense_h_to_4h.weight"], bias=W[pre + "mlp.dense_h_to_4h.bias"], act=ACT_GELU_TANH)
        x = ops.gemm(h, W[pre + "mlp.dense_4h_to_h.weight"], bias=W[pre + "mlp.dense_4h_to_h.bias"], residual=x1,
                     out_dtype=torch.float32)
    return x


def _last_hidden(W, x, g, B, n):
    """Final-LayerNorm hidden state of the last of each sequence's n rows of x [B*n, H]: [B, H]."""
    last = torch.arange(B, device=x.device, dtype=torch.int32) * n + (n - 1)
    hid, _, _ = ops.layernorm_fwd(x, W[GPT + "encoder.final_layernorm.weight"], W[GPT + "encoder.final_layernorm.bias"], g.eps,
                                  in_rows=last, stats=False)
    return hid


def lm_head_fwd(W, hid, labels):
    """Tied LM head + per-token CE on fp32 math (modeling_distributed_gpt3.py:1348-1359).
    Returns (logits [B*S, V] bf16, losses [B*S] fp32, lse)."""
    logits = ops.gemm(hid, W[GPT + "embedding.word_embeddings.weight"])
    losses, lse = ops.ce_fwd(logits, labels.reshape(-1).contiguous())
    return logits, losses, lse


def lm_head_bwd(W, G, hid, logits, labels, lse, grad_rows, keep_logits=False):
    """grad_rows [B*S] fp32 = d loss / d losses.  Overwrites `logits` with dlogits unless keep_logits."""
    dlogits = ops.ce_bwd(logits, labels.reshape(-1).contiguous(), lse, grad_rows.contiguous(),
                         dlogits=torch.empty_like(logits) if keep_logits else None)
    emb = GPT + "embedding.word_embeddings.weight"
    if emb in G:
        ops.gemm(dlogits, hid, a_t=True, b_t=True, out=G[emb].view(dlogits.shape[1], hid.shape[1]), accumulate=True)
    return linear_dgrad(dlogits, W[emb])
