"""TEST INFRASTRUCTURE - CPU oracle: a plain-PyTorch fp32 restatement of the reference hot path.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this file.  It is the CHECKER, never the product: the product path (youku-mplug_b200/)
has no dependency on it and fails loudly when its CUDA library is missing.

Parity status: PINNED.  The reference ships no tests or golden vectors (SURVEY.md section 4), so
the pin is generated from the reference itself: oracle/make_golden.py runs the unmodified
reference modules (through oracle/ref_shims.py) and this port on identical seeded inputs and
weights, asserts they agree to fp32 round-off, and commits the reference outputs as fixtures
under tests/golden/.  tests/test_oracle_golden.py re-checks the port against those fixtures on
every run (CPU, no reference tree needed).

Every function cites the reference lines it restates (paths relative to the reference root).
Weights are addressed by the reference's own state_dict keys (SURVEY.md section 8b).
"""
import math
import re

import torch
import torch.nn.functional as F


def layer_norm(x, w, b, eps):
    """LayerNormWithForceFP32.forward - models/vision_transformer.py:69-71 (fp32 statistics);
    megatron LayerNorm - models/modeling_distributed_gpt3.py:1002-1020."""
    return F.layer_norm(x.float(), (x.shape[-1],), w.float(), b.float(), eps).to(x.dtype)


def vit_attention(x, sd, pre, heads):
    """Attention.forward - models/vision_transformer.py:169-207.
    bias = cat(q_bias, 0, v_bias); q scaled by head_dim**-0.5; softmax over fp32 scores."""
    B, N, C = x.shape
    bias = torch.cat([sd[pre + "q_bias"], torch.zeros_like(sd[pre + "v_bias"]), sd[pre + "v_bias"]])
    qkv = F.linear(x, sd[pre + "qkv.weight"], bias).reshape(B, N, 3, heads, -1).permute(2, 0, 3, 1, 4)
    q, k, v = qkv[0], qkv[1], qkv[2]
    q = q * ((C // heads) ** -0.5)
    attn = (q.float() @ k.float().transpose(-2, -1)).softmax(dim=-1).to(x.dtype)
    out = (attn @ v).transpose(1, 2).reshape(B, N, -1)
    return F.linear(out, sd[pre + "proj.weight"], sd[pre + "proj.bias"])


def mlp(x, sd, pre):
    """Mlp.forward - models/vision_transformer.py:103-110 (exact-erf GELU)."""
    h = F.gelu(F.linear(x, sd[pre + "fc1.weight"], sd[pre + "fc1.bias"]))
    return F.linear(h, sd[pre + "fc2.weight"], sd[pre + "fc2.bias"])


def timesformer_block(x, cls, sd, pre, heads, eps=1e-6):
    """Block.forward - models/vision_transformer.py:243-275.  x [B,T,N,D], cls [B,D]."""
    B, T, N, D = x.shape
    # temporal attention over T for every patch, then temporal_fc, residual in (n t) order
    xt = x.permute(0, 2, 1, 3).reshape(B * N, T, D)
    xt = vit_attention(layer_norm(xt, sd[pre + "temporal_ln.weight"], sd[pre + "temporal_ln.bias"], eps),
                       sd, pre + "temporal_attn.", heads)
    xt = F.linear(xt.reshape(B, N * T, D), sd[pre + "temporal_fc.weight"], sd[pre + "temporal_fc.bias"])
    xt = x.permute(0, 2, 1, 3).reshape(B, N * T, D) + xt
    # spatial attention per frame with the (shared) cls token prepended
    cls_rep = cls[:, None, :].expand(B, T, D).reshape(B * T, 1, D)
    xs = xt.reshape(B, N, T, D).permute(0, 2, 1, 3).reshape(B * T, N, D)
    xs = torch.cat([cls_rep, xs], dim=1)
    xs = vit_attention(layer_norm(xs, sd[pre + "norm1.weight"], sd[pre + "norm1.bias"], eps),
                       sd, pre + "attn.", heads)
    cls_new = xs[:, 0].reshape(B, T, D).mean(dim=1, keepdim=True)  # averaged over frames
    xs = xs[:, 1:].reshape(B, T, N, D).permute(0, 2, 1, 3).reshape(B, N * T, D)
    y = torch.cat([cls[:, None, :], xt], dim=1) + torch.cat([cls_new, xs], dim=1)
    y = y + mlp(layer_norm(y, sd[pre + "norm2.weight"], sd[pre + "norm2.bias"], eps), sd, pre + "mlp.")
    cls_out, y = y[:, 0], y[:, 1:]
    return y.reshape(B, N, T, D).permute(0, 2, 1, 3), cls_out


def timesformer(video, sd, cfg, pre="visual_encoder."):
    """TimeSformer.forward_features - models/vision_transformer.py:544-587 (CLIP mode: conv
    without bias, norm_pre after the position embeddings).  video [B,3,T,H,W] ->
    image_embeds [B, 1+T*N, D] in (t n) order."""
    B, C, T, H, W = video.shape
    P, D, heads, eps = cfg["patch_size"], cfg["embed_dim"], cfg["num_heads"], 1e-6
    x = video.permute(0, 2, 1, 3, 4).reshape(B * T, C, H, W)
    x = F.conv2d(x, sd[pre + "patch_embed.proj.weight"], sd.get(pre + "patch_embed.proj.bias"), stride=P)
    x = x.flatten(2).transpose(1, 2)  # [(b t), n, D]
    N = x.shape[1]
    x = x.reshape(B, T * N, D)
    x = torch.cat([sd[pre + "cls_token"].expand(B, -1, -1), x], dim=1)
    pos = sd[pre + "pos_embed"]
    total = torch.cat([pos[:, :1], pos[:, 1:].repeat(1, T, 1) +
                       sd[pre + "temporal_embed"].repeat_interleave(N, 1)], dim=1)
    x = x + total
    if pre + "norm_pre.weight" in sd:
        x = layer_norm(x, sd[pre + "norm_pre.weight"], sd[pre + "norm_pre.bias"], eps)
    cls, x = x[:, 0], x[:, 1:].reshape(B, T, N, D)
    for i in range(cfg["depth"]):
        x, cls = timesformer_block(x, cls, sd, f"{pre}blocks.{i}.", heads, eps)
    x = torch.cat([cls[:, None, :], x.reshape(B, T * N, D)], dim=1)
    return layer_norm(x, sd[pre + "norm.weight"], sd[pre + "norm.bias"], eps)


def eva_vit(image, sd, cfg, pre="visual_encoder.", eps=1e-6):
    """EVA VisionTransformer.forward_features - models/eva_vit.py:334-350 with Block.forward :174-181 (no layer
    scale, drop_path 0), Attention.forward :117-145 (bias = cat(q_bias, 0, v_bias), q scaled, softmax), PatchEmbed
    :200-207 (Conv2d with bias), final `norm` (use_mean_pooling=False: create_eva_vit_g :413-436).
    image [B,3,H,W] -> tokens [B, 1+N, D] (cls first)."""
    B = image.shape[0]
    P, heads = cfg["patch_size"], cfg["num_heads"]
    x = F.conv2d(image, sd[pre + "patch_embed.proj.weight"], sd[pre + "patch_embed.proj.bias"], stride=P).flatten(2).transpose(1, 2)
    x = torch.cat([sd[pre + "cls_token"].expand(B, -1, -1), x], dim=1) + sd[pre + "pos_embed"]
    for i in range(cfg["depth"]):
        b = f"{pre}blocks.{i}."
        x = x + vit_attention(layer_norm(x, sd[b + "norm1.weight"], sd[b + "norm1.bias"], eps), sd, b + "attn.", heads)
        x = x + mlp(layer_norm(x, sd[b + "norm2.weight"], sd[b + "norm2.bias"], eps), sd, b + "mlp.")
    return layer_norm(x, sd[pre + "norm.weight"], sd[pre + "norm.bias"], eps)


def eva_state_dict(cfg, gcfg, num_query, seed=0):
    """Random state dict with the keys / shapes of DistributedGPT3_Pretrain_Image(use_eva_g) - EVA encoder
    (models/eva_vit.py:245-300), abstractor, visual_fc, decoder - every tensor non-trivial."""
    g = torch.Generator().manual_seed(seed)
    D, depth, P = cfg["embed_dim"], cfg["depth"], cfg["patch_size"]
    N = (cfg["img_size"] // P) ** 2
    hid = int(D * cfg["mlp_ratio"])
    rn = lambda *s, std=0.02: torch.randn(*s, generator=g) * std  # noqa: E731
    ln = lambda n: (1.0 + 0.1 * torch.randn(n, generator=g), 0.02 * torch.randn(n, generator=g))  # noqa: E731
    ve = "visual_encoder."
    sd = {ve + "cls_token": rn(1, 1, D), ve + "pos_embed": rn(1, N + 1, D), ve + "patch_embed.proj.weight": rn(D, 3, P, P),
          ve + "patch_embed.proj.bias": rn(D)}
    for i in range(depth):
        b = f"{ve}blocks.{i}."
        for nm in ("norm1", "norm2"):
            sd[b + nm + ".weight"], sd[b + nm + ".bias"] = ln(D)
        sd[b + "attn.q_bias"], sd[b + "attn.v_bias"] = rn(D), rn(D)
        sd[b + "attn.qkv.weight"], sd[b + "attn.proj.weight"], sd[b + "attn.proj.bias"] = rn(3 * D, D), rn(D, D), rn(D)
        sd[b + "mlp.fc1.weight"], sd[b + "mlp.fc1.bias"] = rn(hid, D), rn(hid)
        sd[b + "mlp.fc2.weight"], sd[b + "mlp.fc2.bias"] = rn(D, hid), rn(D)
    sd[ve + "norm.weight"], sd[ve + "norm.bias"] = ln(D)
    base = init_state_dict(dict(VCFG_TINY, embed_dim=D, mlp_ratio=cfg["mlp_ratio"], num_heads=cfg["num_heads"]), gcfg, num_query,
                           seed=seed + 1, randomize=True)
    for k, v in base.items():
        if not k.startswith(ve):
            sd[k] = v
    return sd


def pretrain_image_forward(image, input_ids, attention_mask, sd, cfg, gcfg, return_all=False):
    """DistributedGPT3_Pretrain_Image.forward (use_eva_g, no contrastive) - models/distributed_gpt3.py:347-385."""
    image_embeds = eva_vit(image, sd, cfg)
    B = image.shape[0]
    image_query = attention_pool(sd["learnable_queries"].expand(B, -1, -1), image_embeds, sd, cfg["num_heads"])
    query_features = F.linear(image_query, sd["visual_fc.weight"], sd["visual_fc.bias"])
    Q = query_features.shape[1]
    targets, loss_mask = build_targets(input_ids, attention_mask, Q)
    emb_w = sd[GPT_PRE + "embedding.word_embeddings.weight"]
    hidden = gpt3_decoder(torch.cat([query_features, emb_w[input_ids]], dim=1), sd, gcfg)
    logits, losses = lm_head_losses(hidden, emb_w, targets)
    loss = masked_mean_loss(losses, loss_mask)
    if return_all:
        return dict(loss=loss, logits=logits, losses=losses, image_embeds=image_embeds, query_features=query_features)
    return loss


ECFG_TINY = dict(img_size=28, patch_size=14, embed_dim=176, depth=2, num_heads=2, mlp_ratio=4.3637)   # head_dim 88 as in EVA-g
ECFG_EVA_G = dict(img_size=224, patch_size=14, embed_dim=1408, depth=40, num_heads=16, mlp_ratio=4.3637)


def attention_pool(q, k, sd, heads, pre="attn_pool.", eps=1e-6):
    """AttentionPool.forward - models/vision_transformer.py:368-374 with nn.MultiheadAttention
    (bias=True, add_bias_kv=True): one learned key/value row is appended; the residual is taken
    from the already-normalised query."""
    B, Q, D = q.shape
    hd = D // heads
    x = layer_norm(q, sd[pre + "norm1.weight"], sd[pre + "norm1.bias"], eps)
    kv = layer_norm(k, sd[pre + "normk.weight"], sd[pre + "normk.bias"], eps)
    w, b = sd[pre + "attn.in_proj_weight"], sd[pre + "attn.in_proj_bias"]
    qp = F.linear(x, w[:D], b[:D])
    kp = F.linear(kv, w[D:2 * D], b[D:2 * D])
    vp = F.linear(kv, w[2 * D:], b[2 * D:])
    kp = torch.cat([kp, sd[pre + "attn.bias_k"].reshape(1, 1, D).expand(B, 1, D)], dim=1)
    vp = torch.cat([vp, sd[pre + "attn.bias_v"].reshape(1, 1, D).expand(B, 1, D)], dim=1)
    S = kp.shape[1]
    qh = qp.reshape(B, Q, heads, hd).transpose(1, 2) * (hd ** -0.5)
    kh = kp.reshape(B, S, heads, hd).transpose(1, 2)
    vh = vp.reshape(B, S, heads, hd).transpose(1, 2)
    att = (qh @ kh.transpose(-2, -1)).softmax(dim=-1)
    o = (att @ vh).transpose(1, 2).reshape(B, Q, D)
    x = x + F.linear(o, sd[pre + "attn.out_proj.weight"], sd[pre + "attn.out_proj.bias"])
    return x + mlp(layer_norm(x, sd[pre + "norm2.weight"], sd[pre + "norm2.bias"], eps), sd, pre + "mlp.")


def gelu_tanh(x):
    """bias_gelu_impl (megatron_util, un-vendored; tanh approximation) -
    call site models/modeling_distributed_gpt3.py:586-588."""
    return x * 0.5 * (1.0 + torch.tanh(0.79788456 * x * (1 + 0.044715 * x * x)))


GPT_PRE = "text_decoder.dist_model.language_model."


def _drop(t2d, drop, site, p):
    """Dropout with the H100 kernels' Philox mask convention (oracle/philox.py) on a [rows, cols] view."""
    if drop is None or p <= 0.0:
        return t2d
    from oracle import philox
    return philox.dropout(t2d, drop["seed"], drop["offset"], site, p)


def gpt3_layer(x, sd, pre, heads, layer_number, eps, drop=None):
    """GPT3ParallelTransformerLayer.forward - models/modeling_distributed_gpt3.py:1034-1089 with
    GPT3ParallelAttention (:868-938) and GPT3CoreAttention (:734-817).  x is [B,S,h] here (the
    reference uses [S,B,h]; the arithmetic per (b, head) is identical).  QKV rows are grouped per
    head as [q|k|v]; scores = q.k / (sqrt(hn)*layer) * layer; causal fill value -10000.
    drop = dict(seed, offset, p_hidden, p_attn): train-mode dropout of the attention probabilities (:772-780)
    and the two bias-dropout-adds (:1051-1078), masks as the H100 kernels draw them (site = 4*layer + 1/2/3)."""
    B, S, H = x.shape
    li = layer_number - 1
    ph = drop["p_hidden"] if drop else 0.0
    pa = drop["p_attn"] if drop else 0.0
    hn = H // heads
    ln1 = layer_norm(x, sd[pre + "input_layernorm.weight"], sd[pre + "input_layernorm.bias"], eps)
    qkv = F.linear(ln1, sd[pre + "self_attention.query_key_value.weight"],
                   sd[pre + "self_attention.query_key_value.bias"]).reshape(B, S, heads, 3 * hn)
    q, k, v = qkv.split(hn, dim=-1)
    q, k, v = q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2)  # [B,np,S,hn]
    coeff = max(1, layer_number)
    scores = (q @ k.transpose(-2, -1)) * (1.0 / (math.sqrt(hn) * coeff))
    scores = scores.float() * coeff
    mask = torch.ones(S, S, dtype=torch.bool, device=x.device).triu(1)
    scores = scores.masked_fill(mask, -10000.0)
    probs = scores.softmax(dim=-1).to(x.dtype)
    probs = _drop(probs.reshape(B * heads * S, S), drop, 4 * li + 1, pa).reshape(B, heads, S, S)
    ctx = (probs @ v).transpose(1, 2).reshape(B, S, H)
    attn_out = F.linear(ctx, sd[pre + "self_attention.dense.weight"]) + sd[pre + "self_attention.dense.bias"]
    x = x + _drop(attn_out.reshape(B * S, H), drop, 4 * li + 2, ph).reshape(B, S, H)  # bias-dropout-add (:1051-1062)
    ln2 = layer_norm(x, sd[pre + "post_attention_layernorm.weight"], sd[pre + "post_attention_layernorm.bias"], eps)
    h = gelu_tanh(F.linear(ln2, sd[pre + "mlp.dense_h_to_4h.weight"]) + sd[pre + "mlp.dense_h_to_4h.bias"])
    mlp_out = F.linear(h, sd[pre + "mlp.dense_4h_to_h.weight"]) + sd[pre + "mlp.dense_4h_to_h.bias"]
    return x + _drop(mlp_out.reshape(B * S, H), drop, 4 * li + 3, ph).reshape(B, S, H)


def gpt3_decoder(input_embeds, sd, gcfg, pre=GPT_PRE, drop=None):
    """GPT3Embedding.forward (:640-666, position ids = arange(S) incl. the visual prefix; embedding dropout :631
    at site 0 when `drop` is given) + GPT3ParallelTransformer.forward (:1140-1186).  Returns final-LN hidden
    states [B,S,h]."""
    B, S, H = input_embeds.shape
    eps = gcfg.get("layernorm_epsilon", 1e-12)
    x = input_embeds + sd[pre + "embedding.position_embeddings.weight"][:S][None]
    if drop is not None:
        x = _drop(x.reshape(B * S, H), drop, 0, drop["p_hidden"]).reshape(B, S, H)
    for i in range(gcfg["num_hidden_layers"]):
        x = gpt3_layer(x, sd, f"{pre}encoder.layers.{i}.", gcfg["num_attention_heads"], i + 1, eps, drop)
    return layer_norm(x, sd[pre + "encoder.final_layernorm.weight"], sd[pre + "encoder.final_layernorm.bias"], eps)


def lm_head_losses(hidden, emb_w, labels):
    """GPT3Model.forward tail - models/modeling_distributed_gpt3.py:1348-1364: tied LM head, CE on
    fp32 logits, unreduced per-token losses [B,S]."""
    logits = F.linear(hidden, emb_w)
    B, S, V = logits.shape
    losses = F.cross_entropy(logits.float().reshape(-1, V), labels.reshape(-1), reduction="none").view(B, S)
    return logits, losses


def build_targets(input_ids, attention_mask, num_query):
    """models/distributed_gpt3.py:142-159 - integer work, bit-exact.  Visual-prefix labels are
    100 (not -100) and are neutralised by loss_mask, not by ignore_index."""
    B = input_ids.shape[0]
    targets = torch.cat([input_ids[:, 1:], input_ids[:, 1:2]], dim=1)
    targets = torch.cat([torch.full((B, num_query), 100, dtype=torch.long, device=input_ids.device), targets], dim=1)
    loss_mask = torch.cat([torch.zeros((B, num_query), dtype=torch.long, device=input_ids.device),
                           attention_mask[:, 1:]], dim=1)
    return targets, loss_mask


def masked_mean_loss(losses, loss_mask):
    """DistributedGPT3.forward - models/modeling_distributed_gpt3.py:1612-1617."""
    lm = loss_mask.reshape(-1).float()
    return torch.sum(losses[:, :-1].reshape(-1).float() * lm) / lm.sum()


def pretrain_forward(video, input_ids, attention_mask, sd, vcfg, gcfg, return_all=False, drop=None):
    """DistributedGPT3_Pretrain.forward (use_contrastive=False) - models/distributed_gpt3.py:130-166.
    drop: see gpt3_layer (decoder dropout in train() mode)."""
    image_embeds = timesformer(video, sd, vcfg)
    B = video.shape[0]
    image_query = attention_pool(sd["learnable_queries"].expand(B, -1, -1), image_embeds, sd, vcfg["num_heads"])
    query_features = F.linear(image_query, sd["visual_fc.weight"], sd["visual_fc.bias"])
    Q = query_features.shape[1]
    targets, loss_mask = build_targets(input_ids, attention_mask, Q)
    emb_w = sd[GPT_PRE + "embedding.word_embeddings.weight"]
    input_embeds = torch.cat([query_features, emb_w[input_ids]], dim=1)
    hidden = gpt3_decoder(input_embeds, sd, gcfg, drop=drop)
    logits, losses = lm_head_losses(hidden, emb_w, targets)
    loss = masked_mean_loss(losses, loss_mask)
    if return_all:
        return dict(loss=loss, logits=logits, losses=losses, hidden=hidden, image_embeds=image_embeds,
                    image_query=image_query, query_features=query_features, targets=targets,
                    loss_mask=loss_mask)
    return loss


# ------------------------------------------------------------------------------------------
# Random-init state dicts with the reference's keys / shapes / init laws (for benches & tests)
# ------------------------------------------------------------------------------------------
def init_state_dict(vcfg, gcfg, num_query, seed=0, dtype=torch.float32, randomize=False, fast=False):
    """Same parameter names, shapes and init distributions as the reference constructors
    (TimeSformer.__init__ models/vision_transformer.py:441-519, DistributedGPT3_Pretrain.__init__
    models/distributed_gpt3.py:96-116, GPT3 init_method_normal / scaled models/
    modeling_distributed_gpt3.py:1253-1269).  Not bit-identical to the reference's RNG stream -
    use oracle/make_golden.py fixtures when exact reference weights are needed."""
    g = torch.Generator().manual_seed(seed)
    D, depth, P = vcfg["embed_dim"], vcfg["depth"], vcfg["patch_size"]
    T, N = vcfg["num_frames"], (vcfg["img_size"] // P) ** 2
    hid = int(D * vcfg["mlp_ratio"])
    sd = {}

    def tn(*shape, std=0.015):
        if fast:  # timing-only weights: same scale, vectorised fill (not reproducible across runs)
            return torch.empty(*shape).uniform_(-1.7 * std, 1.7 * std)
        return torch.nn.init.trunc_normal_(torch.empty(*shape), std=std, generator=g)

    def nrm(*shape, std):
        if fast:
            return torch.empty(*shape).uniform_(-1.7 * std, 1.7 * std)
        return torch.empty(*shape).normal_(0.0, std, generator=g)

    ve = "visual_encoder."
    sd[ve + "cls_token"] = tn(1, 1, D)
    sd[ve + "pos_embed"] = tn(1, N + 1, D)
    sd[ve + "temporal_embed"] = torch.zeros(1, T, D)
    sd[ve + "patch_embed.proj.weight"] = tn(D, 3, P, P)
    for nm in ("norm_pre", "norm"):
        sd[ve + nm + ".weight"], sd[ve + nm + ".bias"] = torch.ones(D), torch.zeros(D)
    for i in range(depth):
        b = f"{ve}blocks.{i}."
        for nm in ("norm1", "norm2", "temporal_ln"):
            sd[b + nm + ".weight"], sd[b + nm + ".bias"] = torch.ones(D), torch.zeros(D)
        for at in ("attn.", "temporal_attn."):
            sd[b + at + "qkv.weight"] = tn(3 * D, D)
            sd[b + at + "q_bias"], sd[b + at + "v_bias"] = torch.zeros(D), torch.zeros(D)
            sd[b + at + "proj.weight"], sd[b + at + "proj.bias"] = tn(D, D), torch.zeros(D)
        sd[b + "attn.proj.weight"] /= math.sqrt(2.0 * (i + 1))
        sd[b + "temporal_fc.weight"] = tn(D, D) if i == 0 else torch.zeros(D, D)
        sd[b + "temporal_fc.bias"] = torch.zeros(D)
        sd[b + "mlp.fc1.weight"], sd[b + "mlp.fc1.bias"] = tn(hid, D), torch.zeros(hid)
        sd[b + "mlp.fc2.weight"], sd[b + "mlp.fc2.bias"] = tn(D, hid) / math.sqrt(2.0 * (i + 1)), torch.zeros(D)
    sd["learnable_queries"] = tn(1, num_query, D)
    ap = "attn_pool."
    for nm in ("norm1", "normk", "norm2"):
        sd[ap + nm + ".weight"], sd[ap + nm + ".bias"] = torch.ones(D), torch.zeros(D)
    sd[ap + "attn.in_proj_weight"] = torch.nn.init.xavier_uniform_(torch.empty(3 * D, D), generator=g)
    sd[ap + "attn.in_proj_bias"] = torch.zeros(3 * D)
    sd[ap + "attn.bias_k"] = torch.nn.init.xavier_normal_(torch.empty(1, 1, D), generator=g)
    sd[ap + "attn.bias_v"] = torch.nn.init.xavier_normal_(torch.empty(1, 1, D), generator=g)
    bound = 1.0 / math.sqrt(D)
    sd[ap + "attn.out_proj.weight"] = torch.empty(D, D).uniform_(-bound, bound, generator=g)
    sd[ap + "attn.out_proj.bias"] = torch.zeros(D)
    sd[ap + "mlp.fc1.weight"] = torch.empty(hid, D).uniform_(-bound, bound, generator=g)
    sd[ap + "mlp.fc1.bias"] = torch.empty(hid).uniform_(-bound, bound, generator=g)
    b2 = 1.0 / math.sqrt(hid)
    sd[ap + "mlp.fc2.weight"] = torch.empty(D, hid).uniform_(-b2, b2, generator=g)
    sd[ap + "mlp.fc2.bias"] = torch.empty(D).uniform_(-b2, b2, generator=g)
    H, V, Lyr = gcfg["hidden_size"], gcfg["vocab_size"], gcfg["num_hidden_layers"]
    F4 = gcfg.get("ffn_hidden_size") or 4 * H
    sd["visual_fc.weight"] = tn(H, D)
    sd["visual_fc.bias"] = torch.empty(H).uniform_(-bound, bound, generator=g)
    std = gcfg.get("init_method_std", 0.02)
    std_out = std / math.sqrt(2.0 * Lyr)
    sd[GPT_PRE + "embedding.word_embeddings.weight"] = nrm(V, H, std=std)
    sd[GPT_PRE + "embedding.position_embeddings.weight"] = nrm(gcfg["max_position_embeddings"], H, std=std)
    for i in range(Lyr):
        b = f"{GPT_PRE}encoder.layers.{i}."
        for nm in ("input_layernorm", "post_attention_layernorm"):
            sd[b + nm + ".weight"], sd[b + nm + ".bias"] = torch.ones(H), torch.zeros(H)
        sd[b + "self_attention.query_key_value.weight"] = nrm(3 * H, H, std=std)
        sd[b + "self_attention.query_key_value.bias"] = torch.zeros(3 * H)
        sd[b + "self_attention.dense.weight"] = nrm(H, H, std=std_out)
        sd[b + "self_attention.dense.bias"] = torch.zeros(H)
        sd[b + "mlp.dense_h_to_4h.weight"] = nrm(F4, H, std=std)
        sd[b + "mlp.dense_h_to_4h.bias"] = torch.zeros(F4)
        sd[b + "mlp.dense_4h_to_h.weight"] = nrm(H, F4, std=std_out)
        sd[b + "mlp.dense_4h_to_h.bias"] = torch.zeros(H)
    sd[GPT_PRE + "encoder.final_layernorm.weight"] = torch.ones(H)
    sd[GPT_PRE + "encoder.final_layernorm.bias"] = torch.zeros(H)
    if randomize:
        # parity fixtures: make every zero/one-initialised tensor non-trivial so that all code
        # paths (biases, LN affine, temporal_fc of blocks > 0, temporal_embed) are exercised
        for k in sorted(sd):
            v = sd[k]
            if k.endswith("norm.weight") or k.endswith("layernorm.weight") or \
                    re.search(r"(norm1|norm2|normk|norm_pre|temporal_ln)\.weight$", k):
                sd[k] = 1.0 + 0.1 * torch.randn(v.shape, generator=g)
            elif float(v.abs().max()) == 0.0:
                sd[k] = 0.02 * torch.randn(v.shape, generator=g)
    return {k: v.to(dtype) for k, v in sd.items()}


def trainable_keys(sd, freeze_vit=False):
    """Parameters with requires_grad in the reference (models/distributed_gpt3.py:86-93):
    everything except the GPT-3 decoder; with freeze_vit only names containing time/temporal."""
    out = []
    for k in sd:
        if k.startswith("text_decoder."):
            continue
        if freeze_vit and k.startswith("visual_encoder.") and not any(s in k for s in ("time", "temporal")):
            continue
        out.append(k)
    return out


VCFG_CLIP_B16 = dict(img_size=224, patch_size=16, embed_dim=768, depth=12, num_heads=8, mlp_ratio=4,
                     num_frames=8, clip_model=True)
GCFG_1_3B = dict(vocab_size=51200, hidden_size=2048, ffn_hidden_size=8192, num_hidden_layers=24,
                 num_attention_heads=32, max_position_embeddings=2048, layernorm_epsilon=1e-5,
                 init_method_std=0.02)
# configs/models/config_gpt3_2.7B.json (32 layers x 2560, 32 heads x 80: BASELINE config-4)
GCFG_2_7B = dict(vocab_size=51200, hidden_size=2560, ffn_hidden_size=10240, num_hidden_layers=32,
                 num_attention_heads=32, max_position_embeddings=2048, layernorm_epsilon=1e-5,
                 init_method_std=0.02)
VCFG_TINY = dict(img_size=32, patch_size=16, embed_dim=192, depth=2, num_heads=2, mlp_ratio=4,
                 num_frames=2, clip_model=True)
GCFG_TINY = dict(vocab_size=512, hidden_size=128, ffn_hidden_size=512, num_hidden_layers=2,
                 num_attention_heads=2, max_position_embeddings=64, layernorm_epsilon=1e-5,
                 init_method_std=0.02)


# ------------------------------------------------------------------------------------------
# Downstream forwards (SURVEY.md section 8a rows a20-a23), restated on the same primitives
# ------------------------------------------------------------------------------------------
def visual_prefix(video, sd, vcfg):
    """image -> (pooled cls feature, image_embeds, image_query, query_features)
    (models/distributed_gpt3.py:532-537 and the identical preambles of the other task models)."""
    image_embeds = timesformer(video, sd, vcfg)
    B = video.shape[0]
    image_query = attention_pool(sd["learnable_queries"].expand(B, -1, -1), image_embeds, sd, vcfg["num_heads"])
    query_features = F.linear(image_query, sd["visual_fc.weight"], sd["visual_fc.bias"])
    return image_embeds[:, 0], image_embeds, image_query, query_features


def prefix_decoder_pass(query_features, input_ids, attention_mask, prompt_lengths, sd, gcfg):
    """Decoder over [prefix | text] with prompt tokens masked out of the loss
    (models/distributed_gpt3.py:540-567).  Returns dict(loss, losses [B,S-1], loss_mask, hidden)."""
    Q = query_features.shape[1]
    att = attention_mask.clone()
    text_loss_atts = att[:, 1:].clone()
    if prompt_lengths is not None:
        for i, ln in enumerate(prompt_lengths.tolist()):
            text_loss_atts[i, :ln] = 0
    targets, _ = build_targets(input_ids, att, Q)
    loss_mask = torch.cat([torch.zeros((att.shape[0], Q), dtype=torch.long), text_loss_atts], dim=1)
    emb_w = sd[GPT_PRE + "embedding.word_embeddings.weight"]
    hidden = gpt3_decoder(torch.cat([query_features, emb_w[input_ids]], dim=1), sd, gcfg)
    logits, losses = lm_head_losses(hidden, emb_w, targets)
    return dict(loss=masked_mean_loss(losses, loss_mask), losses=losses[:, :-1], loss_mask=loss_mask, hidden=hidden,
                logits=logits)


def cls_eval_scores(query_features, input_ids, attention_mask, prompt_lengths, sd, gcfg, num_cls):
    """DistributedGPT3_Cls eval branch - models/distributed_gpt3.py:598-625: prefix repeated per class,
    generation_logits = softmax(-sum(losses * loss_mask))."""
    B, Q, H = query_features.shape
    qf = query_features.unsqueeze(1).repeat(1, num_cls, 1, 1).reshape(B * num_cls, Q, H)
    out = prefix_decoder_pass(qf, input_ids, attention_mask, prompt_lengths, sd, gcfg)
    return (-(out["losses"] * out["loss_mask"]).sum(-1)).view(B, num_cls).softmax(-1)


def pretrain_contrastive_loss(video, input_ids, attention_mask, sd, vcfg, gcfg, temp):
    """Contrastive branch of DistributedGPT3_Pretrain.forward (use_contrastive=True) - models/distributed_gpt3.py:168-217,
    single process: query-token features [B,Q,E] against the text feature of a text-only decoder pass [B,E],
    similarity = max over the Q queries, label-smoothed (0.1) CE in both directions with targets arange(B)."""
    _, _, image_query, _ = visual_prefix(video, sd, vcfg)
    vfeat = F.normalize(F.linear(image_query, sd["vision_proj.weight"], sd["vision_proj.bias"]), dim=-1)
    emb_w = sd[GPT_PRE + "embedding.word_embeddings.weight"]
    hidden = gpt3_decoder(emb_w[input_ids], sd, gcfg)
    pooled = hidden[torch.arange(hidden.shape[0]), attention_mask.sum(-1) - 1]
    tfeat = F.normalize(F.linear(pooled, sd["text_proj.weight"], sd["text_proj.bias"]), dim=-1)
    sim_i2t = torch.einsum("bqe,je->bjq", vfeat, tfeat).max(-1)[0] / temp
    sim_t2i = torch.einsum("be,jqe->bjq", tfeat, vfeat).max(-1)[0] / temp
    tgt = torch.arange(video.shape[0])
    return (F.cross_entropy(sim_i2t, tgt, label_smoothing=0.1) + F.cross_entropy(sim_t2i, tgt, label_smoothing=0.1)) / 2


def cls_head(x, sd):
    """nn.Sequential(Linear, ReLU, Linear) head of the Cls / Retrieval_Cls models (models/distributed_gpt3.py:523-529)."""
    return F.linear(torch.relu(F.linear(x, sd["cls_head.0.weight"], sd["cls_head.0.bias"])), sd["cls_head.2.weight"], sd["cls_head.2.bias"])


def prompt_pooled_hidden(query_features, prompt_ids, prompt_att, sd, gcfg):
    """Hidden state of the last attended prompt token after a [prefix | prompt] decoder pass
    (models/distributed_gpt3.py:569-588): position Q + attention_mask.sum(-1) - 1."""
    Q = query_features.shape[1]
    hidden = prefix_decoder_pass(query_features, prompt_ids, prompt_att, None, sd, gcfg)["hidden"]
    return hidden[torch.arange(hidden.shape[0]), Q + prompt_att.sum(-1) - 1]


def cls_train_losses(query_features, input_ids, attention_mask, prompt_lengths, prompt_ids, prompt_att, labels, sd, gcfg):
    """DistributedGPT3_Cls.forward(train=True, use_cls=True) - models/distributed_gpt3.py:540-592:
    (caption-style loss with the prompt masked out, CE of cls_head on the prompt pass)."""
    loss_caption = prefix_decoder_pass(query_features, input_ids, attention_mask, prompt_lengths, sd, gcfg)["loss"]
    logits = cls_head(prompt_pooled_hidden(query_features, prompt_ids, prompt_att, sd, gcfg), sd)
    return loss_caption, F.cross_entropy(logits, labels)


def retrieval_cls_train_losses(query_features, negative_indices, input_ids, attention_mask, prompt_lengths, prompt_ids, prompt_att,
                               labels, sd, gcfg):
    """DistributedGPT3_Retrieval_Cls.forward(train=True) - models/distributed_gpt3.py:1105-1157: the prefix of every video
    followed by the prefixes of its negatives (query_features[negative_indices])."""
    qf = torch.cat([query_features, query_features[negative_indices]], dim=0)
    return cls_train_losses(qf, input_ids, attention_mask, prompt_lengths, prompt_ids, prompt_att, labels, sd, gcfg)


def retrieval_cls_eval(query_features, input_ids, attention_mask, prompt_lengths, prompt_ids, prompt_att, sd, gcfg):
    """DistributedGPT3_Retrieval_Cls.forward(train=False) - :1159-1213: every video against t texts;
    (-(losses * mask).sum [v, t], softmax(cls_head)[:, 1] [v, t])."""
    v = query_features.shape[0]
    t = input_ids.shape[0] // v
    qf = query_features.repeat_interleave(t, dim=0)
    out = prefix_decoder_pass(qf, input_ids, attention_mask, prompt_lengths, sd, gcfg)
    gen = (-(out["losses"] * out["loss_mask"]).sum(-1)).view(v, t)
    cls = torch.softmax(cls_head(prompt_pooled_hidden(qf, prompt_ids, prompt_att, sd, gcfg), sd), dim=-1)[:, 1].view(v, t)
    return gen, cls


def retrieval_features(video, input_ids, attention_mask, sd, vcfg, gcfg):
    """DistributedGPT3_Retrieval.extract_{vision,text}_feature - models/distributed_gpt3.py:909-945:
    CLS-pooled ViT feature -> vision_proj -> L2 ; GPT hidden at the last valid token -> text_proj -> L2."""
    pooled = timesformer(video, sd, vcfg)[:, 0]
    vfeat = F.normalize(F.linear(pooled, sd["vision_proj.weight"], sd["vision_proj.bias"]), dim=-1)
    emb_w = sd[GPT_PRE + "embedding.word_embeddings.weight"]
    hidden = gpt3_decoder(emb_w[input_ids], sd, gcfg)
    last = hidden[torch.arange(hidden.shape[0]), attention_mask.sum(-1) - 1]
    tfeat = F.normalize(F.linear(last, sd["text_proj.weight"], sd["text_proj.bias"]), dim=-1)
    return vfeat, tfeat


def retrieval_loss(vfeat, tfeat, idx, temp):
    """models/distributed_gpt3.py:966-980 (single process: the gathered features are the local ones)."""
    sim_i2t = vfeat @ tfeat.t() / temp
    sim_t2i = tfeat @ vfeat.t() / temp
    pos = torch.eq(idx.view(-1, 1), idx.view(1, -1)).float()
    tgt = pos / pos.sum(1, keepdim=True)
    return (-(F.log_softmax(sim_i2t, 1) * tgt).sum(1).mean() - (F.log_softmax(sim_t2i, 1) * tgt).sum(1).mean()) / 2


# ------------------------------------------------------------------------------------------
# Generation (SURVEY.md section 8f, row N2): greedy / top-k / top-p sampling and beam search with
# the visual prefix.  The reference decodes incrementally over a KV cache
# (models/modeling_distributed_gpt3.py:868-923); the oracle recomputes the whole [prefix | tokens]
# sequence at every step, which is the same arithmetic for a causal decoder.
# ------------------------------------------------------------------------------------------
def next_token_logits(query_features, tokens, sd, gcfg):
    """Logits [B, V] of the position after `tokens` [B, n] (prefix [B, Q, h] optional)."""
    emb_w = sd[GPT_PRE + "embedding.word_embeddings.weight"]
    x = emb_w[tokens]
    if query_features is not None:
        x = torch.cat([query_features, x], dim=1)
    hidden = gpt3_decoder(x, sd, gcfg)
    return F.linear(hidden[:, -1], emb_w)


def filter_top_k(logits, top_k):
    """modify_logits_for_top_k_filtering (:1369-1373), out of place."""
    kth = torch.topk(logits, top_k)[0][..., -1, None]
    return logits.masked_fill(logits < kth, float("-inf"))


def filter_top_p(logits, top_p):
    """modify_logits_for_top_p_filtering (:1376-1395): nucleus with the historical shift-by-one."""
    sorted_logits, sorted_idx = torch.sort(logits, descending=True)
    cum = sorted_logits.softmax(dim=-1).cumsum(dim=-1)
    drop = cum > top_p
    drop[:, 1:] = drop[:, :-1].clone()
    drop[..., 0] = False
    drop = drop.scatter(1, sorted_idx, drop)
    return logits.masked_fill(drop, float("-inf"))


def pick_token(logits, top_k=0, top_p=0.0, temperature=1.0, vocab_size=None, generator=None):
    """sample() (:1398-1446): argmax for top_k == 1, otherwise temperature -> top-k | top-p -> multinomial."""
    assert logits.ndim == 2
    if top_k == 1:
        assert top_p == 0.0
        out = torch.argmax(logits, dim=-1)
    else:
        lg = logits.clone()
        if temperature != 1.0:
            lg = lg / temperature
        if top_k > 1:
            assert top_p == 0.0 and top_k <= lg.size(1)
            lg = filter_top_k(lg, top_k)
        elif top_p > 0.0:
            assert top_p <= 1.0
            lg = filter_top_p(lg, top_p)
        out = torch.multinomial(lg.softmax(dim=-1), num_samples=1, generator=generator).view(-1)
    if vocab_size:
        out = torch.clamp(out, min=0, max=vocab_size - 1)
    return out


def sample_generate(tokens, sd, gcfg, query_features=None, prompt_length=None, tokens_to_generate=100, eod_id=7,
                    top_k=0, top_p=0.9, temperature=1.0, termination_id=None, early_stop=True, generator=None):
    """DistributedGPT3.sample (:1620-1741) for the default stop rule (termination id).  tokens [B, n];
    prompt_length [B] (tokens beyond a sample's prompt are overwritten as soon as generation reaches them)."""
    B = tokens.size(0)
    lengths = prompt_length if prompt_length is not None else torch.tensor([tokens.size(1)])
    tokens = torch.cat([tokens, torch.full((B, tokens_to_generate), eod_id, dtype=torch.long)], dim=-1)
    max_len = min(tokens.size(1), gcfg["max_position_embeddings"])
    min_prompt = int(lengths.min())
    if min_prompt >= max_len:
        raise ValueError("context length + tokens_to_generate too large")
    if termination_id is None:
        termination_id = eod_id
    done = torch.zeros(B, dtype=torch.bool)
    ctx = min_prompt
    for ctx in range(min_prompt, max_len):
        new = pick_token(next_token_logits(query_features, tokens[:, :ctx], sd, gcfg), top_k, top_p, temperature,
                         gcfg["vocab_size"], generator)
        started = lengths <= ctx
        tokens[started, ctx] = new[started]
        done |= (new == termination_id) & started
        if early_stop and bool(done.all()):
            break
    # the reference slices with the context length that still counts the prefix positions (:1740), so with a
    # visual prefix the returned rows keep (most of) their stop-token padding
    nq = query_features.size(1) if query_features is not None else 0
    return tokens[:, :ctx + nq + 1]


def generation_state_dict(vcfg, gcfg, num_query, seed, pos_gain, ln_gain):
    """Weights of the generation fixtures: a random tiny decoder with tied embeddings only repeats its last
    input token, so the learned position embeddings (x pos_gain) and the final LayerNorm affine (x ln_gain)
    are scaled up - continuations then change from step to step and have usable top-2 margins."""
    sd = init_state_dict(vcfg, gcfg, num_query, seed=seed, randomize=True)
    kp = GPT_PRE + "embedding.position_embeddings.weight"
    sd[kp] = sd[kp] * pos_gain
    for kk in ("encoder.final_layernorm.weight", "encoder.final_layernorm.bias"):
        sd[GPT_PRE + kk] = sd[GPT_PRE + kk] * ln_gain
    return sd


class BeamPool:
    """BeamHypotheses (:1908-1961): n-best list; the score is sum_logprobs / len(hyp) ** length_penalty where
    hyp is the PADDED token row the caller hands in (so every hypothesis is normalised by the same length)."""

    def __init__(self, num_beams, length_penalty=1.0, early_stopping=False):
        self.num_beams, self.length_penalty, self.early_stopping = num_beams, length_penalty, early_stopping
        self.beams, self.worst_score = [], 1e9

    def add(self, hyp, sum_logprobs):
        score = sum_logprobs / (hyp.shape[-1] ** self.length_penalty)
        if len(self.beams) < self.num_beams or score > self.worst_score:
            self.beams.append((score, hyp))
            if len(self.beams) > self.num_beams:
                order = sorted((s, i) for i, (s, _) in enumerate(self.beams))
                del self.beams[order[0][1]]
                self.worst_score = order[1][0]
            else:
                self.worst_score = min(score, self.worst_score)

    def is_done(self, best_sum_logprobs, cur_len):
        if len(self.beams) < self.num_beams:
            return False
        if self.early_stopping:
            return True
        return self.worst_score >= best_sum_logprobs / cur_len ** self.length_penalty


def beam_search_generate(tokens, sd, gcfg, query_features=None, prompt_length=None, beam_size=5, num_return_gen=1,
                         stop_token=None, tokens_to_generate=100, eod_id=7):
    """DistributedGPT3.beam_search (:1743-1875), batch size 1.  Returns (sequences [n, len], scores [n])."""
    assert tokens.size(0) == 1
    plen = int(prompt_length) if prompt_length is not None else tokens.size(1)
    if stop_token is None:
        stop_token = eod_id
    tokens = torch.cat([tokens, torch.full((1, tokens_to_generate), stop_token, dtype=torch.long)], dim=-1)
    final_len = min(tokens.size(1), gcfg["max_position_embeddings"])
    if plen >= final_len:
        raise ValueError("context length + tokens_to_generate too large")
    pool = BeamPool(beam_size)
    scores = torch.zeros(beam_size, 1)
    tokens = tokens.repeat(beam_size, 1)
    qf = query_features.repeat(beam_size, 1, 1) if query_features is not None else None
    done = False
    ctx = plen
    for ctx in range(plen, final_len):
        logp = F.log_softmax(next_token_logits(qf, tokens[:, :ctx], sd, gcfg), dim=-1)
        V = logp.size(1)
        cand = logp + scores
        flat = cand[0] if ctx == plen else cand.view(-1)   # all beams are identical at the first step
        best_scores, idx = torch.sort(flat, descending=True)
        idx, best_scores = idx[:2 * beam_size], best_scores[:2 * beam_size]
        beam_ids, words = torch.div(idx, V, rounding_mode="floor"), idx % V
        nxt = []
        for rank, (w, sc, b) in enumerate(zip(words.tolist(), best_scores, beam_ids.tolist())):
            if w == stop_token:
                if rank >= beam_size:
                    continue
                pool.add(tokens[b].clone(), sc)
            else:
                nxt.append((w, sc, b))
            if len(nxt) == beam_size:
                break
        if pool.is_done(float(best_scores.max()), ctx + 1 - plen):
            done = True
            break
        keep = torch.tensor([b for _, _, b in nxt])
        tokens = tokens[keep]
        tokens[:, ctx] = torch.tensor([w for w, _, _ in nxt])
        scores = torch.stack([sc for _, sc, _ in nxt]).reshape(-1, 1)
    if not done:
        for b in range(beam_size):
            pool.add(tokens[b].clone(), scores[b])
    hyps = sorted(pool.beams, key=lambda x: float(x[0]), reverse=True)[:num_return_gen]
    return torch.stack([h for _, h in hyps]), torch.stack([torch.as_tensor(s).reshape(()) for s, _ in hyps])


# ------------------------------------------------------------------------------------------
# Input pipeline tail (SURVEY.md section 8f, row N4)
# ------------------------------------------------------------------------------------------
CLIP_MEAN = [0.48145466, 0.4578275, 0.40821073]   # dataset/__init__.py:69-72
CLIP_STD = [0.26862954, 0.26130258, 0.27577711]


def clip_to_model_input(frames, mean=CLIP_MEAN, std=CLIP_STD):
    """uint8 [B,T,H,W,C] -> bf16 [B,C,T,H,W]: volume_transforms.ClipToTensor (`torch.from_numpy(clip) / 255.` after the
    (3,0,1,2) transpose, dataset/video_utils/volume_transforms.py:25-37), functional.normalize (`sub_(mean).div_(std)`
    with fp32 mean/std tensors, dataset/video_utils/functional.py:125-137), default collate, bf16 cast."""
    out = []
    for clip in frames:
        x = clip.permute(3, 0, 1, 2) / 255.
        m = torch.as_tensor(mean, dtype=x.dtype)
        s = torch.as_tensor(std, dtype=x.dtype)
        x.sub_(m[:, None, None, None]).div_(s[:, None, None, None])
        out.append(x)
    return torch.stack(out).to(torch.bfloat16)
