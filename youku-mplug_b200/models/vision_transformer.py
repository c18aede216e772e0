"""TimeSformer video encoder + AttentionPool visual abstractor on the H100 kernels.

Mirrors the reference module `models/vision_transformer.py` for the classes the GPT-3 path uses:
TimeSformer (:440-592), AttentionPool (:341-374), LayerNormWithForceFP32 (:43-75),
resize_pos_embed (:731-749), resize_temporal_embed (:752-764), _convert_pretrained_vit (:719-728).
Parameter names / shapes / init follow the reference constructors so released checkpoints load with
load_state_dict.  Only divided space-time attention with absolute position embeddings (the shipped
configs) is implemented; relative position bias raises.
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from ymp import functional as YF

from ._params import Holder, add_param, linear_default, named_param_list, trunc_normal, xavier_uniform


class LayerNormWithForceFP32(nn.LayerNorm):
    """Kept for API compatibility (norm_layer=partial(LayerNormWithForceFP32, eps=1e-6) in the
    reference constructors); the fused kernels always use fp32 statistics."""

    def forward(self, x):
        return F.layer_norm(x.float(), self.normalized_shape, self.weight.float(), self.bias.float(), self.eps).type_as(x)


def _block_params(root, pre, D, hid, std, layer_id, first):
    for nm in ("norm1", "norm2", "temporal_ln"):
        add_param(root, f"{pre}{nm}.weight", torch.ones(D))
        add_param(root, f"{pre}{nm}.bias", torch.zeros(D))
    for at in ("attn", "temporal_attn"):
        add_param(root, f"{pre}{at}.q_bias", torch.zeros(D))
        add_param(root, f"{pre}{at}.v_bias", torch.zeros(D))
        add_param(root, f"{pre}{at}.qkv.weight", trunc_normal((3 * D, D), std))
        w = trunc_normal((D, D), std)
        if at == "attn":
            w = w / math.sqrt(2.0 * layer_id)  # fix_init_weight (:513-519)
        add_param(root, f"{pre}{at}.proj.weight", w)
        add_param(root, f"{pre}{at}.proj.bias", torch.zeros(D))
    # temporal_fc is zero-initialised for every block but the first (:491-498)
    add_param(root, f"{pre}temporal_fc.weight", trunc_normal((D, D), std) if first else torch.zeros(D, D))
    add_param(root, f"{pre}temporal_fc.bias", torch.zeros(D))
    add_param(root, f"{pre}mlp.fc1.weight", trunc_normal((hid, D), std))
    add_param(root, f"{pre}mlp.fc1.bias", torch.zeros(hid))
    add_param(root, f"{pre}mlp.fc2.weight", trunc_normal((D, hid), std) / math.sqrt(2.0 * layer_id))
    add_param(root, f"{pre}mlp.fc2.bias", torch.zeros(D))


class TimeSformer(nn.Module):
    def __init__(self, img_size=224, num_frames=4, patch_size=16, in_chans=3, embed_dim=768, depth=12,
                 num_heads=12, mlp_ratio=4., qkv_bias=True, qk_scale=None, drop_rate=0., attn_drop_rate=0.,
                 drop_path_rate=0., norm_layer=None, init_values=None, attn_head_dim=None,
                 use_abs_pos_emb=True, use_rel_pos_bias=False, use_shared_rel_pos_bias=False, init_std=0.02,
                 grad_ckpt=False, stop_grad_conv1=False, postnorm=False, clip_model=False,
                 add_temporal_module=False, **kwargs):
        super().__init__()
        if use_rel_pos_bias or use_shared_rel_pos_bias or not use_abs_pos_emb:
            raise NotImplementedError("only absolute position embeddings are supported (all shipped configs)")
        if not qkv_bias or postnorm or stop_grad_conv1 or in_chans != 3:
            raise NotImplementedError("unsupported TimeSformer option for the H100 path")
        if init_values:  # layer scale (gamma_1 / gamma_2): no shipped config sets it
            raise NotImplementedError("layer_scale_init_value > 0 is not supported on the H100 path")
        # drop_path_rate is accepted and has no effect, exactly like the reference: Block.forward
        # (models/vision_transformer.py:243-275) never applies self.drop_path.
        self.num_features = self.embed_dim = embed_dim
        self.num_frames = num_frames
        self.img_size, self.patch_size = img_size, patch_size
        self.num_patches = (img_size // patch_size) ** 2
        # grad_ckpt (reference :575-577, one checkpoint per block): the training backward re-runs each block's forward
        # from its saved input instead of keeping the block's activations (ymp.engine.vit_fwd recompute)
        self.grad_ckpt = grad_ckpt
        self.vcfg = dict(img_size=img_size, patch_size=patch_size, embed_dim=embed_dim, depth=depth,
                         num_heads=num_heads, mlp_ratio=mlp_ratio, num_frames=num_frames, clip_model=clip_model,
                         grad_ckpt=bool(grad_ckpt))
        D, hid, std = embed_dim, int(embed_dim * mlp_ratio), init_std
        add_param(self, "cls_token", trunc_normal((1, 1, D), std))
        add_param(self, "pos_embed", trunc_normal((1, self.num_patches + 1, D), std))
        add_param(self, "temporal_embed", torch.zeros(1, num_frames, D))
        add_param(self, "patch_embed.proj.weight", trunc_normal((D, in_chans, patch_size, patch_size), std))
        if not clip_model:
            add_param(self, "patch_embed.proj.bias", torch.zeros(D))
        else:
            add_param(self, "norm_pre.weight", torch.ones(D))
            add_param(self, "norm_pre.bias", torch.zeros(D))
        for i in range(depth):
            _block_params(self, f"blocks.{i}.", D, hid, std, i + 1, i == 0)
        add_param(self, "norm.weight", torch.ones(D))
        add_param(self, "norm.bias", torch.zeros(D))

    @torch.jit.ignore
    def no_weight_decay(self):
        return {'temporal_embed', 'pos_embed', 'cls_token'}

    def get_num_layers(self):
        return self.vcfg["depth"]

    def forward_features(self, x):
        B, C, T, H, W = x.shape
        assert H == self.img_size and W == self.img_size, \
            f"Input image size ({H}*{W}) doesn't match model ({self.img_size}*{self.img_size})."
        keys, params = named_param_list(self, "visual_encoder.")
        return YF.VitFn.apply(x, self.vcfg, torch.is_grad_enabled(), keys, *params)

    def forward(self, image_input):
        feats = self.forward_features(image_input)
        return feats[:, 0], feats


class AttentionPool(nn.Module):
    def __init__(self, dim, num_heads, mlp_ratio=4., qkv_bias=True, qk_scale=None, drop=0., attn_drop=0.,
                 drop_path=0., init_values=None, act_layer=nn.GELU, norm_layer=None, window_size=None,
                 attn_head_dim=None, postnorm=False, kdim=None):
        super().__init__()
        if kdim not in (None, dim) or not qkv_bias or (init_values is not None and init_values > 0) or postnorm:
            raise NotImplementedError("unsupported AttentionPool option for the H100 path")
        self.dim, self.num_heads = dim, num_heads
        hid = int(dim * mlp_ratio)
        for nm in ("norm1", "normk", "norm2"):
            add_param(self, f"{nm}.weight", torch.ones(dim))
            add_param(self, f"{nm}.bias", torch.zeros(dim))
        add_param(self, "attn.in_proj_weight", xavier_uniform((3 * dim, dim)))
        add_param(self, "attn.in_proj_bias", torch.zeros(3 * dim))
        add_param(self, "attn.bias_k", nn.init.xavier_normal_(torch.empty(1, 1, dim)))
        add_param(self, "attn.bias_v", nn.init.xavier_normal_(torch.empty(1, 1, dim)))
        w, _ = linear_default(dim, dim)
        add_param(self, "attn.out_proj.weight", w)
        add_param(self, "attn.out_proj.bias", torch.zeros(dim))
        w, b = linear_default(hid, dim)
        add_param(self, "mlp.fc1.weight", w)
        add_param(self, "mlp.fc1.bias", b)
        w, b = linear_default(dim, hid)
        add_param(self, "mlp.fc2.weight", w)
        add_param(self, "mlp.fc2.bias", b)

    def forward(self, x, k, rel_pos_bias=None, attn_mask=None, queries_param=None):
        """x: learnable_queries.repeat(B,1,1) in the reference call (models/distributed_gpt3.py:134).
        The kernels exploit that every sample shares the same query block, so the un-repeated
        parameter is passed as `queries_param` by the task models; a generic x is accepted only when
        every sample holds the same query block (checked), anything else raises."""
        if queries_param is None:
            if x.shape[0] > 1 and not bool((x == x[:1]).all()):
                raise NotImplementedError("AttentionPool on the H100 path needs one query block shared by all samples "
                                          "(learnable_queries.repeat(B,1,1), models/distributed_gpt3.py:134)")
            queries_param = x[:1]
        keys, params = named_param_list(self, "attn_pool.")
        keys = ["learnable_queries"] + keys
        return YF.AttnPoolFn.apply(k, self.num_heads, torch.is_grad_enabled(), keys, queries_param, *params)


def _convert_pretrained_vit(vit_pretrained_weights):
    """qkv.bias -> (q_bias, v_bias); drop classifier heads (reference :719-728)."""
    for key in list(vit_pretrained_weights.keys()):
        if 'qkv.bias' in key:
            q, _, v = vit_pretrained_weights[key].chunk(3)
            vit_pretrained_weights[key.replace('qkv.bias', 'q_bias')] = q
            vit_pretrained_weights[key.replace('qkv.bias', 'v_bias')] = v
            del vit_pretrained_weights[key]
        elif 'head' in key:
            del vit_pretrained_weights[key]
    return vit_pretrained_weights


def resize_pos_embed(posemb, posemb_new):
    """Bilinear resize of the patch grid of a [1, 1+g*g, D] position embedding (reference :731-749)."""
    n_new = posemb_new.shape[1] - 1
    tok, grid = posemb[:, :1], posemb[0, 1:]
    g_old, g_new = int(math.sqrt(len(grid))), int(math.sqrt(n_new))
    grid = grid.reshape(1, g_old, g_old, -1).permute(0, 3, 1, 2)
    dt = grid.dtype
    grid = F.interpolate(grid.float(), size=(g_new, g_new), mode='bilinear').to(dt)
    grid = grid.permute(0, 2, 3, 1).reshape(1, g_new * g_new, -1)
    return torch.cat([tok, grid], dim=1)


def resize_temporal_embed(posemb, posemb_new, mode='interpolate'):
    """Linear interpolation (or padding) of [1, T, D] temporal embeddings (reference :752-764)."""
    t_new, t_old = posemb_new.shape[1], posemb.shape[1]
    if mode == 'padding':
        if t_old <= t_new:
            posemb_new[:, :t_old] = posemb
            return posemb_new
        return posemb[:, :t_new]
    return F.interpolate(posemb.permute(0, 2, 1), t_new, mode="linear").permute(0, 2, 1)
