"""EVA image encoder on the H100 kernels - mirrors the classes of the reference `models/eva_vit.py` that
`DistributedGPT3_Pretrain_Image` uses (SURVEY.md 8f N3): VisionTransformer (:245-350), create_eva_vit_g (:413-436:
224 px, 14 x 14 patches, 1408 wide, 40 blocks, 16 heads of 88, mlp 4.3637), interpolate_pos_embed (:372-392).
Parameter names follow the reference (`blocks.{i}.attn.{q_bias,v_bias,qkv.weight,proj.*}`, `patch_embed.proj.*`, ...),
so EVA checkpoints load with load_state_dict.  Relative position bias, layer scale and stochastic depth are not
implemented (the shipped visual configs leave them off) and raise."""
import math

import torch
import torch.nn as nn

from ymp import functional as YF

from ._params import add_param, named_param_list, trunc_normal


class VisionTransformer(nn.Module):
    def __init__(self, img_size=224, patch_size=16, in_chans=3, num_classes=1000, embed_dim=768, depth=12, num_heads=12,
                 mlp_ratio=4., qkv_bias=False, qk_scale=None, drop_rate=0., attn_drop_rate=0., drop_path_rate=0.,
                 norm_layer=nn.LayerNorm, init_values=None, use_abs_pos_emb=True, use_rel_pos_bias=False,
                 use_shared_rel_pos_bias=False, use_mean_pooling=True, init_scale=0.001, use_checkpoint=False):
        super().__init__()
        if use_rel_pos_bias or use_shared_rel_pos_bias or not use_abs_pos_emb or (init_values is not None and init_values > 0):
            raise NotImplementedError("EVA encoder on the H100 path: absolute position embeddings, no layer scale")
        if not qkv_bias or use_mean_pooling or in_chans != 3 or drop_rate or attn_drop_rate:
            raise NotImplementedError("EVA encoder on the H100 path: qkv_bias=True, use_mean_pooling=False, no dropout")
        if drop_path_rate:
            raise NotImplementedError("stochastic depth (drop_path > 0) is not implemented on the H100 path")
        self.image_size, self.num_features, self.embed_dim = img_size, embed_dim, embed_dim
        eps = 1e-5
        if norm_layer is not None:
            probe = norm_layer(8)
            eps = getattr(probe, "eps", 1e-5)
        n = (img_size // patch_size) ** 2
        hid = int(embed_dim * mlp_ratio)
        self.ecfg = dict(img_size=img_size, patch_size=patch_size, embed_dim=embed_dim, depth=depth, num_heads=num_heads,
                         mlp_ratio=mlp_ratio, eps=eps)
        D = embed_dim
        add_param(self, "cls_token", trunc_normal((1, 1, D), 0.02))
        add_param(self, "pos_embed", trunc_normal((1, n + 1, D), 0.02))
        add_param(self, "patch_embed.proj.weight", trunc_normal((D, in_chans, patch_size, patch_size), 0.02))
        add_param(self, "patch_embed.proj.bias", torch.zeros(D))
        for i in range(depth):
            pre = f"blocks.{i}."
            for nm in ("norm1", "norm2"):
                add_param(self, pre + nm + ".weight", torch.ones(D))
                add_param(self, pre + nm + ".bias", torch.zeros(D))
            add_param(self, pre + "attn.q_bias", torch.zeros(D))
            add_param(self, pre + "attn.v_bias", torch.zeros(D))
            add_param(self, pre + "attn.qkv.weight", trunc_normal((3 * D, D), 0.02))
            add_param(self, pre + "attn.proj.weight", trunc_normal((D, D), 0.02) / math.sqrt(2.0 * (i + 1)))   # fix_init_weight
            add_param(self, pre + "attn.proj.bias", torch.zeros(D))
            add_param(self, pre + "mlp.fc1.weight", trunc_normal((hid, D), 0.02))
            add_param(self, pre + "mlp.fc1.bias", torch.zeros(hid))
            add_param(self, pre + "mlp.fc2.weight", trunc_normal((D, hid), 0.02) / math.sqrt(2.0 * (i + 1)))
            add_param(self, pre + "mlp.fc2.bias", torch.zeros(D))
        add_param(self, "norm.weight", torch.ones(D))
        add_param(self, "norm.bias", torch.zeros(D))

    @torch.jit.ignore
    def no_weight_decay(self):
        return {'pos_embed', 'cls_token'}

    def forward_features(self, x):
        B, C, H, W = x.shape
        assert H == self.image_size and W == self.image_size, \
            f"Input image size ({H}*{W}) doesn't match model ({self.image_size}*{self.image_size})."
        keys, params = named_param_list(self, "visual_encoder.")
        return YF.EvaFn.apply(x, self.ecfg, keys, *params)

    def forward(self, x):
        x = self.forward_features(x)
        return x[:, 0], x


def interpolate_pos_embed(model, checkpoint_model):
    """Bicubic resize of a checkpoint's patch-grid position embedding to the model's grid (reference :372-392)."""
    if 'pos_embed' in checkpoint_model:
        pos = checkpoint_model['pos_embed'].float()
        D = pos.shape[-1]
        n_new = model.pos_embed.shape[-2] - 1
        g_old, g_new = int((pos.shape[-2] - 1) ** 0.5), int(n_new ** 0.5)
        if g_old != g_new:
            print("Position interpolate from %dx%d to %dx%d" % (g_old, g_old, g_new, g_new))
            tok = pos[:, 1:].reshape(-1, g_old, g_old, D).permute(0, 3, 1, 2)
            tok = torch.nn.functional.interpolate(tok, size=(g_new, g_new), mode='bicubic', align_corners=False)
            checkpoint_model['pos_embed'] = torch.cat((pos[:, :1], tok.permute(0, 2, 3, 1).flatten(1, 2)), dim=1)


def create_eva_vit_g(img_size=224, drop_path_rate=0.4, norm_layer=nn.LayerNorm, use_checkpoint=True, precision="fp16"):
    """EVA-g (reference :413-436).  use_checkpoint is accepted; activations stay resident (180 GB HBM)."""
    return VisionTransformer(img_size=img_size, patch_size=14, use_mean_pooling=False, embed_dim=1408, depth=40,
                             num_heads=1408 // 88, mlp_ratio=4.3637, qkv_bias=True, drop_path_rate=drop_path_rate,
                             norm_layer=norm_layer, use_checkpoint=use_checkpoint)
