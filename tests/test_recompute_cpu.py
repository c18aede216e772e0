"""Host-side plumbing of activation recompute: the TimeSformer's grad_ckpt and megatron_cfg.checkpoint_activations
reach the configs that the autograd functions hand to the engine, and the shipped yamls select them as intended."""
import json
import os

import pytest

from oracle import port
from helpers import build_pretrain, make_model_dir, pretrain_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "youku-mplug_b200")

TRAINING_YAMLS = ["caption/caption_gpt3_1.3B_youku_v0.yaml", "caption/caption_gpt3_2.7B_youku_v0.yaml",
                  "cls/cls_gpt3_1.3B_youku_v0_sharp_2.yaml", "cls/cls_gpt3_2.7B_youku_v0_sharp_2.yaml",
                  "retrieval/retrieval_gpt3_1.3B_youku_v0.yaml", "retrieval/retrieval_gpt3_2.7B_youku_v0.yaml",
                  "retrieval/retrieval_itm_gpt3_1.3B_youku_v0.yaml", "retrieval/retrieval_itm_gpt3_2.7B_youku_v0.yaml",
                  "pretrain/gpt3_1.3B/pretrain_gpt3_freezeGPT_youku_v0.yaml",
                  "pretrain/gpt3_2.7B/pretrain_gpt3_freezeGPT_youku_v0.yaml"]


@pytest.mark.parametrize("flag", [True, False])
def test_timesformer_carries_grad_ckpt(flag):
    from models.vision_transformer import TimeSformer
    vit = TimeSformer(img_size=32, num_frames=2, patch_size=16, embed_dim=64, depth=1, num_heads=2, grad_ckpt=flag)
    assert vit.vcfg["grad_ckpt"] is flag and vit.grad_ckpt is flag


def test_package_clip_b16_turns_vit_recompute_on():
    """Every shipped training yaml uses configs/models/clip-b16.json, which sets grad_ckpt like the reference's."""
    os.environ["YMP_ALLOW_RANDOM_INIT"] = "1"
    import models.distributed_gpt3 as D
    vis = os.path.join(PKG, "configs", "models", "clip-b16.json")
    assert json.load(open(vis))["grad_ckpt"] is True
    td = make_model_dir(port.VCFG_TINY, port.GCFG_TINY)
    tiny_vis = dict(json.load(open(vis)), depth=1, embed_dim=64, num_heads=2, img_size=32, pretrained_ckpt=None)
    with open(os.path.join(td, "clip.json"), "w") as f:
        json.dump(tiny_vis, f)
    model = D.DistributedGPT3_Pretrain(config=pretrain_config(td, 8, visual_cfg=os.path.join(td, "clip.json")), tokenizer=None)
    assert model.visual_encoder.vcfg["grad_ckpt"] is True
    # the test and bench model dirs write grad_ckpt: false, so their code path is the resident one
    assert build_pretrain(port.VCFG_TINY, port.GCFG_TINY, 8).visual_encoder.vcfg["grad_ckpt"] is False


def test_checkpoint_activations_reaches_engine_cfg():
    mc = {"world_size": 1, "model_parallel_size": 1, "tensor_model_parallel_size": 1}
    on = build_pretrain(port.VCFG_TINY, port.GCFG_TINY, 8, megatron_cfg=dict(mc, checkpoint_activations=True))
    assert on.text_decoder.config.engine_cfg(True)["checkpoint_activations"] is True
    assert on.text_decoder.config.engine_cfg(False)["checkpoint_activations"] is True
    off = build_pretrain(port.VCFG_TINY, port.GCFG_TINY, 8, megatron_cfg=mc)
    assert off.text_decoder.config.engine_cfg(True)["checkpoint_activations"] is False
    with pytest.raises(ValueError):   # the tensor-parallel check still runs on the same block
        build_pretrain(port.VCFG_TINY, port.GCFG_TINY, 8, megatron_cfg=dict(mc, tensor_model_parallel_size=2,
                                                                               checkpoint_activations=True))


def test_recompute_flag_lookup():
    from ymp import functional as YF
    assert YF._vit_recompute({"grad_ckpt": True}) and not YF._vit_recompute({})
    assert YF._gpt_recompute({"checkpoint_activations": True}) and not YF._gpt_recompute({"training": True})


def test_only_the_itm_yamls_recompute_the_decoder():
    import importlib
    import sys
    compat = os.path.join(PKG, "compat")
    sys.path.append(compat)
    try:
        ryaml = importlib.import_module("ruamel.yaml")
    finally:
        sys.path.remove(compat)
        for k in [k for k in sys.modules if k == "ruamel" or k.startswith("ruamel.")]:
            del sys.modules[k]
    for n in TRAINING_YAMLS:
        cfg = ryaml.load(open(os.path.join(PKG, "configs", n)), Loader=ryaml.Loader)
        want = "retrieval_itm_" in n
        assert cfg["megatron_cfg"].get("checkpoint_activations", False) is want, n
        assert cfg["megatron_cfg"]["tensor_model_parallel_size"] == 1, n
