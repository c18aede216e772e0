"""TEST INFRASTRUCTURE - makes the UNMODIFIED reference modules importable on CPU.

The reference ($YMP_REFERENCE, X-PLUG/Youku-mPLUG @ 9d3dd3f) imports packages that are not in
this image.  This module installs minimal stand-ins into ``sys.modules`` so that
``models/{vision_transformer,modeling_distributed_gpt3,distributed_gpt3}.py`` import and run on
CPU exactly as written.  It is used ONLY to (a) validate oracle/port.py and (b) generate the golden
vectors under tests/golden/ (oracle/make_golden.py).  Nothing in the product or the tests imports it, and it
needs a checkout of the reference.

Un-vendored arithmetic restated here (source absent from the reference checkout):
  * megatron_util==1.3.0 (README.md:60): tensor-parallel linears / embedding / vocab-parallel CE /
    FusedScaleMaskSoftmax / MixedFusedLayerNorm / bias_gelu_impl.  Stand-ins implement TP=1
    semantics following upstream Megatron-LM: linear = x @ W^T (+ b unless skip_bias_add, in which
    case the bias is returned separately), CE = logsumexp(logits) - logits[label], softmax torch
    path = (optional fp32 upcast) * scale -> masked_fill(-10000) -> softmax, LayerNorm = affine LN,
    bias_gelu = tanh approximation 0.5 x (1 + tanh(0.79788456 x (1 + 0.044715 x^2))).
    Call sites: models/modeling_distributed_gpt3.py:562-578,586-588,619-620,724-727,843-857,
    1002-1020,1348-1357.
  * timm==0.6.7 (drop_path / to_2tuple / trunc_normal_), addict.Dict, sh: init/utility only.
"""
import contextlib
import enum
import importlib.machinery
import json
import os
import sys
import tempfile
import types

import torch
import torch.nn as nn
import torch.nn.functional as F

REFERENCE_ROOT = os.environ.get("YMP_REFERENCE", "reference")


def _module(name, **attrs):
    m = types.ModuleType(name)
    m.__spec__ = importlib.machinery.ModuleSpec(name, loader=None)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


def _install_timm():
    def drop_path(x, drop_prob=0.0, training=False):
        return x

    def to_2tuple(v):
        return v if isinstance(v, tuple) else (v, v)

    _module("timm", create_model=None)
    _module("timm.models")
    _module("timm.models.layers", drop_path=drop_path, to_2tuple=to_2tuple,
            trunc_normal_=torch.nn.init.trunc_normal_)
    _module("timm.models.registry", register_model=lambda fn: fn)
    _module("timm.utils", get_state_dict=lambda m: m.state_dict())


class _AttrDict(dict):
    __getattr__ = dict.get
    __setattr__ = dict.__setitem__


class _TPLinear(nn.Module):
    """Column/RowParallelLinear at tensor-parallel size 1: returns (output, bias_or_None)."""

    def __init__(self, in_f, out_f, init_method=None, skip_bias_add=False, **_unused):
        super().__init__()
        self.weight = nn.Parameter(torch.empty(out_f, in_f))
        self.bias = nn.Parameter(torch.zeros(out_f))
        self.skip_bias_add = skip_bias_add
        (init_method or nn.init.xavier_normal_)(self.weight)

    def forward(self, x):
        if self.skip_bias_add:
            return F.linear(x, self.weight), self.bias
        return F.linear(x, self.weight, self.bias), None


class _VocabEmbedding(nn.Embedding):
    def __init__(self, num, dim, init_method=None):
        super().__init__(num, dim)
        if init_method is not None:
            init_method(self.weight)


class _LinearFn:
    @staticmethod
    def apply(x, w, b, *_flags):
        return F.linear(x, w, b)


def _vocab_ce(logits, labels):  # logits [s,b,V] fp32, labels [s,b]
    s, b, v = logits.shape
    return F.cross_entropy(logits.reshape(-1, v), labels.reshape(-1), reduction="none").view(s, b)


class _RngTracker:
    def fork(self):
        return contextlib.nullcontext()


class _MemBuf:
    def get_tensor(self, shape, dtype, name):
        return torch.empty(shape, dtype=dtype)


class _AttnMaskType(enum.Enum):
    padding = 1
    causal = 2


def _bias_gelu(x, bias):
    x = x + bias
    return x * 0.5 * (1.0 + torch.tanh(0.79788456 * x * (1 + 0.044715 * x * x)))


class _MegatronLayerNorm(nn.LayerNorm):
    def __init__(self, hidden, eps=1e-5, no_persist_layer_norm=True, sequence_parallel=False):
        super().__init__(hidden, eps=eps)


class _ScaleMaskSoftmax(nn.Module):
    def __init__(self, fp16, bf16, mask_type, fusion, mask_func, softmax_in_fp32, scale):
        super().__init__()
        self.mask_func, self.in_fp32, self.scale = mask_func, softmax_in_fp32, scale

    def forward(self, x, mask):
        dt = x.dtype
        if self.in_fp32:
            x = x.float()
        if self.scale is not None:
            x = x * self.scale
        if mask is not None:
            x = self.mask_func(x, mask)
        p = torch.softmax(x, dim=-1)
        return p.to(dt) if self.in_fp32 else p


def _install_megatron():
    def viewless(*a, **k):
        return a[0] if a else k["inp"]

    mpu = _module(
        "megatron_util.mpu",
        ColumnParallelLinear=_TPLinear, RowParallelLinear=_TPLinear,
        VocabParallelEmbedding=_VocabEmbedding,
        LinearWithGradAccumulationAndAsyncCommunication=_LinearFn,
        vocab_parallel_cross_entropy=_vocab_ce,
        gather_from_tensor_model_parallel_region=lambda t: t,
        get_tensor_model_parallel_world_size=lambda: 1,
        get_tensor_model_parallel_rank=lambda: 0,
        divide=lambda a, b: a // b,
        split_tensor_along_last_dim=lambda t, n: torch.split(t, t.size(-1) // n, dim=-1),
        make_viewless_tensor=viewless,
        get_cuda_rng_tracker=lambda: _RngTracker(),
        set_defaults_if_not_set_tensor_model_parallel_attributes=lambda p: None)
    gv = _module("megatron_util.global_vars", get_global_memory_buffer=lambda: _MemBuf())
    model = _module("megatron_util.model", AttnMaskType=_AttnMaskType, Float16Module=nn.Module,
                    LayerNorm=_MegatronLayerNorm, bias_gelu_impl=_bias_gelu)
    _module("megatron_util.model.fused_softmax", FusedScaleMaskSoftmax=_ScaleMaskSoftmax)
    _module("megatron_util", mpu=mpu, global_vars=gv, model=model,
            initialize_megatron=lambda cfg: None)


_installed = False


def install():
    """Install the stand-ins and put the reference on sys.path (idempotent)."""
    global _installed
    if _installed:
        return
    if not os.path.isdir(REFERENCE_ROOT):
        raise RuntimeError(f"reference tree not found at {REFERENCE_ROOT}")
    import transformers  # noqa: F401  (must be imported before the timm stand-in exists)
    import transformers.modeling_utils  # noqa: F401
    _install_timm()
    _module("addict", Dict=_AttrDict)
    _module("sh")
    _install_megatron()
    torch.cuda.current_device = lambda: "cpu"
    nn.Module.cuda = lambda self, device=None: self
    _installed = True


def import_reference():
    """Returns the reference's (vision_transformer, modeling_distributed_gpt3, distributed_gpt3).

    The reference's top-level package is called ``models`` - the same name as this repo's drop-in
    package - and transformers looks modules up by name at construction time, so the reference
    modules stay registered in sys.modules: a process that calls this must not import the
    product's ``models`` package (oracle/make_golden.py does not)."""
    install()
    if "models" in sys.modules and not getattr(sys.modules["models"], "__file__", "").startswith(REFERENCE_ROOT):
        raise RuntimeError("a different `models` package is already imported in this process")
    sys.path.insert(0, REFERENCE_ROOT)
    try:
        import models.vision_transformer as V
        import models.modeling_distributed_gpt3 as G
        import models.distributed_gpt3 as D
    finally:
        sys.path.remove(REFERENCE_ROOT)
    G.pre_load = lambda rank, d, tag="": None
    G.split_state_dict = lambda sd, model, parts: model.state_dict()
    return V, G, D


def build_reference_model(cls_name, visual_cfg, gpt_cfg, num_learnable_token, seed=0, dropout=(0.0, 0.0), **config_extra):
    """Instantiate one of the reference's task models (models/distributed_gpt3.py: DistributedGPT3_Pretrain / _Cls /
    _Caption / _Retrieval / _Retrieval_Cls) on CPU (fp32, eval; dropout = (hidden, attention), 0 by default)."""
    V, G, D = import_reference()
    td = tempfile.mkdtemp(prefix="ymp_ref_")
    gpt_cfg = dict(gpt_cfg, hidden_dropout=dropout[0], attention_dropout=dropout[1])
    with open(os.path.join(td, "config.json"), "w") as f:
        json.dump(gpt_cfg, f)
    vis = dict(visual_cfg, pretrained_ckpt=None, grad_ckpt=False)
    with open(os.path.join(td, "vis.json"), "w") as f:
        json.dump(vis, f)
    config = dict(visual_cfg=os.path.join(td, "vis.json"), text_cfg=os.path.join(td, "config.json"),
                  text_decoder=td, megatron_cfg={}, num_learnable_token=num_learnable_token,
                  use_contrastive=False, freeze_text_decoder=True, num_frames=visual_cfg["num_frames"])
    config.update(config_extra)
    torch.manual_seed(seed)
    model = getattr(D, cls_name)(config=config, tokenizer=None).eval()
    return model, G


def build_reference_pretrain(visual_cfg, gpt_cfg, num_learnable_token, seed=0, use_contrastive=False):
    """Instantiate the reference's DistributedGPT3_Pretrain on CPU (fp32, eval, dropout 0)."""
    return build_reference_model("DistributedGPT3_Pretrain", visual_cfg, gpt_cfg, num_learnable_token, seed=seed,
                                 use_contrastive=use_contrastive)


class philox_dropout:
    """Context manager: while active, torch.nn.functional.dropout (hence nn.Dropout and the reference's
    bias_dropout_add, models/modeling_distributed_gpt3.py:1056-1078) draws its masks from the H100 kernels' Philox
    convention (oracle/philox.py) instead of torch's generator, so the UNMODIFIED reference can be run in train()
    mode with exactly the masks the kernels will use.  Call sites of one decoder pass are identified by call order:
    embedding dropout ([s,b,h], :631) -> site 0, then per layer attention probabilities ([b,np,sq,sk], :732) ->
    4l+1, bias-dropout-add after attention ([s,b,h]) -> 4l+2, after the MLP -> 4l+3."""

    def __init__(self, seed, offset):
        self.seed, self.offset, self.calls = seed, offset, 0

    def _dropout(self, input, p=0.5, training=True, inplace=False):
        from oracle import philox
        if not training or p <= 0.0:
            return input
        n = self.calls
        self.calls += 1
        site = 0 if n == 0 else 4 * ((n - 1) // 3) + 1 + (n - 1) % 3
        if input.dim() == 4:                     # attention probabilities [b, np, sq, sk]
            assert (n - 1) % 3 == 0, "call order: attention dropout expected"
            b, h, sq, sk = input.shape
            return philox.dropout(input.reshape(b * h * sq, sk), self.seed, self.offset, site, p).reshape(input.shape)
        assert input.dim() == 3                  # hidden states [s, b, h]: logical row = b*S + s
        S, B, H = input.shape
        x = input.permute(1, 0, 2).reshape(B * S, H)
        return philox.dropout(x, self.seed, self.offset, site, p).reshape(B, S, H).permute(1, 0, 2)

    def __enter__(self):
        import torch.nn.functional as F
        self._orig = F.dropout
        F.dropout = self._dropout
        return self

    def __exit__(self, *exc):
        import torch.nn.functional as F
        F.dropout = self._orig
        return False
