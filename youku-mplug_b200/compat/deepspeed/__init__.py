"""Stand-in for the part of DeepSpeed the reference scripts use (run_pretrain_distributed_gpt3.py:385-396,
257-267; downstream/run_*_gpt3.py alike): `add_config_arguments(parser)` and `initialize(...)`.

`initialize` reads the `ds_config.json` the script wrote (utils.py:483-562: Adam(adam_w_mode) hyper-parameters,
gradient_clipping, bf16 flag, train_batch_size / train_micro_batch_size_per_gpu -> gradient accumulation) and
returns `ymp.train.TrainEngine` - fused clip + AdamW on flat buffers, bucketed overlapped NCCL all-reduce, no
ZeRO partitioning (130 M trainable parameters = 1.6 GB of state per GPU).
"""
import json

import torch
import torch.distributed as dist

__version__ = "0.8.0+ymp_b200"


def add_config_arguments(parser):
    group = parser.add_argument_group("DeepSpeed", "DeepSpeed configurations")
    group.add_argument("--deepspeed", default=False, action="store_true")
    group.add_argument("--deepspeed_config", default=None, type=str)
    group.add_argument("--deepscale", default=False, action="store_true")
    group.add_argument("--deepscale_config", default=None, type=str)
    group.add_argument("--deepspeed_mpi", default=False, action="store_true")
    return parser


def init_distributed(dist_backend="nccl", **kwargs):
    if not dist.is_initialized():
        dist.init_process_group(backend=dist_backend)


def initialize(args=None, model=None, optimizer=None, model_parameters=None, training_data=None, lr_scheduler=None,
               mpu=None, dist_init_required=None, collate_fn=None, config=None, config_params=None):
    from ymp.train import TrainEngine
    if not torch.cuda.is_available():
        raise RuntimeError("deepspeed.initialize (ymp_b200 engine): needs a CUDA device - the H100 path has no CPU fallback")
    cfg = config if config is not None else config_params
    if cfg is None:
        cfg = getattr(args, "deepspeed_config", None)
    if isinstance(cfg, str):
        with open(cfg) as f:
            cfg = json.load(f)
    cfg = cfg or {}
    if cfg.get("fp16", {}).get("enabled", False):
        raise NotImplementedError("the H100 engine trains in bf16 (pass --bf16): fp16 + dynamic loss scaling is not implemented")
    if dist_init_required and not dist.is_initialized():
        init_distributed()
    if mpu is not None and mpu.get_tensor_model_parallel_world_size() != 1:
        raise ValueError("tensor model parallel size must be 1 on the H100 path (pure data parallel)")
    dev = torch.device("cuda", torch.cuda.current_device())
    model = model.to(dev)
    if cfg.get("bf16", {}).get("enabled", True):
        model = model.to(torch.bfloat16)
    world = dist.get_world_size() if dist.is_initialized() else 1
    opt = cfg.get("optimizer", {}).get("params", {})
    micro = cfg.get("train_micro_batch_size_per_gpu")
    total = cfg.get("train_batch_size")
    gas = cfg.get("gradient_accumulation_steps")
    if gas is None:
        gas = max(1, int(total // (micro * world))) if (micro and total) else 1
    engine = TrainEngine(model, optimizer_params=model_parameters, lr=opt.get("lr", 1e-4), betas=tuple(opt.get("betas", (0.9, 0.999))),
                         eps=opt.get("eps", 1e-8), weight_decay=opt.get("weight_decay", 0.0),
                         clip_grad=cfg.get("gradient_clipping", 0.0), gradient_accumulation_steps=gas)
    return engine, engine.optimizer, None, None
