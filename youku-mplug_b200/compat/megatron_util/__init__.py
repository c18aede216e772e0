"""Stand-in for `megatron_util` (ModelScope wheel, ==1.3.0, not a dependency of this package).  The H100 `models` package does
not use it; the scripts only alias a few `mpu` getters and pass `mpu=` to deepspeed.initialize
(run_pretrain_distributed_gpt3.py:36-40,263-267).  Tensor model parallel size is 1 by construction."""
from . import mpu  # noqa: F401


def initialize_megatron(cfg=None, **kwargs):
    return None
