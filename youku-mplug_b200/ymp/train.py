"""Data-parallel training engine for the drop-in models: the part of `deepspeed.initialize(...)`
the reference scripts rely on (run_pretrain_distributed_gpt3.py:257-267,134-138; utils.py:483-562),
rebuilt for one-process-per-GPU H100 training.

  engine = TrainEngine(model, optimizer_params, lr=..., betas=..., eps=..., clip_grad=...)
  loss, _ = engine(video, text); engine.backward(loss); engine.step()

* trainable parameters live in ONE flat bf16 buffer (module parameters are views of it) with fp32
  master weights and Adam moments beside it (ZeRO-free: 130 M trainable params = 1.6 GB of state);
* weight gradients are accumulated by the kernels directly into one flat fp32 buffer (the GEMM
  split-K epilogue adds into it), so there is no per-parameter .grad tensor and no copy;
* step(): one NCCL all-reduce of the flat gradient over NVLink/NVSwitch, device-side global-norm
  clipping, fused AdamW - no host synchronisation anywhere in backward/step.
"""
import contextlib

import torch
import torch.distributed as dist

from . import functional as YF
from . import ops


def default_param_groups(model, weight_decay, skip_list=(), visual_backbone_scale=False):
    """Same grouping rule as the reference's optim/optim_factory.py:219-265 (no decay for 1-D / `.bias` /
    skip_list names / any name containing "bias" or "LayerNorm.weight" - check_keywords_in_name, :226 - so the
    3-D attn_pool.attn.bias_k / bias_v rows are decay-free too; optional 0.1 lr scale for non-temporal
    visual_encoder weights)."""
    groups = {}
    for name, p in model.named_parameters():
        if not p.requires_grad:
            continue
        no_decay = (p.dim() == 1 or name.endswith(".bias") or name in skip_list
                    or "bias" in name or "LayerNorm.weight" in name)
        scaled = visual_backbone_scale and "visual_encoder." in name and "temporal" not in name
        key = (no_decay, scaled)
        g = groups.setdefault(key, dict(params=[], names=[], weight_decay=0.0 if no_decay else weight_decay,
                                        lr_scale=0.1 if scaled else 1.0))
        g["params"].append(p)
        g["names"].append(name)
    return list(groups.values())


class _Optimizer:
    """What the reference loop touches on `model.optimizer` (run_pretrain...py:46-53,88-96)."""

    def __init__(self, groups):
        self.param_groups = groups
        self.cur_scale = 1.0
        self._global_grad_norm = None


BUCKET_MIN_ELEMS = 1 << 18   # 1 MB of fp32 gradients: smaller ranges are left to the single reduction in step()


def plan_buckets(spans, min_elems=BUCKET_MIN_ELEMS, pattern=r"(visual_encoder\.blocks\.\d+\.)"):
    """In-backward all-reduce buckets: spans = [(parameter name, begin, end)] in flat-buffer order; a bucket is a maximal
    run of ADJACENT spans that belong to the same TimeSformer block (same `pattern` prefix) and holds at least
    `min_elems` elements.  Returns {block prefix: [(begin, end), ...]} - what TrainEngine reduces the moment the
    backward reports that block final (pure host logic, CPU-tested over gloo in tests/test_dist_cpu.py)."""
    import re
    buckets, cur = {}, None

    def close(c):
        if c is not None and c[0] is not None and c[2] - c[1] >= min_elems:
            buckets.setdefault(c[0], []).append((c[1], c[2]))

    for name, a, b in spans:
        m = re.match(pattern, name)
        key = m.group(1) if m else None
        if cur is not None and key is not None and cur[0] == key and cur[2] == a:
            cur[2] = b
        else:
            close(cur)
            cur = [key, a, b]
    close(cur)
    return buckets


def gap_ranges(reduced, total):
    """The parts of [0, total) that the ranges in `reduced` (any order, possibly touching) do not cover."""
    gaps, pos = [], 0
    for a, b in sorted(reduced) + [(total, total)]:
        if a > pos:
            gaps.append((pos, a))
        pos = max(pos, b)
    return gaps


class TrainEngine:
    def __init__(self, model, optimizer_params=None, lr=1e-4, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.05,
                 clip_grad=3.0, process_group=None, gradient_accumulation_steps=1, overlap_comm=True):
        self.module = model
        self.gas = max(1, int(gradient_accumulation_steps))
        self.group = process_group
        self.world = dist.get_world_size(process_group) if dist.is_initialized() else 1
        if optimizer_params is None:
            optimizer_params = default_param_groups(model, weight_decay, getattr(model, "no_weight_decay", lambda: ())())
        self.clip_grad = clip_grad
        params = [p for g in optimizer_params for p in g["params"]]
        assert params, "no trainable parameters"
        dev = params[0].device
        if dev.type != "cuda":
            raise RuntimeError("TrainEngine needs the model on a CUDA device (no CPU fallback)")
        total = sum((p.numel() + 7) // 8 * 8 for p in params)
        self.flat_param = torch.zeros(total, device=dev, dtype=torch.bfloat16)
        self.flat_grad = torch.zeros(total, device=dev, dtype=torch.float32)
        # fp32 master weights come from the parameters as handed in (an fp32 model keeps its low bits; a
        # bf16 model gives exactly its bf16 values)
        self.master = torch.zeros(total, device=dev, dtype=torch.float32)
        self._sink = {}
        self._params = params
        names = {id(p): n for n, p in model.named_parameters()}
        spans = []  # (name, start, end) in flat order
        off = 0
        groups = []
        for g in optimizer_params:
            start = off
            for p in g["params"]:
                n = p.numel()
                spans.append((names.get(id(p), ""), off, off + (n + 7) // 8 * 8))
                self.master[off:off + n].copy_(p.data.reshape(-1))
                view = self.flat_param[off:off + n].view(p.shape)
                view.copy_(p.data)
                p.data = view
                self._sink[id(p)] = self.flat_grad[off:off + n]
                off += (n + 7) // 8 * 8
            groups.append(dict(params=g["params"], weight_decay=g.get("weight_decay", weight_decay),
                               lr_scale=g.get("lr_scale", 1.0), lr=lr * g.get("lr_scale", 1.0), betas=list(betas),
                               eps=eps, _range=(start, off)))
        YF.note_weight_write()   # the parameters now live in flat_param (in this dtype)
        self.exp_avg = torch.zeros_like(self.master)
        self.exp_avg_sq = torch.zeros_like(self.master)
        self._sumsq = torch.zeros(1, device=dev, dtype=torch.float32)
        self.optimizer = _Optimizer(groups)
        self.micro_steps = 0
        self.global_steps = 0
        self._graphs = {}
        # ---- bucketed, overlapped gradient all-reduce (SURVEY 8e; the reference's ZeRO-1 reduce buckets,
        # utils.py:528-529): the contiguous flat ranges of each TimeSformer block (>= 1 MB) are all-reduced as
        # soon as the block's backward has produced them, on NCCL's own stream, while the remaining blocks still
        # run; everything else (abstractor, embeddings, biases: the gaps) goes in step().
        self.overlap_comm = overlap_comm and self.world > 1
        self._buckets, self._pending, self._reduced = {}, [], []
        if self.overlap_comm:
            self._buckets = plan_buckets(spans)

    # ---- nn.Module-like surface -----------------------------------------------------------
    def __call__(self, *args, **kwargs):
        return self.module(*args, **kwargs)

    def train(self, mode=True):
        self.module.train(mode)
        return self

    def eval(self):
        self.module.eval()
        return self

    def parameters(self):
        return self.module.parameters()

    def named_parameters(self):
        return self.module.named_parameters()

    def state_dict(self):
        return self.module.state_dict()

    # ---- training step ----------------------------------------------------------------------
    def _on_ready(self, prefix):
        """Called from inside the backward when the weight gradients under `prefix` are final."""
        if (self.micro_steps + 1) % self.gas:      # not the boundary micro-step: keep accumulating locally
            return
        for a, b in self._buckets.get(prefix, ()):
            self._pending.append(dist.all_reduce(self.flat_grad[a:b], op=dist.ReduceOp.SUM, group=self.group, async_op=True))
            self._reduced.append((a, b))

    def _join_comm(self):
        for w in self._pending:
            w.wait()   # stream-level: the compute stream waits for NCCL's stream, the host does not block
        self._pending = []

    def allreduce_gradients(self):
        """Sum the flat gradient over the data-parallel ranks: whatever the in-backward buckets have not
        already covered (all of it without overlap_comm)."""
        if self.world == 1:
            return
        self._join_comm()
        for a, b in gap_ranges(self._reduced, self.flat_grad.numel()):
            dist.all_reduce(self.flat_grad[a:b], op=dist.ReduceOp.SUM, group=self.group)
        self._reduced = []

    def _backward(self, loss):
        with YF.grad_sink(self._sink, self._on_ready if self.overlap_comm else None):
            loss.backward()
        # Parameters whose gradient comes from ordinary autograd rather than from the ymp Functions (the
        # contrastive `temp`, classifier heads too narrow for the 16-byte-aligned GEMM, ...) arrive in
        # p.grad: fold them into the flat buffer so that step() sees every trainable parameter.
        for p in self._params:
            if p.grad is not None:
                self._sink[id(p)].add_(p.grad.reshape(-1))
                p.grad = None

    def backward(self, loss):
        """DeepSpeed engine semantics (the reference calls model.backward(loss / update_freq),
        run_pretrain_distributed_gpt3.py:134-136): the loss is additionally scaled by
        1 / gradient_accumulation_steps and gradients accumulate until the boundary micro-step."""
        if self.gas > 1:
            loss = loss / self.gas
        self._backward(loss)
        self.micro_steps += 1

    def zero_grad(self):
        self.flat_grad.zero_()

    def is_gradient_accumulation_boundary(self):
        return self.micro_steps % self.gas == 0

    def step(self):
        if not self.is_gradient_accumulation_boundary():
            return  # keep accumulating: no all-reduce, no AdamW, no zeroing
        self.allreduce_gradients()
        self.global_steps += 1
        self._sumsq.zero_()
        ops.sumsq(self.flat_grad, self._sumsq)  # always: the loop logs the norm even without clipping
        scale = 1.0 / self.world
        for g in self.optimizer.param_groups:
            a, b = g["_range"]
            if b == a:
                continue
            ops.adamw(self.master[a:b], self.flat_param[a:b], self.flat_grad[a:b], self.exp_avg[a:b],
                      self.exp_avg_sq[a:b], step=self.global_steps, lr=g["lr"], beta1=g["betas"][0], beta2=g["betas"][1],
                      eps=g["eps"], weight_decay=g["weight_decay"], grad_scale=scale,
                      max_grad_norm=self.clip_grad or 0.0, sumsq_t=self._sumsq if self.clip_grad else None, zero_grad=True)
        YF.note_weight_write()
        self.optimizer._global_grad_norm = _LazyNorm(self._sumsq.clone(), scale)
        # every group range was reset by its AdamW pass (the ranges tile the flat buffer)

    def train_step(self, *inputs, use_graph=True, graph_warmup=2):
        """One full iteration (forward + backward + step) of `self.module(*inputs)`; returns the detached loss -
        for models that return several losses their sum, e.g. loss_caption + loss_contrastive
        (run_pretrain_distributed_gpt3.py:113).

        Shapes are static in pre-training (`padding='max_length'`, run_pretrain_distributed_gpt3.py:100),
        so after `graph_warmup` eager iterations the ~900 kernel launches of forward+backward are
        captured ONCE into a CUDA graph per input signature and replayed; with overlap_comm the bucketed gradient
        all-reduces are part of the graph (fork/join on NCCL's stream); the remaining all-reduce, the
        grad-norm and the fused AdamW (6 launches) stay outside the graph.  Inputs are copied into the graph's static buffers (the copy
        also casts fp32 frames to bf16), so callers may pass fresh tensors every step."""
        key = graph_key(inputs)
        st = self._graphs.setdefault(key, dict(calls=0))
        if self.gas > 1:
            use_graph = False   # boundary / non-boundary micro-steps differ (all-reduce, step): run eagerly

        def total(out):
            return sum(out[1:], out[0]) if isinstance(out, (tuple, list)) else out

        if not use_graph or st["calls"] < graph_warmup:
            loss = total(self.module(*inputs))
            self.backward(loss)
            self.step()
            st["calls"] += 1
            return loss.detach()
        if "graph" not in st:
            # the eager warm-up steps left their activations in the caching allocator; the graph gets a private pool of
            # the same size, so hand the cached blocks back first (B = 96 retrieval / 2.7B caption steps would not fit twice)
            torch.cuda.empty_cache()
            st["static"] = [_static_like(x) for x in inputs]
            for s_, x in zip(st["static"], inputs):
                _copy_into(s_, x)
            torch.cuda.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                loss = total(self.module(*st["static"]))
                self._backward(loss / self.gas if self.gas > 1 else loss)
                self._join_comm()   # the bucket all-reduces are part of the graph (fork/join on NCCL's stream)
            st["graph"], st["loss"], st["reduced"] = g, loss.detach(), list(self._reduced)
        else:
            for s_, x in zip(st["static"], inputs):
                _copy_into(s_, x)
        st["graph"].replay()
        self._reduced = list(st["reduced"])
        self.micro_steps += 1
        self.step()
        return st["loss"]

    # ---- checkpointing (utils.py:476-480,441-455) ----------------------------------------------
    def save_checkpoint(self, save_dir, tag=None, client_state=None):
        import os
        tag = tag or f"global_step{self.global_steps}"
        os.makedirs(os.path.join(save_dir, str(tag)), exist_ok=True)
        if not dist.is_initialized() or dist.get_rank() == 0:
            torch.save(dict(module=self.module.state_dict(), master=self.master, exp_avg=self.exp_avg,
                            exp_avg_sq=self.exp_avg_sq, global_steps=self.global_steps,
                            client_state=client_state or {}),
                       os.path.join(save_dir, str(tag), "mp_rank_00_model_states.pt"))
            with open(os.path.join(save_dir, "latest"), "w") as f:
                f.write(str(tag))
        if dist.is_initialized():
            dist.barrier(group=self.group)  # nobody reads `latest` / the tag directory before it is complete

    def load_checkpoint(self, load_dir, tag=None):
        import os
        if tag is None:
            with open(os.path.join(load_dir, "latest")) as f:
                tag = f.read().strip()
        ck = torch.load(os.path.join(load_dir, str(tag), "mp_rank_00_model_states.pt"), map_location="cpu", weights_only=False)
        self.module.load_state_dict(ck["module"])   # parameters are views of flat_param: refreshed in place
        self.master.copy_(ck["master"])
        self.exp_avg.copy_(ck["exp_avg"])
        self.exp_avg_sq.copy_(ck["exp_avg_sq"])
        self.global_steps = ck["global_steps"]
        YF.note_weight_write()
        return load_dir, ck.get("client_state", {})


def _tensors_of(x):
    """(container kind, {name: tensor}) of a model input: a tensor, or a BatchEncoding-like object with a dict
    `data` of tensors (the tokenizer's output, models/modeling_distributed_gpt3.py:139-178)."""
    if torch.is_tensor(x):
        return {"": x}
    if hasattr(x, "data") and isinstance(x.data, dict):
        return {k: v for k, v in x.data.items() if torch.is_tensor(v)}
    raise TypeError(f"train_step: unsupported input type {type(x).__name__}")


def graph_key(inputs):
    """Key of train_step's CUDA graphs: the library's deterministic mode (from torch.use_deterministic_algorithms;
    a graph replays the kernels of the mode it was captured under) and the input signature."""
    from . import lib
    return (lib.deterministic_mode(torch.are_deterministic_algorithms_enabled(),
                                   torch.is_deterministic_algorithms_warn_only_enabled()),) + tuple(_signature(x) for x in inputs)


def _signature(x):
    if x is None:
        return None
    # floating inputs of any dtype share one graph: their static buffer is bf16 (the copy casts)
    return tuple((k, tuple(v.shape), "float" if v.is_floating_point() else str(v.dtype)) for k, v in sorted(_tensors_of(x).items()))


def _static_like(x):
    if x is None:
        return None
    mk = lambda v: torch.empty(v.shape, device=v.device, dtype=torch.bfloat16 if v.is_floating_point() else v.dtype)  # noqa: E731
    if torch.is_tensor(x):
        return mk(x)
    return type(x)({k: (mk(v) if torch.is_tensor(v) else v) for k, v in x.data.items()})


def _copy_into(static, x):
    if x is None:
        return
    for k, v in _tensors_of(x).items():
        (static if k == "" else static.data[k]).copy_(v, non_blocking=True)


class _LazyNorm:
    """Global grad norm that only synchronises when somebody actually reads it."""

    def __init__(self, sumsq, scale):
        self._s, self._scale = sumsq, scale

    def __float__(self):
        return float(self._s.sqrt().item() * self._scale)

    def item(self):
        return float(self)

    def __repr__(self):
        return f"{float(self):.4f}"
