"""GPU: the deterministic mode (torch.use_deterministic_algorithms(True) -> ymp_set_deterministic).

1. Split-K GEMM: the wgrad shapes of the step at split_k 2, 3, 4, 8 and the library's choice, into a non-zero fp32
   destination, at each tile shape: bit for bit ((D + P0) + P1) + ..., P_k the split_k = 1 product over slice k's
   k-blocks (the kernel's kb_per_split partition), summed in fp32 in slice order; within the float64 bound of
   gemm_bounds.py; three calls equal.
2. LayerNorm gamma / beta gradients, colsum, sumsq: bit for bit the per-block arithmetic of misc_bounds.py's simulators
   combined in block order, and within their bounds.  The simulators add the block partials in a shuffled order (the
   atomics); here torch.randperm is replaced by the identity while they run.  dgamma and sumsq accumulate with fused
   multiply-adds on the device (dg = fma(dy, xh, dg); per four-element group fma(x, x, y y) then z, w), which the
   simulators, written for bounds, round separately: those two partials are restated below with the fma.
3. Training steps: two runs from one state give equal loss, flat gradient, master weights, Adam moments and logged grad
   norm (pre-training at the tiny and at ViT-B / 1.3B widths, dropout with recompute, the CUDA-graph train_step,
   gradient accumulation, Retrieval_Cls with checkpoint_activations, the contrastive Retrieval model).
4. The mode-on step is within the atomics tolerance of the mode-off step on the same inputs.
"""
import json
import os

import pytest
import torch

import gemm_bounds as GB
import misc_bounds as MB
from helpers import make_model_dir, pretrain_config
from oracle import port
from oracle.make_golden import make_inputs

# cuBLAS (the contrastive head's matmuls) is deterministic with a fixed workspace configuration (PyTorch's
# reproducibility notes); torch raises under use_deterministic_algorithms without it
os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")

pytestmark = pytest.mark.gpu
bf16, f32 = torch.bfloat16, torch.float32
VC, GC, Q = port.VCFG_TINY, port.GCFG_TINY, 8
VC_VITB = dict(VC, img_size=64, embed_dim=768, num_heads=12, depth=2)
GC_1P3B = dict(port.GCFG_1_3B, vocab_size=512, num_hidden_layers=2, max_position_embeddings=64)
GRAD_TOL = 1e-5   # of each gradient's max |value|, as test_recompute_gpu.py: sums reordered


@pytest.fixture
def deterministic():
    from ymp import lib
    prev = (torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled())
    torch.use_deterministic_algorithms(True)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(prev[0], warn_only=prev[1])
        lib.sync_deterministic()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _bits_equal(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _cdiv(a, b):
    return -(-a // b)


# ------------------------------------------------------------------------------------------ 1. split-K GEMM
# (M, N) of dW = dy^T x: ViT-B qkv, proj, fc1, fc2; abstractor 1024 x 1024; visual_fc 2048 x 1024
WGRAD = [(2304, 768), (768, 768), (3072, 768), (768, 3072), (1024, 1024), (2048, 1024)]
TILES = [(128, 128), (128, 256), (192, 256)]   # (tile_m, tile_n): every tile the planner can give a wgrad launch


@pytest.mark.parametrize("M,N", WGRAD)
@pytest.mark.parametrize("K", [3152, 8192])   # 16 x 197 tokens (ragged last k-block), 128 k-blocks
def test_split_k_gemm_fixed_order(cuda, deterministic, monkeypatch, M, N, K):
    from ymp import lib as L
    from ymp import ops
    g = torch.Generator(device=cuda).manual_seed(M + N + K)
    dy = torch.randn(K, M, device=cuda, generator=g).to(bf16)
    x = torch.randn(K, N, device=cuda, generator=g).to(bf16)
    d0 = torch.randn(M, N, device=cuda, generator=g) * 4
    ref = GB.reference(dy.T, x.T, d0=d0)
    asked = []
    alloc = L.workspace
    monkeypatch.setattr(L, "workspace", lambda nbytes, device: (asked.append(nbytes), alloc(nbytes, device))[1])
    kb_total = _cdiv(K, 64)
    for tile_m, tile_n in TILES:
        for split_k in (2, 3, 4, 8, 0):
            outs = []
            for _ in range(3):
                asked.clear()
                d = d0.clone()
                ops.gemm(dy, x, a_t=True, b_t=True, out=d, accumulate=True, split_k=split_k, tile_m=tile_m, tile_n=tile_n)
                outs.append(d)
            what = f"M={M} N={N} K={K} tile={tile_m}x{tile_n} split_k={split_k}"
            assert asked and asked[0] % (M * N * 4) == 0, what
            split = asked[0] // (M * N * 4)          # the launch's K slices (the library's choice for split_k = 0)
            assert split_k == 0 or split == split_k, what
            assert all(_bits_equal(outs[0], o) for o in outs[1:]), what + ": three calls differ"
            want = d0.clone()
            if split:
                per = _cdiv(kb_total, split)
                for k in range(split):
                    r0, r1 = k * per * 64, min(K, (k + 1) * per * 64)
                    p = torch.zeros(M, N, device=cuda)
                    ops.gemm(dy[r0:r1], x[r0:r1], a_t=True, b_t=True, out=p, accumulate=True, split_k=1,
                             tile_m=tile_m, tile_n=tile_n)
                    want = want + p
            else:
                ops.gemm(dy, x, a_t=True, b_t=True, out=want, accumulate=True, split_k=1, tile_m=tile_m, tile_n=tile_n)
            assert _bits_equal(outs[0], want), what + ": not ((D + P0) + P1) + ..."
            e_out, _ = GB.bounds(ref, K, split=max(split, 1), out_bf16=False)
            assert GB.worst_ratio(outs[0], ref["out"], e_out) <= 1, what


# ------------------------------------------------------------------------------------------ 2. reductions
@pytest.fixture
def block_order(monkeypatch):
    """The simulators' shuffled block order replaced by the block index."""
    monkeypatch.setattr(torch, "randperm", lambda n, generator=None: torch.arange(n))


def _fma(a, b, c):
    return MB._fma(a, b, c)


def _ln_wgrad_block_order(dy, x, mean, rstd, dgamma0, dbeta0, blocks):
    """ln_bwd_kernel's dgamma (fma) and dbeta per block, added to dgamma0 / dbeta0 in block order."""
    dy, x = dy.float().cpu(), x.float().cpu()
    xh = (x - mean.float().cpu()[:, None]) * rstd.float().cpu()[:, None]
    rows, D = x.shape
    nw = MB.LN_WARPS * blocks
    passes = _cdiv(rows, nw)
    pdy, pxh = torch.zeros(passes * nw, D), torch.zeros(passes * nw, D)
    pdy[:rows], pxh[:rows] = dy, xh
    ag, ab = torch.zeros(nw, D), torch.zeros(nw, D)
    for k in range(passes):
        s = slice(k * nw, (k + 1) * nw)
        ag = _fma(pdy[s], pxh[s], ag)
        ab = ab + pdy[s]
    out = []
    for acc, init in ((ag, dgamma0), (ab, dbeta0)):
        acc = acc.view(blocks, MB.LN_WARPS, D)
        part = torch.zeros(blocks, D)
        for w in range(MB.LN_WARPS):
            part = part + acc[:, w]
        o = init.float().cpu().clone()
        for b in range(blocks):
            o = o + part[b]
        out.append(o)
    return out


def _sumsq_block_order(g, out0, sms):
    """sumsq_kernel with its fmas (t = fma(x, x, y y), then z, then w; the tail fma(g, g, acc)), blocks in order."""
    g = g.float().cpu()
    n = g.numel()
    B = MB.sumsq_blocks(n, sms)
    nt, n4 = B * 256, n // 4
    k = _cdiv(n4, nt)
    v = torch.zeros(k * nt, 4)
    v[:n4] = g[:n4 * 4].view(n4, 4)
    acc = torch.zeros(nt)
    for i in range(k):
        c = v[i * nt:(i + 1) * nt]
        t = c[:, 1] * c[:, 1]
        for e in (0, 2, 3):
            t = _fma(c[:, e], c[:, e], t)
        acc = acc + t
    for j in range(n4 * 4, n):
        acc[j - n4 * 4] = _fma(g[j], g[j], acc[j - n4 * 4])
    w = MB._butterfly(acc.view(B, 8, 32))
    idx = torch.arange(8)
    for o in (4, 2, 1):
        w = w + w[:, idx ^ o]
    out = torch.tensor(float(out0), dtype=f32)
    for b in range(B):
        out = out + w[b, 0]
    return out


@pytest.mark.parametrize("D", [768, 1024, 2048, 2560])
@pytest.mark.parametrize("rows", [3000, 9001])
def test_layernorm_wgrad_fixed_order(cuda, deterministic, block_order, D, rows):
    from ymp import ops
    g = torch.Generator(device=cuda).manual_seed(D + rows)
    x = (torch.randn(rows, D, device=cuda, generator=g) * 2 + 1).to(bf16)
    gamma = (1 + 0.5 * torch.randn(D, device=cuda, generator=g)).to(bf16)
    beta = (0.5 * torch.randn(D, device=cuda, generator=g)).to(bf16)
    dy = torch.randn(rows, D, device=cuda, generator=g).to(bf16)
    _, mean, rstd = ops.layernorm_fwd(x, gamma, beta, 1e-5)
    dg0 = torch.randn(D, device=cuda, generator=g) * 10
    db0 = dg0.flip(0).clone()
    got = []
    for _ in range(3):
        dg, db = dg0.clone(), db0.clone()
        dx = ops.layernorm_bwd(dy, x, gamma, mean, rstd, dgamma=dg, dbeta=db)
        got.append((dg, db, dx))
    for dg, db, dx in got[1:]:
        assert _bits_equal(dg, got[0][0]) and _bits_equal(db, got[0][1]) and torch.equal(dx, got[0][2])
    dg, db, _ = got[0]
    blocks = MB.ln_bwd_blocks(rows, D, _sms())
    want_g, want_b = _ln_wgrad_block_order(dy, x, mean, rstd, dg0, db0, blocks)
    sim = MB.simulate_ln_bwd(dy.cpu(), x.cpu(), gamma.cpu(), mean.cpu(), rstd.cpu(), dgamma0=dg0.cpu(), dbeta0=db0.cpu(),
                             blocks=blocks)
    assert _bits_equal(sim["dbeta"], want_b)
    assert _bits_equal(dg.cpu(), want_g), f"dgamma D={D} rows={rows}"
    assert _bits_equal(db.cpu(), want_b), f"dbeta D={D} rows={rows}"
    ref = MB.ln_bwd_reference(dy, x, gamma, mean.double(), rstd.double(), dgamma0=dg0, dbeta0=db0)
    b = MB.ln_bwd_bounds(ref, blocks, rows=rows)
    assert MB.worst_ratio(dg, ref["dgamma"], b["dgamma"]) <= 1
    assert MB.worst_ratio(db, ref["dbeta"], b["dbeta"]) <= 1


@pytest.mark.parametrize("D", [768, 2560])
@pytest.mark.parametrize("xdt", [bf16, f32])
def test_layernorm_bwd_dx_same_in_both_modes(cuda, D, xdt):
    """ln_bwd_partial_kernel (mode on) is a copy of ln_bwd_kernel with another final store: dx (with the skip gradient
    added) and dx_drop must be bit-identical to the mode-off kernel's, and dgamma / dbeta within reordering."""
    from ymp import lib, ops
    g = torch.Generator(device=cuda).manual_seed(D + 7)
    rows = 5000
    x = (torch.randn(rows, D, device=cuda, generator=g) * 2 + 1).to(xdt)
    gamma = (1 + 0.5 * torch.randn(D, device=cuda, generator=g)).to(bf16)
    beta = (0.5 * torch.randn(D, device=cuda, generator=g)).to(bf16)
    dy = torch.randn(rows, D, device=cuda, generator=g).to(bf16)
    add = torch.randn(rows, D, device=cuda, generator=g).to(bf16)
    _, mean, rstd = ops.layernorm_fwd(x, gamma, beta, 1e-5)
    rng = torch.tensor([0x1234567812345, 7], dtype=torch.int64, device=cuda)
    out = {}
    for on in (False, True):
        torch.use_deterministic_algorithms(on)
        try:
            dg, db = torch.zeros(D, device=cuda), torch.zeros(D, device=cuda)
            dx, dxd = ops.layernorm_bwd(dy, x, gamma, mean, rstd, add=add, dgamma=dg, dbeta=db, drop=ops.Drop(rng, 3, 0.1))
            dx_plain = ops.layernorm_bwd(dy, x, gamma, mean, rstd, dgamma=torch.zeros(D, device=cuda),
                                         dbeta=torch.zeros(D, device=cuda))
        finally:
            torch.use_deterministic_algorithms(False)
            lib.sync_deterministic()
        out[on] = (dx, dxd, dx_plain, dg, db)
    for i, name in enumerate(("dx", "dx_drop", "dx without add / dropout")):
        assert torch.equal(out[False][i].view(torch.int16), out[True][i].view(torch.int16)), f"{name} D={D} {xdt}"
    for i in (3, 4):
        a, b = out[False][i], out[True][i]
        assert float((a - b).abs().max()) <= 1e-5 * float(a.abs().max())


@pytest.mark.parametrize("Cc", [768, 1024, 2048, 2560])
@pytest.mark.parametrize("R", [4096, 50208])
def test_colsum_fixed_order(cuda, deterministic, block_order, R, Cc):
    from ymp import ops
    g = torch.Generator(device=cuda).manual_seed(R + Cc)
    x = torch.randn(R, Cc, device=cuda, generator=g).to(bf16)
    out0 = torch.randn(Cc, device=cuda, generator=g) * 10
    got = [ops.colsum(x, out0.clone()) for _ in range(3)]
    assert all(_bits_equal(o, got[0]) for o in got[1:])
    _, splits, _ = MB.colsum_grid(R, Cc, _sms())
    assert splits > 1
    want = MB.simulate_colsum(x.cpu(), out0.cpu(), _sms())
    assert _bits_equal(got[0].cpu(), want), f"colsum {R}x{Cc}"
    assert MB.worst_ratio(got[0], out0.double() + x.double().sum(0), MB.colsum_bound(x, out0, _sms())) <= 1


@pytest.mark.parametrize("n", [4097, 5 * 2 ** 20 + 3])
def test_sumsq_fixed_order(cuda, deterministic, n):
    from ymp import ops
    g = torch.Generator(device=cuda).manual_seed(n)
    x = torch.randn(n, device=cuda, generator=g)
    out0 = 3.25
    got = [ops.sumsq(x, torch.full((1,), out0, device=cuda)) for _ in range(3)]
    assert all(_bits_equal(o, got[0]) for o in got[1:])
    assert MB.sumsq_blocks(n, _sms()) > 1
    want = _sumsq_block_order(x, out0, _sms())
    assert _bits_equal(got[0].cpu(), want[None]), f"sumsq n={n}: {got[0].item()!r} != {want.item()!r}"
    assert MB.worst_ratio(got[0], (out0 + (x.double() ** 2).sum())[None], MB.sumsq_bound(x, out0, _sms())[None]) <= 1


# ------------------------------------------------------------------------------------------ 3. training steps
def _text(dev, **kw):
    import models.modeling_distributed_gpt3 as G
    return G.BatchEncoding({k: v.to(dev) for k, v in kw.items()})


def _model(dev, sd, vcfg=VC, gcfg=GC, cls_name="DistributedGPT3_Pretrain", grad_ckpt=False, ckpt_act=False,
           dropout=(0.0, 0.0), **extra):
    os.environ["YMP_ALLOW_RANDOM_INIT"] = "1"
    import models.distributed_gpt3 as D
    td = make_model_dir(vcfg, gcfg, dropout)
    with open(os.path.join(td, "vis.json"), "w") as f:
        json.dump(dict(vcfg, pretrained_ckpt=None, grad_ckpt=grad_ckpt), f)
    mc = {"world_size": 1, "model_parallel_size": 1, "tensor_model_parallel_size": 1, "checkpoint_activations": ckpt_act}
    m = getattr(D, cls_name)(config=pretrain_config(td, Q, megatron_cfg=mc, **extra), tokenizer=None)
    _, unexpected = m.load_state_dict(sd, strict=False)
    assert not unexpected, unexpected
    return m.to(dev).to(bf16)


def _sd(vcfg, gcfg, extra=None, seed=21):
    sd = port.init_state_dict(vcfg, gcfg, Q, seed=seed, randomize=True)
    g = torch.Generator().manual_seed(seed + 1)
    for k, shape in (extra or {}).items():
        sd[k] = 0.05 * torch.randn(shape, generator=g)
    return sd


def _pretrain_inputs(dev, vcfg, gcfg):
    def inputs(i):
        video, ids, att = make_inputs(2, vcfg, 8, gcfg["vocab_size"], 100 + i)
        return video.to(dev).bfloat16(), _text(dev, input_ids=ids, attention_mask=att)
    return inputs


def _retrieval_cls_inputs(dev):
    def inputs(i):
        B, L = 2, 8
        video, _, _ = make_inputs(B, VC, L, GC["vocab_size"], 51 + i)
        _, ids, att = make_inputs(3 * B, VC, L, GC["vocab_size"], 52 + i)
        text = _text(dev, input_ids=ids, attention_mask=att, prompt_lengths=torch.tensor([2, 2, 3, 1, 2, 3]))
        prompt = _text(dev, input_ids=ids, attention_mask=att)
        return (video.to(dev).bfloat16(), text, prompt, torch.tensor([1, 0, 1, 0], device=dev),
                torch.tensor([1, 1, 0, 0, 0, 0], device=dev))
    return inputs


def _retrieval_inputs(dev):
    def inputs(i):
        video, ids, att = make_inputs(3, VC, 8, GC["vocab_size"], 41 + i)
        return video.to(dev).bfloat16(), _text(dev, input_ids=ids, attention_mask=att), torch.tensor([7, 9, 7], device=dev)
    return inputs


def _case(name, dev):
    """(model factory, inputs(i), kwargs of the model call, run options)."""
    if name in ("tiny", "tiny_graph", "tiny_gas2", "tiny_dropout_ckpt"):
        sd = _sd(VC, GC)
        kw = dict(grad_ckpt=True, ckpt_act=True, dropout=(0.1, 0.1)) if name == "tiny_dropout_ckpt" else {}
        return (lambda: _model(dev, sd, **kw)), _pretrain_inputs(dev, VC, GC), {}, \
            dict(graph=name == "tiny_graph", gas=2 if name == "tiny_gas2" else 1, dropout=name == "tiny_dropout_ckpt")
    if name == "vitb_1p3b":
        sd = _sd(VC_VITB, GC_1P3B)
        return (lambda: _model(dev, sd, VC_VITB, GC_1P3B)), _pretrain_inputs(dev, VC_VITB, GC_1P3B), {}, {}
    if name == "retrieval_cls_ckpt":
        sd = _sd(VC, GC, {"cls_head.0.weight": (128, 128), "cls_head.0.bias": (128,), "cls_head.2.weight": (2, 128),
                          "cls_head.2.bias": (2,)})
        return (lambda: _model(dev, sd, cls_name="DistributedGPT3_Retrieval_Cls", ckpt_act=True, num_frames=VC["num_frames"],
                               use_cls=True)), _retrieval_cls_inputs(dev), dict(train=True), {}
    if name == "retrieval":
        sd = _sd(VC, GC, {"vision_proj.weight": (32, 192), "vision_proj.bias": (32,), "text_proj.weight": (32, 128),
                          "text_proj.bias": (32,)})
        sd["temp"] = torch.tensor(0.07)
        return (lambda: _model(dev, sd, cls_name="DistributedGPT3_Retrieval", num_frames=VC["num_frames"],
                               contrastive_embed_dim=32)), _retrieval_inputs(dev), {}, {}
    raise KeyError(name)


def _total(out):
    return sum(out[1:], out[0]) if isinstance(out, (tuple, list)) else out


def _run(dev, make, inputs, call_kw, graph=False, gas=1, dropout=False, steps=3):
    """Steps from the model's initial state: {loss, grad (eager: the flat gradient before AdamW consumes it), norm (the
    logged grad norm's sum of squares)} of every step, then the master weights and both Adam moments."""
    from ymp import functional as YF
    from ymp.train import TrainEngine
    eng = TrainEngine(make(), lr=1e-3, gradient_accumulation_steps=gas)
    eng.train()
    rec = []
    for i in range(steps):
        if graph:
            rec.append(("loss", eng.train_step(*inputs(i), use_graph=True, graph_warmup=1).clone()))
        else:
            for mi in range(gas):
                if dropout:
                    YF.set_dropout_seed(77 + i * gas + mi, dev)
                loss = _total(eng(*inputs(i * gas + mi), **call_kw))
                eng.backward(loss)
                rec.append(("loss", loss.detach().clone()))
            rec.append(("grad", eng.flat_grad.clone()))
            eng.step()
        rec.append(("norm", eng.optimizer._global_grad_norm._s.clone()))
    if graph:
        assert any("graph" in st for st in eng._graphs.values())
    return rec + [("master", eng.master.clone()), ("m", eng.exp_avg.clone()), ("v", eng.exp_avg_sq.clone())]


CASES = ["tiny", "tiny_graph", "tiny_gas2", "tiny_dropout_ckpt", "vitb_1p3b", "retrieval_cls_ckpt", "retrieval"]


@pytest.mark.parametrize("name", CASES)
def test_training_step_is_reproducible(cuda, deterministic, name):
    make, inputs, call_kw, opts = _case(name, cuda)
    a = _run(cuda, make, inputs, call_kw, **opts)
    b = _run(cuda, make, inputs, call_kw, **opts)
    assert [k for k, _ in a] == [k for k, _ in b]
    for i, ((k, x), (_, y)) in enumerate(zip(a, b)):
        assert torch.isfinite(x).all(), f"{name}: {k} (record {i}) not finite"
        assert torch.equal(x, y), f"{name}: {k} (record {i}) differs between two runs"


@pytest.mark.parametrize("name", ["tiny", "tiny_graph", "retrieval"])
def test_mode_on_matches_mode_off(cuda, name):
    """Same inputs, same initial state: the deterministic steps stay within the tolerances test_recompute_gpu.py gives
    steps whose fp32 sums are reordered (the first gradient within GRAD_TOL; after an AdamW step the weights differ by
    up to lr where an update's sign flips, and the later gradients and moments with them)."""
    from ymp import lib
    make, inputs, call_kw, opts = _case(name, cuda)
    off = _run(cuda, make, inputs, call_kw, **opts)
    torch.use_deterministic_algorithms(True)
    try:
        on = _run(cuda, make, inputs, call_kw, **opts)
    finally:
        torch.use_deterministic_algorithms(False)
        lib.sync_deterministic()
    lr, steps, grads = 1e-3, 3, 0
    for (k, x), (_, y) in zip(off, on):
        d, scale = (x - y).abs(), float(x.abs().max())
        if k == "loss":
            assert float(d) <= 1e-3 * abs(float(x)), (name, k, float(x), float(y))
        elif k == "norm":
            assert float(d) <= 4e-2 * float(x), (name, k, float(x), float(y))
        elif k == "grad":
            assert float(d.max()) <= (GRAD_TOL if grads == 0 else 2e-2) * scale, (name, k, grads)
            grads += 1
        elif k == "master":
            assert (d > 0.05 * lr).float().mean().item() < 2e-3 and d.max().item() <= 2.0 * lr * steps, name
        else:
            assert float(d.max()) <= 5e-2 * scale, (name, k)


def _dp_det_worker(rank, world, port_no, q):
    """One rank of the two-GPU data-parallel setup of test_train_gpu.py, deterministic mode on: the CUDA-graph step
    (the bucketed all-reduces captured in the graph) run twice from one state on this rank's own batches."""
    import sys
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port_no), RANK=str(rank), WORLD_SIZE=str(world),
                      YMP_ALLOW_RANDOM_INIT="1")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for p in (root, os.path.join(root, "youku-mplug_b200"), os.path.join(root, "tests")):
        if p not in sys.path:
            sys.path.insert(0, p)
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        torch.use_deterministic_algorithms(True)
        make, inputs, call_kw, opts = _case("tiny_graph", dev)
        runs = [_run(dev, make, lambda i: inputs(i + 100 * rank), call_kw, **opts) for _ in range(2)]
        diff = [k for (k, x), (_, y) in zip(*runs) if not torch.equal(x, y)]
        master = runs[0][-3][1]
        other = [torch.empty_like(master) for _ in range(world)]
        dist.all_gather(other, master)
        q.put((rank, dict(diff=diff, records=len(runs[0]), replicas=all(torch.equal(o, other[0]) for o in other))))
    finally:
        dist.destroy_process_group()


def test_two_gpu_training_step_is_reproducible(cuda):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    from test_train_gpu import _free_port
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port_no = _free_port()
    procs = [ctx.Process(target=_dp_det_worker, args=(r, 2, port_no, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=900) for _ in procs]
    for p in procs:
        p.join(timeout=120)
    for rank, r in res:
        assert r["records"] > 0 and not r["diff"], (rank, r)
        assert r["replicas"], (rank, r)
