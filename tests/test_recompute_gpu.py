"""GPU: activation recompute (TimeSformer grad_ckpt, megatron_cfg.checkpoint_activations).

The recompute re-issues the forward kernels of one block / layer in the backward.  The forward kernels are
deterministic, so the rebuilt activations must equal the kept ones bit for bit; gradients may differ only by the
order of the fp32 atomics that accumulate weight gradients.  Also: the CUDA-graph step, the memory it saves, and the
two-GPU bucketed all-reduce with recompute on."""
import json
import os

import pytest
import torch

from oracle import port
from oracle.make_golden import make_inputs
from helpers import make_model_dir, pretrain_config

pytestmark = pytest.mark.gpu
VC, GC, Q = port.VCFG_TINY, port.GCFG_TINY, 8
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GRAD_TOL = 1e-5   # of each gradient's max |value|: fp32 split-K / LayerNorm atomics accumulate in any order


def _text(dev, **kw):
    import models.modeling_distributed_gpt3 as G
    return G.BatchEncoding({k: v.to(dev) for k, v in kw.items()})


def _model(dev, sd, grad_ckpt, ckpt_act=False, cls_name="DistributedGPT3_Pretrain", vcfg=VC, gcfg=GC, q=Q,
           dropout=(0.0, 0.0), dtype=None, **extra):
    """A task model built through its public constructor, with the two switches set the way a user sets them: grad_ckpt
    in the visual json, checkpoint_activations in megatron_cfg.  dtype None keeps fp32 parameters (fp32 .grad)."""
    os.environ["YMP_ALLOW_RANDOM_INIT"] = "1"
    import models.distributed_gpt3 as D
    td = make_model_dir(vcfg, gcfg, dropout)
    with open(os.path.join(td, "vis.json"), "w") as f:
        json.dump(dict(vcfg, pretrained_ckpt=None, grad_ckpt=grad_ckpt), f)
    mc = {"world_size": 1, "model_parallel_size": 1, "tensor_model_parallel_size": 1, "checkpoint_activations": ckpt_act}
    m = getattr(D, cls_name)(config=pretrain_config(td, q, megatron_cfg=mc, **extra), tokenizer=None)
    if sd is not None:
        _, unexpected = m.load_state_dict(sd, strict=False)
        assert not unexpected, unexpected
    m = m.to(dev)
    if dtype is not None:
        m = m.to(dtype)
    assert m.visual_encoder.vcfg["grad_ckpt"] is grad_ckpt
    assert m.text_decoder.config.engine_cfg(True)["checkpoint_activations"] is ckpt_act
    return m


def _assert_grads_close(m_on, m_off):
    off = dict(m_off.named_parameters())
    n = 0
    for k, p in m_on.named_parameters():
        q = off[k]
        if q.grad is None:
            assert p.grad is None, k
            continue
        assert p.grad is not None, k
        scale = q.grad.abs().max().item()
        err = (p.grad - q.grad).abs().max().item()
        assert err <= GRAD_TOL * scale, (k, err, scale)
        n += 1
    assert n > 0


def _assert_ctx_equal(a, b, what, vit_dims=None):
    assert set(a) == set(b), (what, set(a) ^ set(b))
    for k in a:
        if not torch.is_tensor(a[k]):
            continue
        x, y = a[k], b[k]
        if k == "lse_t":
            # temporal attention packs the T-frame groups into tiles of P rows: lse rows past R are padding that no
            # kernel writes or reads
            from ymp import ops
            n_seq, P = ops.temporal_pack(vit_dims.R, vit_dims.T)
            x, y = (t.view(n_seq, -1, P).transpose(1, 2).reshape(n_seq * P, -1)[:vit_dims.R] for t in (x, y))
        assert torch.equal(x, y), (what, k)


# ------------------------------------------------------------------------------------------ 1. bit-identical rebuilds
@pytest.mark.parametrize("vcfg", [dict(port.VCFG_CLIP_B16, depth=2, num_frames=8), VC], ids=["full_width_T8", "tiny"])
def test_vit_recomputed_block_activations_are_bit_identical(cuda, vcfg):
    from ymp import engine
    sd = port.init_state_dict(vcfg, GC, Q, seed=5, randomize=True)
    W = {k: v.to(cuda).bfloat16() for k, v in sd.items() if k.startswith(engine.VE)}
    video = torch.randn(2, 3, vcfg["num_frames"], vcfg["img_size"], vcfg["img_size"],
                        generator=torch.Generator().manual_seed(6)).to(cuda).bfloat16()
    out_res, c_res = engine.vit_fwd(W, video, vcfg, save=True)
    out_rec, c_rec = engine.vit_fwd(W, video, vcfg, save=True, recompute=True)
    assert c_rec.recompute and not c_res.recompute
    assert torch.equal(out_res, out_rec)
    for i in range(vcfg["depth"]):
        assert torch.is_tensor(c_rec.blocks[i]) and c_rec.blocks[i].dtype == torch.float32   # only the block input is kept
        _assert_ctx_equal(engine.vit_block_saved(W, c_res, i), engine.vit_block_saved(W, c_rec, i), f"block {i}", c_res.d)


@pytest.mark.parametrize("train_w", [False, True])
def test_decoder_recomputed_layer_activations_and_dgrad_are_bit_identical(cuda, train_w):
    """1.3B width, 2 layers, B = 2, S = 256, hidden and attention dropout 0.1 (train mode)."""
    from ymp import engine
    gcfg = dict(port.GCFG_1_3B, num_hidden_layers=2)
    B, S, H = 2, 256, gcfg["hidden_size"]
    g = torch.Generator(device=cuda).manual_seed(11)
    W = {}
    for i in range(2):
        pre = f"{engine.GPT}encoder.layers.{i}."
        for nm, shape in (("input_layernorm", (H,)), ("post_attention_layernorm", (H,))):
            W[pre + nm + ".weight"] = (1 + 0.1 * torch.randn(shape, device=cuda, generator=g)).bfloat16()
            W[pre + nm + ".bias"] = (0.1 * torch.randn(shape, device=cuda, generator=g)).bfloat16()
        for nm, (n, k) in (("self_attention.query_key_value", (3 * H, H)), ("self_attention.dense", (H, H)),
                           ("mlp.dense_h_to_4h", (4 * H, H)), ("mlp.dense_4h_to_h", (H, 4 * H))):
            W[pre + nm + ".weight"] = (torch.randn(n, k, device=cuda, generator=g) * k ** -0.5).bfloat16()
            W[pre + nm + ".bias"] = (0.02 * torch.randn(n, device=cuda, generator=g)).bfloat16()
    W[engine.GPT + "encoder.final_layernorm.weight"] = torch.ones(H, device=cuda).bfloat16()
    W[engine.GPT + "encoder.final_layernorm.bias"] = torch.zeros(H, device=cuda).bfloat16()
    x = torch.randn(B * S, H, device=cuda, generator=g)
    rng = torch.tensor([1234, 0], dtype=torch.int64, device=cuda)
    ctxs, hids = [], []
    for recompute in (False, True):
        hid, c = engine.gpt_fwd(W, x.clone(), gcfg, B, S, train_w=train_w, drop=engine.GptDrop(rng.clone(), 0.1, 0.1),
                                recompute=recompute)
        hids.append(hid)
        ctxs.append(c)
    assert torch.equal(hids[0], hids[1])
    for i in range(2):
        a, b = engine.gpt_layer_saved(W, ctxs[0], i), engine.gpt_layer_saved(W, ctxs[1], i)
        assert ("h" in b) is train_w and ("ln1" in b) is train_w
        _assert_ctx_equal(a, b, f"layer {i}")
        del a, b
    if train_w:
        return
    dhid = (0.1 * torch.randn(B * S, H, device=cuda, generator=g)).bfloat16()
    dx = [engine.gpt_bwd(W, {}, c, dhid) for c in ctxs]      # frozen weights: dgrad only, no atomics
    assert torch.equal(dx[0], dx[1])


# ------------------------------------------------------------------------------------------ 2. model level
def _pretrain_pair(cuda, seed=3, **kw):
    sd = port.init_state_dict(VC, GC, Q, seed=seed, randomize=True)
    return sd, [_model(cuda, sd, on, **kw) for on in (True, False)]


def test_pretrain_grad_ckpt_same_loss_and_grads(cuda):
    sd, (m_on, m_off) = _pretrain_pair(cuda)
    video, ids, att = make_inputs(2, VC, 8, GC["vocab_size"], 12)
    losses = []
    for m in (m_on, m_off):
        loss, _ = m(video.to(cuda).bfloat16(), _text(cuda, input_ids=ids, attention_mask=att))
        loss.backward()
        losses.append(loss.detach())
    assert torch.equal(losses[0], losses[1])
    _assert_grads_close(m_on, m_off)


def test_pretrain_grad_ckpt_matches_reference_fixture(cuda):
    """tiny_pretrain.pt at the thresholds of test_model_gpu.py::test_fused_pretrain_matches_reference_fixture."""
    fx = torch.load(os.path.join(GOLD, "tiny_pretrain.pt"), weights_only=False)
    sd = port.init_state_dict(fx["vcfg"], fx["gcfg"], fx["Q"], seed=fx["wseed"], randomize=fx["randomize"])
    m = _model(cuda, sd, True, vcfg=fx["vcfg"], gcfg=fx["gcfg"], q=fx["Q"], dtype=torch.bfloat16)
    video, ids, att = make_inputs(fx["B"], fx["vcfg"], fx["L"], fx["gcfg"]["vocab_size"], fx["iseed"])
    loss, _ = m(video.to(cuda).bfloat16(), _text(cuda, input_ids=ids, attention_mask=att))
    loss.backward()
    Q_ = fx["Q"]

    def rel(a, b):
        return ((a.float().cpu() - b.float().cpu()).abs().max() / (b.float().abs().max() + 1e-12)).item()

    assert abs(loss.item() - fx["loss"].item()) < 1e-2 * abs(fx["loss"].item())
    assert rel(m.last_losses[:, Q_:-1], fx["losses"][:, Q_:]) < 2e-2
    train = set(port.trainable_keys(sd))
    psd = {k: v.bfloat16().float().requires_grad_(k in train) for k, v in sd.items()}
    res = port.pretrain_forward(video.bfloat16().float(), ids, att, psd, fx["vcfg"], fx["gcfg"], return_all=True)
    res["loss"].backward()
    assert abs(loss.item() - res["loss"].item()) < 5e-3 * abs(res["loss"].item())
    for k, p in m.named_parameters():
        if k.startswith("text_decoder."):
            assert p.grad is None, k
            continue
        if psd[k].grad.abs().max().item() < 1e-7:
            continue
        assert rel(p.grad, psd[k].grad) < 6e-2, k
    for k, (stride, vals) in fx["grads"].items():
        g = dict(m.named_parameters())[k].grad.float().cpu().flatten()[::stride]
        if vals.abs().max() > 1e-7:
            assert rel(g, vals) < 8e-2, k


# ------------------------------------------------------------------------------------------ 3. downstream, both switches
def _head_sd(n_out, seed=21):
    sd = port.init_state_dict(VC, GC, Q, seed=seed, randomize=True)
    g = torch.Generator().manual_seed(seed + 1)
    for k, shape in (("cls_head.0.weight", (128, 128)), ("cls_head.0.bias", (128,)), ("cls_head.2.weight", (n_out, 128)),
                     ("cls_head.2.bias", (n_out,))):
        sd[k] = 0.05 * torch.randn(shape, generator=g)
    return sd


def test_retrieval_cls_with_both_switches(cuda):
    sd = _head_sd(2)
    ms = [_model(cuda, sd, on, on, cls_name="DistributedGPT3_Retrieval_Cls", num_frames=VC["num_frames"], use_cls=True,
                 dropout=(0.1, 0.1)) for on in (True, False)]
    B, L = 2, 8
    video, _, _ = make_inputs(B, VC, L, GC["vocab_size"], 51)
    _, ids, att = make_inputs(3 * B, VC, L, GC["vocab_size"], 52)      # positives, then two negatives per video
    text = _text(cuda, input_ids=ids, attention_mask=att, prompt_lengths=torch.tensor([2, 2, 3, 1, 2, 3]))
    prompt = _text(cuda, input_ids=ids, attention_mask=att)
    neg = torch.tensor([1, 0, 1, 0], device=cuda)
    labels = torch.tensor([1, 1, 0, 0, 0, 0], device=cuda)
    out = []
    for m in ms:
        from ymp import functional as YF
        YF.set_dropout_seed(77, cuda)                 # same dropout masks for both models
        m.train()
        lc, lcls = m(video.to(cuda).bfloat16(), text, prompt, neg, labels, train=True)
        (lc + lcls).backward()
        out.append((lc.detach(), lcls.detach()))
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])
    _assert_grads_close(*ms)


def test_caption_with_both_switches_dropout(cuda):
    sd = port.init_state_dict(VC, GC, Q, seed=8, randomize=True)
    ms = [_model(cuda, sd, on, on, cls_name="DistributedGPT3_Caption", num_frames=VC["num_frames"], dropout=(0.1, 0.1))
          for on in (True, False)]
    video, ids, att = make_inputs(2, VC, 8, GC["vocab_size"], 61)
    text = _text(cuda, input_ids=ids, attention_mask=att, prompt_lengths=torch.tensor([2, 3]))
    losses = []
    for m in ms:
        from ymp import functional as YF
        YF.set_dropout_seed(78, cuda)
        m.train()
        loss = m(video.to(cuda).bfloat16(), text)
        loss.backward()
        losses.append(loss.detach())
    assert torch.equal(losses[0], losses[1])
    _assert_grads_close(*ms)


# ------------------------------------------------------------------------------------------ 4. CUDA graph
def test_graph_train_step_with_recompute_equals_eager_loop(cuda):
    """The criterion of test_train_gpu.py::test_graph_train_step_equals_eager_loop, both switches on."""
    from ymp.train import TrainEngine
    lr = 1e-3
    sd = port.init_state_dict(VC, GC, Q, seed=3, randomize=True)
    eng_g = TrainEngine(_model(cuda, sd, True, True, dtype=torch.bfloat16), lr=lr)
    eng_e = TrainEngine(_model(cuda, sd, True, True, dtype=torch.bfloat16), lr=lr)
    losses_g, losses_e = [], []
    for i in range(4):
        video, ids, att = make_inputs(2, VC, 8, GC["vocab_size"], 100 + i)
        video, text = video.to(cuda).bfloat16(), _text(cuda, input_ids=ids, attention_mask=att)
        losses_g.append(eng_g.train_step(video, text, use_graph=True, graph_warmup=1).item())
        loss, zero = eng_e(video, text)
        eng_e.backward(loss + zero)
        eng_e.step()
        losses_e.append(loss.item())
    assert any("graph" in st for st in eng_g._graphs.values())
    for a, b in zip(losses_g, losses_e):
        assert abs(a - b) <= 1e-3 * abs(b), (losses_g, losses_e)
    assert losses_e[0] != losses_e[1]
    d = (eng_g.master - eng_e.master).abs()
    assert (d > 0.05 * lr).float().mean().item() < 2e-3
    assert d.max().item() <= 2.0 * lr * 4
    assert eng_g.global_steps == eng_e.global_steps == 4
    assert float(eng_g.flat_grad.abs().max()) == 0.0
    gn_g, gn_e = float(eng_g.optimizer._global_grad_norm), float(eng_e.optimizer._global_grad_norm)
    assert abs(gn_g - gn_e) <= 2e-2 * gn_e


# ------------------------------------------------------------------------------------------ 5. memory
def _growth(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def test_vit_recompute_memory(cuda):
    """Full-width 12-block ViT, 8 frames, B = 2, tiny decoder: 1.50 GB of block activations resident against 0.12 GB of
    block inputs plus one rebuilt block (0.13 GB).  Gradients go to the engine's preallocated flat buffer."""
    from ymp.train import TrainEngine
    vcfg = dict(port.VCFG_CLIP_B16, num_frames=8)
    video, ids, att = make_inputs(2, vcfg, 8, GC["vocab_size"], 71)
    video, text = video.to(cuda).bfloat16(), _text(cuda, input_ids=ids, attention_mask=att)
    growth = {}
    for on in (False, True):
        eng = TrainEngine(_model(cuda, None, on, vcfg=vcfg, dtype=torch.bfloat16), lr=1e-4)

        def step():
            loss, _ = eng(video, text)
            eng.backward(loss)

        step()   # warm-up: lazily built tables and caches are not activations
        eng.zero_grad()
        growth[on] = _growth(step)
        del eng, step
        torch.cuda.empty_cache()
    print("ViT fwd+bwd peak growth (bytes): resident", growth[False], "recompute", growth[True])
    assert growth[True] <= 0.4 * growth[False], growth


def test_decoder_recompute_memory(cuda):
    """1.3B-width 4-layer frozen decoder, B = 8, S = 208, through gpt_fwd / gpt_bwd."""
    from ymp import engine
    gcfg = dict(port.GCFG_1_3B, num_hidden_layers=4)
    B, S, H = 8, 208, gcfg["hidden_size"]
    g = torch.Generator(device=cuda).manual_seed(3)
    W = {}
    for i in range(4):
        pre = f"{engine.GPT}encoder.layers.{i}."
        for nm in ("input_layernorm", "post_attention_layernorm"):
            W[pre + nm + ".weight"] = torch.ones(H, device=cuda).bfloat16()
            W[pre + nm + ".bias"] = torch.zeros(H, device=cuda).bfloat16()
        for nm, (n, k) in (("self_attention.query_key_value", (3 * H, H)), ("self_attention.dense", (H, H)),
                           ("mlp.dense_h_to_4h", (4 * H, H)), ("mlp.dense_4h_to_h", (H, 4 * H))):
            W[pre + nm + ".weight"] = (torch.randn(n, k, device=cuda, generator=g) * k ** -0.5).bfloat16()
            W[pre + nm + ".bias"] = torch.zeros(n, device=cuda).bfloat16()
    W[engine.GPT + "encoder.final_layernorm.weight"] = torch.ones(H, device=cuda).bfloat16()
    W[engine.GPT + "encoder.final_layernorm.bias"] = torch.zeros(H, device=cuda).bfloat16()
    x0 = torch.randn(B * S, H, device=cuda, generator=g)
    dhid = (0.1 * torch.randn(B * S, H, device=cuda, generator=g)).bfloat16()
    growth = {}
    for recompute in (False, True):
        x = x0.clone()

        def step():
            c = engine.gpt_fwd(W, x, gcfg, B, S, recompute=recompute)[1]
            engine.gpt_bwd(W, {}, c, dhid)

        step()
        growth[recompute] = _growth(step)
    print("decoder fwd+bwd peak growth (bytes): resident", growth[False], "recompute", growth[True])
    assert growth[True] <= 0.5 * growth[False], growth


# ------------------------------------------------------------------------------------------ 6. two GPUs
def _dp_worker(rank, world, port_no, q):
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
        from ymp.train import TrainEngine
        res = {}
        sd = port.init_state_dict(VC, GC, Q, seed=3, randomize=True)
        video, ids, att = make_inputs(2 * world, VC, 8, GC["vocab_size"], 77)
        video = video.to(dev).bfloat16()
        shard = lambda r: (video[2 * r:2 * r + 2], _text(dev, input_ids=ids[2 * r:2 * r + 2], attention_mask=att[2 * r:2 * r + 2]))  # noqa: E731
        eng = TrainEngine(_model(dev, sd, True, dtype=torch.bfloat16), lr=1e-3, overlap_comm=True)
        loss, _ = eng(*shard(rank))
        eng.backward(loss)
        eng.allreduce_gradients()
        got = eng.flat_grad.clone() / world
        single = TrainEngine(_model(dev, sd, True, dtype=torch.bfloat16), lr=1e-3, overlap_comm=False)
        single.world = 1
        for r in range(world):
            l, _ = single(*shard(r))
            single.backward(l)
        ref = single.flat_grad / world
        res["dp_grad"] = (got - ref).abs().max().item() / ref.abs().max().item()
        res["buckets"] = len(eng._buckets)
        eng = TrainEngine(_model(dev, sd, True, dtype=torch.bfloat16), lr=1e-3, overlap_comm=True)
        for i in range(4):
            v, i2, a2 = make_inputs(2, VC, 8, GC["vocab_size"], 500 + 10 * i + rank)
            eng.train_step(v.to(dev).bfloat16(), _text(dev, input_ids=i2, attention_mask=a2), use_graph=True, graph_warmup=1)
        flat = eng.master.clone()
        other = [torch.empty_like(flat) for _ in range(world)]
        dist.all_gather(other, flat)
        res["replicas_identical"] = bool(all(torch.equal(o, other[0]) for o in other))
        res["graph_used"] = any("graph" in st for st in eng._graphs.values())
        q.put((rank, res))
    finally:
        dist.destroy_process_group()


def test_two_gpu_grad_ckpt_bucketed_allreduce(cuda):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import socket
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port_no = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_dp_worker, args=(r, 2, port_no, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=600) for _ in procs]
    for p in procs:
        p.join(timeout=120)
    for rank, r in res:
        assert r["dp_grad"] < 2e-2, r
        assert r["replicas_identical"] and r["graph_used"], r
