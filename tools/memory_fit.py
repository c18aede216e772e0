"""Peak device memory of the shipped training configs at their own per-GPU batch, and the cost of ViT recompute.

    python tools/memory_fit.py [--configs caption/caption_gpt3_2.7B_youku_v0.yaml ...] [--iters 2]
    python tools/memory_fit.py --compare [--rounds 3] [--steps 5]

Main mode: for each training yaml under youku-mplug_b200/configs/ (the ten the task scripts run), build the model
class its script builds with random bf16 weights (the decoder's dropout at the reference default 0.1, train mode), the
vis json's grad_ckpt and the yaml's megatron_cfg, and run `--iters` eager iterations of model(...) ->
TrainEngine.backward -> step on synthetic inputs at the yaml's batch_size, frame count and max_length.  Each config
runs in a fresh process.  One JSON line per config: card, power limit, max SM clock, peak max_memory_allocated /
max_memory_reserved, ms per iteration, and the activation bytes the forward keeps for the backward, counted from
shapes with and without recompute.  A config whose counted bytes do not fit the card is reported and not run.

--compare: the bench's `pretrain` shape (1.3B decoder, B = 32, 8 frames, text 128, 128 queries), one engine with the
ViT activations resident and one with grad_ckpt, same weights and inputs, CUDA-graph steps as bench.py times them.
The arms alternate, `--rounds` windows of `--steps` steps each; before every window both engines are reset to the same
state, so their losses compare bit for bit.
"""
import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "youku-mplug_b200")
for _p in (ROOT, PKG, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

YAMLS = ["caption/caption_gpt3_1.3B_youku_v0.yaml", "caption/caption_gpt3_2.7B_youku_v0.yaml",
         "cls/cls_gpt3_1.3B_youku_v0_sharp_2.yaml", "cls/cls_gpt3_2.7B_youku_v0_sharp_2.yaml",
         "retrieval/retrieval_gpt3_1.3B_youku_v0.yaml", "retrieval/retrieval_gpt3_2.7B_youku_v0.yaml",
         "retrieval/retrieval_itm_gpt3_1.3B_youku_v0.yaml", "retrieval/retrieval_itm_gpt3_2.7B_youku_v0.yaml",
         "pretrain/gpt3_1.3B/pretrain_gpt3_freezeGPT_youku_v0.yaml", "pretrain/gpt3_2.7B/pretrain_gpt3_freezeGPT_youku_v0.yaml"]
GB = 1e9


def card_info():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip()
    name, plim, clk = [x.strip() for x in out.split(",")]
    return dict(name=name, power_limit=plim, max_sm_clock=clk)


def load_yaml(path):
    """The yaml as the task scripts read it (the package's ruamel.yaml stand-in)."""
    import importlib
    compat = os.path.join(PKG, "compat")
    sys.path.append(compat)
    try:
        ryaml = importlib.import_module("ruamel.yaml")
        with open(path) as f:
            return dict(ryaml.load(f, Loader=ryaml.Loader))
    finally:
        sys.path.remove(compat)


def model_class(name):
    if name.startswith("caption/"):
        return "DistributedGPT3_Caption"
    if name.startswith("cls/"):
        return "DistributedGPT3_Cls"
    if name.startswith("retrieval/retrieval_itm_"):
        return "DistributedGPT3_Retrieval_Cls"
    if name.startswith("retrieval/"):
        return "DistributedGPT3_Retrieval"
    return "DistributedGPT3_Pretrain"


def counted_bytes(cls, vis, gcfg, B, T, L, Q):
    """Activation bytes that the forward keeps for the backward (ymp.engine), from shapes.  ViT block: fp32 x, xt, y;
    bf16 ln_t, att_t, proj_t, ln_s, att_s, ln_m (D columns), qkv_t, qkv_s (3D), dact, h (4D): 52 D bytes per token row;
    its fp32 input alone is 4 D.  Frozen decoder layer: fp32 x, x1; bf16 qkv, att, dact: 24 H bytes per token (with
    ffn 4H); its fp32 input alone is 4 H.  Recompute keeps the inputs and rebuilds one block / layer at a time."""
    D, depth = vis["embed_dim"], vis["depth"]
    N = (vis["img_size"] // vis["patch_size"]) ** 2
    hid = int(D * vis["mlp_ratio"])
    RB = B * N * T + B
    vit_block = RB * (3 * 4 * D + 6 * 2 * D + 2 * 2 * 3 * D + 2 * 2 * hid)
    vit_in = RB * 4 * D
    H, F, layers = gcfg["hidden_size"], gcfg.get("ffn_hidden_size") or 4 * gcfg["hidden_size"], gcfg["num_hidden_layers"]
    S = Q + L
    # decoder passes that need a backward (their input comes from the trainable visual prefix)
    seqs = {"DistributedGPT3_Pretrain": [B], "DistributedGPT3_Caption": [B], "DistributedGPT3_Cls": [B, B],
            "DistributedGPT3_Retrieval_Cls": [3 * B, 3 * B], "DistributedGPT3_Retrieval": []}[cls]
    tok = sum(seqs) * S
    layer = tok * (4 * H + 4 * H + 2 * 3 * H + 2 * H + 2 * F)
    dec_in = tok * 4 * H
    one_layer = max(seqs, default=0) * S * (4 * H + 4 * H + 2 * 3 * H + 2 * H + 2 * F)
    return dict(vit_resident=depth * vit_block, vit_recompute=depth * vit_in + vit_block,
                decoder_resident=layers * layer, decoder_recompute=layers * dec_in + one_layer)


def make_text(B, L, vocab, seed, prompt=None):
    import torch
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(3, vocab, (B, L), generator=g)
    ids[:, 0] = 1
    lens = torch.randint(L // 2, L + 1, (B,), generator=g)
    att = (torch.arange(L)[None, :] < lens[:, None]).long()
    ids = torch.where(att.bool(), ids, torch.zeros_like(ids))
    d = dict(input_ids=ids, attention_mask=att)
    if prompt is not None:
        d["prompt_lengths"] = torch.full((B,), prompt, dtype=torch.long)
    return d


def derangement(n, rng):
    while True:
        p = list(range(n))
        rng.shuffle(p)
        if all(i != v for i, v in enumerate(p)):
            return p


def build(name, cfg, dev, grad_ckpt=None, dropout=0.1):
    """The script's model (random bf16 weights) and its TrainEngine."""
    import torch
    os.environ["YMP_ALLOW_RANDOM_INIT"] = "1"
    from helpers import make_model_dir
    import models.distributed_gpt3 as D
    from ymp.train import TrainEngine
    with open(os.path.join(PKG, cfg["visual_cfg"])) as f:
        vis = json.load(f)
    with open(os.path.join(PKG, cfg["text_cfg"])) as f:
        gcfg = json.load(f)
    td = make_model_dir(vis, gcfg, dropout=(dropout, dropout))
    with open(os.path.join(td, "vis.json"), "w") as f:   # make_model_dir writes grad_ckpt: false
        json.dump(dict(vis, pretrained_ckpt=None, grad_ckpt=vis.get("grad_ckpt", True) if grad_ckpt is None else grad_ckpt), f)
    config = dict(cfg, visual_cfg=os.path.join(td, "vis.json"), text_cfg=os.path.join(td, "config.json"), text_decoder=td)
    torch.manual_seed(0)
    with torch.device(dev):
        model = getattr(D, model_class(name))(config=config, tokenizer=None)
    model = model.to(torch.bfloat16).train()
    o = cfg.get("optimizer", {})
    eng = TrainEngine(model, lr=float(o.get("lr", 1e-4)), betas=tuple(o.get("opt_betas", (0.9, 0.999))),
                      eps=float(o.get("opt_eps", 1e-8)), weight_decay=float(o.get("weight_decay", 0.05)),
                      clip_grad=float(o.get("clip_grad", 3.0)))
    return eng, vis, gcfg


def inputs(name, cfg, vis, gcfg, dev, B, T, L, seed=0):
    """Synthetic arguments of the script's model(...) call at the yaml's shapes."""
    import torch
    import models.modeling_distributed_gpt3 as G

    def enc(d):
        return G.BatchEncoding({k: v.to(dev) for k, v in d.items()})

    V = gcfg["vocab_size"]
    video = torch.randn(B, 3, T, vis["img_size"], vis["img_size"], generator=torch.Generator().manual_seed(seed)).to(dev).bfloat16()
    cls = model_class(name)
    if cls in ("DistributedGPT3_Pretrain", "DistributedGPT3_Caption"):
        return (video, enc(make_text(B, L, V, seed + 1, prompt=None if cls.endswith("Pretrain") else 8)))
    if cls == "DistributedGPT3_Retrieval":
        return (video, enc(make_text(B, L, V, seed + 1)), torch.arange(B, device=dev))
    if cls == "DistributedGPT3_Cls":
        labels = torch.randint(0, int(cfg.get("num_classes", 45)), (B,), generator=torch.Generator().manual_seed(seed + 3))
        return (video, enc(make_text(B, L, V, seed + 1, prompt=12)), enc(make_text(B, L, V, seed + 2)), labels.to(dev))
    rng = random.Random(seed)   # run_retrieval_distributed_gpt3_itm.py: two derangements of hard negatives per batch
    neg = derangement(B, rng) + derangement(B, rng)
    labels = torch.cat([torch.ones(B), torch.zeros(2 * B)]).long()
    return (video, enc(make_text(3 * B, L, V, seed + 1, prompt=16)), enc(make_text(3 * B, L, V, seed + 2)),
            torch.tensor(neg, device=dev), labels.to(dev))


def total_loss(out):
    return sum(out[1:], out[0]) if isinstance(out, (tuple, list)) else out


def run_one(name, iters):
    import torch
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    cfg = load_yaml(os.path.join(PKG, "configs", name))
    with open(os.path.join(PKG, cfg["visual_cfg"])) as f:
        vis = json.load(f)
    with open(os.path.join(PKG, cfg["text_cfg"])) as f:
        gcfg = json.load(f)
    B, L, Q = int(cfg["batch_size"]), int(cfg["max_length"]), int(cfg.get("num_learnable_token", 256))
    T = int(cfg.get("num_frames") or vis["num_frames"])
    cls = model_class(name)
    vit_on = bool(vis.get("grad_ckpt", True))
    dec_on = bool((cfg.get("megatron_cfg") or {}).get("checkpoint_activations", False))
    cnt = counted_bytes(cls, vis, gcfg, B, T, L, Q)
    configured = (cnt["vit_recompute"] if vit_on else cnt["vit_resident"]) + \
        (cnt["decoder_recompute"] if dec_on else cnt["decoder_resident"])
    line = dict(config=name, model=cls, card=card_info(), batch_per_gpu=B, frames=T, text_len=L, queries=Q,
                vit_recompute=vit_on, decoder_recompute=dec_on,
                counted_activation_gb={k: round(v / GB, 2) for k, v in cnt.items()},
                counted_activation_gb_as_configured=round(configured / GB, 2))
    cap = torch.cuda.get_device_properties(dev).total_memory
    if configured > 0.9 * cap:
        line.update(ran=False, reason=f"counted activations {configured / GB:.1f} GB do not fit {cap / GB:.0f} GB")
        print(json.dumps(line), flush=True)
        return
    eng, vis, gcfg = build(name, cfg, dev)
    args = inputs(name, cfg, vis, gcfg, dev, B, T, L)
    torch.cuda.synchronize()
    state_gb = torch.cuda.memory_allocated(dev) / GB
    torch.cuda.reset_peak_memory_stats(dev)
    ms, losses = [], []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        loss = total_loss(eng(*args))
        eng.backward(loss)
        eng.step()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
        losses.append(float(loss.item()))
    line.update(ran=True, iters=iters, ms_per_iter=[round(x, 1) for x in ms], losses=losses,
                weights_and_optimizer_gb=round(state_gb, 2),
                peak_allocated_gb=round(torch.cuda.max_memory_allocated(dev) / GB, 2),
                peak_reserved_gb=round(torch.cuda.max_memory_reserved(dev) / GB, 2),
                total_gb=round(cap / GB, 2), note="eager iterations (model -> TrainEngine.backward -> step); first one includes warm-up")
    print(json.dumps(line), flush=True)


def compare(rounds, steps):
    import torch
    from bench import VCFG_CLIP_B16, GCFG, make_text as bench_text
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    B, T, L, Q = 32, 8, 128, 128
    vcfg = dict(VCFG_CLIP_B16, num_frames=T, drop_path=0)
    vdir = tempfile.mkdtemp(prefix="memfit_")
    with open(os.path.join(vdir, "vis.json"), "w") as f:
        json.dump(vcfg, f)
    with open(os.path.join(vdir, "gpt.json"), "w") as f:
        json.dump(GCFG["1.3B"], f)
    cfg = dict(visual_cfg=os.path.join(vdir, "vis.json"), text_cfg=os.path.join(vdir, "gpt.json"), num_frames=T,
               megatron_cfg={"world_size": 1, "model_parallel_size": 1, "tensor_model_parallel_size": 1},
               num_learnable_token=Q, use_contrastive=False, freeze_text_decoder=True,
               optimizer=dict(lr=1e-4, opt_betas=[0.9, 0.999], opt_eps=1e-6, weight_decay=0.05, clip_grad=3.0))
    import models.modeling_distributed_gpt3 as G
    g = torch.Generator().manual_seed(1234)
    video = torch.randn(B, 3, T, 224, 224, generator=g).to(dev).bfloat16()
    ids, att = bench_text(G, B, L, 51200, 4321)
    text = G.BatchEncoding(dict(input_ids=ids.to(dev), attention_mask=att.to(dev)))
    arms = {}
    for name, on in (("resident", False), ("recompute", True)):
        eng, _, _ = build("pretrain/bench", cfg, dev, grad_ckpt=on, dropout=0.0)   # bench.py default: no decoder dropout
        assert eng.module.visual_encoder.vcfg["grad_ckpt"] is on
        arms[name] = dict(eng=eng, snap=[t.clone() for t in (eng.flat_param, eng.master, eng.exp_avg, eng.exp_avg_sq)],
                          ms=[], losses=[])
    snap0 = arms["resident"]["snap"]
    assert all(torch.equal(a, b) for a, b in zip(snap0, arms["recompute"]["snap"])), "arms must start from the same weights"

    def reset(eng):
        for t, s in zip((eng.flat_param, eng.master, eng.exp_avg, eng.exp_avg_sq), snap0):
            t.copy_(s)
        eng.flat_grad.zero_()
        eng.global_steps = 0

    # activation growth of one eager forward + backward, then graph capture (two eager warm-up steps each)
    for name, a in arms.items():
        eng = a["eng"]
        reset(eng)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        base = torch.cuda.memory_allocated(dev)
        loss = total_loss(eng(video, text))
        eng.backward(loss)
        torch.cuda.synchronize()
        a["eager_fwd_bwd_growth_gb"] = (torch.cuda.max_memory_allocated(dev) - base) / GB
        del loss
        eng.flat_grad.zero_()
        torch.cuda.empty_cache()
    for name, a in arms.items():
        reset(a["eng"])
        for _ in range(3):
            a["eng"].train_step(video, text, use_graph=True, graph_warmup=2)
        torch.cuda.synchronize()
    for r in range(rounds):
        for name, a in arms.items():
            eng = a["eng"]
            reset(eng)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            # a replayed step returns the graph's static loss tensor: keep a copy of each step's value
            ls = [eng.train_step(video, text, use_graph=True).clone() for _ in range(steps)]
            e1.record()
            torch.cuda.synchronize()
            a["ms"].append(e0.elapsed_time(e1) / steps)
            a["losses"].append([float(x.item()) for x in ls])
    res, rec = arms["resident"], arms["recompute"]
    med = {n: statistics.median(a["ms"]) for n, a in arms.items()}
    first_equal = all(x[0] == y[0] for x, y in zip(res["losses"], rec["losses"]))
    all_equal = res["losses"] == rec["losses"]
    line = dict(mode="compare", card=card_info(), shape=dict(model="DistributedGPT3_Pretrain", decoder="GPT-3 1.3B", batch=B,
                                                              frames=T, text_len=L, queries=Q),
                rounds=rounds, steps_per_window=steps, cuda_graph=True,
                ms_per_step={n: [round(x, 2) for x in a["ms"]] for n, a in arms.items()},
                median_ms_per_step={n: round(v, 2) for n, v in med.items()},
                step_time_overhead=round(med["recompute"] / med["resident"] - 1.0, 4),
                samples_per_s={n: round(B * 1000.0 / v, 1) for n, v in med.items()},
                eager_fwd_bwd_growth_gb={n: round(a["eager_fwd_bwd_growth_gb"], 2) for n, a in arms.items()},
                memory_saved_gb=round(res["eager_fwd_bwd_growth_gb"] - rec["eager_fwd_bwd_growth_gb"], 2),
                losses={n: a["losses"] for n, a in arms.items()},
                first_step_loss_bit_equal=first_equal, all_losses_bit_equal=all_equal,
                note="first step of every window: same weights, same inputs, identical forward; later steps follow "
                     "updates whose fp32 gradient sums are accumulated by atomics in any order")
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="+", default=YAMLS, help="yamls under youku-mplug_b200/configs/")
    ap.add_argument("--iters", type=int, default=2)
    ap.add_argument("--compare", action="store_true", help="resident vs ViT recompute at the bench's pretrain shape")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--one", default=None, help=argparse.SUPPRESS)   # child process: one config
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("memory_fit.py needs a GPU")
    if args.compare:
        compare(args.rounds, args.steps)
        return
    if args.one:
        run_one(args.one, args.iters)
        return
    failed = []
    for name in args.configs:
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--one", name, "--iters", str(args.iters)])
        if r.returncode:
            failed.append(name)
            print(json.dumps(dict(config=name, ran=False, reason=f"exit code {r.returncode}")), flush=True)
    if failed:
        sys.exit(1)


if __name__ == "__main__":
    main()
