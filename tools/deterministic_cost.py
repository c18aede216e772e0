"""Cost of the deterministic mode (torch.use_deterministic_algorithms(True)) on the training step of bench.py's configs.

    python tools/deterministic_cost.py [--configs pretrain caption27b retrieval] [--rounds 3] [--steps 8] [--warmup 3]
                                       [--json OUT]

One process, one GPU.  Per config the model and TrainEngine of bench.py are built once (seed 0, the same synthetic
batch every step) and their initial state kept; then three arms alternate for --rounds rounds: mode off, mode on, and
mode on with torch.utils.deterministic.fill_uninitialized_memory off ("on, no fill").  The last arm splits the cost
between what PyTorch itself does under the flag (the NaN fill of every uninitialised allocation) and the library's
fixed-order sums.  Each arm restores the initial state, runs --warmup CUDA-graph train_steps (eager warm-up and the
capture included) and times --steps more with CUDA events around work that ends in a synchronise; it reports the
median ms/step over the rounds and the peak allocated memory of its steps.  Only the current arm's graph is kept (two
graphs of the large configs do not fit together).  Every mode-on round (either fill setting) starts from the same
state and runs the same steps, so each must end with the same loss and the same fixed sample of parameters
(bench.py --dump-outputs' sample) bit for bit; the script asserts it.
The card's name and power limit are read in the same call.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
os.environ.setdefault("CUBLAS_WORKSPACE_CONFIG", ":4096:8")   # the contrastive head's cuBLAS matmuls


def card_info():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip()
    name, plim, clk = [x.strip() for x in out.split(",")]
    return dict(name=name, power_limit=plim, max_sm_clock=clk)


def run_config(name, rounds, steps, warmup):
    import torch
    import bench
    from helpers import make_model_dir, pretrain_config
    import models.distributed_gpt3 as D
    import models.modeling_distributed_gpt3 as G
    from ymp import functional as YF
    from ymp import lib, train

    os.environ["YMP_ALLOW_RANDOM_INIT"] = "1"
    dev = torch.device("cuda:0")
    cfg = bench.CONFIGS[name]
    B, T, L, Q = cfg["batch"], cfg["frames"], cfg["text_len"], 128
    vcfg = dict(bench.VCFG_CLIP_B16, num_frames=T)
    td = make_model_dir(vcfg, bench.GCFG[cfg["gpt"]])
    torch.manual_seed(0)
    with torch.device(dev):
        model = getattr(D, cfg["cls"])(config=pretrain_config(td, Q, num_frames=T), tokenizer=None)
    model = model.to(torch.bfloat16)
    model.train()
    eng = train.TrainEngine(model, lr=1e-4, betas=(0.9, 0.999), eps=1e-6, weight_decay=0.05, clip_grad=3.0)
    g = torch.Generator().manual_seed(1234)
    video = torch.randn(B, 3, T, 224, 224, generator=g).to(dev).bfloat16()
    ids, att = bench.make_text(G, B, L, 51200, 4321)
    extra = {"prompt_lengths": torch.full((B,), 4, dtype=torch.long, device=dev)} if name == "caption27b" else {}
    text = G.BatchEncoding(dict(input_ids=ids.to(dev), attention_mask=att.to(dev), **extra))
    tail = (torch.arange(B, dtype=torch.long, device=dev),) if name == "retrieval" else ()
    state0 = [t.clone() for t in (eng.flat_param, eng.master)]
    n = eng.master.numel()
    gs = torch.Generator().manual_seed(20240)
    idx = torch.randint(0, n, (min(n, bench.DUMP_SAMPLE),), generator=gs).sort().values.to(dev)

    def restore():
        eng._graphs.clear()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        eng.flat_param.copy_(state0[0])
        eng.master.copy_(state0[1])
        for t in (eng.exp_avg, eng.exp_avg_sq, eng.flat_grad):
            t.zero_()
        eng.global_steps = eng.micro_steps = 0
        YF.note_weight_write()

    import torch.utils.deterministic as det
    fill0 = det.fill_uninitialized_memory

    def arm(mode):
        on = mode != "off"
        torch.use_deterministic_algorithms(on)
        det.fill_uninitialized_memory = mode != "on_nofill"
        lib.sync_deterministic()
        restore()
        torch.cuda.reset_peak_memory_stats(dev)
        for _ in range(warmup):
            eng.train_step(video, text, *tail)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            loss = eng.train_step(video, text, *tail)
        e1.record()
        torch.cuda.synchronize()
        out = dict(ms=e0.elapsed_time(e1) / steps, peak_gb=torch.cuda.max_memory_allocated(dev) / 2 ** 30,
                   loss=loss.clone(), params=(eng.flat_param[idx].clone(), eng.master[idx].clone()))
        torch.use_deterministic_algorithms(False)
        det.fill_uninitialized_memory = fill0
        lib.sync_deterministic()
        return out

    modes = ("off", "on", "on_nofill")
    res = {m: [] for m in modes}
    for _ in range(rounds):
        for m in modes:
            res[m].append(arm(m))
    first = res["on"][0]
    for r in res["on"][1:] + res["on_nofill"]:     # the fill touches no value the step reads
        assert torch.equal(r["loss"], first["loss"]), f"{name}: mode-on loss differs between rounds"
        assert all(torch.equal(a, b) for a, b in zip(r["params"], first["params"])), f"{name}: mode-on parameters differ"
    row = dict(config=name)
    for m in modes:
        row[f"{m}_ms"] = statistics.median(r["ms"] for r in res[m])
        row[f"{m}_peak_gb"] = max(r["peak_gb"] for r in res[m])
    row["cost_pct"] = 100.0 * (row["on_ms"] / row["off_ms"] - 1.0)
    row["cost_nofill_pct"] = 100.0 * (row["on_nofill_ms"] / row["off_ms"] - 1.0)
    row["on_loss"] = float(first["loss"])
    row["off_loss"] = float(res["off"][0]["loss"])
    del model, eng
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="+", default=["pretrain", "caption27b", "retrieval"])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    assert args.rounds >= 3 and args.warmup >= 3, "at least 3 rounds after a warm-up of 3 steps (eager, capture, replay)"
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("deterministic_cost.py needs a GPU (nothing is estimated without one)")
    card = card_info()
    rows = [run_config(c, args.rounds, args.steps, args.warmup) for c in args.configs]
    print(f"{card['name']}, power limit {card['power_limit']}, max SM clock {card['max_sm_clock']}")
    print(f"{'config':<12} {'off ms/step':>12} {'on ms/step':>11} {'cost':>7} {'on, no fill':>12} {'cost':>7} "
          f"{'off peak GB':>12} {'on peak GB':>11}")
    for r in rows:
        print(f"{r['config']:<12} {r['off_ms']:>12.2f} {r['on_ms']:>11.2f} {r['cost_pct']:>6.1f}% {r['on_nofill_ms']:>12.2f} "
              f"{r['cost_nofill_pct']:>6.1f}% {r['off_peak_gb']:>12.2f} {r['on_peak_gb']:>11.2f}")
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=card, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
