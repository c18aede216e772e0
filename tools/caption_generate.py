"""Time caption generation: the per-clip beam-search loop against the batched and streaming beam searches.

    python tools/caption_generate.py [--shapes caption_1.3B caption_2.7B] [--rounds 3] [--workloads full varied]
                                     [--stop-scale 4] [--kernel] [--counts] [--profile]

Each shape builds DistributedGPT3_Caption with the shipped decoder json, random bf16 weights in eval mode, 128 queries
and 16 frames, and decodes the caption eval's batch (24 clips at 1.3B, 36 at 2.7B): prompt ids [B, 20] with one
common prompt length, beam 5, 100 tokens to generate.  Four arms, alternating in one process after a warm-up call of
each, every call ending in a device synchronise; the median of --rounds calls is reported:
  per_clip       - the composition before batching: the visual prefix, then one beam search per clip;
  batched_moving - the chunked batched search with the beams permuted by moving the cached K/V rows (KVCache.reorder);
  batched        - the chunked batched search (chunks of 64 // beam clips per decode step, each running until its
                   slowest clip is done), beams permuted through the cache's row table (KVCache.reindex);
  stream         - model.generate(video, text): the streaming search (run_beam_search over the per-row decode state),
                   a finished clip's beam slots take the next clip while the others keep decoding.
Two workloads: `full` (random weights almost never emit the stop token, so every caption runs all 100 tokens: the
stream arm must do the batched arm's steps) and `varied` (the stop token's row of the tied word embedding scaled by
--stop-scale, so captions end at varying steps: where the stream arm saves steps).
One JSON line per shape and workload: card name, power limit and max SM clock, ms per call, single-token decode steps,
rows stepped that no beam search reads (rows stepped minus beam x the per-clip arm's steps), peak allocated memory,
the distribution of per-clip decode steps and whether the four arms' sequences and scores are bit-equal.
--profile prints the device-time share of each kernel family in one batched 12-clip, 40-token call of each batched arm.
--kernel times ymp_gemm_skinny_wide alone per decoder linear and for the LM head at M in {5, 8, 16, 32, 60, 64} rows (CUDA
events over many launches, weights rotated through copies larger than L2): microseconds and GB/s next to the H100
SXM data sheet's 3.35 TB/s.  --counts prints the weight and KV-cache bytes counted from shapes, without a GPU.
"""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "youku-mplug_b200")
for _p in (ROOT, PKG, os.path.join(ROOT, "tests")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

Q, L, FRAMES, BEAM, NEW = 128, 20, 16, 5, 100   # queries, prompt ids, frames per clip, beam, tokens to generate
MAX_ROWS = 64                                   # ops.SKINNY_WIDE_MAX_ROWS: rows of one batched decode step
HBM_TBS = 3.35                                  # H100 SXM data sheet
# name: (decoder json, clips per call: the caption yamls' per-GPU eval batch)
SHAPES = {"caption_1.3B": ("config_gpt3_1.3B.json", 24), "caption_2.7B": ("config_gpt3_2.7B.json", 36)}
M_KERNEL = (5, 8, 16, 32, 60, 64)


def gpt_cfg(name):
    with open(os.path.join(PKG, "configs", "models", SHAPES[name][0])) as f:
        return json.load(f)


def linears(name):
    """(name, N, K) of the decoder's skinny GEMMs: the four linears of a layer, and the LM head."""
    g = gpt_cfg(name)
    h, V = g["hidden_size"], g["vocab_size"]
    return [("qkv", 3 * h, h), ("dense", h, h), ("h_to_4h", 4 * h, h), ("4h_to_h", h, 4 * h), ("lm_head", V, h)]


def counts(name, clips=None):
    """Weight bytes one decode step streams, weight passes per eval batch of each arm (one per token step; the prefill
    passes are not counted), the KV-cache bytes of one batched chunk, and the bytes one beam reorder moves at the mean
    cached length of a full-length decode: the moving KVCache.reorder (index_select into a temporary, copy back: each
    cached [q|k|v] row read twice and written twice) against KVCache.reindex (the same four passes over the int32 row
    table's cached columns)."""
    g = gpt_cfg(name)
    h, layers = g["hidden_size"], g["num_hidden_layers"]
    B = clips or SHAPES[name][1]
    per_chunk = MAX_ROWS // BEAM
    chunks = -(-B // per_chunk)
    step_bytes = sum(N * K * 2 for nm, N, K in linears(name) if nm != "lm_head") * layers + \
        [N * K * 2 for nm, N, K in linears(name) if nm == "lm_head"][0]
    positions = Q + L + NEW   # KV-cache positions of one sequence
    rows = min(B, per_chunk) * BEAM
    mean_len = Q + L + NEW / 2
    moving = 4 * layers * rows * mean_len * 3 * h * 2
    indexed = 4 * rows * mean_len * 4
    return dict(clips=B, beam=BEAM, tokens_to_generate=NEW, weight_gb_per_step=round(step_bytes / 1e9, 3),
                passes_per_clip_arm=B * NEW, passes_batched_arm=chunks * NEW, chunks=chunks, rows_per_chunk=rows,
                weight_tb_per_clip_arm=round(B * NEW * step_bytes / 1e12, 2),
                weight_tb_batched_arm=round(chunks * NEW * step_bytes / 1e12, 2),
                kv_cache_gb_per_chunk=round(layers * rows * positions * 3 * h * 2 / 1e9, 2), kv_positions=positions,
                reorder_mean_len=mean_len, reorder_moving_gb=round(moving / 1e9, 2), reorder_indexed_kb=round(indexed / 1e3, 1),
                reorder_moving_min_ms_at_3_35_tb_s=round(moving / (HBM_TBS * 1e12) * 1e3, 2))


def card_info():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip()
    name, plim, clk = [x.strip() for x in out.split(",")]
    return dict(card=name, power_limit=plim, max_sm_clock=clk)


def build(name, dev):
    import torch
    os.environ["YMP_ALLOW_RANDOM_INIT"] = "1"
    from helpers import make_model_dir, pretrain_config
    import models.distributed_gpt3 as D
    with open(os.path.join(PKG, "configs", "models", "clip-b16.json")) as f:
        vis = json.load(f)
    td = make_model_dir(vis, gpt_cfg(name), dropout=(0.1, 0.1))
    torch.manual_seed(0)
    with torch.device(dev):
        model = D.DistributedGPT3_Caption(config=pretrain_config(td, Q, num_frames=FRAMES), tokenizer=None)
    model = model.to(torch.bfloat16).eval()
    model.text_decoder.config.tokens_to_generate = NEW
    return model, vis


def per_clip_generate(model, video, text):
    """DistributedGPT3_Caption.generate as it was before batching: one beam search per clip."""
    import torch
    with torch.no_grad():
        return _per_clip(model, video, text)


def _per_clip(model, video, text):
    _, _, _, qf = model.visual_prefix(video)
    eos = model.text_decoder.config.eod_id
    res = []
    for i in range(len(text.input_ids)):
        out = model.text_decoder.generate(text.input_ids[i:i + 1], query_embeds=qf[i:i + 1], termination_id=eos,
                                          do_sample=False, prompt_length=text.attention_mask.sum(-1)[i] - 1)
        res.append(out.sequences.cpu())
    return res


def moving_generate(model, video, text):
    """The batched call with the beam loop's reorder callback moving the cached rows (KVCache.reorder: every cached
    [q|k|v] row of every layer permuted in place) instead of gathering the row table (KVCache.reindex)."""
    dec = model.text_decoder
    callbacks = dec._decode_callbacks

    def moving(query_embeds):
        step, _ = callbacks(query_embeds)
        return step, lambda idx: dec.inference_params.cache.reorder(idx)
    dec._decode_callbacks = moving
    try:
        return model.generate(video, text)
    finally:
        del dec._decode_callbacks


def inputs(vis, name, B):
    import torch
    import models.modeling_distributed_gpt3 as G
    dev = torch.device("cuda:0")
    vocab = gpt_cfg(name)["vocab_size"]
    gen = torch.Generator().manual_seed(1)
    video = torch.randn(B, 3, FRAMES, vis["img_size"], vis["img_size"], generator=gen).to(dev).bfloat16()
    ids = torch.randint(3, vocab, (B, L), generator=gen)
    text = G.BatchEncoding(dict(input_ids=ids.to(dev), attention_mask=torch.ones(B, L, dtype=torch.long, device=dev)))
    return video, text


def chunked_generate(model, video, text, moving=False):
    """model.generate through the chunked batched beam search: streams_beam_search answers no, so beam_search runs
    its chunks over fixed-length decode states."""
    import models.modeling_distributed_gpt3 as G
    streams = G.streams_beam_search
    G.streams_beam_search = lambda *a: False
    try:
        return moving_generate(model, video, text) if moving else model.generate(video, text)
    finally:
        G.streams_beam_search = streams


def run(model, vis, name, rounds, workload="full", stop_scale=4.0):
    import torch
    from ymp import engine
    B = SHAPES[name][1]
    video, text = inputs(vis, name, B)
    dec = model.text_decoder
    emb = dec.dist_model.language_model.embedding.word_embeddings.weight
    eod_row = emb[dec.config.eod_id].clone()
    if workload == "varied":
        with torch.no_grad():
            emb[dec.config.eod_id] *= stop_scale
    orig = dec.beam_search
    found, steps = [], [0]
    tok_steps, tok_rows, clip_steps = [0], [0], []
    ts_run = engine.TokenStep.run

    def counting_run(self, emb_in):   # single-token steps and the rows they step
        tok_steps[0] += 1
        tok_rows[0] += self.cache.B
        return ts_run(self, emb_in)
    engine.TokenStep.run = counting_run

    def beam_search(*a, **k):   # keeps every beam search's results (sequences and scores) for the comparison
        n0 = tok_steps[0]
        out = orig(*a, **k)
        found.extend(out if isinstance(out, list) else [out])
        clip_steps.append(tok_steps[0] - n0)
        return out
    dec.beam_search = beam_search
    orig_decode = dec._decode

    def counting_decode(*a, **k):
        steps[0] += 1
        return orig_decode(*a, **k)
    dec._decode = counting_decode
    arms = dict(per_clip=lambda: per_clip_generate(model, video, text),
                batched_moving=lambda: chunked_generate(model, video, text, moving=True),
                batched=lambda: chunked_generate(model, video, text), stream=lambda: model.generate(video, text))
    ms = {a: [] for a in arms}
    peak = {a: 0 for a in arms}
    n_steps, outs, n_tok, n_rows, per_clip_steps = {}, {}, {}, {}, []
    for r in range(rounds + 1):   # round 0 warms up every arm
        for a, fn in arms.items():
            found.clear()
            clip_steps.clear()
            outs.pop(a, None)
            steps[0] = tok_steps[0] = tok_rows[0] = 0
            # the decoder pools one KV cache + captured step per shape on the model: every arm allocates (and counts in
            # its peak) and captures its own, rather than one arm inheriting the cache of the arm before it
            dec.__dict__.pop("_decode_pool", None)
            gc.collect()   # a dropped cache and its captured step reference each other: free them before the next arm
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            dt = (time.perf_counter() - t0) * 1e3
            outs[a] = [(o.sequences.cpu(), o.scores.cpu()) for o in found]
            n_steps[a] = steps[0]
            n_tok[a], n_rows[a] = tok_steps[0], tok_rows[0]
            if a == "per_clip":
                per_clip_steps = list(clip_steps)
            if r > 0:
                ms[a].append(dt)
                peak[a] = max(peak[a], torch.cuda.max_memory_allocated() - base)
    del dec.beam_search, dec._decode
    engine.TokenStep.run = ts_run
    with torch.no_grad():
        emb[dec.config.eod_id] = eod_row
    equal = all(len(outs[a]) == B and all(torch.equal(s0, s1) and torch.equal(c0, c1)
                                          for (s0, c0), (s1, c1) in zip(outs["per_clip"], outs[a])) for a in arms)
    res = dict(shape=name, workload=workload, stop_scale=stop_scale if workload == "varied" else 1.0, clips=B,
               frames=FRAMES, queries=Q, beam=BEAM, tokens_to_generate=NEW, **card_info())
    read_rows = BEAM * sum(per_clip_steps)
    for a in arms:
        res[f"{a}_ms"] = round(statistics.median(ms[a]), 1)
        res[f"{a}_ms_all"] = [round(x, 1) for x in ms[a]]
        res[f"{a}_decoder_calls"] = n_steps[a]
        res[f"{a}_decode_steps"] = n_tok[a]
        res[f"{a}_unread_rows"] = n_rows[a] - read_rows
        res[f"{a}_peak_gb"] = round(peak[a] / 1e9, 2)
    res["clip_steps"] = dict(min=min(per_clip_steps), median=statistics.median(per_clip_steps), max=max(per_clip_steps),
                             all=per_clip_steps)
    res["speedup"] = round(res["per_clip_ms"] / res["batched_ms"], 2)
    res["speedup_over_moving"] = round(res["batched_moving_ms"] / res["batched_ms"], 2)
    res["stream_over_batched"] = round(res["batched_ms"] / res["stream_ms"], 2)
    res["bit_equal"] = bool(equal)
    res["counts"] = counts(name)
    print(json.dumps(res), flush=True)
    return res


def profile(model, vis, name, clips=12, new=40):
    """torch.profiler over one batched call of each batched arm (one 60-row chunk, `new` tokens), after a warm-up call:
    device time per kernel family - decode / prefill attention, skinny GEMMs, and the index_select / copy kernels
    (the moving reorder's two passes, or the indexed arm's table gather, with the step's small copies)."""
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile
    dec = model.text_decoder
    dec.config.tokens_to_generate = new
    video, text = inputs(vis, name, clips)
    arms = dict(batched_moving=lambda: chunked_generate(model, video, text, moving=True),
                batched=lambda: chunked_generate(model, video, text))
    info = card_info()
    try:
        for a, fn in arms.items():
            with torch.no_grad():
                fn()
                torch.cuda.synchronize()
                with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
                    fn()
                    torch.cuda.synchronize()
            fam, per_kernel = {}, {}
            for e in prof.events():
                if e.device_type != torch.autograd.DeviceType.CUDA:
                    continue
                k = e.name
                per_kernel[k] = per_kernel.get(k, 0.0) + e.time_range.elapsed_us()
                f = ("attn_decode" if "attn_decode_kernel" in k else "attn_other" if "attn_" in k else
                     "gemm_skinny" if "gemm_skinny" in k else
                     "index_select_copy" if any(w in k.lower() for w in ("index", "gather", "copy")) else "other")
                fam[f] = fam.get(f, 0.0) + e.time_range.elapsed_us()
            total = sum(fam.values())
            top = sorted(per_kernel.items(), key=lambda kv: -kv[1])[:6]
            print(json.dumps(dict(shape=name, arm=a, clips=clips, tokens_to_generate=new, device_ms=round(total / 1e3, 1),
                                  **{f"{f}_ms": round(v / 1e3, 1) for f, v in sorted(fam.items())},
                                  **{f"{f}_share": round(v / total, 3) for f, v in sorted(fam.items())},
                                  top_kernels_ms={k[:80]: round(v / 1e3, 1) for k, v in top}, **info)), flush=True)
    finally:
        dec.config.tokens_to_generate = NEW


def kernel(name, iters=50):
    """ymp_gemm_skinny_wide alone (M <= 8: the ymp_gemm_skinny launch): per (linear, M), microseconds per launch and
    algorithmic GB/s (weights + x + y)."""
    import torch
    from ymp import ops
    dev = torch.device("cuda:0")
    info = card_info()
    for lin, N, K in linears(name):
        wbytes = N * K * 2
        copies = max(2, -(-200_000_000 // wbytes))   # rotate through > 200 MB of weights: nothing stays in L2
        ws = [torch.randn(N, K, device=dev).bfloat16() for _ in range(copies)]
        for M in M_KERNEL:
            x = torch.randn(M, K, device=dev).bfloat16()
            y = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
            for w in ws:
                ops.gemm_skinny_wide(x, w, out=y)
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            ev0.record()
            for i in range(iters):
                ops.gemm_skinny_wide(x, ws[i % copies], out=y)
            ev1.record()
            torch.cuda.synchronize()
            us = ev0.elapsed_time(ev1) * 1e3 / iters
            gbs = (wbytes + M * (K + N) * 2) / us / 1e3
            print(json.dumps(dict(shape=name, linear=lin, N=N, K=K, M=M, us=round(us, 2), gb_s=round(gbs, 1),
                                  share_of_3_35_tb_s=round(gbs / (HBM_TBS * 1e3), 3), **info)), flush=True)
        del ws


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--shapes", nargs="*", default=list(SHAPES), choices=list(SHAPES))
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--workloads", nargs="*", default=["full", "varied"], choices=["full", "varied"])
    ap.add_argument("--stop-scale", type=float, default=4.0, help="varied workload: factor on the stop token's embedding row")
    ap.add_argument("--kernel", action="store_true", help="time ymp_gemm_skinny_wide per decoder linear and M")
    ap.add_argument("--counts", action="store_true", help="print the counted bytes only (no GPU)")
    ap.add_argument("--profile", action="store_true", help="device-time shares of one batched 12-clip, 40-token call per "
                                                           "batched arm (torch.profiler)")
    args = ap.parse_args()
    if args.counts:
        for s in args.shapes:
            print(json.dumps(dict(shape=s, **counts(s))))
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("caption_generate.py times the H100 kernels: no CUDA device found")
    for s in args.shapes:
        if args.kernel:
            kernel(s)
            continue
        model, vis = build(s, torch.device("cuda:0"))
        if args.profile:
            profile(model, vis, s)
        else:
            for w in args.workloads:
                run(model, vis, s, args.rounds, w, args.stop_scale)
        del model
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
