"""Replay the ITM retrieval evaluation's text-chunk loop and time the eval calls with and without the prefix cache.

    python tools/itm_eval.py [--shapes itm_1.3B cls_1.3B ...] [--chunks 4] [--rounds 2] [--counts]

downstream/run_retrieval_distributed_gpt3_itm.py (`evaluation`) moves one video batch to the device and scores it
against all test texts in chunks of 8, one model(video, text, prompt_text, train=False) call per chunk on the same
clip tensor.  Each ITM shape builds DistributedGPT3_Retrieval_Cls with random bf16 weights at the shipped yaml's shape
(96 videos at 1.3B, 64 at 2.7B, 4 frames, 128 queries, 80-token texts) and runs that loop over --chunks chunks of fresh
random texts per arm, the arms alternating in one process after a warm-up loop of each:
  current - what every eval call did before the prefix cache: the visual encoder, then the generation and the cls pass,
            each computing the video prefixes through every decoder layer (the shared passes without a PrefixKV);
  cached  - model(..., train=False): the first chunk runs the encoder, its generation pass computes the prefixes and
            keeps their keys and values (a PrefixKV) that its cls pass reads; the later chunks reuse the clip's query
            features and PrefixKV.
The Cls shapes (3 / 2 videos x 45 title-structured class prompts, 8 frames) make one call per video batch, so only
the sharing within a call applies there: one loop of one chunk per arm, the cache dropped before each call.
One JSON line per shape: card name, power limit and max SM clock (read in the same process), per arm the ms of the
first chunk, the median ms of the later ones, the whole loop's ms and peak allocated memory (medians over --rounds
loops), and whether the two arms' outputs are bit-equal in every row of every chunk.  --counts prints, without a GPU,
the decoder rows, the prefix rows among them, and the encoder GEMM GFLOP of one call per arm and chunk position.
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import eval_prefix as EP  # noqa: E402  (model shapes, builder, text makers and card query shared with that tool)

Q, L = EP.Q, EP.L
SHAPES = ("itm_1.3B", "itm_2.7B", "cls_1.3B", "cls_2.7B")


def chunk_texts(name, c):
    """(text, prompt_text) dicts of chunk c (CPU tensors): ITM pairs of 80-token texts, fresh per chunk; the Cls shapes'
    title-structured class prompts."""
    if name.startswith("cls"):
        return EP.make_texts(name, "titles")
    _, _, _, V, t = EP.SHAPES[name]
    vocab = EP.gpt_cfg(name)["vocab_size"]
    return EP.make_text(V * t, vocab, L, 10 + c, True), EP.make_text(V * t, vocab, L, 1000 + c, False)


def encoder_gflop(name):
    """GEMM GFLOP of one call's visual side, counted from shapes: per TimeSformer block and token, the temporal and
    spatial attention in / out projections, temporal_fc and the MLP (34 D^2 flop); the patch embedding; visual_fc
    (2 D H per query).  The attention products and the abstractor are not counted."""
    with open(os.path.join(EP.PKG, "configs", "models", "clip-b16.json")) as f:
        vis = json.load(f)
    _, _, frames, V, _ = EP.SHAPES[name]
    D, P, depth = vis["embed_dim"], vis["patch_size"], vis["depth"]
    tokens = V * frames * (vis["img_size"] // P) ** 2
    flop = tokens * (2 * 3 * P * P * D + depth * 34 * D * D) + 2 * V * Q * D * EP.gpt_cfg(name)["hidden_size"]
    return flop / 1e9


def call_counts(name, c):
    """Decoder rows of one eval call at chunk c per arm: (rows, prefix rows) of the current and the cached arm, with the
    cached arm's prefix rows those of its generation pass (first chunk) or none (later chunks of the ITM loop)."""
    import torch
    from models.distributed_gpt3 import build_targets, mask_prompt, shared_text_columns
    from ymp import functional as YF
    _, _, _, V, t = EP.SHAPES[name]
    text, prompt = chunk_texts(name, c)
    _, loss_mask = build_targets(text["input_ids"], mask_prompt(text["attention_mask"][:, 1:].clone(), text["prompt_lengths"]), Q)
    passes = [(text, torch.nn.functional.pad(loss_mask[:, Q:], (0, 1)))]
    att = prompt["attention_mask"]
    passes.append((prompt, torch.arange(L)[None, :] == att.sum(-1, keepdim=True) - 1))   # the cls pass reads one column
    own = 0
    for d, read in passes:
        shared, used = shared_text_columns(d["input_ids"], d["attention_mask"], read, V)
        _, Ls, Pmax = YF.shared_title_layout(V, max(used), shared, used)
        own += d["input_ids"].shape[0] * Ls + V * Pmax
    first = name.startswith("cls") or c == 0
    return dict(current=(own + 2 * V * Q, 2 * V * Q), cached=(own + (V * Q if first else 0), V * Q if first else 0))


def print_counts(shapes, chunks):
    print(f"{'shape':10s} {'arm':8s} {'call':6s} {'decoder_rows':>12s} {'prefix_rows':>11s} {'encoder_gflop':>13s}")
    for name in shapes:
        enc = encoder_gflop(name)
        for c in ([0] if name.startswith("cls") else [0, 1]):
            cc = call_counts(name, c)
            for arm in ("current", "cached"):
                rows, prefix = cc[arm]
                e = enc if (arm == "current" or c == 0) else 0
                print(f"{name:10s} {arm:8s} {'first' if c == 0 else 'later':6s} {rows:12d} {prefix:11d} {round(e):13d}")
        if not name.startswith("cls"):
            print(f"{name:10s} (the later-chunk rows hold for every chunk after the first; {chunks} chunks per loop)")


def current_call(model, video, text, prompt_text):
    """The eval branch as it ran before the prefix cache: encoder, then both shared passes computing the prefixes."""
    _, _, _, qf = model.visual_prefix(video)
    V = qf.shape[0]
    t = text.input_ids.shape[0] // V
    losses, loss_mask = model._gen_pass_shared(qf, text)
    gen = (-(losses * loss_mask).sum(dim=-1)).view(V, t)
    cls = model._cls_pass_shared(qf, prompt_text)
    if type(model).__name__ == "DistributedGPT3_Cls":
        return gen.softmax(dim=-1), cls
    return gen, cls.float().softmax(dim=-1)[:, 1].view(V, t)


def run(name, chunks, rounds):
    import torch
    import models.modeling_distributed_gpt3 as G
    dev = torch.device("cuda:0")
    model, vis = EP.build(name, dev)
    _, gjson, frames, V, t = EP.SHAPES[name]
    is_cls = name.startswith("cls")
    n_chunks = 1 if is_cls else chunks

    def enc(d):
        return G.BatchEncoding({k: v.to(dev) for k, v in d.items()})

    texts = [tuple(enc(d) for d in chunk_texts(name, c)) for c in range(n_chunks)]
    video = torch.randn(V, 3, frames, vis["img_size"], vis["img_size"], generator=torch.Generator().manual_seed(1)).to(dev).bfloat16()

    def cached_call(video, text, prompt_text):
        if is_cls:
            model._prefix_cache = None   # a Cls batch is scored in one call: nothing to reuse across calls
        return model(video, text, prompt_text, train=False)

    arms = dict(current=lambda tx: current_call(model, video, *tx), cached=lambda tx: cached_call(video, *tx))
    stats = {a: dict(first=[], later=[], loop=[], peak=[]) for a in arms}
    outs = {}
    with torch.no_grad():
        for r in range(rounds + 1):   # round 0 warms up both arms
            for a, fn in arms.items():
                model._prefix_cache = None   # each loop starts on a new video batch
                outs[a] = None
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                per, res = [], []
                t_loop = time.perf_counter()
                for tx in texts:
                    t0 = time.perf_counter()
                    res.append(fn(tx))
                    torch.cuda.synchronize()
                    per.append((time.perf_counter() - t0) * 1e3)
                loop_ms = (time.perf_counter() - t_loop) * 1e3
                outs[a] = res
                if r > 0:
                    s = stats[a]
                    s["first"].append(per[0])
                    s["later"] += per[1:]
                    s["loop"].append(loop_ms)
                    s["peak"].append(torch.cuda.max_memory_allocated() - base)
    model._prefix_cache = None
    equal = all(torch.equal(x, y) for ca, cb in zip(outs["current"], outs["cached"]) for x, y in zip(ca, cb))
    res = dict(shape=name, videos=V, texts_per_video=t, frames=frames, chunks=n_chunks, decoder=gjson, **EP.card_info())
    for a, s in stats.items():
        res[f"{a}_first_ms"] = round(statistics.median(s["first"]), 2)
        res[f"{a}_later_ms"] = round(statistics.median(s["later"]), 2) if s["later"] else None
        res[f"{a}_loop_ms"] = round(statistics.median(s["loop"]), 2)
        res[f"{a}_peak_gb"] = round(max(s["peak"]) / 1e9, 3)
    res["loop_speedup"] = round(res["current_loop_ms"] / res["cached_loop_ms"], 3)
    res["bit_equal"] = bool(equal)
    print(json.dumps(res), flush=True)
    del model
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--shapes", nargs="*", default=list(SHAPES), choices=list(SHAPES))
    ap.add_argument("--chunks", type=int, default=4, help="text chunks per ITM video batch (at least 2)")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--counts", action="store_true", help="print the counted rows and encoder work only (no GPU)")
    args = ap.parse_args()
    if args.chunks < 2:
        ap.error("--chunks must be at least 2: the later chunks are what the cache serves")
    if args.counts:
        print_counts(args.shapes, args.chunks)
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("itm_eval.py times the H100 kernels: no CUDA device found")
    for s in args.shapes:
        run(s, args.chunks, args.rounds)


if __name__ == "__main__":
    main()
