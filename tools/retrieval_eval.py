"""Time the retrieval evaluation's text features with and without padding rows: DistributedGPT3_Retrieval
extract_text_feature at the retrieval yamls' eval shape.

    python tools/retrieval_eval.py [--models 1.3B 2.7B] [--chunks 8] [--rounds 3] [--counts]

The evaluation (downstream/run_retrieval_distributed_gpt3.py) encodes its texts in chunks of 32, each padded to
max(64, max_length) = 80 tokens.  Each model builds the yaml's DistributedGPT3_Retrieval with its full decoder and random
bf16 weights (eval mode) and times two arms on the same chunks, alternating in one process after a warm-up round of each,
every timed call ending in a device synchronise:
  padded - the training-step pass over the padded texts (decoder, tied LM head and per-token CE on every row), then the
           pooled row (DistributedGPT3_Retrieval._pooled_text_padded);
  packed - extract_text_feature: the texts packed back to back, no padding rows and no LM head.
Length sets: all 80 tokens, and lengths U[8, 80] from a fixed seed.  One JSON line per (model, length set): card name,
power limit and max SM clock, median ms per chunk of each arm over --rounds rounds of --chunks chunks, peak allocated
memory of each arm above what the model holds, decoder rows per chunk, and whether the two arms' features are bit-equal
(asserted).  --counts prints the decoder rows and the work counted from shapes, without a GPU.
"""
import argparse
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

B, L = 32, 80   # texts per chunk (text_bs) and their padded length max(64, max_length) of the retrieval yamls
MODELS = {"1.3B": "config_gpt3_1.3B.json", "2.7B": "config_gpt3_2.7B.json"}
LENGTHS = ("all80", "uniform8_80")


def gpt_cfg(name):
    with open(os.path.join(PKG, "configs", "models", MODELS[name])) as f:
        return json.load(f)


def make_chunk(vocab, lengths, seed):
    """input_ids / attention_mask [B, L] (CPU) of one chunk: bos, random ids, right padding with 0."""
    import torch
    g = torch.Generator().manual_seed(seed)
    lens = torch.full((B,), L) if lengths == "all80" else torch.randint(8, L + 1, (B,), generator=g)
    att = (torch.arange(L)[None, :] < lens[:, None]).long()
    ids = torch.randint(3, vocab, (B, L), generator=g)
    ids[:, 0] = 1
    return dict(input_ids=torch.where(att.bool(), ids, torch.zeros_like(ids)), attention_mask=att)


def counts(name, lengths, chunks=1):
    """Decoder rows and work per chunk (averaged over `chunks` chunks): layer GEMMs 24 h^2 flop per row per layer
    (QKV 6, dense 2, MLP 16), tied LM head 2 h V per row (the padded pass runs it on every padded row, the packed one
    not at all)."""
    from ymp import functional as YF
    g = gpt_cfg(name)
    h, layers, vocab = g["hidden_size"], g["num_hidden_layers"], g["vocab_size"]
    packed = sum(int(YF.packed_text_rows(make_chunk(vocab, lengths, 100 + c)["attention_mask"])[0][-1])
                 for c in range(chunks)) / chunks
    padded = B * L
    return dict(model=name, lengths=lengths, texts=B, padded_len=L, rows_padded=padded, rows_packed=packed,
                layer_tf_padded=round(24 * h * h * padded * layers / 1e12, 4),
                layer_tf_packed=round(24 * h * h * packed * layers / 1e12, 4),
                lm_head_tf_padded=round(2 * h * vocab * padded / 1e12, 4), lm_head_tf_packed=0.0)


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
    td = make_model_dir(vis, gpt_cfg(name), dropout=(0.1, 0.1))   # the shipped decoder's dropout (off in eval mode)
    torch.manual_seed(0)
    with torch.device(dev):
        model = D.DistributedGPT3_Retrieval(config=pretrain_config(td, 128, num_frames=4, contrastive_embed_dim=256),
                                            tokenizer=None)
    return model.to(torch.bfloat16).eval()


def run(model, name, lengths, chunks, rounds):
    import torch
    import torch.nn.functional as F
    import models.modeling_distributed_gpt3 as G
    dev = torch.device("cuda:0")
    vocab = gpt_cfg(name)["vocab_size"]
    texts = [G.BatchEncoding({k: v.to(dev) for k, v in make_chunk(vocab, lengths, 100 + c).items()}) for c in range(chunks)]
    arms = dict(padded=lambda t: F.normalize(model.text_proj(model._pooled_text_padded(t)).float(), dim=-1),
                packed=model.extract_text_feature)
    ms = {a: [] for a in arms}
    peak = {a: 0 for a in arms}
    outs = {}
    with torch.no_grad():
        for r in range(rounds + 1):   # round 0 warms up both arms
            for a, fn in arms.items():
                outs[a] = None
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                t0 = time.perf_counter()
                outs[a] = [fn(t) for t in texts]
                torch.cuda.synchronize()
                dt = (time.perf_counter() - t0) * 1e3 / chunks
                if r > 0:
                    ms[a].append(dt)
                    peak[a] = max(peak[a], torch.cuda.max_memory_allocated() - base)
    equal = all(torch.equal(x, y) for x, y in zip(outs["padded"], outs["packed"]))
    res = dict(model=name, lengths=lengths, chunks=chunks, **card_info())
    for a in arms:
        res[f"{a}_ms_per_chunk"] = round(statistics.median(ms[a]), 3)
        res[f"{a}_ms_all"] = [round(x, 3) for x in ms[a]]
        res[f"{a}_peak_gb"] = round(peak[a] / 1e9, 3)
    res["speedup"] = round(res["padded_ms_per_chunk"] / res["packed_ms_per_chunk"], 3)
    res["bit_equal"] = bool(equal)
    res["counts"] = counts(name, lengths, chunks)
    print(json.dumps(res), flush=True)
    assert equal, "the packed and padded text features differ"
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--models", nargs="*", default=list(MODELS), choices=list(MODELS))
    ap.add_argument("--chunks", type=int, default=8, help="chunks of 32 texts per timed round")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--counts", action="store_true", help="print the counted rows and work only (no GPU)")
    args = ap.parse_args()
    if args.counts:
        for m in args.models:
            for lengths in LENGTHS:
                print(json.dumps(counts(m, lengths, args.chunks)))
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("retrieval_eval.py times the H100 kernels: no CUDA device found")
    for m in args.models:
        model = build(m, torch.device("cuda:0"))
        for lengths in LENGTHS:
            run(model, m, lengths, args.chunks, args.rounds)
        del model
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
