"""Time the shared-prefix evaluation against the repeated one: DistributedGPT3_Cls and DistributedGPT3_Retrieval_Cls
eval calls at the shipped yamls' shapes.

    python tools/eval_prefix.py [--shapes cls_1.3B itm_2.7B ...] [--rounds 3] [--counts]

Each shape builds the yaml's model class with random bf16 weights (eval mode, 128 queries, the yaml's frame count) and
times one eval model(...) call per arm, the arms alternating in one process after a warm-up call of each, every
call ending in a device synchronise:
  repeated    - every video's query features copied once per text, then _gen_pass / _cls_pass;
  prefix_only - every text against one copy of its video's prefix, each text's own columns all computed
                (forward_shared_prefix without shared_cols);
  shared      - model(..., train=False): one copy of the prefix and of the text columns a video's texts have in common.
Text shapes: all 80 tokens; uniform lengths in [16, 80]; and (Cls shapes) `titles`: per video a title prompt of
U[12, 60] tokens, its t class labels of 1-4 tokens and eos, padded to 80, laid out as
DistributedGPT3Tokenizer._fit_prompt does.  One JSON line per (shape, text shape): card name, power limit and max SM
clock, median ms per call, peak allocated memory of each arm (of the whole call, and of its decoder passes: from the
end of the visual prefix, which every arm computes alike), the decoder rows of each arm's generation pass, and whether
the arms' outputs are bit-equal.  --counts prints the decoder rows and GEMM work counted from shapes, and the rows of
each arm per text shape, without a GPU.
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

Q, L = 128, 80   # num_learnable_token and max_length of the four yamls
# name: (model class, decoder json, frames, videos per call, texts per video).  Cls: the reference's validation batch
# (3 / 2 videos) x 45 class prompts; ITM: run_retrieval_distributed_gpt3_itm.py scores 96 / 64 videos x 8 texts.
SHAPES = {
    "cls_1.3B": ("DistributedGPT3_Cls", "config_gpt3_1.3B.json", 8, 3, 45),
    "cls_2.7B": ("DistributedGPT3_Cls", "config_gpt3_2.7B.json", 8, 2, 45),
    "itm_1.3B": ("DistributedGPT3_Retrieval_Cls", "config_gpt3_1.3B.json", 4, 96, 8),
    "itm_2.7B": ("DistributedGPT3_Retrieval_Cls", "config_gpt3_2.7B.json", 4, 64, 8),
}


def gpt_cfg(name):
    with open(os.path.join(PKG, "configs", "models", SHAPES[name][1])) as f:
        return json.load(f)


def counts(name):
    """Decoder rows and work of one eval call's generation pass, before any column is trimmed: layer GEMMs
    24 h^2 flop per row per layer (QKV 6, dense 2, MLP 16), LM head 2 h V per text row (the repeated pass computes it on
    the prefix rows too)."""
    g = gpt_cfg(name)
    _, _, _, V, t = SHAPES[name]
    h, layers, vocab = g["hidden_size"], g["num_hidden_layers"], g["vocab_size"]
    N = V * t
    rows_rep, rows_sh = N * (Q + L), N * L + V * Q
    return dict(sequences=N, rows_repeated=rows_rep, rows_shared=rows_sh,
                layer_tf_repeated=24 * h * h * rows_rep * layers / 1e12, layer_tf_shared=24 * h * h * rows_sh * layers / 1e12,
                lm_head_tf_repeated=2 * h * vocab * rows_rep / 1e12, lm_head_tf_shared=2 * h * vocab * N * L / 1e12)


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
    cls, _, frames, _, _ = SHAPES[name]
    with open(os.path.join(PKG, "configs", "models", "clip-b16.json")) as f:
        vis = json.load(f)
    td = make_model_dir(vis, gpt_cfg(name), dropout=(0.1, 0.1))
    torch.manual_seed(0)
    with torch.device(dev):
        model = getattr(D, cls)(config=pretrain_config(td, Q, num_frames=frames, use_cls=True, num_classes=45), tokenizer=None)
    return model.to(torch.bfloat16).eval(), vis


def make_text(n, vocab, lo, seed, prompt):
    import torch
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(3, vocab, (n, L), generator=g)
    ids[:, 0] = 1
    lens = torch.randint(lo, L + 1, (n,), generator=g)
    att = (torch.arange(L)[None, :] < lens[:, None]).long()
    ids = torch.where(att.bool(), ids, torch.zeros_like(ids))
    d = dict(input_ids=ids, attention_mask=att)
    if prompt:
        d["prompt_lengths"] = torch.minimum(torch.randint(1, 12, (n,), generator=g), lens - 1)
    return d


def make_titles(V, t, vocab, seed, cls):
    """The `titles` text shape: (text, prompt_text) dicts.  Video v's texts are [bos | title prompt | label | eos] for the
    t class labels (one class list for every video), prompt_lengths as _fit_prompt sets them; prompt_text is
    [bos | title prompt | eos], one row per video (Cls) or per pair (ITM)."""
    import torch
    g = torch.Generator().manual_seed(seed)
    labels = [torch.randint(3, vocab, (int(torch.randint(1, 5, (1,), generator=g)),), generator=g).tolist() for _ in range(t)]
    ids, plen, pids = [], [], []
    for _ in range(V):
        prompt = torch.randint(3, vocab, (int(torch.randint(12, 61, (1,), generator=g)),), generator=g).tolist()
        for lab in labels:
            pr = prompt[:L - len(lab) - 2] if 2 + len(prompt) + len(lab) > L else prompt
            ids.append([1] + pr + lab + [2])
            plen.append(len(pr))
        pids += [([1] + prompt + [2])[:L]] * (1 if cls == "DistributedGPT3_Cls" else t)

    def pad(rows):
        return dict(input_ids=torch.tensor([r + [0] * (L - len(r)) for r in rows]),
                    attention_mask=torch.tensor([[1] * len(r) + [0] * (L - len(r)) for r in rows]))
    return dict(pad(ids), prompt_lengths=torch.tensor(plen)), pad(pids)


def make_texts(name, lengths):
    """(text, prompt_text) dicts of one text shape (CPU tensors)."""
    cls, _, _, V, t = SHAPES[name]
    vocab = gpt_cfg(name)["vocab_size"]
    if lengths == "titles":
        return make_titles(V, t, vocab, 2, cls)
    lo = L if lengths == "all80" else 16
    n_prompt = V if cls == "DistributedGPT3_Cls" else V * t   # Cls: one cls prompt per video; ITM: one per pair
    return make_text(V * t, vocab, lo, 2, True), make_text(n_prompt, vocab, lo, 3, False)


def text_shapes(name):
    return ("all80", "uniform16_80") + (("titles",) if SHAPES[name][0] == "DistributedGPT3_Cls" else ())


def arm_rows(name, lengths):
    """Decoder rows of each arm's generation pass at one text shape (the same host arithmetic as the model)."""
    from models.distributed_gpt3 import build_targets, mask_prompt, shared_text_columns
    from ymp import functional as YF
    import torch
    _, _, _, V, t = SHAPES[name]
    text, _ = make_texts(name, lengths)
    _, loss_mask = build_targets(text["input_ids"], mask_prompt(text["attention_mask"][:, 1:].clone(), text["prompt_lengths"]), Q)
    shared, used = shared_text_columns(text["input_ids"], text["attention_mask"], torch.nn.functional.pad(loss_mask[:, Q:], (0, 1)), V)
    _, Ls, Pmax = YF.shared_title_layout(V, max(used), shared, used)
    N = V * t
    return dict(rows_repeated=N * (Q + L), rows_prefix_only=N * max(used) + V * Q, rows_shared=N * Ls + V * (Q + Pmax),
                shared_cols_min=min(shared), shared_cols_max=Pmax)


def prefix_only_call(model, video, text, prompt_text):
    """The eval branch with every text against one copy of its video's prefix and all of its own columns computed:
    forward_shared_prefix without shared_cols, composed as the model's shared passes are."""
    import torch
    from models.distributed_gpt3 import build_targets, mask_prompt, used_columns
    _, _, _, qf = model.visual_prefix(video)
    V, Q_ = qf.shape[:2]
    N, Lt = text.input_ids.shape
    t = N // V
    dec, wemb = model.text_decoder, model._word_embedding()
    targets, loss_mask = build_targets(text.input_ids, mask_prompt(text.attention_mask[:, 1:].clone(), text.prompt_lengths), Q_)
    Le = used_columns(text.attention_mask)
    out = dec.forward_shared_prefix(qf, wemb(text.input_ids[:, :Le]).to(qf.dtype), labels=targets[:, Q_:Q_ + Le])
    losses = torch.zeros((N, Q_ + Lt), device=qf.device, dtype=torch.float32)
    losses[:, Q_:Q_ + Le] = out.losses
    gen = (-(losses[:, :-1] * loss_mask).sum(dim=-1)).view(V, t)
    att = prompt_text.attention_mask
    Lp = used_columns(att)
    rows = torch.arange(att.shape[0], device=att.device) * Lp + att.sum(dim=-1) - 1
    cls = model.cls_head(dec.forward_shared_prefix(qf, wemb(prompt_text.input_ids[:, :Lp]).to(qf.dtype), hidden_rows=rows).hidden)
    if type(model).__name__ == "DistributedGPT3_Cls":
        return gen.softmax(dim=-1), cls
    return gen, cls.float().softmax(dim=-1)[:, 1].view(V, t)


def repeated_call(model, video, text, prompt_text):
    """The eval branch with every video's query features copied once per text (the composition before the shared pass)."""
    _, _, _, qf = model.visual_prefix(video)
    V = qf.shape[0]
    t = text.input_ids.shape[0] // V
    qr = qf.repeat_interleave(t, dim=0)
    out, loss_mask = model._gen_pass(qr, text)
    gen = (-(out.losses * loss_mask).sum(dim=-1)).view(V, t)
    if type(model).__name__ == "DistributedGPT3_Cls":
        return gen.softmax(dim=-1), model._cls_pass(qf, prompt_text, False)
    return gen, model._cls_pass(qr, prompt_text, False).float().softmax(dim=-1)[:, 1].view(V, t)


def run(model, vis, name, rounds, lengths):
    import torch
    import models.modeling_distributed_gpt3 as G
    dev = torch.device("cuda:0")
    cls, gjson, frames, V, t = SHAPES[name]

    def enc(d):
        return G.BatchEncoding({k: v.to(dev) for k, v in d.items()})

    video = torch.randn(V, 3, frames, vis["img_size"], vis["img_size"], generator=torch.Generator().manual_seed(1)).to(dev).bfloat16()
    text, prompt_text = (enc(d) for d in make_texts(name, lengths))
    arms = dict(repeated=lambda: repeated_call(model, video, text, prompt_text),
                prefix_only=lambda: prefix_only_call(model, video, text, prompt_text),
                shared=lambda: model(video, text, prompt_text, train=False))
    ms = {a: [] for a in arms}
    peak = {a: 0 for a in arms}
    dec_peak = {a: 0 for a in arms}
    outs = {}
    vis = {}
    visual_prefix = model.visual_prefix

    def visual_prefix_then_reset(video):
        """Both arms call this: the peak of the visual side (common to the arms) is taken here and the counter restarts,
        so that what follows is the decoder passes' own peak."""
        out = visual_prefix(video)
        torch.cuda.synchronize()
        vis["peak"] = torch.cuda.max_memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        return out

    model.visual_prefix = visual_prefix_then_reset
    with torch.no_grad():
        for r in range(rounds + 1):   # round 0 warms up both arms
            for a, fn in arms.items():
                outs[a] = None
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                t0 = time.perf_counter()
                outs[a] = fn()
                torch.cuda.synchronize()
                dt = (time.perf_counter() - t0) * 1e3
                if r > 0:
                    ms[a].append(dt)
                    dec = torch.cuda.max_memory_allocated()
                    peak[a] = max(peak[a], vis["peak"] - base, dec - base)
                    dec_peak[a] = max(dec_peak[a], dec - base)
    del model.visual_prefix
    equal = all(torch.equal(x, y) for a in ("prefix_only", "shared") for x, y in zip(outs["repeated"], outs[a]))
    res = dict(shape=name, lengths=lengths, videos=V, texts_per_video=t, frames=frames, decoder=gjson, **card_info())
    for a in arms:
        res[f"{a}_ms"] = round(statistics.median(ms[a]), 2)
        res[f"{a}_ms_all"] = [round(x, 2) for x in ms[a]]
        res[f"{a}_peak_gb"] = round(peak[a] / 1e9, 3)
        res[f"{a}_decoder_peak_gb"] = round(dec_peak[a] / 1e9, 3)
    res["speedup"] = round(res["repeated_ms"] / res["shared_ms"], 3)
    res["speedup_vs_prefix_only"] = round(res["prefix_only_ms"] / res["shared_ms"], 3)
    res["bit_equal"] = bool(equal)
    res["counts"] = counts(name)
    res["rows"] = arm_rows(name, lengths)
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--shapes", nargs="*", default=list(SHAPES), choices=list(SHAPES))
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--counts", action="store_true", help="print the counted rows and work only (no GPU)")
    args = ap.parse_args()
    if args.counts:
        for s in args.shapes:
            print(json.dumps(dict(shape=s, **counts(s))))
            for lengths in text_shapes(s):
                print(json.dumps(dict(shape=s, lengths=lengths, **arm_rows(s, lengths))))
        return
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("eval_prefix.py times the H100 kernels: no CUDA device found")
    for s in args.shapes:
        model, vis = build(s, torch.device("cuda:0"))
        for lengths in text_shapes(s):
            run(model, vis, s, args.rounds, lengths)
        del model
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
