"""Fixed cost per output tile of the wgmma GEMM: µs per wave = k_blocks x t + f, fitted per launch class.

    python tools/gemm_tile_cost.py [--root TREE [TREE ...]] [--tile-n 256 [128]] [--tile-m 128 [192]] [--rounds 3]
                                   [--json OUT]

A launch runs ceil(units / SMs) waves of tile_m x tile_n tiles, one CTA per SM.  For each launch class (M, N, operand
layouts and epilogue of a launch of the training step, DESIGN.md §5) `ops.gemm` is timed at K = 64, 256, 768, 2048 and
8192 (1 to 128 k-blocks of 64), warm, with CUDA events over enough repeats for at least 0.2 s per point, and
time / waves is fitted by least squares to k_blocks x t + f: t is the cost of one tile's k-block of MMAs, f what a tile
costs whatever its K (pipeline fill, epilogue, turnover between tiles).  Every tile shape of --tile-n x --tile-m (192
rows only with 256 columns) is an arm; the arms alternate at every point.  The classes:

    the ViT's fc1 (GELU, act' stored), its dgrad (B MN-major, x act'), qkv (plain bf16), proj / fc2 (fp32 residual; one
    class, they differ in K only), GPT h->4h (GELU, act' stored), 4h->h (fp32 residual), its dgrad (B MN-major), the LM
    head (plain bf16), and one wgrad (both operands MN-major, fp32 accumulate, split_k = 1).

Every --root is a built repository tree; each is measured in a process of its own (they hold different builds of the
same library), the trees alternate --rounds times, and the medians over the rounds are fitted.  Card name, power limit
and maximum SM clock are printed with the table.  Needs a GPU.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(HERE, "tools"))
from gemm_ab import card_info, time_fn  # noqa: E402

KS = (64, 256, 768, 2048, 8192)
BK = 64
# name, M, N, a_t, b_t, epilogue
CLASSES = [
    ("vit fc1: GELU, act' stored", 50208, 3072, 0, 0, "gelu_aux"),
    ("vit fc1 dgrad: B MN-major, x act'", 50208, 3072, 0, 1, "mul"),
    ("vit qkv: plain bf16", 50208, 2304, 0, 0, "plain"),
    ("vit proj / fc2: fp32 residual", 50208, 768, 0, 0, "res32"),
    ("gpt h->4h: GELU, act' stored", 8192, 8192, 0, 0, "gelu_aux"),
    ("gpt 4h->h: fp32 residual", 8192, 2048, 0, 0, "res32"),
    ("gpt 4h->h dgrad: B MN-major", 8192, 2048, 0, 1, "plain"),
    ("lm head: plain bf16", 4096, 51200, 0, 0, "plain"),
    ("wgrad: A, B MN-major, fp32 accumulate", 8192, 2048, 1, 1, "acc"),
]


def waves(M, N, sms, bm, bn):
    return -(-(-(-M // bm) * -(-N // bn)) // sms)


def fit(kbs, ys):
    """Least squares y = kb t + f; returns t, f and the rms residual."""
    n = len(kbs)
    mx, my = sum(kbs) / n, sum(ys) / n
    t = sum((x - mx) * (y - my) for x, y in zip(kbs, ys)) / sum((x - mx) ** 2 for x in kbs)
    f = my - t * mx
    return t, f, math.sqrt(sum((y - (x * t + f)) ** 2 for x, y in zip(kbs, ys)) / n)


def worker(root, out_path, min_s, arms):
    for p in (root, os.path.join(root, "youku-mplug_b200")):
        sys.path.insert(0, p)
    import torch
    if not torch.cuda.is_available():
        sys.exit("gemm_tile_cost.py needs a GPU")
    from ymp import ops
    dev = torch.device("cuda")
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    g = torch.Generator(device=dev).manual_seed(5)
    res = []
    for name, M, N, a_t, b_t, epi in CLASSES:
        us = {arm: [] for arm in arms}
        for K in KS:
            rnd = lambda *s: (torch.randn(*s, device=dev, generator=g) / K ** 0.25).to(torch.bfloat16)  # noqa: E731
            a = rnd(K, M) if a_t else rnd(M, K)
            b = rnd(K, N) if b_t else rnd(N, K)
            kw = dict(a_t=bool(a_t), b_t=bool(b_t))
            f32 = epi in ("res32", "acc")
            kw["out"] = torch.zeros(M, N, device=dev, dtype=torch.float32 if f32 else torch.bfloat16)
            if epi == "gelu_aux":
                kw.update(act=ops.ACT_GELU_ERF, aux_out=torch.empty(M, N, device=dev, dtype=torch.bfloat16))
            elif epi == "mul":
                kw["aux_in"] = rnd(M, N)
            elif epi == "res32":
                kw["residual"] = torch.randn(M, N, device=dev, generator=g)
            elif epi == "acc":
                kw.update(accumulate=True, split_k=1)
            for bm, bn in arms:
                fn = lambda: ops.gemm(a, b, tile_m=bm, tile_n=bn, **kw)  # noqa: E731
                est = time_fn(fn, 3) * 1e-6
                us[(bm, bn)].append(time_fn(fn, max(5, int(min_s / est) + 1)))
            del a, b, kw, fn
            torch.cuda.empty_cache()
        res.append(dict(name=name, M=M, N=N, arms={f"{bm}x{bn}": dict(waves=waves(M, N, sms, bm, bn), us=us[(bm, bn)])
                                                  for bm, bn in arms}))
    with open(out_path, "w") as fh:
        json.dump(dict(root=root, sms=sms, classes=res), fh)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--root", nargs="+", default=[HERE], help="built repository trees to measure, alternated")
    ap.add_argument("--tile-n", type=int, nargs="+", default=[256], choices=(128, 256))
    ap.add_argument("--tile-m", type=int, nargs="+", default=[128], choices=(128, 192))
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--min-seconds", type=float, default=0.2, help="timed window per (class, K) point")
    ap.add_argument("--json", default=None, help="also write the samples and fits as json")
    ap.add_argument("--worker", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    arms = [(bm, bn) for bn in args.tile_n for bm in args.tile_m if bm == 128 or bn == 256]
    if args.worker:
        return worker(os.path.abspath(args.root[0]), args.worker, args.min_seconds, arms)

    import tempfile
    import torch
    if not torch.cuda.is_available():
        sys.exit("gemm_tile_cost.py needs a GPU")
    info = card_info()
    roots = [os.path.abspath(r) for r in args.root]
    samples = {r: [] for r in roots}
    with tempfile.TemporaryDirectory(prefix="gemm_tile_cost_") as td:
        for rnd in range(args.rounds):
            for r in roots:
                out = os.path.join(td, f"r{rnd}.json")
                subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", out, "--root", r,
                                "--min-seconds", str(args.min_seconds), "--tile-n", *map(str, args.tile_n),
                                "--tile-m", *map(str, args.tile_m)], check=True)
                with open(out) as fh:
                    samples[r].append(json.load(fh))
    print(f"# {info['name']}, power limit {info['power_limit']}, max SM clock {info['max_sm_clock']}; "
          f"K = {', '.join(map(str, KS))}; medians of {args.rounds} rounds; µs per wave = k_blocks x t + f")
    kbs = [K // BK for K in KS]
    result = dict(card=info, ks=KS, roots={})
    for r in roots:
        print(f"\n## {r}")
        print(f"{'class':40s} {'M':>6s} {'N':>6s} tile    waves " + " ".join(f"K={K:<5d}us" for K in KS)
              + "   t_us    f_us  resid_us")
        rows = []
        for i, (name, M, N, *_rest) in enumerate(CLASSES):
            for bm, bn in arms:
                arm = f"{bm}x{bn}"
                got = [s["classes"][i]["arms"][arm] for s in samples[r]]
                w = got[0]["waves"]
                us = [statistics.median(g["us"][j] for g in got) for j in range(len(KS))]
                t, f, resid = fit(kbs, [u / w for u in us])
                print(f"{name:40s} {M:6d} {N:6d} {arm:7s} {w:5d} " + " ".join(f"{u:9.1f}" for u in us)
                      + f" {t:6.3f} {f:7.2f} {resid:9.2f}")
                rows.append(dict(name=name, M=M, N=N, tile=arm, waves=w, us=us, t_us=t, f_us=f, resid_us=resid,
                                 samples_us=[g["us"] for g in got]))
        result["roots"][r] = rows
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
