"""Per-shape timing of the GEMM launches of one training step, next to cuBLAS on the same operands.

    python tools/gemm_ab.py [--configs pretrain caption27b retrieval] [--reports-dir DIR] [--arms 0] [--json OUT]

The distinct launches (shape, operand layouts, epilogue flags) come from `bench.py --gemm-report` of each config:
DIR/gemm_<config>.json is read when it exists, otherwise bench.py is run once (1 step) to write it.  Every launch is
then rebuilt on seeded random operands and timed through `ops.gemm` with CUDA events, once per arm in --arms (an arm
is `tile_n` or `tile_n:tile_m`, e.g. `0,256:128,256:192`; the arms alternate, three rounds each) and once as
`torch.matmul` on the same bf16 operands (cuBLAS, a reference for what a plain GEMM of that shape reaches on the card).  Operands and outputs are allocated once per
launch, so a timed window is the kernel alone.

Not reproduced from the report (it does not record them): bias, row-mod residual broadcast, row re-blocking of D,
dropout and the fused im2col A operand.  The patch embedding is timed as the plain GEMM of the same shape.

Each arm's non-accumulating output is fingerprinted (sums of its raw bits), so runs of two builds on the same card
can be checked for bit-identical results; arms of one run are compared directly.  --root selects the tree whose
`ymp` package is imported (default: the one this script lives in).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card_info():
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip()
    name, plim, clk = [x.strip() for x in out.split(",")]
    return dict(name=name, power_limit=plim, max_sm_clock=clk)


def load_report(root, cfg, rdir):
    path = os.path.join(rdir, f"gemm_{cfg}.json")
    if not os.path.exists(path):
        subprocess.run([sys.executable, os.path.join(root, "bench.py"), "--gpus", "1", "--config", cfg, "--steps", "1",
                        "--warmup", "1", "--no-cpu-baseline", "--gemm-report", path], check=True,
                       stdout=subprocess.DEVNULL)
    with open(path) as fh:
        return json.load(fh)


def fingerprint(t):
    """Two wrapping int64 sums over the raw bits of t: equal outputs give equal fingerprints."""
    import torch
    v = t.contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32).long()
    return [int(v.sum().item()), int((v * v).sum().item())]


def build_case(row, seed):
    import torch
    M, N, K = row["M"], row["N"], row["K"]
    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(seed)

    def rnd(*shape, dtype=torch.bfloat16, scale=1.0):
        return (torch.randn(*shape, device=dev, generator=g) * scale).to(dtype)

    a = rnd(K, M) if row["a_t"] else rnd(M, K)
    b = rnd(K, N) if row["b_t"] else rnd(N, K)
    a, b = a / K ** 0.25, b / K ** 0.25
    kw = dict(a_t=bool(row["a_t"]), b_t=bool(row["b_t"]), act=row["act"])
    out_dtype = torch.float32 if row["out_f32"] else torch.bfloat16
    kw["out"] = torch.zeros(M, N, device=dev, dtype=out_dtype)
    if row["acc"]:
        kw["accumulate"] = True
    if row["aux_out"]:
        kw["aux_out"] = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    if row["aux_in"]:
        kw["aux_in"] = rnd(M, N)
    if row["res"]:
        kw["residual"] = rnd(M, N, dtype=torch.float32 if row["res_f32"] else torch.bfloat16)
    return a, b, kw


def time_fn(fn, reps):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / reps  # us per launch


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="+", default=["pretrain", "caption27b", "retrieval"])
    ap.add_argument("--reports-dir", default=None, help="where gemm_<config>.json live (written by bench.py if missing)")
    ap.add_argument("--arms", default="0", help="comma-separated tile_n or tile_n:tile_m arms timed alternately")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--window-ms", type=float, default=20.0, help="target length of one timed window")
    ap.add_argument("--root", default=HERE, help="repository tree whose ymp package is imported")
    ap.add_argument("--json", default=None, help="also write the table as json")
    args = ap.parse_args()

    root = os.path.abspath(args.root)
    for p in (root, os.path.join(root, "youku-mplug_b200")):
        sys.path.insert(0, p)
    import torch
    from ymp import ops
    if not torch.cuda.is_available():
        sys.exit("gemm_ab.py needs a GPU")
    arms = args.arms.split(",")
    tiles = {arm: dict(tile_n=int(arm.split(":")[0]), tile_m=int(arm.split(":")[1]) if ":" in arm else 0) for arm in arms}
    rdir = args.reports_dir or tempfile.mkdtemp(prefix="gemm_ab_")
    os.makedirs(rdir, exist_ok=True)
    info = card_info()
    print(f"# {info['name']}, power limit {info['power_limit']}, max SM clock {info['max_sm_clock']}; "
          f"ymp from {root}; arms tile_n[:tile_m]={arms}", flush=True)

    result = dict(card=info, root=root, arms=arms, configs={})
    for cfg in args.configs:
        rows = load_report(root, cfg, rdir)
        print(f"\n## {cfg}: {len(rows)} distinct launches, {sum(r['n'] for r in rows)} per step")
        hdr = "   M     N     K at bt acc act ax ai res r32 o32   n  step_us " + \
              " ".join(f" {a:>8}us   TF/s" for a in arms) + "  cublas_us   TF/s  same"
        print(hdr)
        out_rows = []
        tot = {a: 0.0 for a in arms}
        tot_cb = 0.0
        for i, row in enumerate(rows):
            a, b, kw = build_case(row, 1000 + i)
            flop = 2.0 * row["M"] * row["N"] * row["K"]
            reps = max(5, min(500, int(args.window_ms * 1e-3 / (flop / 4e14 + 4e-6))))
            fns = {arm: (lambda arm=arm: ops.gemm(a, b, **tiles[arm], **kw)) for arm in arms}
            am = a.t() if row["a_t"] else a
            bm = b if row["b_t"] else b.t()
            cb_out = torch.empty(row["M"], row["N"], device=a.device, dtype=torch.bfloat16)
            fns["cublas"] = lambda: torch.matmul(am, bm, out=cb_out)
            samples = {k: [] for k in fns}
            for _ in range(args.rounds):
                for k, fn in fns.items():
                    samples[k].append(time_fn(fn, reps))
            us = {k: statistics.median(v) for k, v in samples.items()}
            fps, same = {}, None
            if not row["acc"]:
                outs = {}
                for arm in arms:
                    kw["out"].zero_()
                    ops.gemm(a, b, **tiles[arm], **kw)
                    outs[arm] = kw["out"].clone()
                    fps[arm] = fingerprint(outs[arm])
                same = all(torch.equal(outs[arms[0]], outs[x]) for x in arms[1:])
                del outs
            for arm in arms:
                tot[arm] += us[arm] * row["n"]
            tot_cb += us["cublas"] * row["n"]
            print(f"{row['M']:5d} {row['N']:5d} {row['K']:5d} {row['a_t']:2d} {row['b_t']:2d} {row['acc']:3d} {row['act']:3d} "
                  f"{row['aux_out']:2d} {row['aux_in']:2d} {row['res']:3d} {row['res_f32']:3d} {row['out_f32']:3d} "
                  f"{row['n']:3d} {row['ms'] * 1e3 / row['n']:8.1f} "
                  + " ".join(f"{us[arm]:10.1f} {flop / us[arm] / 1e6:6.1f}" for arm in arms)
                  + f" {us['cublas']:10.1f} {flop / us['cublas'] / 1e6:6.1f}  {'-' if same is None else 'yes' if same else 'NO'}",
                  flush=True)
            out_rows.append(dict(row, step_us=row["ms"] * 1e3 / row["n"], us={str(k): v for k, v in us.items()},
                                 samples_us={str(k): v for k, v in samples.items()},
                                 tflops={str(k): flop / v / 1e6 for k, v in us.items()},
                                 fingerprint={str(k): v for k, v in fps.items()}, arms_identical=same))
            del a, b, kw, cb_out, fns
            torch.cuda.empty_cache()
        print(f"# {cfg}: sum over one step's launches (ms): "
              + ", ".join(f"{a}: {tot[a] / 1e3:.2f}" for a in arms) + f", cuBLAS: {tot_cb / 1e3:.2f}")
        result["configs"][cfg] = dict(rows=out_rows, step_ms={str(a): tot[a] / 1e3 for a in arms}, cublas_step_ms=tot_cb / 1e3)
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, "w") as fh:
            json.dump(result, fh, indent=1)


if __name__ == "__main__":
    main()
