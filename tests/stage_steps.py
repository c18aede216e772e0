"""Float64 step programs of the hand-scheduled model stages, and the trace recorder and walker that check
ymp/engine.py and ymp/functional.py against them one kernel call at a time.

A *step program* restates one stage of the reference layer (oracle/port.py: timesformer, attention_pool,
gpt3_layer / gpt3_decoder, lm_head_losses, pretrain_forward) as the sequence of kernel calls that computes it:
every step names the kernel (`gemm`, `layernorm_fwd`, `attn_bwd`, ...), the quantities it consumes (a stage
input, a weight, an earlier step's output, or an exactly stated transform of one, such as bf16(colsum)), and where
an accumulating output goes (a gradient key of G, or a fresh zeroed temporary).  Programs are written against an
executor `X` and run in three modes:

  exact  every step returns its float64 value: the composition of a stage's steps is the float64 reference layer
         (test_stage_steps_cpu.py compares it with autograd through oracle/port.py);
  synth  every step returns its float64 value rounded to the dtype the engine stores it in, and appends the call
         to a synthetic trace (the walker's own test);
  walk   every step consumes the next call of a recorded trace.  It checks the kernel name (schedule), that every
         operand equals, bit for bit, the value the step names (dataflow), and that every output element is within
         the kernel's derived bound of the float64 value computed from those operands (value); it then returns the
         recorded outputs, so the next steps are checked on the GPU's own values (teacher forcing).

The bounds are the per-kernel ones of gemm_bounds.py, attn_bounds.py and misc_bounds.py, unchanged: with teacher
forcing every step's operands are exact, so each kernel is held to its own bound.  Torch-side glue between kernels
(slices, copies, `.to(bf16)`, sums into G) is checked through the values that reach the next kernel, or, for the
sums that land in G, by the final-value check below.

Gradient accumulators.  A step that accumulates (GEMM with accumulate, colsum, LayerNorm dgamma / dbeta) names its
target: a gradient key and element offset of G, or a temporary that must start at zero.  The recorder resolves the
output pointer to its G key, so a wgrad into the wrong key or into a scratch buffer fails.  The walker keeps, per
key, the float64 value G should hold and a bound on it: a kernel step sets them to its reference and bound (the
operand d0 is the recorded before-value, checked against them), a torch-side sum of n fp32 terms into G adds
C (n + 1) u32 (|G| + sum |terms|) to the bound (one rounding per term, each relative to a partial sum).  After the
walk every key of G must hold its value within its bound, and G must contain exactly the keys the program writes.

Bounds this module adds (C, u, u32, TINY as in gemm_bounds.py; each is one rounding of an exact float64 value y):
  group_reduce broadcast   out = bf16(fl32(x scale)): the product rounds once to fp32 and once to bf16,
                           |out - y| <= (u32 + u) |y| (1 + u32), covered by C (u32 + u) |y| + TINY.
  dropout (fp32, in place) y = x k on kept elements, k = fl32(1 / (1 - p)) exact in the reference: one fp32 product,
                           C u32 |y| + TINY; dropped elements are exact zeros.
  embed_gather (fp32 out)  y = table[id] + pos, both bf16 and exact in fp32: one fp32 add, C u32 |y| + TINY.
  im2col                   a gather (zeros in the padded columns): exact, TINY.
  accumulating GEMM        gemm_bounds.bounds takes the number of K-splits.  With split_k = 0, ymp_gemm's heuristic
                           (gemm_wgmma.cu) tries sp <= 64 with 8 sp <= kb_total and then caps split at kb_total =
                           ceil(K/64), so split = min(64, ceil(K/64)) bounds the chains and the atomic adds onto D0
                           from above, and the bound grows with split.

Row layouts are those of the kernels' interfaces: ViT tokens row (b N + n) T + t, then B cls rows; decoder row
b S + s; attention operands are gathered per (sequence, head) through the calls' own sequence maps.

Decoding (decode_session: DistributedGPT3's sample / beam_search over the KV cache).  Host events drive the program:
decode entries (new token ids, whether query embeddings were fed), KVCache.reindex / reorder / share_prefill, and the
logits each decode returned, which must be the last step's value bit for bit.  The program keeps each sequence's
history of cached QKV rows (KVHistory) and applies the events to it; every attention step's K / V operands, gathered
through the call's row table (kv_rows, min(s_kv, *s_kv_dev) keys), must equal that history bit for bit, and a skinny
QKV GEMM's cache copy must land in slot b max_len + len and equal its output row bit for bit.  The GPU walks fill each
new cache store with a finite +-3e4 poison, so a read of a slot no step wrote fails.  The skinny GEMMs use
gemm_bounds.bounds with split = skinny_slices(N, K) (each K slice is its own chain); the table gather is exact.  No
bound is added.
"""
import json
import math
import os

import numpy as np
import torch

import attn_bounds as AB
import gemm_bounds as GB
import misc_bounds as MB

F64 = torch.float64
BF16 = torch.bfloat16
F32 = torch.float32
U32, C, TINY = GB.U32, GB.C, GB.TINY
ACT_NONE, ACT_GELU_ERF, ACT_GELU_TANH = GB.ACT_NONE, GB.ACT_GELU_ERF, GB.ACT_GELU_TANH

GPT = "text_decoder.dist_model.language_model."
VE = "visual_encoder."
AP = "attn_pool."


class StepFailure(AssertionError):
    """A trace disagrees with its step program at `step`."""

    def __init__(self, step, what):
        super().__init__(f"{step}: {what}")
        self.step, self.what = step, what


def f32(x):
    return float(torch.tensor(float(x), dtype=F32))


def drop_mult(spec, rows, cols, dev):
    """float64 [len(rows), cols] multiplier keep / (1 - p) of a dropout spec (seed, offset, site, p) with the kernels'
    Philox convention (oracle/philox.py); rows: the logical row indices."""
    from oracle import philox
    seed, off, site, p = spec
    keep = philox.keep_mask(seed, off, site, np.asarray(rows, dtype=np.int64), cols, p)
    return torch.from_numpy(keep).to(dev).to(F64) * philox.scale(p)


def _same(a, b):
    if a is None or b is None:
        return a is None and b is None
    if isinstance(a, torch.Tensor) or isinstance(b, torch.Tensor):
        a, b = torch.as_tensor(a), torch.as_tensor(b)
        return a.shape == b.shape and torch.equal(a.to(F64), b.to(device=a.device, dtype=F64))
    if isinstance(a, float) or isinstance(b, float):
        return f32(a) == f32(b)
    return a == b


def _ratio(got, want, bound):
    err = (got.to(F64) - want.to(F64)).abs() / bound
    err = torch.where(torch.isnan(err), torch.full_like(err, math.inf), err)
    return float(err.max()) if err.numel() else 0.0


# ---------------------------------------------------------------------------------- per-kernel references and bounds
# Each returns {output: (float64 value, bound)} from the logical operands `a` and the scalar arguments `kw`.
ACC_D0 = {"D": "d0", "out": "d0", "dgamma": "dgamma0", "dbeta": "dbeta0"}


def _k_gemm(a, kw, sms):
    # patch_embed_gemm reads the patch rows straight from the video
    A = patch_rows(a["video"], kw["P"]) if "video" in a else a["A"]
    B = a["B"]
    aux_in = a.get("aux_in")
    if kw.get("drop") is not None:
        aux_in = drop_mult(kw["drop"], range(A.shape[0]), B.shape[0], A.device)
    ref = GB.reference(A, B, alpha=kw.get("alpha", 1.0), bias=a.get("bias"), act=kw.get("act", 0), aux_in=aux_in,
                       residual=a.get("residual"), d0=a.get("d0"))
    K = A.shape[1]
    split = min(64, -(-K // 64)) if a.get("d0") is not None else 1
    e_out, e_aux = GB.bounds(ref, K, split=split, out_bf16=kw["out_dtype"] == BF16)
    r = dict(D=(ref["out"], e_out))
    if kw.get("aux"):
        r["aux"] = (ref["aux"], e_aux)
    return r


def _k_skinny(a, kw, sms):
    # out2 (the KV-cache copy) holds the same bf16 value as D; the walker also checks that bit for bit
    A, B = a["A"], a["B"]
    ref = GB.reference(A, B, bias=a.get("bias"), act=kw.get("act", 0), residual=a.get("residual"))
    e_out, _ = GB.bounds(ref, A.shape[1], split=GB.skinny_slices(B.shape[0], A.shape[1]), out_bf16=kw["out_dtype"] == BF16)
    return dict(D=(ref["out"], e_out), out2=(ref["out"], e_out))


def _k_im2col(a, kw, sms):
    p = patch_rows(a["video"], kw["P"])
    out = torch.zeros(p.shape[0], kw["ld"], dtype=F64, device=p.device)
    out[:, :p.shape[1]] = p
    return dict(out=(out, torch.full_like(out, TINY)))


def _k_ln_fwd(a, kw, sms):
    x, g, b = a["x"], a["gamma"], a["beta"]
    pad = kw.get("pad")
    y, mean, rstd = MB.ln_fwd_reference(x, g, b, kw["eps"])
    e_y, e_m, e_r = MB.ln_fwd_bounds(x, g, b, kw["eps"], y_bf16=kw["y_dtype"] == BF16)
    if pad is not None:                                # padding slots: zero row, mean = rstd = 0, exactly
        pm = pad.to(x.device)
        y, mean, rstd = (t.masked_fill(pm[:, None] if t.dim() == 2 else pm, 0.0) for t in (y, mean, rstd))
        e_y, e_m, e_r = (t.masked_fill(pm[:, None] if t.dim() == 2 else pm, TINY) for t in (e_y, e_m, e_r))
    return dict(y=(y, e_y), mean=(mean, e_m), rstd=(rstd, e_r))


def _k_ln_bwd(a, kw, sms):
    dy, x = a["dy"], a["x"]
    rows, D = dy.shape
    keep, p = None, 0.0
    if kw.get("drop") is not None:
        m = drop_mult(kw["drop"], kw["xrows"], D, dy.device)
        keep, p = m > 0, kw["drop"][3]
    ref = MB.ln_bwd_reference(dy, x, a["gamma"], a["mean"], a["rstd"], add=a.get("add"), dgamma0=a.get("dgamma0"),
                              dbeta0=a.get("dbeta0"), keep=keep, p=p)
    bd = MB.ln_bwd_bounds(ref, MB.ln_bwd_blocks(rows, D, sms, wgrad="dgamma0" in a), rows=rows)
    r = dict(dx=(ref["dx"], bd["dx"]))
    if keep is not None:
        r["dx_drop"] = (ref["dx_drop"], bd["dx_drop"])
    if "dgamma0" in a:
        r["dgamma"], r["dbeta"] = (ref["dgamma"], bd["dgamma"]), (ref["dbeta"], bd["dbeta"])
    return r


def _attn_mult(kw, n, H, sq, skv, dev):
    if kw.get("drop") is None:
        return None
    return drop_mult(kw["drop"], range(n * H * sq), skv, dev).view(n, H, sq, skv)


def _k_attn_fwd(a, kw, sms):
    q, k, v = a["q"], a["k"], a["v"]
    n, H, sq, _ = q.shape
    vis = AB.visible(n, sq, k.shape[2], kw["mask"])
    ref = AB.reference(q, k, v, vis, kw["scale"], mult=_attn_mult(kw, n, H, sq, k.shape[2], q.device))
    e_o, e_lse = AB.fwd_bounds(q, k, v, kw["scale"], ref)
    return dict(o=(ref["O"], e_o), lse=(ref["lse"], e_lse))


def _k_attn_bwd(a, kw, sms):
    q, k, v, do = a["q"], a["k"], a["v"], a["do"]
    n, H, sq, _ = q.shape
    vis = AB.visible(n, sq, k.shape[2], kw["mask"])
    ref = AB.reference(q, k, v, vis, kw["scale"], dout=do, mult=_attn_mult(kw, n, H, sq, k.shape[2], q.device))
    # the backward is given the kernel's O and lse: their forward bounds enter its own (attn_bounds, E_O / E_lse)
    e_o, e_lse = AB.fwd_bounds(q, k, v, kw["scale"], ref)
    e_dq, e_dk, e_dv = AB.bwd_bounds(q, k, v, do, kw["scale"], ref, e_o=e_o, e_lse=e_lse)
    return dict(dq=(ref["dQ"], e_dq), dk=(ref["dK"], e_dk), dv=(ref["dV"], e_dv))


def _k_group_reduce(a, kw, sms):
    x = a["x"]
    if kw["broadcast"]:
        want = (x.to(F64) * f32(kw["scale"])).repeat_interleave(kw["T"], 0)
        return dict(out=(want, C * (U32 + GB.U) * want.abs() + TINY))
    want = MB.group_reduce_reference(x, kw["G"], kw["T"], kw["scale"])
    return dict(out=(want, MB.group_reduce_bound(x, kw["G"], kw["T"], kw["scale"])))


def _k_colsum(a, kw, sms):
    x, d0 = a["x"], a["d0"]
    return dict(out=(d0.to(F64) + x.to(F64).sum(0), MB.colsum_bound(x, d0, sms)))


def _k_dropout(a, kw, sms):
    x = a["x"].to(F64)
    want = x * drop_mult(kw["drop"], range(x.shape[0]), x.shape[1], x.device)
    return dict(y=(want, C * U32 * want.abs() + TINY))


def _k_embed(a, kw, sms):
    ids = a["ids"].reshape(-1).long()
    S, off = kw["S"], kw["row_offset"]
    L = a["ids"].shape[1]
    pos = a["pos"][off:off + L].to(F64).repeat(a["ids"].shape[0], 1)
    want = a["table"].to(F64)[ids] + pos
    return dict(out=(want, C * U32 * want.abs() + TINY))


def _k_ce_fwd(a, kw, sms):
    loss, lse = MB.ce_reference(a["logits"], a["labels"])
    e_loss, e_lse, _ = MB.ce_fwd_bounds(a["logits"], a["labels"])
    return dict(loss=(loss, e_loss), lse=(lse, e_lse))


def _k_ce_bwd(a, kw, sms):
    want, bound = MB.ce_bwd_bounds(a["logits"], a["labels"], a["lse"], a["g"])
    return dict(dlogits=(want, bound))


KERNELS = dict(gemm=_k_gemm, patch_embed_gemm=_k_gemm, im2col=_k_im2col, layernorm_fwd=_k_ln_fwd, layernorm_bwd=_k_ln_bwd,
               attn_fwd=_k_attn_fwd, attn_bwd=_k_attn_bwd, attn_temporal_fwd=_k_attn_fwd, attn_temporal_bwd=_k_attn_bwd,
               group_reduce=_k_group_reduce, colsum=_k_colsum, dropout=_k_dropout, embed_gather=_k_embed,
               ce_fwd=_k_ce_fwd, ce_bwd=_k_ce_bwd, gemm_skinny=_k_skinny, gemm_skinny_wide=_k_skinny)


def patch_rows(video, P):
    """video [B, C, T, H, W] -> patch matrix [(b n t), C P P] (Conv2d(k = stride = P) as a GEMM, n row-major)."""
    B, Cc, T, H, Wd = video.shape
    x = video.to(F64).reshape(B, Cc, T, H // P, P, Wd // P, P)
    return x.permute(0, 3, 5, 2, 1, 4, 6).reshape(B * (H // P) * (Wd // P) * T, Cc * P * P)


# ---------------------------------------------------------------------------------- executor
class Rec:
    """One recorded (or synthesised) kernel call: op name, logical operands, scalar arguments, logical outputs, and
    for accumulating outputs the gradient key and offset their buffer lies in (None: not in G)."""
    __slots__ = ("op", "ins", "kw", "outs", "targets")

    def __init__(self, op, ins, kw, outs, targets):
        self.op, self.ins, self.kw, self.outs, self.targets = op, ins, kw, outs, targets


class Exec:
    """Runs a step program.  mode: "exact" | "synth" | "walk".  G0: {key: fp32 values} the gradient buffers held
    before the stage (walk / synth); trace: the recorded calls (walk); tamper: {step: fn(ins, kw, vals) -> (ins, kw)}
    (synth; None drops a torch-side sum).  sms: SM count of the device (grid-dependent bounds)."""

    def __init__(self, mode, *, G0=None, trace=None, tamper=None, sms=MB.SMS_H100, dev="cpu"):
        self.mode, self.trace, self.tamper, self.sms, self.dev = mode, list(trace or []), dict(tamper or {}), sms, dev
        self.pos = 0
        self.G = {k: v.to(F64).reshape(-1).clone() for k, v in (G0 or {}).items()}
        self.Gb = {k: torch.zeros_like(v) for k, v in self.G.items()}
        self.touched = set()
        self.vals = {}
        self.out_trace = []
        self.report = {}

    # ---- values
    def rnd(self, t, dtype):
        """t as the engine stores it in `dtype` (exact mode: unrounded)."""
        return t if self.mode == "exact" else t.to(dtype).to(F64)

    def zeros_g(self, key, numel):
        """Exact mode starts from G = 0 and grows each key to the extent its steps write."""
        if key not in self.G:
            self.G[key] = torch.zeros(0, dtype=F64, device=self.dev)
            self.Gb[key] = torch.zeros_like(self.G[key])
        if self.G[key].numel() < numel:
            pad = torch.zeros(numel - self.G[key].numel(), dtype=F64, device=self.dev)
            self.G[key], self.Gb[key] = torch.cat([self.G[key], pad]), torch.cat([self.Gb[key], pad])

    # ---- one kernel call
    def call(self, name, op, ins, kw, outs, acc=None):
        """ins: {operand: float64 tensor or None}; kw: scalar arguments; outs: {output: dtype}; acc: {output: (key,
        offset) or None for a zeroed temporary}.  Returns {output: float64 value}."""
        ins = {k: v for k, v in ins.items() if v is not None}
        kw = dict(kw)
        acc = dict(acc or {})
        for o, tgt in acc.items():
            shape = self._out_shape(op, o, ins, kw)
            n = int(np.prod(shape))
            if tgt is None:
                ins[ACC_D0[o]] = torch.zeros(shape, dtype=F64, device=self.dev)
            else:
                key, off = tgt
                self.zeros_g(key, off + n)
                self.touched.add(key)
                ins[ACC_D0[o]] = self.G[key][off:off + n].view(shape)
        if self.mode == "walk":
            res = self._walk(name, op, ins, kw, outs, acc)
        else:
            if self.mode == "synth" and name in self.tamper:
                ins, kw = self.tamper[name](dict(ins), dict(kw), self.vals)
            refs = KERNELS[op](ins, kw, self.sms)
            res = {o: (refs[o][0] if self.mode == "exact" else self.rnd(refs[o][0], outs[o])) for o in outs}
            if self.mode == "synth":
                targets = {o: (acc[o] if (o in acc and acc[o] is not None) else None) for o in outs}
                self.out_trace.append(Rec(op, {k: v.clone() for k, v in ins.items()}, kw,
                                          {o: res[o].to(outs[o]) for o in outs}, targets))
        for o, tgt in acc.items():
            if tgt is not None:
                key, off = tgt
                n = res[o].numel()
                self.G[key][off:off + n] = res[o].reshape(-1)
        self.vals[name] = res
        return res

    def _out_shape(self, op, o, ins, kw):
        if op in ("gemm", "patch_embed_gemm"):
            return (ins["A"].shape[0], ins["B"].shape[0])
        if op == "colsum":
            return (ins["x"].shape[1],)
        return (ins["dy"].shape[1],)          # layernorm_bwd dgamma / dbeta

    def _walk(self, name, op, ins, kw, outs, acc):
        if self.pos >= len(self.trace):
            raise StepFailure(name, f"schedule: the trace ends before this {op} call")
        rec = self.trace[self.pos]
        self.pos += 1
        if rec.op != op:
            raise StepFailure(name, f"schedule: expected {op}, the trace has {rec.op}")
        for k in set(kw) | set(rec.kw):
            if not _same(kw.get(k), rec.kw.get(k)):
                raise StepFailure(name, f"argument {k}: expected {kw.get(k)}, got {rec.kw.get(k)}")
        d0names = {ACC_D0[o] for o in acc}
        for k in set(ins) | set(rec.ins):
            if k in d0names:
                continue
            if k not in ins or k not in rec.ins:
                raise StepFailure(name, f"operand {k}: {'missing' if k in ins else 'unexpected'} in the trace")
            if not _same(ins[k], rec.ins[k]):
                g, w = rec.ins[k], ins[k]
                detail = f"shape {tuple(g.shape)} vs {tuple(w.shape)}" if g.shape != w.shape else \
                    f"max |diff| {float((g.to(F64) - w.to(F64).to(g.device)).abs().max()):.3e}"
                raise StepFailure(name, f"dataflow: operand {k} is not the named quantity ({detail})")
        for o in acc:
            want_t = acc[o]
            got_t = rec.targets.get(o)
            if want_t is None:
                if got_t is not None:
                    raise StepFailure(name, f"accumulator {o} lands in G[{got_t[0]}], expected a temporary")
                if not torch.equal(rec.ins[ACC_D0[o]].to(F64), ins[ACC_D0[o]]):
                    raise StepFailure(name, f"accumulator {o}: the temporary does not start at zero")
            else:
                if got_t is None or tuple(got_t) != tuple(want_t):
                    raise StepFailure(name, f"accumulator {o} lands in {got_t}, expected G[{want_t[0]}] at {want_t[1]}")
                key, off = want_t
                d0 = rec.ins[ACC_D0[o]].to(F64)
                n = d0.numel()
                r = _ratio(d0.reshape(-1), self.G[key][off:off + n], self.Gb[key][off:off + n] + TINY)
                if r > 1:
                    raise StepFailure(name, f"accumulator {o}: G[{key}] before the call is off by {r:.3g} x its bound")
            ins[ACC_D0[o]] = rec.ins[ACC_D0[o]].to(F64)
        refs = KERNELS[op](ins, kw, self.sms)
        res = {}
        for o, dt in outs.items():
            if o not in rec.outs:
                raise StepFailure(name, f"output {o} missing from the trace")
            got = rec.outs[o]
            want, bound = refs[o]
            if o == "out2" and not torch.equal(got, rec.outs["D"].to(got.dtype)):
                raise StepFailure(name, "value out2: the cache row is not the output row bit for bit")
            if got.dtype != dt:
                raise StepFailure(name, f"output {o} stored as {got.dtype}, expected {dt}")
            if tuple(got.shape) != tuple(want.shape):
                raise StepFailure(name, f"output {o} shape {tuple(got.shape)} vs {tuple(want.shape)}")
            r = _ratio(got, want, bound)
            self.report[f"{name}.{o}"] = max(r, self.report.get(f"{name}.{o}", 0.0))
            if not r <= 1.0:
                raise StepFailure(name, f"value {o}: err/bound {r:.3g}")
            res[o] = got.to(F64)
            if o in acc and acc[o] is not None:
                key, off = acc[o]
                n = got.numel()
                self.Gb[key][off:off + n] = bound.reshape(-1)
        return res

    # ---- torch-side sums into G
    def grad_add(self, name, key, off, terms):
        """G[key][off:] += terms.sum(0) in fp32 (torch glue); terms [n, ...] float64."""
        if self.mode == "synth" and name in self.tamper:
            terms = self.tamper[name](terms, None, self.vals)
            if terms is None:
                return
        n = terms[0].numel()
        self.zeros_g(key, off + n)
        self.touched.add(key)
        s = terms.to(F64).sum(0).reshape(-1)
        g = self.G[key][off:off + n]
        new = g + s
        if self.mode == "walk":
            self.Gb[key][off:off + n] += C * (terms.shape[0] + 1) * U32 * (g.abs() + terms.abs().sum(0).reshape(-1) + new.abs())
        self.G[key][off:off + n] = new if self.mode == "exact" else new.to(F32).to(F64)

    # ---- after the stage
    def finish(self, G_final=None):
        """walk: every call consumed, every key of G within its bound, no key missing or extra."""
        if self.mode != "walk":
            return
        if self.pos != len(self.trace):
            raise StepFailure(f"after {self.pos} calls", f"schedule: {len(self.trace) - self.pos} extra kernel calls, "
                                                         f"next {self.trace[self.pos].op}")
        if G_final is None:
            return
        extra = set(G_final) - self.touched
        missing = self.touched - set(G_final)
        if extra or missing:
            raise StepFailure("G", f"gradient keys: extra {sorted(extra)}, missing {sorted(missing)}")
        for k in sorted(self.touched):
            got = G_final[k].to(F64).reshape(-1)
            r = _ratio(got, self.G[k].to(got.device), self.Gb[k].to(got.device) + TINY)
            self.report[f"G[{k}]"] = r
            if not r <= 1.0:
                raise StepFailure(f"G[{k}]", f"final gradient off by {r:.3g} x its bound")

    def returned(self, name, got, want):
        """A tensor the stage returns must be the step program's value, bit for bit."""
        if self.mode == "walk" and not _same(got, want):
            raise StepFailure(name, "the returned tensor is not the last step's value")

    # ---- host events (decoding: cache table updates, decode entries, returned logits)
    def next_host(self, name, script):
        """The next host event (kind, payload) that drives a program: walk reads it from the trace (None at its end),
        exact / synth take it from the iterator `script` (synth logs it).  A synth tamper named `name.kind` changes
        what the program applies, not what is logged (an event the product logs but does not carry out)."""
        if self.mode == "walk":
            if self.pos >= len(self.trace):
                return None
            rec = self.trace[self.pos]
            if rec.op != "event":
                raise StepFailure(f"after {self.pos} calls", f"schedule: expected a host event, the trace has {rec.op}")
            self.pos += 1
            return rec.kw["kind"], rec.ins
        ev = next(script, None)
        if ev is None:
            return None
        kind, payload = ev
        return kind, self._log_event(f"{name}.{kind}", kind, payload)

    def host(self, name, kind, payload):
        """A host event the program expects here with this payload (walk: the recorded one must match it)."""
        if self.mode == "walk":
            if self.pos >= len(self.trace):
                raise StepFailure(name, f"schedule: the trace ends before this {kind} event")
            rec = self.trace[self.pos]
            self.pos += 1
            if rec.op != "event" or rec.kw["kind"] != kind:
                raise StepFailure(name, f"schedule: expected a {kind} event, the trace has {rec.kw.get('kind', rec.op)}")
            for k in set(payload) | set(rec.ins):
                if not _same(payload.get(k), rec.ins.get(k)):
                    raise StepFailure(name, f"event {kind}: {k} is not the value the program names")
            return payload
        return self._log_event(name, kind, payload)

    def _log_event(self, name, kind, payload):
        if self.mode == "synth":
            self.out_trace.append(Rec("event", dict(payload), dict(kind=kind), {}, {}))
            if name in self.tamper:
                return self.tamper[name](dict(payload), None, self.vals)
        return payload


def write_report(ex, stage):
    """Merge the walk's largest err/bound per step into the JSON file named by YMP_STAGE_BOUNDS_REPORT."""
    path = os.environ.get("YMP_STAGE_BOUNDS_REPORT")
    if not path:
        return
    data = {}
    if os.path.exists(path):
        with open(path) as f:
            data = json.load(f)
    cur = data.setdefault(stage, {})
    for k, v in ex.report.items():
        cur[k] = max(v, cur.get(k, 0.0))
    with open(path, "w") as f:
        json.dump(data, f, indent=1, sort_keys=True)


# ---------------------------------------------------------------------------------- step sugar
TMP = "tmp"


def gemm(X, name, A, B, *, bias=None, residual=None, act=ACT_NONE, aux=False, aux_in=None, out=BF16, drop=None,
         acc=False, alpha=1.0):
    """D = epilogue(A B^T) with A [M, K], B [N, K] as the kernel reads them; acc: False (plain store), (key, offset)
    of G, or TMP (a zeroed temporary) for an accumulating call."""
    outs = dict(D=out)
    if aux:
        outs["aux"] = BF16
    kw = dict(act=act, alpha=alpha, accumulate=acc is not False, drop=drop, aux=aux, out_dtype=out)
    r = X.call(name, "gemm", dict(A=A, B=B, bias=bias, residual=residual, aux_in=aux_in), kw, outs,
               acc=None if acc is False else dict(D=None if acc == TMP else acc))
    return (r["D"], r["aux"]) if aux else r["D"]


def wgrad(X, name, dy, x, wkey, bkey, T):
    """G[wkey] += dy^T x, G[bkey] += colsum(dy) for the trainable keys in T (linear_wgrad's pair of kernels)."""
    if wkey in T:
        gemm(X, name + ".wgrad", dy.T, x.T, out=F32, acc=(wkey, 0))
    if bkey is not None and bkey in T:
        colsum(X, name + ".bgrad", dy, (bkey, 0))


def colsum(X, name, x, tgt):
    return X.call(name, "colsum", dict(x=x), {}, dict(out=F32), acc=dict(out=tgt))["out"]


def ln_fwd(X, name, x, W, pre, eps, y=BF16, in_rows=None, pad=None, stats=True):
    r = X.call(name, "layernorm_fwd", dict(x=x, gamma=W[pre + ".weight"], beta=W[pre + ".bias"]),
               dict(eps=eps, y_dtype=y, in_rows=in_rows, pad=pad), dict(y=y, mean=F32, rstd=F32) if stats else dict(y=y))
    return r["y"], r.get("mean"), r.get("rstd")


def ln_bwd(X, name, dy, x, W, pre, mean, rstd, T, add=None, drop=None, in_rows=None, xrows=None):
    """dx (+ add) of LN(x); dgamma / dbeta into G when trainable; with drop also dx_drop (mask rows = x rows)."""
    acc = dict(dgamma=(pre + ".weight", 0), dbeta=(pre + ".bias", 0)) if pre + ".weight" in T else {}
    outs = dict(dx=BF16)
    if drop is not None:
        outs["dx_drop"] = BF16
    if acc:
        outs.update(dgamma=F32, dbeta=F32)
    if xrows is None:
        xrows = list(range(dy.shape[0]))
    r = X.call(name, "layernorm_bwd", dict(dy=dy, x=x, gamma=W[pre + ".weight"], mean=mean, rstd=rstd, add=add),
               dict(drop=drop, in_rows=in_rows, xrows=torch.as_tensor(list(xrows))), outs, acc=acc)
    return r["dx"], r.get("dx_drop", r["dx"])


def attn(X, name, q, k, v, *, scale, causal=False, drop=None, temporal=False, keys=None):
    """keys: the key count of a call that reads its keys through a row table (kv_rows), as the device held it."""
    r = X.call(name, "attn_temporal_fwd" if temporal else "attn_fwd", dict(q=q, k=k, v=v),
               dict(mask=AB.MASK_CAUSAL if causal else AB.MASK_NONE, scale=scale, drop=drop, keys=keys),
               dict(o=BF16, lse=F32))
    return r["o"], r["lse"]


def skinny(X, name, op, A, B, *, bias=None, residual=None, act=ACT_NONE, out=BF16, out2_rows=None):
    """ymp_gemm_skinny(_wide): D = act(A B^T + bias) + residual.  out2_rows: the KV-cache rows the result is also
    written to (the step names them)."""
    ins = dict(A=A, B=B, bias=bias, residual=residual)
    kw = dict(act=act, out_dtype=out, out2_rows=out2_rows)
    outs = dict(D=out)
    if out2_rows is not None:
        outs["out2"] = BF16
    return X.call(name, op, ins, kw, outs)["D"]


def attn_b(X, name, q, k, v, o, lse, do, *, scale, causal=False, drop=None, temporal=False):
    r = X.call(name, "attn_temporal_bwd" if temporal else "attn_bwd", dict(q=q, k=k, v=v, o=o, lse=lse, do=do),
               dict(mask=AB.MASK_CAUSAL if causal else AB.MASK_NONE, scale=scale, drop=drop),
               dict(dq=BF16, dk=BF16, dv=BF16))
    return r["dq"], r["dk"], r["dv"]


def heads(t, n, S, H, hd, col=0, hs=None):
    """Rows [n * S, *] -> [n, H, S, hd]: head h at columns col + h hs."""
    hs = hd if hs is None else hs
    idx = col + (torch.arange(H)[:, None] * hs + torch.arange(hd)[None, :]).reshape(-1).to(t.device)
    return t.reshape(n * S, -1)[:, idx].reshape(n, S, H, hd).permute(0, 2, 1, 3)


def unheads(o):
    """[n, H, S, hd] -> [n * S, H hd]."""
    n, H, S, hd = o.shape
    return o.permute(0, 2, 1, 3).reshape(n * S, H * hd)


def qkv_bias(W, pre):
    """cat(q_bias, 0, v_bias) - the ViT attention has no key bias (port.vit_attention)."""
    return torch.cat([W[pre + "q_bias"], torch.zeros_like(W[pre + "v_bias"]), W[pre + "v_bias"]])


def dims_vit(vcfg, B):
    P, D, T = vcfg["patch_size"], vcfg["embed_dim"], vcfg["num_frames"]
    N = (vcfg["img_size"] // P) ** 2
    R = B * N * T
    return dict(P=P, D=D, T=T, N=N, B=B, R=R, RB=R + B, H=vcfg["num_heads"], hd=D // vcfg["num_heads"],
                depth=vcfg["depth"], eps=1e-6, scale=(D // vcfg["num_heads"]) ** -0.5)


def spatial_rows(d):
    """[B T, N + 1] token rows of the spatial attention's sequences (b, t): the shared cls row R + b, then the patches
    (b N + n) T + t; and the same with the per-frame cls output rows RB + b T + t."""
    B, T, N, R, RB = d["B"], d["T"], d["N"], d["R"], d["RB"]
    b = torch.arange(B)[:, None, None]
    t = torch.arange(T)[None, :, None]
    n = torch.arange(N)[None, None, :]
    tok = ((b * N + n) * T + t).reshape(B * T, N)
    cls_in = (R + torch.arange(B)).repeat_interleave(T)[:, None]
    cls_out = (RB + torch.arange(B * T))[:, None]
    return torch.cat([cls_in, tok], 1), torch.cat([cls_out, tok], 1)


def final_rows(d):
    """Output row (b, 0) = cls row R + b, (b, 1 + t N + n) = token row (b N + n) T + t: the (t n) order of
    port.timesformer's output."""
    B, T, N, R = d["B"], d["T"], d["N"], d["R"]
    b = torch.arange(B).view(B, 1, 1)
    t = torch.arange(T).view(1, T, 1)
    n = torch.arange(N).view(1, 1, N)
    tok = ((b * N + n) * T + t).reshape(B, T * N)
    return torch.cat([(R + torch.arange(B)).view(B, 1), tok], 1).reshape(-1)


# ---------------------------------------------------------------------------------- TimeSformer
def vit_block_fwd(X, W, pre, x, d):
    """port.timesformer_block on rows x [RB, D] (fp32 residual stream)."""
    R, RB, D, B, T, N, H, hd = d["R"], d["RB"], d["D"], d["B"], d["T"], d["N"], d["H"], d["hd"]
    c = dict(x=x)
    # temporal attention over the T frames of each patch: sequences of T consecutive rows
    c["ln_t"], c["m_t"], c["r_t"] = ln_fwd(X, pre + "temporal_ln", x[:R], W, pre + "temporal_ln", d["eps"])
    c["qkv_t"] = gemm(X, pre + "temporal_attn.qkv", c["ln_t"], W[pre + "temporal_attn.qkv.weight"],
                      bias=qkv_bias(W, pre + "temporal_attn."))
    q, k, v = (heads(c["qkv_t"], R // T, T, H, hd, col=i * D) for i in range(3))
    o, c["lse_t"] = attn(X, pre + "temporal_attn", q, k, v, scale=d["scale"], temporal=True)
    c["att_t"] = unheads(o)
    c["proj_t"] = gemm(X, pre + "temporal_attn.proj", c["att_t"], W[pre + "temporal_attn.proj.weight"],
                       bias=W[pre + "temporal_attn.proj.bias"])
    xt_tok = gemm(X, pre + "temporal_fc", c["proj_t"], W[pre + "temporal_fc.weight"], bias=W[pre + "temporal_fc.bias"],
                  residual=x[:R], out=F32)
    c["xt"] = xt = torch.cat([xt_tok, x[R:]])
    # spatial attention per frame; every frame's sequence starts with the sample's cls row
    c["ln_s"], c["m_s"], c["r_s"] = ln_fwd(X, pre + "norm1", xt, W, pre + "norm1", d["eps"])
    c["qkv_s"] = gemm(X, pre + "attn.qkv", c["ln_s"], W[pre + "attn.qkv.weight"], bias=qkv_bias(W, pre + "attn."))
    rin, _ = spatial_rows(d)
    rows = c["qkv_s"][rin.reshape(-1).to(x.device)]
    q, k, v = (heads(rows, B * T, N + 1, H, hd, col=i * D) for i in range(3))
    c["o_s"], c["lse_s"] = attn(X, pre + "attn", q, k, v, scale=d["scale"])
    os_ = c["o_s"].permute(0, 2, 1, 3).reshape(B * T, N + 1, D)
    tok = torch.empty(R, D, dtype=F64, device=x.device)
    tok[rin[:, 1:].reshape(-1).to(x.device)] = os_[:, 1:].reshape(-1, D)
    c["cls_f"] = os_[:, 0]
    # the cls output is the mean of its T per-frame outputs (port: xs[:, 0].reshape(B, T, D).mean(1))
    cls = X.call(pre + "cls_mean", "group_reduce", dict(x=c["cls_f"]), dict(G=B, T=T, scale=1.0 / T, broadcast=False),
                 dict(out=BF16))["out"]
    c["att_s"] = torch.cat([tok, cls])
    c["y"] = gemm(X, pre + "attn.proj", c["att_s"], W[pre + "attn.proj.weight"], bias=W[pre + "attn.proj.bias"],
                  residual=xt, out=F32)
    c["ln_m"], c["m_m"], c["r_m"] = ln_fwd(X, pre + "norm2", c["y"], W, pre + "norm2", d["eps"])
    c["h"], c["dact"] = gemm(X, pre + "mlp.fc1", c["ln_m"], W[pre + "mlp.fc1.weight"], bias=W[pre + "mlp.fc1.bias"],
                             act=ACT_GELU_ERF, aux=True)
    out = gemm(X, pre + "mlp.fc2", c["h"], W[pre + "mlp.fc2.weight"], bias=W[pre + "mlp.fc2.bias"], residual=c["y"],
               out=F32)
    return out, c


def qkv_wgrad(X, name, apre, dqkv, x, D, T):
    wgrad(X, name, dqkv, x, apre + "qkv.weight", None, T)
    if apre + "q_bias" in T:
        colsum(X, name + ".q_bias", dqkv[:, :D], (apre + "q_bias", 0))
    if apre + "v_bias" in T:
        colsum(X, name + ".v_bias", dqkv[:, 2 * D:], (apre + "v_bias", 0))


def vit_block_bwd(X, W, T, pre, c, dout, d):
    R, RB, D, B, Tf, N, H, hd = d["R"], d["RB"], d["D"], d["B"], d["T"], d["N"], d["H"], d["hd"]
    dev = dout.device
    wgrad(X, pre + "mlp.fc2", dout, c["h"], pre + "mlp.fc2.weight", pre + "mlp.fc2.bias", T)
    dpre = gemm(X, pre + "mlp.fc2.dgrad", dout, W[pre + "mlp.fc2.weight"].T, act=ACT_GELU_ERF, aux_in=c["dact"], acc=False)
    wgrad(X, pre + "mlp.fc1", dpre, c["ln_m"], pre + "mlp.fc1.weight", pre + "mlp.fc1.bias", T)
    dln_m = gemm(X, pre + "mlp.fc1.dgrad", dpre, W[pre + "mlp.fc1.weight"].T, acc=False)
    dy, _ = ln_bwd(X, pre + "norm2.bwd", dln_m, c["y"], W, pre + "norm2", c["m_m"], c["r_m"], T, add=dout)
    wgrad(X, pre + "attn.proj", dy, c["att_s"], pre + "attn.proj.weight", pre + "attn.proj.bias", T)
    datt = gemm(X, pre + "attn.proj.dgrad", dy, W[pre + "attn.proj.weight"].T, acc=False)
    # d(cls mean) reaches each frame's cls output scaled by 1/T
    dcls_f = X.call(pre + "cls_mean.bwd", "group_reduce", dict(x=datt[R:]), dict(G=B, T=Tf, scale=1.0 / Tf, broadcast=True),
                    dict(out=BF16))["out"]
    rin, _ = spatial_rows(d)
    ridx = rin[:, 1:].reshape(-1).to(dev)
    do_rows = torch.cat([dcls_f[:, None, :], datt[ridx].view(B * Tf, N, D)], 1)
    rows_qkv = c["qkv_s"][rin.reshape(-1).to(dev)]
    q, k, v = (heads(rows_qkv, B * Tf, N + 1, H, hd, col=i * D) for i in range(3))
    dq, dk, dv = attn_b(X, pre + "attn.bwd", q, k, v, c["o_s"], c["lse_s"], heads(do_rows.reshape(-1, D), B * Tf, N + 1, H, hd),
                        scale=d["scale"])
    dqkv_seq = torch.cat([unheads(t).view(B * Tf, N + 1, D) for t in (dq, dk, dv)], 2)      # [B T, N + 1, 3D]
    dqkv_tok = torch.empty(R, 3 * D, dtype=F64, device=dev)
    dqkv_tok[ridx] = dqkv_seq[:, 1:].reshape(-1, 3 * D)
    # the shared cls row's gradient is the sum over the T frames that read it
    dqkv_cls = X.call(pre + "attn.cls_sum", "group_reduce", dict(x=dqkv_seq[:, 0]), dict(G=B, T=Tf, scale=1.0, broadcast=False),
                      dict(out=BF16))["out"]
    dqkv = torch.cat([dqkv_tok, dqkv_cls])
    qkv_wgrad(X, pre + "attn.qkv", pre + "attn.", dqkv, c["ln_s"], D, T)
    dln_s = gemm(X, pre + "attn.qkv.dgrad", dqkv, W[pre + "attn.qkv.weight"].T, acc=False)
    dxt, _ = ln_bwd(X, pre + "norm1.bwd", dln_s, c["xt"], W, pre + "norm1", c["m_s"], c["r_s"], T, add=dy)
    wgrad(X, pre + "temporal_fc", dxt[:R], c["proj_t"], pre + "temporal_fc.weight", pre + "temporal_fc.bias", T)
    dproj = gemm(X, pre + "temporal_fc.dgrad", dxt[:R], W[pre + "temporal_fc.weight"].T, acc=False)
    wgrad(X, pre + "temporal_attn.proj", dproj, c["att_t"], pre + "temporal_attn.proj.weight", pre + "temporal_attn.proj.bias", T)
    datt_t = gemm(X, pre + "temporal_attn.proj.dgrad", dproj, W[pre + "temporal_attn.proj.weight"].T, acc=False)
    q, k, v = (heads(c["qkv_t"], R // Tf, Tf, H, hd, col=i * D) for i in range(3))
    dq, dk, dv = attn_b(X, pre + "temporal_attn.bwd", q, k, v, heads(c["att_t"], R // Tf, Tf, H, hd), c["lse_t"],
                        heads(datt_t, R // Tf, Tf, H, hd), scale=d["scale"], temporal=True)
    dqkv_t = torch.cat([unheads(t) for t in (dq, dk, dv)], 1)
    qkv_wgrad(X, pre + "temporal_attn.qkv", pre + "temporal_attn.", dqkv_t, c["ln_t"], D, T)
    dln_t = gemm(X, pre + "temporal_attn.qkv.dgrad", dqkv_t, W[pre + "temporal_attn.qkv.weight"].T, acc=False)
    dx_tok, _ = ln_bwd(X, pre + "temporal_ln.bwd", dln_t, c["x"][:R], W, pre + "temporal_ln", c["m_t"], c["r_t"], T,
                       add=dxt[:R])
    return torch.cat([dx_tok, dxt[R:]])


def vit_fwd(X, W, video, vcfg, fused):
    """port.timesformer: patch GEMM with the (pos + temporal) table, cls rows, norm_pre, blocks, final LayerNorm in
    (t n) order.  fused: the patch GEMM gathers its rows from the video (patch_embed_gemm) instead of an im2col."""
    d = dims_vit(vcfg, video.shape[0])
    B, D, T, N, R, P = d["B"], d["D"], d["T"], d["N"], d["R"], d["P"]
    pos, temb = W[VE + "pos_embed"], W[VE + "temporal_embed"]
    table = X.rnd(X.rnd(pos[0, 1:, None, :] + temb[0, None, :, :], F32), BF16).reshape(N * T, D)
    wp = W[VE + "patch_embed.proj.weight"].reshape(D, -1)
    c = dict(d=d, video=video, blocks=[])
    if fused:
        kw = dict(act=ACT_NONE, alpha=1.0, accumulate=False, drop=None, aux=False, out_dtype=F32, P=P)
        xt = X.call("vit.patch_embed", "patch_embed_gemm", dict(video=video, B=wp, bias=W.get(VE + "patch_embed.proj.bias"),
                    residual=table.repeat(B, 1)), kw, dict(D=F32))["D"]
    else:
        patches = X.call("vit.im2col", "im2col", dict(video=video), dict(P=P, ld=(wp.shape[1] + 7) // 8 * 8),
                         dict(out=BF16))["out"]
        c["patches"] = patches
        xt = gemm(X, "vit.patch_embed", patches, wp, bias=W.get(VE + "patch_embed.proj.bias"), residual=table.repeat(B, 1),
                  out=F32, acc=False)
    cls = X.rnd(W[VE + "cls_token"][0, 0] + pos[0, 0], F32)
    x0 = torch.cat([xt, cls.expand(B, D)])
    c["x0"] = x0
    x = x0
    if VE + "norm_pre.weight" in W:
        x, c["m0"], c["r0"] = ln_fwd(X, "vit.norm_pre", x0, W, VE + "norm_pre", d["eps"], y=F32)
    for i in range(d["depth"]):
        x, bc = vit_block_fwd(X, W, f"{VE}blocks.{i}.", x, d)
        c["blocks"].append(bc)
    rows = final_rows(d)
    c["xL"], c["rows"] = x, rows
    out, c["mf"], c["rf"] = ln_fwd(X, "vit.norm", x[rows.to(x.device)], W, VE + "norm", d["eps"], in_rows=rows)
    return out, c


def vit_bwd(X, W, T, c, d_out):
    d = c["d"]
    B, D, Tf, N, R, RB = d["B"], d["D"], d["T"], d["N"], d["R"], d["RB"]
    rows = c["rows"]
    dev = d_out.device
    dxr, _ = ln_bwd(X, "vit.norm.bwd", d_out, c["xL"][rows.to(dev)], W, VE + "norm", c["mf"], c["rf"], T, in_rows=rows,
                    xrows=rows.tolist())
    dx = torch.empty(RB, D, dtype=F64, device=dev)
    dx[rows.to(dev)] = dxr
    for i in reversed(range(d["depth"])):
        dx = vit_block_bwd(X, W, T, f"{VE}blocks.{i}.", c["blocks"][i], dx, d)
    dx0 = dx
    if VE + "norm_pre.weight" in W:
        dx0, _ = ln_bwd(X, "vit.norm_pre.bwd", dx, c["x0"], W, VE + "norm_pre", c["m0"], c["r0"], T)
    # the cls rows carry cls_token + pos_embed[0]; the token rows the (pos_embed[1 + n] + temporal_embed[t]) table
    if VE + "cls_token" in T or VE + "pos_embed" in T:
        dcls = colsum(X, "vit.cls.colsum", dx0[R:], None)
        if VE + "cls_token" in T:
            X.grad_add("vit.cls_token.grad", VE + "cls_token", 0, dcls[None])
        if VE + "pos_embed" in T:
            X.grad_add("vit.pos_embed0.grad", VE + "pos_embed", 0, dcls[None])
    if VE + "pos_embed" in T or VE + "temporal_embed" in T:
        dtab = colsum(X, "vit.table.colsum", dx0[:R].reshape(B, N * Tf * D), None).view(N, Tf, D)
        if VE + "pos_embed" in T:
            X.grad_add("vit.pos_embed.grad", VE + "pos_embed", D, dtab.permute(1, 0, 2))
        if VE + "temporal_embed" in T:
            X.grad_add("vit.temporal_embed.grad", VE + "temporal_embed", 0, dtab)
    pk, bk = VE + "patch_embed.proj.weight", VE + "patch_embed.proj.bias"
    patches = c.get("patches")
    if patches is None and pk in T:
        # the fused forward never formed the patch matrix: the weight gradient's B operand is materialised here
        patches = X.call("vit.im2col.bwd", "im2col", dict(video=c["video"]), dict(P=d["P"], ld=3 * d["P"] ** 2),
                         dict(out=BF16))["out"]
    if patches is not None:
        wgrad(X, "vit.patch_embed", dx0[:R], patches, pk, bk, T)
    elif bk in T:
        colsum(X, "vit.patch_embed.bgrad", dx0[:R], (bk, 0))
    return dx0


# ---------------------------------------------------------------------------------- AttentionPool
def attn_pool_fwd(X, W, img, B, nheads):
    """port.attention_pool on learnable_queries.repeat(B): the query block is normalised and projected once; each
    sample's keys are its K1 normalised image rows and the learned bias_k / bias_v row (one padding slot)."""
    D = img.shape[1]
    K1 = img.shape[0] // B
    KP, hd = K1 + 1, D // nheads
    lq = W["learnable_queries"][0]
    Q = lq.shape[0]
    dev = img.device
    c = dict(B=B, Q=Q, K1=K1, D=D, H=nheads, hd=hd, lq=lq, img=img)
    c["xq"], c["mq"], c["rq"] = ln_fwd(X, "ap.norm1", lq, W, AP + "norm1", 1e-6)
    rows = torch.cat([torch.arange(B * K1).view(B, K1), torch.full((B, 1), -1)], 1).reshape(-1)
    pad = rows < 0
    xin = img[rows.clamp(min=0).to(dev)].masked_fill(pad.to(dev)[:, None], 0.0)
    c["kvn"], c["mk"], c["rk"] = ln_fwd(X, "ap.normk", xin, W, AP + "normk", 1e-6, in_rows=rows, pad=pad)
    c["rows"], c["pad"] = rows, pad
    w, b = W[AP + "attn.in_proj_weight"], W[AP + "attn.in_proj_bias"]
    c["qp"] = gemm(X, "ap.q_proj", c["xq"], w[:D], bias=b[:D], acc=False)
    kvp = gemm(X, "ap.kv_proj", c["kvn"], w[D:], bias=b[D:], acc=False).clone()
    kvp.view(B, KP, 2 * D)[:, K1] = torch.cat([W[AP + "attn.bias_k"].reshape(-1), W[AP + "attn.bias_v"].reshape(-1)])
    c["kvp"] = kvp
    q = heads(c["qp"], 1, Q, nheads, hd).expand(B, -1, -1, -1)
    k, v = heads(kvp, B, KP, nheads, hd), heads(kvp, B, KP, nheads, hd, col=D)
    c["o"], c["lse"] = attn(X, "ap.attn", q, k, v, scale=hd ** -0.5)
    c["att"] = unheads(c["o"])
    # the residual is the normalised query (port: x = x + out_proj(...))
    c["x1"] = gemm(X, "ap.out_proj", c["att"], W[AP + "attn.out_proj.weight"], bias=W[AP + "attn.out_proj.bias"],
                   residual=c["xq"].repeat(B, 1), out=F32, acc=False)
    c["ln2"], c["m2"], c["r2"] = ln_fwd(X, "ap.norm2", c["x1"], W, AP + "norm2", 1e-6)
    c["h"], c["dact"] = gemm(X, "ap.mlp.fc1", c["ln2"], W[AP + "mlp.fc1.weight"], bias=W[AP + "mlp.fc1.bias"],
                             act=ACT_GELU_ERF, aux=True, acc=False)
    out = gemm(X, "ap.mlp.fc2", c["h"], W[AP + "mlp.fc2.weight"], bias=W[AP + "mlp.fc2.bias"], residual=c["x1"], acc=False)
    return out, c


def attn_pool_bwd(X, W, T, c, dout):
    B, Q, K1, D, H, hd = c["B"], c["Q"], c["K1"], c["D"], c["H"], c["hd"]
    KP = K1 + 1
    wgrad(X, "ap.mlp.fc2", dout, c["h"], AP + "mlp.fc2.weight", AP + "mlp.fc2.bias", T)
    dpre = gemm(X, "ap.mlp.fc2.dgrad", dout, W[AP + "mlp.fc2.weight"].T, act=ACT_GELU_ERF, aux_in=c["dact"], acc=False)
    wgrad(X, "ap.mlp.fc1", dpre, c["ln2"], AP + "mlp.fc1.weight", AP + "mlp.fc1.bias", T)
    dln2 = gemm(X, "ap.mlp.fc1.dgrad", dpre, W[AP + "mlp.fc1.weight"].T, acc=False)
    dx1, _ = ln_bwd(X, "ap.norm2.bwd", dln2, c["x1"], W, AP + "norm2", c["m2"], c["r2"], T, add=dout)
    wgrad(X, "ap.out_proj", dx1, c["att"], AP + "attn.out_proj.weight", AP + "attn.out_proj.bias", T)
    datt = gemm(X, "ap.out_proj.dgrad", dx1, W[AP + "attn.out_proj.weight"].T, acc=False)
    q = heads(c["qp"], 1, Q, H, hd).expand(B, -1, -1, -1)
    k, v = heads(c["kvp"], B, KP, H, hd), heads(c["kvp"], B, KP, H, hd, col=D)
    dq, dk, dv = attn_b(X, "ap.attn.bwd", q, k, v, c["o"], c["lse"], heads(datt, B, Q, H, hd), scale=hd ** -0.5)
    dkvp_raw = torch.cat([unheads(dk), unheads(dv)], 1)                       # [B KP, 2D]
    # the learned bias_k / bias_v row: its gradient is the batch sum of that row, which then leaves the projections
    brow = dkvp_raw.view(B, KP, 2 * D)[:, K1]
    if AP + "attn.bias_k" in T:
        X.grad_add("ap.bias_k.grad", AP + "attn.bias_k", 0, brow[:, :D])
    if AP + "attn.bias_v" in T:
        X.grad_add("ap.bias_v.grad", AP + "attn.bias_v", 0, brow[:, D:])
    dkvp = dkvp_raw.clone()
    dkvp.view(B, KP, 2 * D)[:, K1] = 0.0
    # the query block is shared by the batch: its gradients are sums over the samples (query and residual paths)
    dq_sum = colsum(X, "ap.q.colsum", unheads(dq).reshape(B, Q * D), None)
    dqp = X.rnd(dq_sum.view(Q, D), BF16)
    dres = colsum(X, "ap.res.colsum", dx1.reshape(B, Q * D), None)
    if AP + "attn.in_proj_weight" in T:
        gemm(X, "ap.q_proj.wgrad", dqp.T, c["xq"].T, out=F32, acc=(AP + "attn.in_proj_weight", 0))
        gemm(X, "ap.kv_proj.wgrad", dkvp.T, c["kvn"].T, out=F32, acc=(AP + "attn.in_proj_weight", D * D))
    if AP + "attn.in_proj_bias" in T:
        colsum(X, "ap.q_proj.bgrad", dqp, (AP + "attn.in_proj_bias", 0))
        colsum(X, "ap.kv_proj.bgrad", dkvp, (AP + "attn.in_proj_bias", D))
    w_in = W[AP + "attn.in_proj_weight"]
    dxq = gemm(X, "ap.q_proj.dgrad", dqp, w_in[:D].T, out=F32, acc=False)
    dxq = X.rnd(X.rnd(dxq + dres.view(Q, D), F32), BF16)
    dlq, _ = ln_bwd(X, "ap.norm1.bwd", dxq, c["lq"], W, AP + "norm1", c["mq"], c["rq"], T)
    if "learnable_queries" in T:
        X.grad_add("ap.learnable_queries.grad", "learnable_queries", 0, dlq[None])
    dkvn = gemm(X, "ap.kv_proj.dgrad", dkvp, w_in[D:].T, acc=False)
    rows = c["rows"]
    valid = (~c["pad"]).to(dkvn.device)
    xin = c["img"][rows.clamp(min=0).to(dkvn.device)].masked_fill(~valid[:, None], 0.0)
    dxr, _ = ln_bwd(X, "ap.normk.bwd", dkvn, xin, W, AP + "normk", c["mk"], c["rk"], T, in_rows=rows,
                    xrows=rows.clamp(min=0).tolist())
    return dxr[valid]


# ---------------------------------------------------------------------------------- GPT-3 decoder
def dims_gpt(gcfg):
    H, nh = gcfg["hidden_size"], gcfg["num_attention_heads"]
    return dict(H=H, nh=nh, hd=H // nh, layers=gcfg["num_hidden_layers"], F=gcfg.get("ffn_hidden_size") or 4 * H,
                V=gcfg["vocab_size"], eps=gcfg.get("layernorm_epsilon", 1e-12), scale=1.0 / math.sqrt(H // nh))


class Drop:
    """The decoder pass's dropout sites (port.gpt3_layer: attention 4 li + 1, bias-dropout-adds 4 li + 2 / 4 li + 3,
    embedding 0) as (seed, offset, site, p) specs; None where p = 0."""

    def __init__(self, seed, offset, p_hidden, p_attn):
        self.seed, self.offset, self.ph, self.pa = int(seed), int(offset), float(p_hidden), float(p_attn)

    def _s(self, site, p):
        return (self.seed, self.offset, site, f32(p)) if p > 0 else None

    def embed(self):
        return self._s(0, self.ph)

    def attn(self, i):
        return self._s(4 * i + 1, self.pa)

    def bda_attn(self, i):
        return self._s(4 * i + 2, self.ph)

    def bda_mlp(self, i):
        return self._s(4 * i + 3, self.ph)


def _dr(drop, fn, *a):
    return getattr(drop, fn)(*a) if drop is not None else None


def gpt_layer_fwd(X, W, pre, x, g, B, S, drop, li):
    H, nh, hd = g["H"], g["nh"], g["hd"]
    c = dict(x=x)
    c["ln1"], c["m1"], c["r1"] = ln_fwd(X, pre + "input_layernorm", x, W, pre + "input_layernorm", g["eps"])
    c["qkv"] = gemm(X, pre + "qkv", c["ln1"], W[pre + "self_attention.query_key_value.weight"],
                    bias=W[pre + "self_attention.query_key_value.bias"], acc=False)
    q, k, v = (heads(c["qkv"], B, S, nh, hd, col=i * hd, hs=3 * hd) for i in range(3))   # per head [q|k|v]
    c["o"], c["lse"] = attn(X, pre + "attn", q, k, v, scale=g["scale"], causal=True, drop=_dr(drop, "attn", li))
    c["att"] = unheads(c["o"])
    c["x1"] = gemm(X, pre + "dense", c["att"], W[pre + "self_attention.dense.weight"], bias=W[pre + "self_attention.dense.bias"],
                   residual=x, out=F32, drop=_dr(drop, "bda_attn", li), acc=False)
    c["ln2"], c["m2"], c["r2"] = ln_fwd(X, pre + "post_attention_layernorm", c["x1"], W, pre + "post_attention_layernorm", g["eps"])
    c["h"], c["dact"] = gemm(X, pre + "mlp.dense_h_to_4h", c["ln2"], W[pre + "mlp.dense_h_to_4h.weight"],
                             bias=W[pre + "mlp.dense_h_to_4h.bias"], act=ACT_GELU_TANH, aux=True, acc=False)
    out = gemm(X, pre + "mlp.dense_4h_to_h", c["h"], W[pre + "mlp.dense_4h_to_h.weight"], bias=W[pre + "mlp.dense_4h_to_h.bias"],
               residual=c["x1"], out=F32, drop=_dr(drop, "bda_mlp", li), acc=False)
    return out, c


def gpt_layer_bwd(X, W, T, pre, c, dout, dout_d, g, B, S, drop, li, train_w):
    """dout: gradient of the layer output; dout_d: the same through the layer's MLP bias-dropout-add mask.  Returns
    (dx, dx_d), dx_d through the mask of the site that produced the layer input (previous layer's MLP
    bias-dropout-add, or the embedding dropout for layer 0)."""
    nh, hd = g["nh"], g["hd"]
    Tw = T if train_w else set()
    wgrad(X, pre + "mlp.dense_4h_to_h", dout_d, c["h"], pre + "mlp.dense_4h_to_h.weight", pre + "mlp.dense_4h_to_h.bias", Tw)
    dpre = gemm(X, pre + "mlp.dense_4h_to_h.dgrad", dout_d, W[pre + "mlp.dense_4h_to_h.weight"].T, act=ACT_GELU_TANH,
                aux_in=c["dact"], acc=False)
    wgrad(X, pre + "mlp.dense_h_to_4h", dpre, c["ln2"], pre + "mlp.dense_h_to_4h.weight", pre + "mlp.dense_h_to_4h.bias", Tw)
    dln2 = gemm(X, pre + "mlp.dense_h_to_4h.dgrad", dpre, W[pre + "mlp.dense_h_to_4h.weight"].T, acc=False)
    # the residual stream's gradient passes the bias-dropout-add undropped; the attention branch sees it dropped
    dx1, dx1_d = ln_bwd(X, pre + "post_attention_layernorm.bwd", dln2, c["x1"], W, pre + "post_attention_layernorm", c["m2"],
                        c["r2"], T, add=dout, drop=_dr(drop, "bda_attn", li))
    wgrad(X, pre + "dense", dx1_d, c["att"], pre + "self_attention.dense.weight", pre + "self_attention.dense.bias", Tw)
    datt = gemm(X, pre + "dense.dgrad", dx1_d, W[pre + "self_attention.dense.weight"].T, acc=False)
    q, k, v = (heads(c["qkv"], B, S, nh, hd, col=i * hd, hs=3 * hd) for i in range(3))
    dq, dk, dv = attn_b(X, pre + "attn.bwd", q, k, v, c["o"], c["lse"], heads(datt, B, S, nh, hd), scale=g["scale"],
                        causal=True, drop=_dr(drop, "attn", li))
    dqkv = torch.stack([unheads(t).view(B * S, nh, hd) for t in (dq, dk, dv)], 2).reshape(B * S, 3 * nh * hd)
    wgrad(X, pre + "qkv", dqkv, c["ln1"], pre + "self_attention.query_key_value.weight",
          pre + "self_attention.query_key_value.bias", Tw)
    dln1 = gemm(X, pre + "qkv.dgrad", dqkv, W[pre + "self_attention.query_key_value.weight"].T, acc=False)
    d_in = (_dr(drop, "bda_mlp", li - 1) if li > 0 else _dr(drop, "embed")) if drop is not None else None
    return ln_bwd(X, pre + "input_layernorm.bwd", dln1, c["x"], W, pre + "input_layernorm", c["m1"], c["r1"], T,
                  add=dx1, drop=d_in)


def gpt_fwd(X, W, x, gcfg, B, S, drop=None, out_rows=None):
    """port.gpt3_decoder after the position add: x [B S, H] fp32 input embeddings (+ positions); the embedding dropout,
    the layers, the final LayerNorm of out_rows (all rows when None)."""
    g = dims_gpt(gcfg)
    c = dict(g=g, B=B, S=S, drop=drop, layers=[], out_rows=out_rows)
    if drop is not None and drop.embed() is not None:
        x = X.call("gpt.embed_dropout", "dropout", dict(x=x), dict(drop=drop.embed()), dict(y=F32))["y"]
    for i in range(g["layers"]):
        x, lc = gpt_layer_fwd(X, W, f"{GPT}encoder.layers.{i}.", x, g, B, S, drop, i)
        c["layers"].append(lc)
    c["xL"] = x
    xr = x if out_rows is None else x[out_rows.long().to(x.device)]
    hid, c["mf"], c["rf"] = ln_fwd(X, "gpt.final_layernorm", xr, W, GPT + "encoder.final_layernorm", g["eps"], in_rows=out_rows)
    return hid, c


def gpt_bwd(X, W, T, c, dhid, train_w=False):
    g, B, S, drop, out_rows = c["g"], c["B"], c["S"], c["drop"], c["out_rows"]
    xL = c["xL"]
    dev = dhid.device
    rows = torch.arange(xL.shape[0]) if out_rows is None else out_rows.long().cpu()
    r = ln_bwd(X, "gpt.final_layernorm.bwd", dhid, xL[rows.to(dev)], W, GPT + "encoder.final_layernorm", c["mf"], c["rf"], T,
               drop=_dr(drop, "bda_mlp", g["layers"] - 1), in_rows=out_rows, xrows=rows.tolist())
    # rows the final LayerNorm does not emit get an exact zero gradient
    dx, dx_d = (torch.zeros_like(xL).index_copy(0, rows.to(dev), t) for t in r)
    for i in reversed(range(g["layers"])):
        dx, dx_d = gpt_layer_bwd(X, W, T, f"{GPT}encoder.layers.{i}.", c["layers"][i], dx, dx_d, g, B, S, drop, i, train_w)
    return dx_d


def lm_head_fwd(X, W, hid, labels):
    logits = gemm(X, "lm_head", hid, W[GPT + "embedding.word_embeddings.weight"], acc=False)
    r = X.call("ce", "ce_fwd", dict(logits=logits, labels=labels.reshape(-1)), {}, dict(loss=F32, lse=F32))
    return logits, r["loss"], r["lse"]


def lm_head_bwd(X, W, T, hid, logits, labels, lse, grow):
    dl = X.call("ce.bwd", "ce_bwd", dict(logits=logits, labels=labels.reshape(-1), lse=lse, g=grow), {},
                dict(dlogits=BF16))["dlogits"]
    emb = GPT + "embedding.word_embeddings.weight"
    if emb in T:
        gemm(X, "lm_head.wgrad", dl.T, hid.T, out=F32, acc=(emb, 0))
    return gemm(X, "lm_head.dgrad", dl, W[emb].T, acc=False)


# ---------------------------------------------------------------------------------- pre-training step
def pretrain_fwd(X, W, video, ids, targets, loss_mask, vcfg, gcfg, Q, drop=None, fused=False):
    """port.pretrain_forward: TimeSformer -> AttentionPool -> visual_fc written into the decoder's prefix rows with
    their positions -> token embeddings + positions in the text rows -> decoder -> LM head and CE over the text rows
    (the prefix rows carry loss_mask 0)."""
    B, L = ids.shape
    S = Q + L
    H = gcfg["hidden_size"]
    img, cv = vit_fwd(X, W, video, vcfg, fused)
    qf, ca = attn_pool_fwd(X, W, img, B, vcfg["num_heads"])
    pos = W[GPT + "embedding.position_embeddings.weight"]
    xq = gemm(X, "visual_fc", qf, W["visual_fc.weight"], bias=W["visual_fc.bias"], residual=pos[:Q].repeat(B, 1), out=F32,
              acc=False)
    xt = X.call("embed_gather", "embed_gather", dict(ids=ids, table=W[GPT + "embedding.word_embeddings.weight"], pos=pos),
                dict(S=S, row_offset=Q), dict(out=F32))["out"]
    x_in = torch.cat([xq.view(B, Q, H), xt.view(B, L, H)], 1).reshape(B * S, H)
    text_rows = (torch.arange(B)[:, None] * S + torch.arange(Q, S)[None, :]).reshape(-1).int()
    hid, cg = gpt_fwd(X, W, x_in, gcfg, B, S, drop=drop, out_rows=text_rows)
    tt = targets[:, Q:].reshape(-1)
    logits, losses, lse = lm_head_fwd(X, W, hid, tt)
    lbs = torch.zeros(B, S, dtype=F64, device=losses.device)
    lbs[:, Q:] = losses.view(B, L)
    lm = loss_mask.reshape(-1).to(F64)
    loss = (lbs[:, :-1].reshape(-1) * lm).sum() / lm.sum()
    c = dict(cv=cv, ca=ca, cg=cg, qf=qf, hid=hid, logits=logits, lse=lse, tt=tt, dims=(B, S, Q, H), x_in=x_in)
    return loss, lbs, c


def pretrain_bwd(X, W, T, c, loss_mask, dloss=1.0):
    """PretrainFn.backward: d loss / d losses = loss_mask / loss_mask.sum() on the text rows, then the stages in reverse;
    the visual_fc gradient comes from the decoder input's prefix rows."""
    B, S, Q, H = c["dims"]
    lm = loss_mask.to(F32)
    grow = torch.zeros(B, S, dtype=F32, device=lm.device)
    grow[:, :-1] = lm * (torch.tensor(float(dloss), dtype=F32) / lm.sum())
    grow = grow.to(F64)
    dhid = lm_head_bwd(X, W, T, c["hid"], c["logits"], c["tt"], c["lse"], grow[:, Q:].reshape(-1))
    dx_in = gpt_bwd(X, W, T, c["cg"], dhid)
    dqf = dx_in.view(B, S, H)[:, :Q].reshape(B * Q, H)
    wgrad(X, "visual_fc", dqf, c["qf"], "visual_fc.weight", "visual_fc.bias", T)
    dq = gemm(X, "visual_fc.dgrad", dqf, W["visual_fc.weight"].T, acc=False)
    d_img = attn_pool_bwd(X, W, T, c["ca"], dq)
    vit_bwd(X, W, T, c["cv"], d_img)
    return d_img


# ---------------------------------------------------------------------------------- EVA image encoder
def dims_eva(ecfg, B):
    P, D, H = ecfg["patch_size"], ecfg["embed_dim"], ecfg["num_heads"]
    N = (ecfg["img_size"] // P) ** 2
    return dict(P=P, D=D, H=H, hd=D // H, N=N, S=N + 1, B=B, depth=ecfg["depth"], eps=ecfg.get("eps", 1e-6),
                scale=(D // H) ** -0.5, K=3 * P * P, Kp=(3 * P * P + 7) // 8 * 8)


def eva_fwd(X, W, image, ecfg):
    """port.eva_vit: Conv2d patch embedding with bias as one GEMM over the im2col rows (K = 3 P P zero-padded to a
    multiple of 8: 588 -> 592 at P = 14), the patch rows stored row-blocked after each sample's cls row with the
    position embeddings added, pre-LN blocks over [cls | patches], final LayerNorm.  Rows b (N + 1) + i."""
    d = dims_eva(ecfg, image.shape[0])
    B, D, N, S, H, hd = d["B"], d["D"], d["N"], d["S"], d["H"], d["hd"]
    dev = image.device
    patches = X.call("eva.im2col", "im2col", dict(video=image[:, :, None]), dict(P=d["P"], ld=d["Kp"]),
                     dict(out=BF16))["out"]
    wp = torch.zeros(D, d["Kp"], dtype=F64, device=dev)
    wp[:, :d["K"]] = W[VE + "patch_embed.proj.weight"].reshape(D, -1)
    pos = W[VE + "pos_embed"][0]
    xp = gemm(X, "eva.patch_embed", patches, wp, bias=W[VE + "patch_embed.proj.bias"], residual=pos[1:].repeat(B, 1), out=F32)
    cls = X.rnd(W[VE + "cls_token"][0, 0] + pos[0], F32)
    x = torch.cat([cls.expand(B, 1, D), xp.view(B, N, D)], 1).reshape(B * S, D)
    c = dict(d=d, patches=patches, blocks=[])
    for i in range(d["depth"]):
        pre = f"{VE}blocks.{i}."
        bc = dict(x=x)
        bc["ln1"], bc["m1"], bc["r1"] = ln_fwd(X, pre + "norm1", x, W, pre + "norm1", d["eps"])
        bc["qkv"] = gemm(X, pre + "attn.qkv", bc["ln1"], W[pre + "attn.qkv.weight"], bias=qkv_bias(W, pre + "attn."))
        q, k, v = (heads(bc["qkv"], B, S, H, hd, col=j * D) for j in range(3))
        bc["o"], bc["lse"] = attn(X, pre + "attn", q, k, v, scale=d["scale"])
        bc["att"] = unheads(bc["o"])
        bc["x1"] = gemm(X, pre + "attn.proj", bc["att"], W[pre + "attn.proj.weight"], bias=W[pre + "attn.proj.bias"],
                        residual=x, out=F32)
        bc["ln2"], bc["m2"], bc["r2"] = ln_fwd(X, pre + "norm2", bc["x1"], W, pre + "norm2", d["eps"])
        bc["h"], bc["dact"] = gemm(X, pre + "mlp.fc1", bc["ln2"], W[pre + "mlp.fc1.weight"], bias=W[pre + "mlp.fc1.bias"],
                                   act=ACT_GELU_ERF, aux=True)
        x = gemm(X, pre + "mlp.fc2", bc["h"], W[pre + "mlp.fc2.weight"], bias=W[pre + "mlp.fc2.bias"], residual=bc["x1"],
                 out=F32)
        c["blocks"].append(bc)
    c["xL"] = x
    out, c["mf"], c["rf"] = ln_fwd(X, "eva.norm", x, W, VE + "norm", d["eps"])
    return out, c


def eva_bwd(X, W, T, c, d_out):
    d = c["d"]
    B, D, N, S, H, hd = d["B"], d["D"], d["N"], d["S"], d["H"], d["hd"]
    dx, _ = ln_bwd(X, "eva.norm.bwd", d_out, c["xL"], W, VE + "norm", c["mf"], c["rf"], T)
    for i in reversed(range(d["depth"])):
        pre, bc = f"{VE}blocks.{i}.", c["blocks"][i]
        wgrad(X, pre + "mlp.fc2", dx, bc["h"], pre + "mlp.fc2.weight", pre + "mlp.fc2.bias", T)
        dpre = gemm(X, pre + "mlp.fc2.dgrad", dx, W[pre + "mlp.fc2.weight"].T, act=ACT_GELU_ERF, aux_in=bc["dact"])
        wgrad(X, pre + "mlp.fc1", dpre, bc["ln2"], pre + "mlp.fc1.weight", pre + "mlp.fc1.bias", T)
        dln2 = gemm(X, pre + "mlp.fc1.dgrad", dpre, W[pre + "mlp.fc1.weight"].T)
        dx1, _ = ln_bwd(X, pre + "norm2.bwd", dln2, bc["x1"], W, pre + "norm2", bc["m2"], bc["r2"], T, add=dx)
        wgrad(X, pre + "attn.proj", dx1, bc["att"], pre + "attn.proj.weight", pre + "attn.proj.bias", T)
        datt = gemm(X, pre + "attn.proj.dgrad", dx1, W[pre + "attn.proj.weight"].T)
        q, k, v = (heads(bc["qkv"], B, S, H, hd, col=j * D) for j in range(3))
        dq, dk, dv = attn_b(X, pre + "attn.bwd", q, k, v, bc["o"], bc["lse"], heads(datt, B, S, H, hd), scale=d["scale"])
        dqkv = torch.cat([unheads(t) for t in (dq, dk, dv)], 1)
        qkv_wgrad(X, pre + "attn.qkv", pre + "attn.", dqkv, bc["ln1"], D, T)
        dln1 = gemm(X, pre + "attn.qkv.dgrad", dqkv, W[pre + "attn.qkv.weight"].T)
        dx, _ = ln_bwd(X, pre + "norm1.bwd", dln1, bc["x"], W, pre + "norm1", bc["m1"], bc["r1"], T, add=dx1)
    dx3 = dx.view(B, S, D)
    # cls_token feeds row 0 of every sample, pos_embed every row of every sample: sums over the batch
    if VE + "cls_token" in T:
        X.grad_add("eva.cls_token.grad", VE + "cls_token", 0, dx3[:, 0])
    if VE + "pos_embed" in T:
        X.grad_add("eva.pos_embed.grad", VE + "pos_embed", 0, dx3)
    dpatch = dx3[:, 1:].reshape(B * N, D)
    pk = VE + "patch_embed.proj.weight"
    if pk in T and d["Kp"] == d["K"]:
        gemm(X, "eva.patch_embed.wgrad", dpatch.T, c["patches"].T, out=F32, acc=(pk, 0))
    elif pk in T:
        # the zero-padded K columns accumulate into a temporary; the real ones are added to the gradient
        tmp = gemm(X, "eva.patch_embed.wgrad", dpatch.T, c["patches"].T, out=F32, acc=TMP)
        X.grad_add("eva.patch_embed.weight.grad", pk, 0, tmp[:, :d["K"]][None])
    if VE + "patch_embed.proj.bias" in T:
        colsum(X, "eva.patch_embed.bgrad", dpatch, (VE + "patch_embed.proj.bias", 0))
    return dx


# ---------------------------------------------------------------------------------- component path
def component_fwd(X, W, video, ids, targets, vcfg, gcfg, Q, drop=None, fused=False):
    """The model's component path (VitFn -> AttnPoolFn -> LinearFn(visual_fc) -> GptFn): the decoder input is
    cat(visual_fc(queries), word_embeddings[ids]) in bf16, positions added in fp32, LM head and CE over every row."""
    B, L = ids.shape
    S, H = Q + L, gcfg["hidden_size"]
    img, cv = vit_fwd(X, W, video, vcfg, fused)
    qa, ca = attn_pool_fwd(X, W, img, B, vcfg["num_heads"])
    qf = gemm(X, "visual_fc", qa, W["visual_fc.weight"], bias=W["visual_fc.bias"])
    emb = W[GPT + "embedding.word_embeddings.weight"][ids.reshape(-1).to(qf.device)]
    inp = torch.cat([qf.view(B, Q, H), emb.view(B, L, H)], 1)
    pos = W[GPT + "embedding.position_embeddings.weight"][:S]
    x_in = X.rnd(inp + pos[None], F32).reshape(B * S, H)
    hid, cg = gpt_fwd(X, W, x_in, gcfg, B, S, drop=drop)
    tt = targets.reshape(-1)
    logits, losses, lse = lm_head_fwd(X, W, hid, tt)
    return losses.view(B, S), dict(cv=cv, ca=ca, cg=cg, qa=qa, hid=hid, logits=logits, lse=lse, tt=tt, dims=(B, S, Q, H))


def component_bwd(X, W, T, c, loss_mask):
    """Autograd of masked_mean_loss hands GptFn d loss / d losses = loss_mask * fl(1 / loss_mask.sum()) on [:, :-1];
    LinearFn's backward runs its dgrad before the weight gradients."""
    B, S, Q, H = c["dims"]
    lm = loss_mask.to(F32)
    g = torch.zeros(B, S, dtype=F32, device=lm.device)
    g[:, :-1] = lm * (torch.tensor(1.0, dtype=F32, device=lm.device) / lm.sum())
    dhid = lm_head_bwd(X, W, T, c["hid"], c["logits"], c["tt"], c["lse"], g.to(F64).reshape(-1))
    dx = gpt_bwd(X, W, T, c["cg"], dhid)
    dqf = dx.view(B, S, H)[:, :Q].reshape(B * Q, H)
    dq = gemm(X, "visual_fc.dgrad", dqf, W["visual_fc.weight"].T)
    wgrad(X, "visual_fc", dqf, c["qa"], "visual_fc.weight", "visual_fc.bias", T)
    d_img = attn_pool_bwd(X, W, T, c["ca"], dq)
    vit_bwd(X, W, T, c["cv"], d_img)
    return d_img


# ---------------------------------------------------------------------------------- GPT-3 decoding
POISON = 3.0e4


def poison_(store):
    """Fill a bf16 KV-cache store with the finite poison +-3e4 in alternating signs (every row starts with +), so
    that a read of a slot no step wrote fails its bound."""
    v = store.view(-1, 2)
    v[:, 0] = POISON
    v[:, 1] = -POISON
    return store


def poison_row(width, dev="cpu"):
    r = torch.full((width,), POISON, dtype=F64, device=dev)
    r[1::2] = -POISON
    return r.to(BF16).to(F64)


class KVHistory:
    """The decoder's KV cache as the decoding programs see it: for each sequence, the ids of the cached QKV rows of its
    positions in order.  Every layer's row of one position has the same id; id 0 is the poison row of a slot that was
    never written.  reindex / reorder permute the sequences' lists; share_prefill starts every beam of a clip from
    its clip's prefill rows."""

    def __init__(self, layers, B, width, dev):
        self.B, self.len = B, 0
        self.pool = [[poison_row(width, dev)[None]] for _ in range(layers)]
        self.n = [1] * layers
        self._cat = [None] * layers
        self.seq = [[] for _ in range(B)]

    def put(self, i, rows):
        """Cache the QKV rows [r, 3H] of layer i; returns their ids."""
        base = self.n[i]
        self.pool[i].append(rows)
        self.n[i] += rows.shape[0]
        self._cat[i] = None
        return list(range(base, self.n[i]))

    def rows(self, i):
        """[B, len, 3H] float64: each sequence's cached rows of layer i, in position order."""
        if self._cat[i] is None:
            self._cat[i] = torch.cat(self.pool[i])
        idx = torch.tensor(self.seq, dtype=torch.long, device=self._cat[i].device)
        return self._cat[i][idx]

    def permute(self, idx):
        """Sequence b continues old sequence idx[b]."""
        self.seq = [list(self.seq[int(j)]) for j in idx]


def _emb_pos(W, ids, p0, n, qf=None):
    """[word_embeddings[ids] (after the prefix qf) | positions p0 .. p0 + n - 1] as DistributedGPT3._decode and
    TokenStep add them: x = fl32(bf16 embedding + bf16 position), [B n, H]."""
    wemb, pos = W[GPT + "embedding.word_embeddings.weight"], W[GPT + "embedding.position_embeddings.weight"]
    B = ids.shape[0]
    emb = wemb[ids.reshape(-1).to(wemb.device)].view(B, -1, wemb.shape[1])
    if qf is not None:
        emb = torch.cat([qf.to(F64), emb], 1)
    return emb + pos[p0:p0 + n][None]


def decode_prefill(X, W, qf, ids, gcfg, stride, hist, name="decode.0"):
    """gpt_decode with an empty cache (off = 0) and the bf16 LM head of DistributedGPT3._decode.  The B / stride
    sequences [qf | ids] of n positions: x = fl32(emb + pos[0:n]); per layer LN1 -> QKV (GEMM row b n + i is cache
    row (b stride) max_len + i) -> causal attention -> dense + fp32 residual -> LN2 -> h->4h tanh-GELU -> 4h->h +
    residual; share_prefill(stride); the final LayerNorm of each sequence's last row b n + n - 1; the LM head.
    Sequence b's rows become the history of cache sequence b stride; the other beams of its group hold poison until
    share_prefill points them at it.  Returns the logits [B / stride, V]."""
    g = dims_gpt(gcfg)
    nh, hd, H = g["nh"], g["hd"], g["H"]
    Bp = ids.shape[0]
    if Bp * stride != hist.B:
        raise StepFailure(name, f"decode entry: {Bp} prefill sequences at stride {stride} for a cache of {hist.B}")
    emb = _emb_pos(W, ids, 0, ids.shape[1] + (0 if qf is None else qf.shape[1]), qf)
    n = emb.shape[1]
    x = X.rnd(emb, F32).reshape(Bp * n, H)
    for i in range(g["layers"]):
        pre, s = f"{GPT}encoder.layers.{i}.", f"{name}.L{i}."
        ln1, _, _ = ln_fwd(X, s + "input_layernorm", x, W, pre + "input_layernorm", g["eps"], stats=False)
        qkv = gemm(X, s + "qkv", ln1, W[pre + "self_attention.query_key_value.weight"],
                   bias=W[pre + "self_attention.query_key_value.bias"])
        new = hist.put(i, qkv)
        if i == 0:
            hist.seq = [new[(b // stride) * n:(b // stride + 1) * n] if b % stride == 0 else [0] * n for b in range(hist.B)]
        q, k, v = (heads(qkv, Bp, n, nh, hd, col=j * hd, hs=3 * hd) for j in range(3))
        o, _ = attn(X, s + "attn", q, k, v, scale=g["scale"], causal=True)
        x1 = gemm(X, s + "dense", unheads(o), W[pre + "self_attention.dense.weight"],
                  bias=W[pre + "self_attention.dense.bias"], residual=x, out=F32)
        ln2, _, _ = ln_fwd(X, s + "post_attention_layernorm", x1, W, pre + "post_attention_layernorm", g["eps"], stats=False)
        h = gemm(X, s + "h_to_4h", ln2, W[pre + "mlp.dense_h_to_4h.weight"], bias=W[pre + "mlp.dense_h_to_4h.bias"],
                 act=ACT_GELU_TANH)
        x = gemm(X, s + "4h_to_h", h, W[pre + "mlp.dense_4h_to_h.weight"], bias=W[pre + "mlp.dense_4h_to_h.bias"],
                 residual=x1, out=F32)
    hist.len = n
    if X.host(name + ".share_prefill", "share_prefill", dict(stride=stride)) is not None and stride > 1:
        hist.seq = [list(hist.seq[b // stride * stride]) for b in range(hist.B)]
    last = torch.arange(Bp, dtype=torch.int32) * n + (n - 1)
    hid, _, _ = ln_fwd(X, name + ".final_layernorm", x[last.long().to(x.device)], W, GPT + "encoder.final_layernorm",
                       g["eps"], in_rows=last, stats=False)
    return gemm(X, name + ".lm_head", hid, W[GPT + "embedding.word_embeddings.weight"])


def decode_token(X, W, tok, hist, gcfg, kind, name, max_len):
    """One single-token step of all B sequences at position len = hist.len, after which len grows by one.
    kind "skinny" is TokenStep: x = fl32(bf16 emb(tok) + bf16 pos[len]), every linear a skinny GEMM (the wide entry
    point above 8 rows); the QKV GEMM writes q to the staging rows and the same row to cache slot b max_len + len;
    attention reads the len + 1 keys of each sequence's history (the new one last) through the row table; the
    LayerNorms are separate calls; fp32 logits.  kind "gemm" is gpt_decode with n = 1: wgmma GEMMs, the QKV rows stored
    straight into the cache slots, share_prefill(1), the final LayerNorm through in_rows, bf16 logits.  Returns the
    logits [B, V]."""
    g = dims_gpt(gcfg)
    nh, hd, H, eps = g["nh"], g["hd"], g["H"], g["eps"]
    B, p = hist.B, hist.len
    x = X.rnd(_emb_pos(W, tok.reshape(B, 1), p, 1), F32).reshape(B, H)
    op = "gemm_skinny" if B <= 8 else "gemm_skinny_wide"

    def lin(nm, a, wname, **k):
        wb = dict(bias=W[wname + ".bias"])
        if kind == "gemm":
            k.pop("out2_rows", None)
            return gemm(X, nm, a, W[wname + ".weight"], **wb, **k)
        return skinny(X, nm, op, a, W[wname + ".weight"], **wb, **k)

    def lin_ln(nm, a, wname, residual, ln_pre, ln_name):
        y = lin(nm, a, wname, residual=residual, out=F32)
        if kind == "gemm":    # gpt_decode normalises at the start of the next layer, the final rows after the loop
            return y, None
        return y, ln_fwd(X, ln_name, y, W, ln_pre, eps, stats=False)[0]

    ln1 = ln_fwd(X, f"{name}.L0.input_layernorm", x, W, f"{GPT}encoder.layers.0.input_layernorm", eps, stats=False)[0]
    for i in range(g["layers"]):
        pre, s = f"{GPT}encoder.layers.{i}.", f"{name}.L{i}."
        if kind == "gemm" and i > 0:
            ln1 = ln_fwd(X, s + "input_layernorm", x, W, pre + "input_layernorm", eps, stats=False)[0]
        qkv = lin(s + "qkv", ln1, pre + "self_attention.query_key_value",
                  out2_rows=torch.arange(B, dtype=torch.int64) * max_len + p)
        new = hist.put(i, qkv)
        if i == 0:
            for b in range(B):
                hist.seq[b].append(new[b])
        q = heads(qkv, B, 1, nh, hd, hs=3 * hd)
        rows = hist.rows(i).reshape(B * (p + 1), 3 * H)
        k, v = (heads(rows, B, p + 1, nh, hd, col=j * hd, hs=3 * hd) for j in (1, 2))
        o, _ = attn(X, s + "attn", q, k, v, scale=g["scale"], keys=p + 1)
        x1, ln2 = lin_ln(s + "dense", unheads(o), pre + "self_attention.dense", x, pre + "post_attention_layernorm",
                         s + "post_attention_layernorm")
        if kind == "gemm":
            ln2 = ln_fwd(X, s + "post_attention_layernorm", x1, W, pre + "post_attention_layernorm", eps, stats=False)[0]
        h = lin(s + "h_to_4h", ln2, pre + "mlp.dense_h_to_4h", act=ACT_GELU_TANH)
        last = i + 1 == g["layers"]
        nxt = GPT + "encoder.final_layernorm" if last else f"{GPT}encoder.layers.{i + 1}.input_layernorm"
        x, ln1 = lin_ln(s + "4h_to_h", h, pre + "mlp.dense_4h_to_h", x1, nxt,
                        f"{name}.final_layernorm" if last else f"{name}.L{i + 1}.input_layernorm")
    hist.len = p + 1
    wemb = W[GPT + "embedding.word_embeddings.weight"]
    if kind != "gemm":
        return skinny(X, name + ".lm_head", op, ln1, wemb, out=F32)
    X.host(name + ".share_prefill", "share_prefill", dict(stride=1))
    hid = ln_fwd(X, name + ".final_layernorm", x, W, GPT + "encoder.final_layernorm", eps,
                 in_rows=torch.arange(B, dtype=torch.int32), stats=False)[0]
    return gemm(X, name + ".lm_head", hid, wemb)


def decode_session(X, W, gcfg, qf, script=None, *, B, max_len, stride=1, kind="skinny"):
    """A decoding run of DistributedGPT3 (sample / beam_search / the batched beam search) over one KV cache of B
    sequences: the host events drive it (exact / synth: `script`, a list of (kind, payload); walk: the trace).
    ("decode", dict(tokens, query)) is a decode entry: the first is the prefill of [qf | tokens] (query embeddings
    fed), every later one a single-token step; ("reindex" | "reorder", dict(idx)) permutes the sequences.  After each
    decode the logits it returned must be the last step's value bit for bit.  Returns every decode's logits."""
    g = dims_gpt(gcfg)
    hist = KVHistory(g["layers"], B, 3 * g["H"], W[GPT + "embedding.word_embeddings.weight"].device)
    it = iter(script or [])
    out = []
    while True:
        name = f"decode.{len(out)}"
        ev = X.next_host(name, it)
        if ev is None:
            return out
        kind_, p = ev
        if kind_ in ("reindex", "reorder"):
            if p is not None:
                hist.permute(p["idx"].tolist())
            continue
        if kind_ != "decode":
            raise StepFailure(name, f"schedule: unexpected host event {kind_}")
        first = hist.len == 0
        if bool(p["query"]) != (first and qf is not None):
            raise StepFailure(name, f"decode entry: query embeddings fed = {bool(p['query'])}")
        if first:
            logits = decode_prefill(X, W, qf, p["tokens"], gcfg, stride, hist, name)
        else:
            if tuple(p["tokens"].shape) != (B, 1):
                raise StepFailure(name, f"decode entry: tokens of shape {tuple(p['tokens'].shape)}, expected ({B}, 1)")
            logits = decode_token(X, W, p["tokens"][:, 0], hist, gcfg, kind, name, max_len)
        X.host(name + ".logits", "logits", dict(logits=logits))
        out.append(logits)


# ---------------------------------------------------------------------------------- trace recorder (GPU)
def _map_dict(m):
    return {f: int(getattr(m, f)) for f in ("seq_div", "n_prefix", "prefix_per_seq", "outer_stride", "inner_stride",
                                            "pos_stride", "prefix_base", "prefix_stride")}


def _gather_view(tv, n, S, H, hd):
    """A TView (tensor, column offset, head stride, seqmap) -> [n, H, S, hd] float64 of what the kernel reads there."""
    rows = AB.map_rows(_map_dict(tv.m), n, S).reshape(-1).to(tv.t.device)
    return heads(tv.t[rows].to(F64), n, S, H, hd, col=tv.col, hs=tv.hs)


def _table_view(tv, rows, H, hd):
    """A TView's keys read through a row table: rows [n, cnt] -> [n, H, cnt, hd] float64."""
    n, cnt = rows.shape
    return heads(tv.t[rows.reshape(-1).to(tv.t.device)].to(F64), n, cnt, H, hd, col=tv.col, hs=tv.hs)


class Recorder:
    """Wraps the ymp.ops entry points that engine.py and functional.py call (installed with monkeypatch.setattr; the
    product is unchanged).  Every outermost call becomes one Rec: operands gathered to their logical layout and copied
    just before the call, outputs copied after a torch.cuda.synchronize(), accumulating outputs with their before-value
    and the key of G their buffer lies in."""

    NAMES = ("gemm", "patch_embed_gemm", "im2col", "layernorm_fwd", "layernorm_bwd", "attn_fwd", "attn_bwd",
             "attn_temporal_fwd", "attn_temporal_bwd", "group_reduce", "colsum", "dropout", "embed_gather", "ce_fwd",
             "ce_bwd", "gemm_skinny", "gemm_skinny_wide")

    def __init__(self, ops, G=None):
        self.ops, self.G = ops, dict(G or {})
        self.trace, self.depth, self.temporal = [], 0, None
        self.orig = {n: getattr(ops, n) for n in self.NAMES}

    def install(self, monkeypatch):
        for n in self.NAMES:
            monkeypatch.setattr(self.ops, n, self._wrap(n))

    def install_decode(self, monkeypatch, cache_cls, model_cls):
        """Also log the host events of decoding as Recs of op "event": KVCache.reindex / reorder (idx) and
        share_prefill (stride), and around every model._decode entry its new token ids and whether query embeddings
        were fed, then the logits [B, V] it returns."""
        for nm, key in (("reindex", "idx"), ("reorder", "idx"), ("share_prefill", "stride")):
            def w(cache, arg, _orig=getattr(cache_cls, nm), _nm=nm, _key=key):
                self._push("event", {_key: arg.detach().cpu().clone() if torch.is_tensor(arg) else arg}, dict(kind=_nm), {})
                return _orig(cache, arg)
            monkeypatch.setattr(cache_cls, nm, w)

        def decode(model, tokens, input_embeds, n_query, _orig=model_cls._decode):
            self._push("event", dict(tokens=tokens.detach().cpu().clone(), query=n_query > 0), dict(kind="decode"), {})
            out = _orig(model, tokens, input_embeds, n_query)
            self._push("event", dict(logits=out.logits.reshape(out.logits.shape[0], -1).clone()), dict(kind="logits"), {})
            return out
        monkeypatch.setattr(model_cls, "_decode", decode)

    def _key_of(self, t):
        p = t.data_ptr()
        for k, g in self.G.items():
            b = g.data_ptr()
            if b <= p < b + g.numel() * g.element_size():
                return (k, (p - b) // g.element_size())
        return None

    def _wrap(self, name):
        fn = self.orig[name]
        rec = getattr(self, "_" + name)

        def w(*a, **kw):
            if self.depth:
                return fn(*a, **kw)
            self.depth += 1
            try:
                return rec(fn, *a, **kw)
            finally:
                self.depth -= 1
        return w

    def _push(self, op, ins, kw, outs, targets=None):
        self.trace.append(Rec(op, ins, kw, outs, targets or {}))

    # ---- GEMM
    def _gemm_common(self, op, fn, a, b, kw, A_logical, extra_kw):
        a_t, b_t = kw.get("a_t", False), kw.get("b_t", False)
        out = kw.get("out")
        bias, residual, aux_in = kw.get("bias"), kw.get("residual"), kw.get("aux_in")
        B = (b.T if b_t else b).to(F64)
        M, N = A_logical.shape[0], B.shape[0]
        acc = bool(kw.get("accumulate", False))
        srows = GB.store_rows(M, kw.get("d_row_block", 0), kw.get("d_row_stride", 0)).to(b.device)
        ins = dict(B=B.clone())
        ins.update(extra_kw.pop("ins"))
        if bias is not None:
            ins["bias"] = bias.to(F64).clone()
        if residual is not None:
            ins["residual"] = residual[GB.res_rows(M, kw.get("res_row_mod", 0)).to(b.device)].to(F64)
        if aux_in is not None:
            ins["aux_in"] = aux_in.to(F64).clone()
        targets = {}
        if acc:
            ins["d0"] = out[srows].to(F64)
            targets["D"] = self._key_of(out)
        drop = kw.get("drop")
        dspec = None
        if drop is not None and drop.p > 0:
            s, o = drop.rng.tolist()
            dspec = (int(s), int(o), drop.site, f32(drop.p))
        r = fn(a, b, **kw) if op == "gemm" else fn(*extra_kw.pop("args"), **kw)
        torch.cuda.synchronize()
        outs = dict(D=r[srows].clone())
        aux_out = kw.get("aux_out")
        if aux_out is not None:
            outs["aux"] = aux_out.clone()
        k = dict(act=kw.get("act", 0), alpha=kw.get("alpha", 1.0), accumulate=acc, drop=dspec, aux=aux_out is not None,
                 out_dtype=r.dtype)
        k.update(extra_kw)
        self._push(op, ins, k, outs, targets)
        return r

    def _gemm(self, fn, a, b, **kw):
        A = (a.T if kw.get("a_t", False) else a).to(F64)
        return self._gemm_common("gemm", fn, a, b, kw, A, dict(ins=dict(A=A.clone())))

    def _patch_embed_gemm(self, fn, video, weight2d, P, **kw):
        A = patch_rows(video, P)
        return self._gemm_common("patch_embed_gemm", fn, None, weight2d, kw, A,
                                 dict(ins=dict(video=video.to(F64).clone()), P=P, args=(video, weight2d, P)))

    def _im2col(self, fn, video, P, out=None):
        ins = dict(video=video.to(F64).clone())
        r = fn(video, P, out=out)
        torch.cuda.synchronize()
        self._push("im2col", ins, dict(P=P, ld=r.shape[1]), dict(out=r.clone()))
        return r

    def _skinny(self, op, fn, x, w, *, bias=None, residual=None, act=ACT_NONE, out=None, out_dtype=BF16, out2=None,
                out2_row_stride=0, out2_off=None):
        """out2: the cache rows m out2_row_stride + *out2_off (offset read after the sync) as output out2 and their
        indices as argument out2_rows."""
        ins = dict(A=x.to(F64).clone(), B=w.to(F64).clone())
        if bias is not None:
            ins["bias"] = bias.to(F64).clone()
        if residual is not None:
            ins["residual"] = residual.to(F64).clone()
        kw = dict(act=act, out2_rows=None)
        y = fn(x, w, bias=bias, residual=residual, act=act, out=out, out_dtype=out_dtype, out2=out2,
               out2_row_stride=out2_row_stride, out2_off=out2_off)
        torch.cuda.synchronize()
        kw["out_dtype"] = y.dtype
        outs = dict(D=y.clone())
        if out2 is not None:
            rows = torch.arange(y.shape[0], dtype=torch.int64) * out2_row_stride + int(out2_off.item())
            kw["out2_rows"] = rows
            outs["out2"] = out2[rows.to(out2.device)].clone()
        self._push(op, ins, kw, outs)
        return y

    def _gemm_skinny(self, fn, x, w, **kw):
        return self._skinny("gemm_skinny", fn, x, w, **kw)

    def _gemm_skinny_wide(self, fn, x, w, **kw):
        return self._skinny("gemm_skinny_wide", fn, x, w, **kw)

    # ---- LayerNorm
    def _rows_of(self, x, in_rows, rows):
        if in_rows is None:
            return x[:rows].to(F64), None, torch.arange(rows)
        ir = in_rows.long()
        pad = ir < 0
        xr = x[ir.clamp(min=0)].to(F64).masked_fill(pad[:, None], 0.0)
        return xr, (pad.cpu() if bool(pad.any()) else None), ir.clamp(min=0).cpu()

    def _layernorm_fwd(self, fn, x, gamma, beta, eps, out=None, in_rows=None, rows=None, stats=True, out_dtype=BF16):
        n = rows if rows is not None else (in_rows.numel() if in_rows is not None else x.shape[0])
        xr, pad, _ = self._rows_of(x, in_rows, n)
        ins = dict(x=xr, gamma=gamma.to(F64).clone(), beta=beta.to(F64).clone())
        y, m, r = fn(x, gamma, beta, eps, out=out, in_rows=in_rows, rows=rows, stats=stats, out_dtype=out_dtype)
        torch.cuda.synchronize()
        outs = dict(y=y.clone())
        if stats:
            outs.update(mean=m.clone(), rstd=r.clone())
        self._push("layernorm_fwd", ins, dict(eps=eps, y_dtype=y.dtype, in_rows=None if in_rows is None else in_rows.cpu(),
                                              pad=pad), outs)
        return y, m, r

    def _layernorm_bwd(self, fn, dy, x, gamma, mean, rstd, add=None, dgamma=None, dbeta=None, in_rows=None, dx=None,
                       drop=None, dx_drop=None):
        rows = dy.shape[0]
        xr, pad, xrows = self._rows_of(x, in_rows, rows)
        ins = dict(dy=dy.to(F64).clone(), x=xr, gamma=gamma.to(F64).clone(), mean=mean.to(F64).clone(),
                   rstd=rstd.to(F64).clone())
        if add is not None:
            ins["add"] = add[xrows.to(add.device)].to(F64)
        targets = {}
        if dgamma is not None:
            ins["dgamma0"], ins["dbeta0"] = dgamma.to(F64).clone(), dbeta.to(F64).clone()
            targets = dict(dgamma=self._key_of(dgamma), dbeta=self._key_of(dbeta))
        dspec = None
        if drop is not None and drop.p > 0:
            s, o = drop.rng.tolist()
            dspec = (int(s), int(o), drop.site, f32(drop.p))
        r = fn(dy, x, gamma, mean, rstd, add=add, dgamma=dgamma, dbeta=dbeta, in_rows=in_rows, dx=dx, drop=drop,
               dx_drop=dx_drop)
        torch.cuda.synchronize()
        dxt, dxd = r if isinstance(r, tuple) else (r, None)
        sel = xrows.to(dxt.device)
        keep = None if pad is None else (~pad).to(dxt.device)[:, None]
        outs = dict(dx=dxt[sel].clone() if keep is None else dxt[sel].masked_fill(~keep, 0))
        if dxd is not None:
            outs["dx_drop"] = dxd[sel].clone() if keep is None else dxd[sel].masked_fill(~keep, 0)
        if dgamma is not None:
            outs["dgamma"], outs["dbeta"] = dgamma.clone(), dbeta.clone()
        self._push("layernorm_bwd", ins, dict(drop=dspec, in_rows=None if in_rows is None else in_rows.cpu(),
                                              xrows=xrows), outs, targets)
        return r

    # ---- attention
    def _attn_kw(self, kw):
        drop = kw.get("drop")
        dspec = None
        if drop is not None and drop.p > 0:
            s, o = drop.rng.tolist()
            dspec = (int(s), int(o), drop.site, f32(drop.p))
        mask = int(kw["causal"])
        return dict(mask=AB.MASK_NONE if mask == AB.MASK_BLOCK else mask, scale=kw["scale"], drop=dspec)

    def _temporal(self, t, R, T, H, hd):
        """Packed block-diagonal tiles of dense rows -> independent length-T sequences [R / T, H, T, hd]."""
        return heads(t[:R].to(F64), R // T, T, H, hd)

    def _lse_temporal(self, lse, R, T, H):
        return lse.permute(0, 2, 1).reshape(-1, H)[:R].reshape(R // T, T, H).permute(0, 2, 1)

    def _attn_fwd(self, fn, q, k, v, o, **kw):
        n, H, hd, sq, skv = kw["n_seq"], kw["n_heads"], kw["head_dim"], kw["s_q"], kw["s_kv"]
        extra = {}
        if self.temporal:
            R, T = self.temporal
            ins = {nm: self._temporal(tv.t[:, tv.col:], R, T, H, hd).clone() for nm, tv in (("q", q), ("k", k), ("v", v))}
        elif kw.get("kv_rows") is not None:
            # keys through the row table: key j of sequence s is row kv_rows[s, j], and min(s_kv, *s_kv_dev) exist
            cnt = skv if kw.get("s_kv_dev") is None else min(skv, int(kw["s_kv_dev"].item()))
            rows = kw["kv_rows"][:, :cnt].long()
            ins = dict(q=_gather_view(q, n, sq, H, hd), k=_table_view(k, rows, H, hd), v=_table_view(v, rows, H, hd))
            extra["keys"] = cnt
        else:
            ins = dict(q=_gather_view(q, n, sq, H, hd), k=_gather_view(k, n, skv, H, hd), v=_gather_view(v, n, skv, H, hd))
        lse = fn(q, k, v, o, **kw)
        torch.cuda.synchronize()
        if self.temporal:
            outs = dict(o=self._temporal(o.t, R, T, H, hd).to(BF16), lse=self._lse_temporal(lse, R, T, H).clone())
        else:
            outs = dict(o=_gather_view(o, n, sq, H, hd).to(BF16), lse=lse.clone())
        self._push("attn_temporal_fwd" if self.temporal else "attn_fwd", ins, dict(self._attn_kw(kw), **extra), outs)
        return lse

    def _attn_bwd(self, fn, q, k, v, o, lse, dout, dq, dk, dv, **kw):
        n, H, hd, sq, skv = kw["n_seq"], kw["n_heads"], kw["head_dim"], kw["s_q"], kw["s_kv"]
        if self.temporal:
            R, T = self.temporal
            g = lambda tv: self._temporal(tv.t[:, tv.col:], R, T, H, hd)  # noqa: E731
            ins = dict(q=g(q), k=g(k), v=g(v), o=g(o), do=g(dout), lse=self._lse_temporal(lse, R, T, H).clone())
        else:
            ins = dict(q=_gather_view(q, n, sq, H, hd), k=_gather_view(k, n, skv, H, hd), v=_gather_view(v, n, skv, H, hd),
                       o=_gather_view(o, n, sq, H, hd), do=_gather_view(dout, n, sq, H, hd), lse=lse.clone())
        fn(q, k, v, o, lse, dout, dq, dk, dv, **kw)
        torch.cuda.synchronize()
        if self.temporal:
            outs = {nm: g(tv).to(BF16) for nm, tv in (("dq", dq), ("dk", dk), ("dv", dv))}
        else:
            outs = dict(dq=_gather_view(dq, n, sq, H, hd).to(BF16), dk=_gather_view(dk, n, skv, H, hd).to(BF16),
                        dv=_gather_view(dv, n, skv, H, hd).to(BF16))
        self._push("attn_temporal_bwd" if self.temporal else "attn_bwd", ins, self._attn_kw(kw), outs)

    def _attn_temporal_fwd(self, fn, qkv, out, *, R, n_heads, T, D, scale):
        self.temporal = (R, T)
        self.depth -= 1            # the inner attn_fwd call is the one recorded
        try:
            return fn(qkv, out, R=R, n_heads=n_heads, T=T, D=D, scale=scale)
        finally:
            self.depth += 1
            self.temporal = None

    def _attn_temporal_bwd(self, fn, qkv, out, lse, dout, dqkv, *, R, n_heads, T, D, scale):
        self.temporal = (R, T)
        self.depth -= 1
        try:
            return fn(qkv, out, lse, dout, dqkv, R=R, n_heads=n_heads, T=T, D=D, scale=scale)
        finally:
            self.depth += 1
            self.temporal = None

    # ---- reductions and the rest
    def _group_reduce(self, fn, x, G, T, out, scale=1.0, broadcast=False):
        n_in = G if broadcast else G * T
        ins = dict(x=x[:n_in].to(F64).clone())
        fn(x, G, T, out, scale=scale, broadcast=broadcast)
        torch.cuda.synchronize()
        self._push("group_reduce", ins, dict(G=G, T=T, scale=scale, broadcast=bool(broadcast)),
                   dict(out=out[:G * T if broadcast else G].clone()))
        return out

    def _colsum(self, fn, x, out):
        ins = dict(x=x.to(F64).clone(), d0=out.to(F64).clone())
        tgt = self._key_of(out)
        fn(x, out)
        torch.cuda.synchronize()
        self._push("colsum", ins, {}, dict(out=out.clone()), dict(out=tgt))
        return out

    def _dropout(self, fn, x, drop, out=None, row0=0):
        ins = dict(x=x.to(F64).clone())
        s, o = drop.rng.tolist()
        r = fn(x, drop, out=out, row0=row0)
        torch.cuda.synchronize()
        self._push("dropout", ins, dict(drop=(int(s), int(o), drop.site, f32(drop.p))), dict(y=r.clone()))
        return r

    def _embed_gather(self, fn, ids, table, pos, out, S, row_offset):
        ins = dict(ids=ids.clone(), table=table.to(F64), pos=pos.to(F64))
        fn(ids, table, pos, out, S, row_offset)
        torch.cuda.synchronize()
        B, L = ids.shape
        rows = (torch.arange(B)[:, None] * S + row_offset + torch.arange(L)[None, :]).reshape(-1).to(out.device)
        self._push("embed_gather", ins, dict(S=S, row_offset=row_offset), dict(out=out[rows].clone()))
        return out

    def _ce_fwd(self, fn, logits, labels):
        ins = dict(logits=logits.to(F64), labels=labels.reshape(-1).clone())
        loss, lse = fn(logits, labels)
        torch.cuda.synchronize()
        self._push("ce_fwd", ins, {}, dict(loss=loss.clone(), lse=lse.clone()))
        return loss, lse

    def _ce_bwd(self, fn, logits, labels, lse, grad_rows, dlogits=None):
        ins = dict(logits=logits.to(F64), labels=labels.reshape(-1).clone(), lse=lse.to(F64).clone(),
                   g=grad_rows.to(F64).clone())
        r = fn(logits, labels, lse, grad_rows, dlogits=dlogits)
        torch.cuda.synchronize()
        self._push("ce_bwd", ins, {}, dict(dlogits=r.clone()))
        return r
