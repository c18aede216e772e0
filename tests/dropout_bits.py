"""Exact readouts of the dropout keep bits of the attention kernels, and the oracle's bits to compare them with.

Used by test_dropout_bits_gpu.py (the kernels) and test_dropout_bits_cpu.py (the same readouts through the CPU
simulation of the kernel arithmetic in attn_bounds.py).  An error bound cannot see one wrong keep bit: it moves O_i by
about |V| / (0.9 n_i), inside the bound once a row sees some 70 keys.  So each readout feeds one kernel inputs under
which an output element is non-zero exactly when one (query, key) pair is kept.

Q = 0 on every addressed element, so every visible score is 0 and P_ij = 1 / n_i (n_i visible keys; no underflow).
With hd the head dim, k = 1 / (1 - p) and the window [base, base + hd):
  fwd    V[j, d] = [d == j - base]                                   O[i, d] = k / n_i * keep(i, base + d)
  dq     K[j, d] = [d == j - base], V[j] = e_0, dO[i] = e_0,
         O = 0 (so delta = 0), lse_i = log n_i                       dQ[i, d] = scale * k / n_i * keep(i, base + d)
  dkdv   dO[i, d] = [d == i - base], V = 0, O = 0, lse_i = log n_i   dV[j, d] = k / n_(base+d) * keep(base + d, j)
Windows step through all keys (fwd, dq) or all queries (dkdv).  The dK / dV kernel multiplies P and dZ by one keep
factor, so dV also shows the bits its dK uses.  Operands nothing depends on (K in fwd and dkdv) hold random values.
"""
import numpy as np
import torch

import attn_bounds as AB
from oracle import philox

KINDS = ("fwd", "dq", "dkdv")
SEED, OFFSET = 0x1234567812345, 7
P_DROP = (0.1, 0.3)


def case(name, hd, s_q, s_kv, *, n=2, H=3, mask=AB.MASK_NONE, mask_block=0, total_rows=0):
    return dict(name=name, hd=hd, s_q=s_q, s_kv=s_kv, n=n, H=H, mask=mask, mask_block=mask_block,
                total_rows=total_rows)


def _cases():
    c = []
    for hd in (64, 80, 88, 96):                    # wgmma forward and backward
        for mask in (AB.MASK_NONE, AB.MASK_CAUSAL):
            for L in (1, 63, 65, 129):
                c.append(case(f"wgmma-hd{hd}-{'causal' if mask else 'self'}-{L}", hd, L, L, mask=mask))
    for hd, sq, skv in ((64, 63, 129), (80, 129, 65), (88, 1, 70), (96, 65, 1)):
        c.append(case(f"wgmma-hd{hd}-cross-{sq}x{skv}", hd, sq, skv))
    for hd, S, total, mask in ((64, 100, 250, AB.MASK_CAUSAL), (96, 65, 131, AB.MASK_NONE)):
        c.append(case(f"wgmma-hd{hd}-ragged-{S}-{total}", hd, S, S, n=(total + S - 1) // S, mask=mask,
                      total_rows=total))
    for sq, skv, mask in ((130, 130, AB.MASK_CAUSAL), (70, 200, AB.MASK_NONE), (129, 64, AB.MASK_NONE)):
        c.append(case(f"mma_sync-hd128-{sq}x{skv}-{'causal' if mask else 'none'}", 128, sq, skv, mask=mask))
    for T in (8, 16, 20, 24):                      # block masks: mma.sync (attention_small.cu takes no dropout)
        for hd in (64, 88, 96):
            P = 96 if T == 24 else 80
            total = 200 if (T, hd) == (8, 88) else 140 if (T, hd) == (20, 96) else 0
            n = 3 if not total else (total + P - 1) // P
            c.append(case(f"mma_sync-hd{hd}-block{T}" + (f"-total{total}" if total else ""), hd, P, P, n=n,
                          mask=AB.MASK_BLOCK, mask_block=T, total_rows=total))
    for sq in (2, 7, 15):                          # forward on mma.sync, backward on wgmma
        for skv in (257, 1000):
            hd = (64, 80, 96)[(sq + skv) % 3]
            c.append(case(f"few-queries-hd{hd}-{sq}x{skv}", hd, sq, skv))
    for i, x in enumerate(c):                      # both probabilities in every group
        x["p"] = P_DROP[i % 2]
    return c


CASES = _cases()


def oracle_keep(c, site, rows=None):
    """bool [n, H, s_q, s_kv]: the oracle's keep bit of every (seq, head, query, key); rows: the dropout row of each
    (seq, head, query), default (seq * H + head) * s_q + query."""
    n, H, sq, skv = c["n"], c["H"], c["s_q"], c["s_kv"]
    r = np.arange(n * H * sq) if rows is None else np.asarray(rows).reshape(-1)
    return torch.from_numpy(philox.keep_mask(SEED, OFFSET, site, r, skv, c["p"])).view(n, H, sq, skv)


def visible(c):
    return AB.visible(c["n"], c["s_q"], c["s_kv"], c["mask"], c["mask_block"], c["total_rows"])


def windows(kind, c):
    return range(0, c["s_q"] if kind == "dkdv" else c["s_kv"], c["hd"])


def inputs(kind, base, c, vis, gen):
    """float64 q, k, v, do, o [n, H, S, hd] and lse [n, H, s_q] of one readout window (module docstring)."""
    n, H, sq, skv, hd = c["n"], c["H"], c["s_q"], c["s_kv"], c["hd"]
    d = torch.arange(hd)

    def onehot(S):      # [S, hd]: row base + d holds e_d
        return (torch.arange(S)[:, None] - base == d[None, :]).double().expand(n, H, S, hd)

    def rand(S):
        return torch.randn(n, H, S, hd, generator=gen).to(torch.bfloat16).double()

    e0 = lambda S: (d == 0).double().expand(n, H, S, hd)
    zero = lambda S: torch.zeros(n, H, S, hd, dtype=torch.float64)
    x = dict(q=zero(sq), k=rand(skv), v=rand(skv), do=rand(sq), o=zero(sq))
    if kind == "fwd":
        x["v"] = onehot(skv)
    elif kind == "dq":
        x.update(k=onehot(skv), v=e0(skv), do=e0(sq))
    else:
        x.update(v=zero(skv), do=onehot(sq))
    cnt = vis.sum(-1).double()[:, None].expand(n, H, sq)
    x["lse"] = torch.where(cnt > 0, cnt.clamp(min=1).log(), torch.zeros_like(cnt))
    return x


class Bits:
    """Keep bits read back window by window: bits [n, H, s_q, s_kv] and the pairs read so far."""

    def __init__(self, c):
        shape = (c["n"], c["H"], c["s_q"], c["s_kv"])
        self.c, self.bits, self.read = c, torch.zeros(shape, dtype=torch.bool), torch.zeros(shape, dtype=torch.bool)

    def add(self, kind, base, out):
        """out: the window's O or dQ [n, H, s_q, hd] (fwd, dq) or dV [n, H, s_kv, hd] (dkdv)."""
        hd = self.c["hd"]
        nz = out.cpu() != 0
        if kind == "dkdv":
            w = min(hd, self.c["s_q"] - base)
            assert not bool(nz[..., w:].any()), f"dV non-zero in a column past the last query (window {base})"
            self.bits[:, :, base:base + w] = nz[..., :w].transpose(-1, -2)
            self.read[:, :, base:base + w] = True
        else:
            w = min(hd, self.c["s_kv"] - base)
            assert not bool(nz[..., w:].any()), f"{kind}: non-zero in a column past the last key (window {base})"
            self.bits[..., base:base + w] = nz[..., :w]
            self.read[..., base:base + w] = True

    def check(self, what, keep, vis):
        """Every pair read back; the bits equal keep on the visible pairs and are 0 on the others."""
        assert bool(self.read.all()), f"{what}: {int((~self.read).sum())} pairs never read back"
        check_bits(what, self.bits, keep & vis[:, None])


def first_wrong(got, want):
    """(seq, head, row, key) of the first pair where got and want differ, in row-major order, and the number of such
    pairs; None when they agree."""
    bad = got != want
    if not bool(bad.any()):
        return None
    return tuple(int(i) for i in bad.nonzero()[0]), int(bad.sum())


def check_bits(what, got, want):
    w = first_wrong(got, want)
    if w is not None:
        pos, cnt = w
        raise AssertionError(f"{what}: {cnt} keep bits differ from the oracle, first at (seq, head, row, key) {pos}: "
                             f"read {int(got[pos])}, oracle {int(want[pos])}")


# ---------------------------------------------------------------------------------- the readouts on the CPU
def simulate(kind, c, x, vis, mult):
    """The window's readout output through attn_bounds' CPU simulation of the kernel arithmetic."""
    scale = c["hd"] ** -0.5
    if kind == "fwd":
        return AB.simulate_fwd(x["q"], x["k"], x["v"], vis, scale, mult=mult)[0]
    dq, _, dv = AB.simulate_bwd(x["q"], x["k"], x["v"], x["o"], x["lse"].float(), x["do"], vis, scale, mult=mult)
    return dq if kind == "dq" else dv


def read_simulated(kind, c, keep, seed=0):
    """Bits read back from the simulated readouts of one kind with the keep mask `keep` [n, H, s_q, s_kv]."""
    vis = visible(c)
    mult = keep.double() * philox.scale(c["p"])
    gen = torch.Generator().manual_seed(seed)
    b = Bits(c)
    for base in windows(kind, c):
        b.add(kind, base, simulate(kind, c, inputs(kind, base, c, vis, gen), vis, mult))
    return b


# ---------------------------------------------------------------------------------- defective masks
def defect_keep(defect, c, site):
    """The keep mask a kernel with one defect would draw."""
    n, H, sq, skv = c["n"], c["H"], c["s_q"], c["s_kv"]
    s, h, i = torch.arange(n).view(n, 1, 1), torch.arange(H).view(1, H, 1), torch.arange(sq).view(1, 1, sq)
    if defect == "s_kv_row":                 # the dropout row built with s_kv in place of s_q
        return oracle_keep(c, site, ((s * H + h) * skv + i).numpy())
    if defect == "head_seq_swap":            # (head * n_seq + seq) instead of (seq * n_heads + head)
        return oracle_keep(c, site, ((h * n + s) * sq + i).numpy())
    rows = np.arange(n * H * sq)
    w = torch.from_numpy(philox.words(SEED, OFFSET, site, rows, skv + 4).astype(np.int64)).view(n, H, sq, skv + 4)
    t = philox.threshold(c["p"])
    if defect == "words_1_2":                # words 1 and 2 of every Philox call exchanged
        j = torch.arange(skv)
        j = torch.where(j % 4 == 1, j + 1, torch.where(j % 4 == 2, j - 1, j))
        return w[..., j] >= t
    if defect == "last_tile_shift":          # the last 64-key tile reads its words 4 columns on
        j = torch.arange(skv)
        j = torch.where(j >= (skv - 1) // 64 * 64, j + 4, j)
        return w[..., j] >= t
    raise ValueError(defect)
