"""Every attention kernel family, element by element, against the float64 reference of attn_bounds.py with the
per-element error bounds derived there (module docstring of attn_bounds.py).

Each case
  - reads Q / K / V / dO in place through the same seqmaps the models use, from buffers with gaps between heads
    (head stride > head_dim), a row stride wider than the view and rows before and after it; every element a kernel
    has no business reading holds finite poison (+-3e4), including cache rows past the key count and rows past
    total_rows;
  - writes O / lse / dQ / dK / dV into buffers filled with a NaN bit pattern: every addressed element must come back
    finite and inside its bound, every other element must still hold the pattern bit for bit;
  - asserts which kernel family served the forward and the backward (lib.attn_last_path);
  - under causal masks gives V geometric growth along the keys, and under block masks block-wise magnitudes, so that
    a key that leaks through the mask moves O by more than the bound;
  - tests the backward in isolation (given the reference O rounded to bf16 and the reference lse), and for one case
    per family chained to the kernel's own forward (with the forward's bounds as the input error).
Under dropout on the probabilities the reference and the bounds take the oracle's multiplier keep / (1 - p).
Set YMP_ATTN_BOUNDS_REPORT=<file> to write the largest err / bound per family and tensor as JSON (the families under
dropout as "<family>+drop", and "mma_sync+drop(per-element)" for the dK / dV kernel's per-element Philox calls).
"""
import json
import math
import os

import pytest
import torch

import attn_bounds as AB
import stage_steps as SS

pytestmark = pytest.mark.gpu
bf16 = torch.bfloat16

SENT16 = 0x7FA5          # bf16 NaN bit pattern of untouched output memory
SENT32 = 0x7FA0BEEF      # fp32 NaN bit pattern of untouched lse memory
POISON = 3.0e4           # finite poison of input memory no kernel may read
ROW0 = 2                 # rows of every buffer before the addressed view
DROP_SEED, DROP_OFFSET, DROP_SITE = 0x1234567812345, 7, 4 * 5 + 1
RATIOS = {}


def _family_name(f):
    from ymp import lib
    return {lib.ATTN_PATH_MMA_SYNC: "mma_sync", lib.ATTN_PATH_WGMMA: "wgmma", lib.ATTN_PATH_SMALL: "small",
            lib.ATTN_PATH_DECODE: "decode"}[f]


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    path = os.environ.get("YMP_ATTN_BOUNDS_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump(RATIOS, f, indent=1, sort_keys=True)


def fwd_family(hd, s_q, s_kv, mask, mask_block=0, total_rows=0, kv_dev=False, drop=False):
    """The family ymp.h documents for a forward call (dense seqmaps under block masks).  Under dropout neither the
    decode kernel nor the warp-per-sequence kernel runs."""
    from ymp import lib
    if mask == AB.MASK_CAUSAL and s_q < s_kv:
        return lib.ATTN_PATH_WGMMA
    if s_q == 1 and mask == AB.MASK_NONE and not total_rows and hd not in (88, 128) and not drop:
        return lib.ATTN_PATH_DECODE
    if mask == AB.MASK_BLOCK and mask_block <= 16 and hd != 88 and not kv_dev and not drop:
        return lib.ATTN_PATH_SMALL
    if hd == 128 or mask == AB.MASK_BLOCK or kv_dev or (s_q < 16 and s_kv > 256):
        return lib.ATTN_PATH_MMA_SYNC
    return lib.ATTN_PATH_WGMMA


def bwd_family(hd, mask, mask_block=0, drop=False):
    from ymp import lib
    if mask == AB.MASK_BLOCK and mask_block <= 16 and hd != 88 and not drop:
        return lib.ATTN_PATH_SMALL
    if hd == 128 or mask == AB.MASK_BLOCK:
        return lib.ATTN_PATH_MMA_SYNC
    return lib.ATTN_PATH_WGMMA


class Operand:
    """One bf16 operand of n_seq x H heads x S positions x hd, addressed through a seqmap in a larger buffer:
    head stride hd + 8, 8 columns before the first head and after the last, ROW0 rows before the view, 3 after."""

    def __init__(self, cuda, m, n, S, H, hd, lens, output, gen=None):
        from ymp import ops
        self.rows = AB.map_rows(m, n, S)
        self.valid = torch.arange(S)[None, :] < lens[:, None]           # [n, S]
        self.H, self.hd, self.hs, self.col = H, hd, hd + 8, 8
        ld = self.col + H * self.hs + 8
        R = int(self.rows.max()) + 1
        cols = self.col + torch.arange(H)[:, None] * self.hs + torch.arange(hd)[None, :]      # [H, hd]
        self.cols = cols
        addr = torch.zeros(ROW0 + R + 3, ld, dtype=torch.bool)
        vr = ROW0 + self.rows[self.valid]                                                     # [k]
        addr[vr[:, None], cols.flatten()[None, :]] = True
        self.addr = addr.to(cuda)
        if output:
            self.base = torch.full((ROW0 + R + 3, ld), SENT16, dtype=torch.int16, device=cuda).view(bf16)
        else:
            sign = torch.randint(0, 2, (ROW0 + R + 3, ld), generator=gen).float() * 2 - 1
            data = torch.randn(ROW0 + R + 3, ld, generator=gen)
            self.base = torch.where(addr, data, sign * POISON).to(bf16).to(cuda)
        self.view = ops.TView(self.base[ROW0:], self.col, self.hs, ops.seqmap(**m))
        self.m = m

    def gather(self):
        """[n, H, S, hd] float64 of the addressed elements (0 at positions that do not exist)."""
        x = self.base[ROW0:][self.rows.to(self.base.device)][..., self.cols.to(self.base.device)]   # [n, S, H, hd]
        x = x.double().permute(0, 2, 1, 3)
        return torch.where(self.valid.to(x.device)[:, None, :, None], x, torch.zeros_like(x))

    def set(self, x):
        """Write [n, H, S, hd] values (rounded to bf16) at the existing positions."""
        rows = (ROW0 + self.rows[self.valid]).to(self.base.device)
        vals = x.permute(0, 2, 1, 3)[self.valid.to(x.device)].to(bf16)                          # [k, H, hd]
        self.base[rows[:, None, None], self.cols.to(self.base.device)[None]] = vals

    def check_untouched(self, what):
        bits = self.base.view(torch.int16)
        bad = (bits != SENT16) & ~self.addr
        assert not bool(bad.any()), f"{what}: {int(bad.sum())} elements outside the view were written, first at " \
                                    f"{bad.nonzero()[0].tolist()} (buffer row, column)"
        got = self.base.float()[self.addr]
        assert bool(torch.isfinite(got).all()), f"{what}: {int((~torch.isfinite(got)).sum())} addressed elements " \
                                                f"not written or not finite"


class Lse:
    """fp32 [n, H, s_q] inside a buffer with 16 elements on either side."""

    def __init__(self, cuda, n, H, s_q, lens, fill_bits=None, values=None):
        N = n * H * s_q
        self.addr = torch.zeros(N + 32, dtype=torch.bool)
        self.addr[16:16 + N] = (torch.arange(s_q)[None, None, :] < lens[:, None, None]).expand(n, H, s_q).flatten()
        self.addr = self.addr.to(cuda)
        if values is None:
            self.buf = torch.full((N + 32,), SENT32, dtype=torch.int32, device=cuda).view(torch.float32)
        else:   # an input: the given values where rows exist, finite poison (exp(s - lse) = inf if read) elsewhere
            self.buf = torch.full((N + 32,), -POISON, dtype=torch.float32, device=cuda)
            self.buf[self.addr] = values.float().flatten()[self.addr[16:16 + N]]
        self.t = self.buf[16:16 + N].view(n, H, s_q)

    def check_untouched(self):
        bad = (self.buf.view(torch.int32) != SENT32) & ~self.addr
        assert not bool(bad.any()), f"lse: {int(bad.sum())} elements outside the view were written"
        assert bool(torch.isfinite(self.buf[self.addr]).all()), "lse: addressed entries not written or not finite"


def _check(fam, what, got, want, bound, where):
    r = AB.worst_ratio(got, want, bound, where)
    key = f"{fam}.{what}"
    RATIOS[key] = max(RATIOS.get(key, 0.0), r)
    if r > 1:
        err = ((got.double() - want.double()).abs() / bound).nan_to_num(math.inf)
        err = torch.where(where.expand_as(err), err, torch.zeros_like(err))
        idx = err.flatten().argmax()
        pos = list(torch.unravel_index(idx, err.shape))
        raise AssertionError(f"{key}: err / bound = {r:.3g} at (seq, head, row, col) {[int(p) for p in pos]}: "
                             f"got {got.flatten()[idx].item():.6g}, want {want.flatten()[idx].item():.6g}, "
                             f"bound {bound.flatten()[idx].item():.3g}")


def _drop_name(name, hd, drop, bwd=False):
    """Report name of a family under dropout; the mma.sync dK / dV kernel draws one Philox call per element at head_dim
    88 and 96 and shares calls within a quad of lanes otherwise."""
    if not drop:
        return name
    return name + ("+drop(per-element)" if bwd and name == "mma_sync" and hd in (88, 96) else "+drop")


def run(cuda, *, hd, s_q, s_kv, n=2, H=2, mask=AB.MASK_NONE, mask_block=0, total_rows=0, kv_count=None, maps=None,
        fwd_path, bwd_path=None, chained=False, probe=None, seed=0, drop=None):
    """One forward (and, with bwd_path, one isolated backward; with chained, also one backward from the kernel's own
    O and lse) checked element-wise, with sentinels and the served family.  drop: the probability of dropout on the
    attention probabilities (the reference and the bounds take the oracle's keep / (1 - p))."""
    from ymp import lib, ops
    gen = torch.Generator().manual_seed(seed)
    maps = dict(dict(q=AB.dense(s_q), kv=AB.dense(s_kv), o=AB.dense(s_q)), **(maps or {}))
    maps.setdefault("dq", maps["o"])
    maps.setdefault("dkv", maps["kv"])
    lq, lkv = AB.lengths(n, s_q, s_kv, total_rows, kv_count)
    Q, K, V = (Operand(cuda, maps[w], n, s, H, hd, l, False, gen) for w, s, l in (("q", s_q, lq), ("kv", s_kv, lkv),
                                                                                 ("kv", s_kv, lkv)))
    dO = Operand(cuda, maps["o"], n, s_q, H, hd, lq, False, gen)
    if probe == "causal":     # V grows geometrically with the key position: a later key leaking in moves O past the bound
        r = math.exp(min(0.2, 30.0 / s_kv))
        v = V.gather()
        sign = torch.sign(torch.randn(1, H, 1, hd, generator=gen)).to(v.device)
        V.set(sign * (v.abs() + 0.5) * r ** torch.arange(s_kv, device=v.device, dtype=torch.float64)[:, None])
    elif probe == "block":    # magnitudes cycle x1, x8, x64 from one diagonal block to the next
        v = V.gather()
        f = 8.0 ** ((torch.arange(s_kv, device=v.device) // mask_block) % 3).double()
        V.set(v * f[:, None])
    q, k, v, do = Q.gather(), K.gather(), V.gather(), dO.gather()
    vis = AB.visible(n, s_q, s_kv, mask, mask_block, total_rows, kv_count)
    scale = hd ** -0.5
    mult = dspec = None
    if drop:
        dspec = ops.Drop(torch.tensor([DROP_SEED, DROP_OFFSET], dtype=torch.int64, device=cuda), DROP_SITE, drop)
        mult = SS.drop_mult((DROP_SEED, DROP_OFFSET, DROP_SITE, drop), range(n * H * s_q), s_kv, cuda)
        mult = mult.view(n, H, s_q, s_kv)
    ref = AB.reference(q, k, v, vis.to(cuda), scale, do, mult=mult)
    rows = ref["vis"].any(-1)                                  # [n, 1, s_q]: query rows that exist
    keys = ref["vis"].any(-2)                                  # [n, 1, s_kv]: keys some query sees
    kw = dict(n_seq=n, n_heads=H, head_dim=hd, s_q=s_q, s_kv=s_kv, causal=mask, scale=scale, mask_block=mask_block,
              total_rows=total_rows, drop=dspec)
    dev = None if kv_count is None else torch.tensor([kv_count], dtype=torch.int32, device=cuda)

    O = Operand(cuda, maps["o"], n, s_q, H, hd, lq, True)
    lse = Lse(cuda, n, H, s_q, lq)
    ops.attn_fwd(Q.view, K.view, V.view, O.view, lse=lse.t, s_kv_dev=dev, **kw)
    fam = lib.attn_last_path()
    assert fam == fwd_path, f"forward served by {_family_name(fam)}, expected {_family_name(fwd_path)}"
    torch.cuda.synchronize()
    name = _drop_name(_family_name(fam), hd, drop)
    O.check_untouched(f"{name} O")
    lse.check_untouched()
    e_o, e_lse = AB.fwd_bounds(q, k, v, scale, ref)
    _check(name, "O", O.gather(), ref["O"], e_o, rows[..., None])
    _check(name, "lse", lse.t.double(), ref["lse"], e_lse, rows)
    if bwd_path is None:
        return

    cases = [("", ref["O"], ref["lse"], None, None)]
    if chained:
        cases.append(("chained ", O.gather(), lse.t, e_o, e_lse))
    for tag, o_in, lse_in, eo, el in cases:
        Oi = Operand(cuda, maps["o"], n, s_q, H, hd, lq, False, gen)
        Oi.set(o_in)
        Li = Lse(cuda, n, H, s_q, lq, values=lse_in.masked_fill(~rows, 0.0))
        dQ = Operand(cuda, maps["dq"], n, s_q, H, hd, lq, True)
        dK, dV = (Operand(cuda, maps["dkv"], n, s_kv, H, hd, lkv, True) for _ in range(2))
        ops.attn_bwd(Q.view, K.view, V.view, Oi.view, Li.t, dO.view, dQ.view, dK.view, dV.view, **kw)
        fam = lib.attn_last_path()
        assert fam == bwd_path, f"{tag}backward served by {_family_name(fam)}, expected {_family_name(bwd_path)}"
        torch.cuda.synchronize()
        bname = _drop_name(_family_name(fam), hd, drop, bwd=True)
        for t, w in ((dQ, "dQ"), (dK, "dK"), (dV, "dV")):
            t.check_untouched(f"{tag}{bname} {w}")
        e_dq, e_dk, e_dv = AB.bwd_bounds(q, k, v, do, scale, ref, eo, el)
        _check(bname, tag + "dQ", dQ.gather(), ref["dQ"], e_dq, rows[..., None])
        _check(bname, tag + "dK", dK.gather(), ref["dK"], e_dk, keys[..., None])
        _check(bname, tag + "dV", dV.gather(), ref["dV"], e_dv, keys[..., None])


# ---------------------------------------------------------------------------------- wgmma
WG_HD = [64, 80, 88, 96]
WG_LEN = [1, 63, 64, 65, 127, 129, 257, 384]
CROSS_KV = {1: 70, 63: 200, 64: 1, 65: 130, 127: 64, 129: 257, 257: 65, 384: 129}


@pytest.mark.parametrize("causal", [False, True], ids=["self", "causal"])
@pytest.mark.parametrize("L", WG_LEN)
@pytest.mark.parametrize("hd", WG_HD)
def test_wgmma_self(cuda, hd, L, causal):
    mask = AB.MASK_CAUSAL if causal else AB.MASK_NONE
    run(cuda, hd=hd, s_q=L, s_kv=L, mask=mask, fwd_path=fwd_family(hd, L, L, mask), bwd_path=bwd_family(hd, mask),
        probe="causal" if causal else None, seed=L + hd)


@pytest.mark.parametrize("L", WG_LEN)
@pytest.mark.parametrize("hd", WG_HD)
def test_wgmma_cross(cuda, hd, L):
    skv = CROSS_KV[L]
    run(cuda, hd=hd, s_q=L, s_kv=skv, fwd_path=fwd_family(hd, L, skv, AB.MASK_NONE), bwd_path=bwd_family(hd, 0),
        seed=3 * L + hd)


@pytest.mark.parametrize("hd", [88, 96])
def test_wgmma_abstractor(cuda, hd):
    """The abstractor's cross attention: 128 queries against 1570 visual tokens."""
    from ymp import lib
    run(cuda, hd=hd, s_q=128, s_kv=1570, fwd_path=lib.ATTN_PATH_WGMMA, bwd_path=lib.ATTN_PATH_WGMMA, seed=hd)


@pytest.mark.parametrize("hd", [64, 96])
def test_wgmma_timesformer_prefix_map(cuda, hd):
    """Per-frame sequences [cls_b ; x[b, :, t]] read in place from the (b n t) + cls row layout; outputs and gradients
    of the cls row go to one row per frame."""
    from ymp import lib
    B, N, T = 2, 9, 3
    R = B * N * T
    base = dict(seq_div=T, outer_stride=N * T, inner_stride=1, pos_stride=T, n_prefix=1, prefix_base=R, prefix_stride=1)
    m_in, m_out = dict(base, prefix_per_seq=0), dict(base, prefix_per_seq=1)
    run(cuda, hd=hd, n=B * T, s_q=N + 1, s_kv=N + 1, maps=dict(q=m_in, kv=m_in, o=m_out, dq=m_out, dkv=m_out),
        fwd_path=lib.ATTN_PATH_WGMMA, bwd_path=lib.ATTN_PATH_WGMMA, seed=hd + 1)


@pytest.mark.parametrize("hd,Q,S", [(96, 70, 330), (64, 128, 65)])
def test_wgmma_shared_query_map(cuda, hd, Q, S):
    """One query block read by every sequence (outer_stride = 0); each sequence gets its own dQ rows."""
    from ymp import lib
    run(cuda, hd=hd, s_q=Q, s_kv=S, maps=dict(q=dict(outer_stride=0, pos_stride=1)),
        fwd_path=lib.ATTN_PATH_WGMMA, bwd_path=lib.ATTN_PATH_WGMMA, seed=hd + Q)


@pytest.mark.parametrize("hd,S,total,causal", [(64, 100, 250, True), (96, 197, 300, False), (88, 129, 300, True),
                                               (80, 64, 150, False), (96, 65, 131, True)])
def test_wgmma_ragged_total_rows(cuda, hd, S, total, causal):
    """The last sequence cut short by total_rows: rows past it are poison on input and untouched on output."""
    from ymp import lib
    mask = AB.MASK_CAUSAL if causal else AB.MASK_NONE
    run(cuda, hd=hd, n=(total + S - 1) // S, s_q=S, s_kv=S, mask=mask, total_rows=total,
        fwd_path=lib.ATTN_PATH_WGMMA, bwd_path=lib.ATTN_PATH_WGMMA, probe="causal" if causal else None, seed=total)


@pytest.mark.parametrize("s_q", [1, 5, 64, 70])
@pytest.mark.parametrize("off", [1, 63, 64, 65, 200])
def test_wgmma_offset_causal(cuda, off, s_q):
    """Causal with s_q < s_kv, bottom-right aligned (forward only)."""
    from ymp import lib
    hd = WG_HD[(off + s_q) % 4]
    run(cuda, hd=hd, s_q=s_q, s_kv=s_q + off, mask=AB.MASK_CAUSAL, fwd_path=lib.ATTN_PATH_WGMMA, probe="causal",
        seed=off * 7 + s_q)


def test_wgmma_chained(cuda):
    from ymp import lib
    run(cuda, hd=80, s_q=129, s_kv=129, mask=AB.MASK_CAUSAL, fwd_path=lib.ATTN_PATH_WGMMA,
        bwd_path=lib.ATTN_PATH_WGMMA, chained=True, probe="causal", seed=5)


# ---------------------------------------------------------------------------------- decode (one query row)
@pytest.mark.parametrize("dev", [False, True], ids=["count", "device_count"])
@pytest.mark.parametrize("skv", [1, 127, 128, 129, 1000])
@pytest.mark.parametrize("hd", [64, 80, 96])
def test_decode(cuda, hd, skv, dev):
    """One query row per sequence; with the device-side key count the cache holds 37 more rows of +-3e4."""
    from ymp import lib
    if dev:
        run(cuda, hd=hd, n=3, s_q=1, s_kv=skv + 37, kv_count=skv, fwd_path=lib.ATTN_PATH_DECODE, seed=skv + hd)
    else:
        run(cuda, hd=hd, n=3, s_q=1, s_kv=skv, fwd_path=lib.ATTN_PATH_DECODE, seed=skv + hd)


def test_decode_chained(cuda):
    """The decoding forward, then the backward of the same call (served by the tensor-core kernels)."""
    from ymp import lib
    run(cuda, hd=64, n=3, s_q=1, s_kv=129, fwd_path=lib.ATTN_PATH_DECODE, bwd_path=lib.ATTN_PATH_WGMMA, chained=True,
        seed=9)


# ---------------------------------------------------------------------------------- small (block-diagonal, T <= 16)
@pytest.mark.parametrize("hd", [64, 80, 96, 128])
@pytest.mark.parametrize("T", [2, 3, 5, 8, 12, 16])
def test_small_block_diagonal(cuda, T, hd):
    """TimeSformer temporal attention packed into (64 // T) * T-row sequences; R rows in all, not a multiple of the
    packed sequence, so the last one is ragged."""
    from ymp import lib, ops
    R = T * (64 // T + 1)
    n, P = ops.temporal_pack(R, T)
    assert R % P
    run(cuda, hd=hd, n=n, s_q=P, s_kv=P, mask=AB.MASK_BLOCK, mask_block=T, total_rows=R, fwd_path=lib.ATTN_PATH_SMALL,
        bwd_path=lib.ATTN_PATH_SMALL, probe="block", seed=T * hd)


def test_small_chained(cuda):
    from ymp import lib, ops
    T, hd = 8, 96
    R = 8 * 21
    n, P = ops.temporal_pack(R, T)
    run(cuda, hd=hd, n=n, s_q=P, s_kv=P, mask=AB.MASK_BLOCK, mask_block=T, total_rows=R, fwd_path=lib.ATTN_PATH_SMALL,
        bwd_path=lib.ATTN_PATH_SMALL, chained=True, probe="block", seed=11)


# ---------------------------------------------------------------------------------- mma.sync
@pytest.mark.parametrize("kind,s_q,s_kv", [("dense", 130, 130), ("causal", 130, 130), ("cross", 70, 200),
                                           ("cross", 129, 64)])
def test_mma_sync_hd128(cuda, kind, s_q, s_kv):
    from ymp import lib
    mask = AB.MASK_CAUSAL if kind == "causal" else AB.MASK_NONE
    run(cuda, hd=128, s_q=s_q, s_kv=s_kv, mask=mask, fwd_path=lib.ATTN_PATH_MMA_SYNC, bwd_path=lib.ATTN_PATH_MMA_SYNC,
        probe="causal" if kind == "causal" else None, seed=s_q + s_kv)


@pytest.mark.parametrize("hd,T,P,total", [(64, 20, 80, 0), (96, 20, 80, 140), (64, 32, 96, 160), (80, 32, 96, 0),
                                          (88, 8, 64, 152), (88, 20, 60, 0), (128, 32, 128, 224)])
def test_mma_sync_block_mask(cuda, hd, T, P, total):
    """Block-diagonal masks the warp-per-sequence kernel declines (T > 16, or head_dim 88)."""
    from ymp import lib
    n = 3 if not total else (total + P - 1) // P
    run(cuda, hd=hd, n=n, s_q=P, s_kv=P, mask=AB.MASK_BLOCK, mask_block=T, total_rows=total,
        fwd_path=lib.ATTN_PATH_MMA_SYNC, bwd_path=lib.ATTN_PATH_MMA_SYNC, probe="block", seed=hd + T + P)


@pytest.mark.parametrize("s_kv", [257, 1000])
@pytest.mark.parametrize("s_q", [2, 7, 15])
def test_mma_sync_few_queries_long_keys(cuda, s_q, s_kv):
    """A few query rows against a long key range (forward)."""
    from ymp import lib
    hd = [64, 80, 96][(s_q + s_kv) % 3]
    run(cuda, hd=hd, s_q=s_q, s_kv=s_kv, fwd_path=lib.ATTN_PATH_MMA_SYNC, seed=s_q * s_kv)


@pytest.mark.parametrize("hd,s_q,ml,cnt", [(64, 5, 300, 200), (96, 16, 200, 131), (128, 3, 200, 64), (80, 2, 129, 1),
                                           (128, 1, 300, 257)])
def test_mma_sync_device_key_count(cuda, hd, s_q, ml, cnt):
    """The device-side key count with more than one query row (or head_dim 128): the cache rows past the count hold
    +-3e4 (forward)."""
    from ymp import lib
    run(cuda, hd=hd, n=3, s_q=s_q, s_kv=ml, kv_count=cnt, fwd_path=lib.ATTN_PATH_MMA_SYNC, seed=cnt + hd)


@pytest.mark.parametrize("kind", ["causal", "block"])
def test_mma_sync_chained(cuda, kind):
    from ymp import lib
    if kind == "causal":
        run(cuda, hd=128, s_q=130, s_kv=130, mask=AB.MASK_CAUSAL, fwd_path=lib.ATTN_PATH_MMA_SYNC,
            bwd_path=lib.ATTN_PATH_MMA_SYNC, chained=True, probe="causal", seed=13)
    else:
        run(cuda, hd=64, n=3, s_q=80, s_kv=80, mask=AB.MASK_BLOCK, mask_block=20, fwd_path=lib.ATTN_PATH_MMA_SYNC,
            bwd_path=lib.ATTN_PATH_MMA_SYNC, chained=True, probe="block", seed=14)


# ---------------------------------------------------------------------------------- dropout on the probabilities
# One isolated and one chained case for each family and keep-bit path: wgmma (s_q == 1 included: no decode kernel
# under dropout; cross attention; total_rows), the mma.sync kernels with the quad exchange (head_dim 64, 128) and with
# one Philox call per element in the dK / dV kernel (88, 96), and the mma.sync forward with the wgmma backward.
@pytest.mark.parametrize("hd,s_q,s_kv,n,mask,mb,total,p,chained", [
    (64, 129, 129, 2, AB.MASK_CAUSAL, 0, 0, 0.1, False), (96, 63, 129, 2, AB.MASK_NONE, 0, 0, 0.3, False),
    (64, 1, 70, 2, AB.MASK_NONE, 0, 0, 0.1, False), (64, 100, 100, 3, AB.MASK_CAUSAL, 0, 250, 0.3, False),
    (80, 129, 129, 2, AB.MASK_CAUSAL, 0, 0, 0.1, True),
    (128, 70, 200, 2, AB.MASK_NONE, 0, 0, 0.3, False), (64, 80, 80, 3, AB.MASK_BLOCK, 20, 0, 0.1, False),
    (128, 130, 130, 2, AB.MASK_CAUSAL, 0, 0, 0.1, True),
    (96, 96, 96, 3, AB.MASK_BLOCK, 24, 0, 0.3, False), (88, 80, 80, 3, AB.MASK_BLOCK, 8, 0, 0.3, True),
    (80, 7, 1000, 2, AB.MASK_NONE, 0, 0, 0.3, False), (96, 15, 257, 2, AB.MASK_NONE, 0, 0, 0.1, True)])
def test_dropout(cuda, hd, s_q, s_kv, n, mask, mb, total, p, chained):
    run(cuda, hd=hd, n=n, s_q=s_q, s_kv=s_kv, mask=mask, mask_block=mb, total_rows=total,
        fwd_path=fwd_family(hd, s_q, s_kv, mask, mb, total, drop=True), bwd_path=bwd_family(hd, mask, mb, drop=True),
        chained=chained, probe="causal" if mask == AB.MASK_CAUSAL else "block" if mask == AB.MASK_BLOCK else None,
        seed=hd + s_q + s_kv, drop=p)
