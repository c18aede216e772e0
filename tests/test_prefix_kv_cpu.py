"""Host side of the evaluation's prefix cache: the row layout of a shared pass that reads its prefixes' keys and values
from a PrefixKV, checked by index arithmetic against the repeated [N, Q + Le] rows; the rule that decides when an eval
call may reuse the kept clip's prefixes; the ctypes mirror of the prefix-cache attention arguments; and the tool's
row and FLOP counts, which need no GPU."""
import os
import re
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _key_row(m, s, i, n0, n_prefix):
    """ymp_attn_fwd_prefix_kv: (source, row) of key i of sequence s; source 'cache' (row of the prefix cache) or 'x'
    (row of the pass's own buffer, through the key seqmap m)."""
    if i < n0:
        return "cache", (s // m.seq_div) * n0 + i
    if i < n_prefix:
        return "x", m.prefix_base + (s // m.seq_div) * m.prefix_stride + (i - n0)
    return "x", (s // m.seq_div) * m.outer_stride + (s % m.seq_div) * m.inner_stride + (i - n_prefix) * m.pos_stride


def _holder(V, t, Q, P, Ls, n, i):
    """Where the cached pass keeps position i of the repeated sequence [prefix n // t | text n]."""
    N, v = V * t, n // t
    if i < Q:
        return "cache", v * Q + i                           # the video's prefix row i, in the PrefixKV
    if i < Q + P[v]:
        return "x", N * Ls + v * max(P) + (i - Q)           # a shared title column: the video's title rows
    return "x", n * Ls + (i - Q - P[v])                     # the text's own suffix row


@pytest.mark.parametrize("V,t,Q,P,Le", [(2, 3, 128, [20, 60], [26, 66]), (3, 2, 8, [0, 1, 5], [8, 3, 7]),
                                          (1, 5, 100, [0], [37]), (2, 4, 64, [63, 1], [64, 65]), (2, 2, 8, [0, 0], [8, 8])])
def test_cached_title_maps_address_the_repeated_rows(V, t, Q, P, Le):
    """Key i of text n (n0 = Q cached keys, n_prefix = Q + P_v) and key i of video v's title rows (n0 = n_prefix = Q)
    are exactly the rows that hold position i of [prefix n // t | text n] in the repeated layout."""
    from ymp import engine, functional as YF
    N = V * t
    L = max(Le)
    _, Ls, Pmax = YF.shared_title_layout(V, L, P, Le)
    m_txt, m_keys, m_title = engine.cached_title_maps(V, t, Ls, Pmax)
    for n in range(N):
        v = n // t
        S = Q + Le[v]
        assert [_key_row(m_keys, n, i, Q, Q + P[v]) for i in range(S)] == [_holder(V, t, Q, P, Ls, n, i) for i in range(S)]
        assert [("x", _key_row(m_txt, n, j, 0, 0)[1]) for j in range(Le[v] - P[v])] == \
            [_holder(V, t, Q, P, Ls, n, Q + P[v] + j) for j in range(Le[v] - P[v])]
    for v in range(V):   # the title call: Q cached keys, then the video's title rows (from row N*Ls on)
        keys = [_key_row(m_title, v, i, Q, Q) for i in range(Q + P[v])]
        keys = [(src, r if src == "cache" else N * Ls + r) for src, r in keys]
        assert keys == [_holder(V, t, Q, P, Ls, v * t, i) for i in range(Q + P[v])]
    # the caller's text row n*L + j is read from the row holding position Q + j; columns from P_v + Ls on do not exist
    p_n = torch.tensor(P).repeat_interleave(t)
    rows, keep = YF.cached_title_rows(p_n, t, L, Ls, Pmax, torch.arange(N * L))
    for n in range(N):
        for j in range(L):
            k = n * L + j
            assert bool(keep[k]) == (j < P[n // t] + Ls)
            if j < Le[n // t]:
                assert keep[k] and ("x", int(rows[k])) == _holder(V, t, Q, P, Ls, n, Q + j)


def test_prefix_cache_hit_rule():
    from models.distributed_gpt3 import prefix_cache_hit
    clip = torch.zeros(2, 3)
    w = (17, 4)
    entry = (clip, (clip._version, w), "query_features", "prefix_kv")
    assert prefix_cache_hit(entry, clip, w, True)
    assert not prefix_cache_hit(entry, clip, w, False)             # grad, dropout or train mode: never read
    assert not prefix_cache_hit(None, clip, w, True)
    assert not prefix_cache_hit(entry, clip.clone(), w, True)      # equal values, another tensor
    assert not prefix_cache_hit(entry, clip.view(2, 3), w, True)   # a view is another tensor object too
    assert not prefix_cache_hit(entry, clip, (18, 4), True)        # a parameter was written in place
    assert not prefix_cache_hit(entry, clip, (17, 5), True)        # an optimizer step or a checkpoint load
    clip.add_(1)                                                   # the clip was edited in place
    assert not prefix_cache_hit(entry, clip, w, True)


def test_train_engine_and_checkpoint_load_count_as_weight_writes():
    src = open(os.path.join(ROOT, "youku-mplug_b200", "ymp", "train.py")).read()
    for fn in ("def step(self)", "def load_checkpoint(self"):
        body = src.split(fn, 1)[1].split("\n    def ", 1)[0]
        assert "YF.note_weight_write()" in body, fn
    from ymp import functional as YF
    n = YF.weight_writes()
    YF.note_weight_write()
    assert YF.weight_writes() == n + 1


def test_prefix_kv_args_mirror_the_header():
    import ctypes
    from ymp import lib as L
    hdr = open(os.path.join(ROOT, "include", "ymp.h")).read()
    body = re.search(r"typedef struct ymp_attn_prefix_kv_args \{(.*?)\} ymp_attn_prefix_kv_args;", hdr, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    decls = [d.strip() for d in body.split(";") if d.strip()]
    fields = [re.findall(r"([A-Za-z_][A-Za-z0-9_]*)\s*$", d)[0] for d in decls]
    assert fields == [f[0] for f in L.AttnPrefixKvArgs._fields_] == \
        ["table", "k_cache", "v_cache", "ld_cache", "cache_head_stride", "n0", "_pad"]
    types = dict(L.AttnPrefixKvArgs._fields_)
    assert types["table"] is L.AttnPrefixTableArgs
    assert all(types[f] is ctypes.c_void_p for f in ("k_cache", "v_cache"))
    assert all(d.startswith("int32_t") for d in decls[3:]) and all(types[f] is ctypes.c_int32 for f in fields[3:])
    assert ctypes.sizeof(L.AttnPrefixKvArgs) == ctypes.sizeof(L.AttnPrefixTableArgs) + 2 * 8 + 4 * 4
    assert re.search(r"int ymp_attn_fwd_prefix_kv\(const ymp_attn_prefix_kv_args\* a, void\* stream\);", hdr)
    assert hasattr(L.lib, "ymp_attn_fwd_prefix_kv")


def test_itm_eval_counts_run_without_a_gpu():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "itm_eval.py"), "--counts"], capture_output=True,
                       text=True, timeout=300, env={**os.environ, "CUDA_VISIBLE_DEVICES": ""})
    assert r.returncode == 0, r.stderr
    out = r.stdout
    for shape in ("itm_1.3B", "itm_2.7B", "cls_1.3B", "cls_2.7B"):
        assert shape in out
    # the ITM chunk calls after the first compute no prefix row and no encoder FLOP
    assert re.search(r"itm_1\.3B\s+cached\s+later\s+\d+\s+0\s+0\b", out), out
