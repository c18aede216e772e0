"""CPU: the packed-text layout of the retrieval text features (ymp.functional.packed_text_rows) against a numpy
restatement of its rule, and the C ABI of ymp_attn_fwd_packed (header declaration, ctypes mirror)."""
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rule(mask):
    """numpy: packed length 1 + max(last attended column, pooled column), pooled column = mask.sum() - 1 read as
    Python indexes (-1: the last column); starts are the running sum of the lengths."""
    mask = np.asarray(mask)
    L = mask.shape[1]
    lens, pooled = [], []
    for row in mask:
        col = int(row.sum()) - 1
        col = col + L if col < 0 else col
        nz = np.nonzero(row)[0]
        last = int(nz[-1]) if len(nz) else -1
        lens.append(1 + max(last, col))
        pooled.append(col)
    starts = np.concatenate([[0], np.cumsum(lens)])
    return starts, np.array(lens), starts[:-1] + np.array(pooled)


def _check(mask):
    from ymp import functional as YF
    starts, lens, rows = YF.packed_text_rows(torch.tensor(mask))
    want = _rule(mask)
    for got, w in zip((starts, lens, rows), want):
        assert got.dtype == torch.int64 and got.tolist() == w.tolist(), (mask, got, w)
    return starts.tolist(), lens.tolist(), rows.tolist()


def test_right_padded_masks():
    mask = [[1] * n + [0] * (8 - n) for n in (3, 5, 2)]
    assert _check(mask) == ([0, 3, 8, 10], [3, 5, 2], [2, 7, 9])


def test_full_length_and_length_one_rows():
    mask = [[1] * 8, [1] + [0] * 7, [1] * 8]
    assert _check(mask) == ([0, 8, 9, 17], [8, 1, 8], [7, 8, 16])


def test_mask_with_a_hole_keeps_the_last_attended_column():
    # sum - 1 = 3 but column 5 is attended: the text keeps columns 0 .. 5 and pools packed row 3
    mask = [[1, 1, 0, 1, 0, 1, 0, 0], [1, 1, 1, 0, 0, 0, 0, 0]]
    assert _check(mask) == ([0, 6, 9], [6, 3], [3, 8])


def test_empty_mask_pools_the_last_column_as_the_padded_pass_reads_it():
    mask = [[0] * 6, [1, 1, 0, 0, 0, 0]]
    assert _check(mask) == ([0, 6, 8], [6, 2], [5, 7])


def test_random_masks_match_the_rule():
    g = np.random.default_rng(5)
    for _ in range(20):
        B, L = int(g.integers(1, 9)), int(g.integers(1, 81))
        lens = g.integers(1, L + 1, B)
        mask = (np.arange(L)[None, :] < lens[:, None]).astype(np.int64)
        mask[g.random((B, L)) < 0.1] = 0   # holes
        _check(mask)


def test_pooled_column_outside_the_mask_is_rejected():
    from ymp import functional as YF
    with pytest.raises(ValueError, match="pooled"):
        YF.packed_text_rows(torch.tensor([[2, 2, 2, 0]]))


def test_packed_args_mirror_the_header():
    from ymp import lib as L
    hdr = open(os.path.join(ROOT, "include", "ymp.h")).read()
    body = re.search(r"typedef struct ymp_attn_packed_args \{(.*?)\} ymp_attn_packed_args;", hdr, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = [re.findall(r"([A-Za-z_][A-Za-z0-9_]*)\s*$", d.strip())[0] for d in body.split(";") if d.strip()]
    assert fields == [f[0] for f in L.AttnPackedArgs._fields_] == ["attn", "starts", "max_len", "_pad"]
    assert L.AttnPackedArgs._fields_[0][1] is L.AttnArgs
    assert re.search(r"int ymp_attn_fwd_packed\(const ymp_attn_packed_args\* a, void\* stream\);", hdr)
    assert hasattr(L.lib, "ymp_attn_fwd_packed")
