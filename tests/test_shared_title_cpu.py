"""Host side of sharing a video's title columns among its texts: the per-video shared column count, the row layout of
the shared pass checked by index arithmetic against the repeated [N, Q + Le] rows, and the ctypes mirror of the
prefix-table attention arguments."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BOS, EOS, PAD = 1, 2, 0


def _fit_prompt(prompt, label, length):
    """DistributedGPT3Tokenizer._fit_prompt on [bos] + prompt + label + [eos], padded to `length`."""
    import models.modeling_distributed_gpt3 as G

    class Tok:
        tokenizer = type("T", (), {"pad": PAD})()
        _fit = G.DistributedGPT3Tokenizer._fit
    arr, plen, n = G.DistributedGPT3Tokenizer._fit_prompt(Tok(), ([BOS], list(prompt), list(label), [EOS]), length)
    return list(arr), plen, n


def _texts(rows, length):
    """rows: (prompt, label) per text -> (input_ids, attention_mask, loss-read columns) as the generation pass sees
    them: loss column j (loss_mask column Q + j) is read when j >= prompt_length and token j + 1 is attended."""
    from models.distributed_gpt3 import build_targets, mask_prompt
    ids, att, plen = [], [], []
    for prompt, label in rows:
        a, p, n = _fit_prompt(prompt, label, length)
        ids.append(a)
        att.append([1] * n + [0] * (length - n))
        plen.append(p)
    ids, att, plen = torch.tensor(ids), torch.tensor(att), torch.tensor(plen)
    Q = 4
    _, loss_mask = build_targets(ids, mask_prompt(att[:, 1:].clone(), plen), Q)
    read = torch.nn.functional.pad(loss_mask[:, Q:], (0, 1))
    return ids, att, read


def _shared(rows, length, V):
    from models.distributed_gpt3 import shared_text_columns
    return shared_text_columns(*_texts(rows, length), V)


def test_common_prompt_is_shared_up_to_the_first_scored_column():
    # video 0: prompt of 5 tokens, labels of 1..3 tokens; video 1: prompt of 9 tokens
    p0, p1 = [10, 11, 12, 13, 14], [20 + i for i in range(9)]
    rows = [(p0, [30]), (p0, [31, 32]), (p0, [33, 34, 35]), (p1, [30]), (p1, [36, 37]), (p1, [38])]
    shared, used = _shared(rows, 20, 2)
    # bos + prompt = 1 + len(prompt) columns in common; the first loss column is len(prompt) (predicts the label)
    assert shared == [5, 9]
    assert used == [1 + 5 + 3 + 1, 1 + 9 + 2 + 1]


def test_labels_sharing_a_first_token_do_not_extend_past_the_scored_column():
    p = [10, 11, 12]
    rows = [(p, [40, 41]), (p, [40, 42]), (p, [40])]
    ids, _, _ = _texts(rows, 12)
    assert torch.equal(ids[:, :5], ids[:1, :5].expand(3, 5))   # bos, prompt and the label's first token agree
    shared, used = _shared(rows, 12, 1)
    assert shared == [3] and used == [7]


def test_prompt_shortened_for_some_rows_only():
    # length 12: a label of 6 tokens leaves room for 12 - 6 - 2 = 4 prompt tokens; the short labels keep all 7
    p = [10, 11, 12, 13, 14, 15, 16]
    rows = [(p, [30]), (p, [31, 32, 33, 34, 35, 36]), (p, [37, 38])]
    ids, _, read = _texts(rows, 12)
    assert ids[1, 1:5].tolist() == p[:4] and ids[1, 5] == 31
    shared, _ = _shared(rows, 12, 1)
    assert shared == [4]   # the truncated row leaves the common ids and is scored from its column 4 on
    assert int(read[1].nonzero()[0]) == 4


def test_one_text_per_video_shares_nothing():
    shared, used = _shared([([10, 11, 12], [30]), ([10, 11], [31, 32])], 10, 2)
    assert shared == [0, 0] and used == [6, 6]


def test_no_read_column_leaves_the_last_used_column_unshared():
    from models.distributed_gpt3 import shared_text_columns
    ids = torch.tensor([[1, 5, 6, 7, 0, 0], [1, 5, 6, 7, 0, 0], [1, 5, 6, 7, 8, 0], [1, 5, 6, 7, 9, 0]])
    att = (ids != 0).long()
    shared, used = shared_text_columns(ids, att, torch.zeros_like(ids), 2)
    assert used == [4, 5]
    assert shared == [3, 4]   # the whole of video 0's rows agree: Le_v - 1; video 1 differs at column 4


def test_read_hidden_columns_limit_the_shared_count():
    from models.distributed_gpt3 import shared_text_columns
    ids = torch.tensor([[1, 5, 6, 7, 8, 3], [1, 5, 6, 7, 8, 4]] * 2)
    att = torch.ones_like(ids)
    read = torch.zeros_like(ids)
    read[0, 4] = 1   # video 0: the hidden state of column 4 of its first text is read (the cls pass)
    read[3, 2] = 1   # video 1: column 2 of its second text
    shared, used = shared_text_columns(ids, att, read, 2)
    assert shared == [4, 2] and used == [6, 6]


def _row(m, s, i, n_prefix=None):
    """include/ymp.h: row(s, i) of a ymp_seqmap; n_prefix: the prefix-table call's key prefix of sequence s."""
    npre = m.n_prefix if n_prefix is None else n_prefix
    if i < npre:
        return m.prefix_base + (s if m.prefix_per_seq else s // m.seq_div) * m.prefix_stride + i
    return (s // m.seq_div) * m.outer_stride + (s % m.seq_div) * m.inner_stride + (i - npre) * m.pos_stride


def _holder(V, t, Q, P, Ls, n, i):
    """The row of the shared pass that computes position i of the repeated sequence [prefix n // t | text n]."""
    N, v = V * t, n // t
    B = Q + max(P)
    if i < Q + P[v]:                 # a query row or a shared text column: video v's block
        return N * Ls + v * B + i
    return n * Ls + (i - Q - P[v])   # text column i - Q >= P_v: text n's suffix row


@pytest.mark.parametrize("V,t,Q,P,Le", [(2, 3, 128, [20, 60], [26, 66]), (3, 2, 8, [0, 1, 5], [8, 3, 7]),
                                          (1, 5, 100, [0], [37]), (2, 4, 64, [63, 1], [64, 65]), (2, 2, 8, [0, 0], [8, 8])])
def test_shared_title_maps_address_the_repeated_rows(V, t, Q, P, Le):
    """Key i of text n (with the per-video prefix Q + P_v of the table call) and its query / block rows are exactly the
    rows that hold position i of [prefix n // t | text n] in the repeated layout."""
    from ymp import engine, functional as YF
    N = V * t
    L = max(Le)
    Pl, Ls, Pmax = YF.shared_title_layout(V, L, P, Le)
    assert Pl == P and Ls == max(u - p for p, u in zip(P, Le)) and Pmax == max(P)
    m_txt, m_keys, m_blk = engine.shared_title_maps(V, t, Q, Ls, Pmax)
    for n in range(N):
        v = n // t
        S = Q + Le[v]
        npre = Q + P[v]
        assert [_row(m_keys, n, i, npre) for i in range(S)] == [_holder(V, t, Q, P, Ls, n, i) for i in range(S)]
        # the text rows (queries and outputs of the table call) are the suffix rows, position Q + P_v + j
        assert [_row(m_txt, n, j) for j in range(Le[v] - P[v])] == [_holder(V, t, Q, P, Ls, n, npre + j)
                                                                  for j in range(Le[v] - P[v])]
    for v in range(V):   # the square causal call over the blocks (on the rows from N*Ls on)
        assert [N * Ls + _row(m_blk, v, i) for i in range(Q + P[v])] == [_holder(V, t, Q, P, Ls, v * t, i)
                                                                       for i in range(Q + P[v])]
    # the caller's text row n*L + j is read from the row holding position Q + j; columns from P_v + Ls on do not exist
    p_n = torch.tensor(P).repeat_interleave(t)
    want = torch.arange(N * L)
    rows, keep = YF.shared_title_rows(p_n, t, Q, L, Ls, Pmax, want)
    for n in range(N):
        for j in range(L):
            k = n * L + j
            assert bool(keep[k]) == (j < P[n // t] + Ls)
            if j < Le[n // t]:
                assert keep[k] and int(rows[k]) == _holder(V, t, Q, P, Ls, n, Q + j)


def test_shared_title_layout_rejects_bad_counts():
    from ymp import functional as YF
    assert YF.shared_title_layout(2, 10) == ([0, 0], 10, 0)
    for shared, used in (([3, 0], [3, 5]), ([0], [5]), ([-1, 0], None), ([0, 0], [0, 4]), ([0, 0], [4, 11])):
        with pytest.raises(ValueError, match="shared"):
            YF.shared_title_layout(2, 10, shared, used)


def test_prefix_table_args_mirror_the_header():
    from ymp import lib as L
    hdr = open(os.path.join(ROOT, "include", "ymp.h")).read()
    body = re.search(r"typedef struct ymp_attn_prefix_table_args \{(.*?)\} ymp_attn_prefix_table_args;", hdr, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    fields = [re.findall(r"([A-Za-z_][A-Za-z0-9_]*)\s*$", d.strip())[0] for d in body.split(";") if d.strip()]
    assert fields == [f[0] for f in L.AttnPrefixTableArgs._fields_] == ["attn", "n_prefix"]
    assert L.AttnPrefixTableArgs._fields_[0][1] is L.AttnArgs
    assert re.search(r"int ymp_attn_fwd_prefix_table\(const ymp_attn_prefix_table_args\* a, void\* stream\);", hdr)
    assert hasattr(L.lib, "ymp_attn_fwd_prefix_table")
