"""Host side of the shared-prefix evaluation: the key maps address the rows the repeated layout holds, the eval branches
choose the shared pass only when no backward and no dropout can be involved, and the tool's counted table."""
import importlib.util
import os

import pytest
import torch

from oracle import port
from helpers import build_pretrain

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _row(m, s, i):
    """include/ymp.h: row(s, i) of a ymp_seqmap."""
    if i < m.n_prefix:
        return m.prefix_base + (s if m.prefix_per_seq else s // m.seq_div) * m.prefix_stride + i
    return (s // m.seq_div) * m.outer_stride + (s % m.seq_div) * m.inner_stride + (i - m.n_prefix) * m.pos_stride


@pytest.mark.parametrize("V,t,Q,L", [(2, 3, 128, 80), (3, 2, 8, 8), (1, 5, 100, 37), (2, 1, 64, 130), (2, 4, 128, 1)])
def test_shared_prefix_maps_address_the_repeated_rows(V, t, Q, L):
    """Key i of sequence n is prefix row i of video n // t (rows N*L + v*Q + i) for i < Q, else text row n*L + i - Q:
    exactly the row that holds position i of [prefix n // t | text n] in the repeated layout."""
    from ymp import engine
    N, T = V * t, V * t * L
    m_txt, m_keys, m_pre = engine.shared_prefix_maps(V, t, Q, L)
    for n in range(N):
        assert [_row(m_keys, n, i) for i in range(Q)] == [T + (n // t) * Q + i for i in range(Q)]
        assert [_row(m_keys, n, Q + j) for j in range(L)] == [n * L + j for j in range(L)]
        assert [_row(m_txt, n, j) for j in range(L)] == [n * L + j for j in range(L)]
    for v in range(V):
        assert [_row(m_pre, v, i) for i in range(Q)] == [v * Q + i for i in range(Q)]   # on the rows from N*L on


def _cls_model(dropout=(0.0, 0.0)):
    return build_pretrain(port.VCFG_TINY, port.GCFG_TINY, 8, cls_name="DistributedGPT3_Cls", num_frames=2, use_cls=True,
                          num_classes=3, dropout=dropout)


def test_routing_predicate():
    m = _cls_model()
    qf_trainable = torch.zeros(2, 8, 128, requires_grad=True)
    qf_const = torch.zeros(2, 8, 128)
    with torch.no_grad():
        assert m._shared_prefix_ok(qf_trainable)                 # no graph is recorded
    with torch.enable_grad():
        assert not m._shared_prefix_ok(qf_trainable)             # a backward may reach the visual side
        assert m._shared_prefix_ok(qf_const)                     # frozen decoder, constant prefix
        m.text_decoder.dist_model.language_model.encoder.final_layernorm.weight.requires_grad_(True)
        assert not m._shared_prefix_ok(qf_const)                 # a trainable decoder parameter
    m = _cls_model(dropout=(0.1, 0.1))
    assert m.text_decoder.training
    with torch.no_grad():
        assert not m._shared_prefix_ok(qf_const)                 # dropout masks would differ per copy
        m.eval()
        assert m._shared_prefix_ok(qf_const)                     # eval mode: dropout off
        m.text_decoder.train()
    m = _cls_model(dropout=(0.0, 0.1))
    with torch.no_grad():
        assert not m._shared_prefix_ok(qf_const)                 # attention dropout alone counts too


def test_used_columns():
    from models.distributed_gpt3 import used_columns
    att = torch.tensor([[1, 1, 1, 0, 0, 0], [1, 1, 0, 0, 0, 0]])
    assert used_columns(att) == 3
    assert used_columns(torch.ones(2, 5, dtype=torch.long)) == 5
    assert used_columns(torch.zeros(2, 5, dtype=torch.long)) == 1


def test_tool_counts_match_the_table():
    spec = importlib.util.spec_from_file_location("eval_prefix", os.path.join(ROOT, "tools", "eval_prefix.py"))
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    table = {  # sequences, rows repeated -> shared, layer-GEMM TF repeated -> shared, LM-head TF repeated -> shared
        "cls_1.3B": (135, 28080, 11184, 67.8, 27.0, 5.9, 2.3),
        "cls_2.7B": (90, 18720, 7456, 94.2, 37.5, 4.9, 1.9),
        "itm_1.3B": (768, 159744, 73728, 385.9, 178.1, 33.5, 12.9),
        "itm_2.7B": (512, 106496, 49152, 536.0, 247.4, 27.9, 10.7),
    }
    for name, want in table.items():
        c = tool.counts(name)
        got = (c["sequences"], c["rows_repeated"], c["rows_shared"], round(c["layer_tf_repeated"], 1),
               round(c["layer_tf_shared"], 1), round(c["lm_head_tf_repeated"], 1), round(c["lm_head_tf_shared"], 1))
        assert got == want, name
