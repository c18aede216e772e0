"""CPU: the host logic of the chunked beam search (models.modeling_distributed_gpt3.run_beam_search over a fixed-length
decode state of several groups, the grouping and chunking of DistributedGPT3.beam_search with B > 1, the torch ops of
its decoding step) and the counted table of tools/caption_generate.py."""
import importlib.util
import os
from collections import Counter

import pytest
import torch
from torch.utils._python_dispatch import TorchDispatchMode

from oracle import port

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


def _fixture():
    fx = torch.load(os.path.join(GOLD, "tiny_generate.pt"), weights_only=False)
    sd = port.generation_state_dict(fx["vcfg"], fx["gcfg"], fx["Q"], fx["wseed"], fx["pos_gain"], fx["ln_gain"])
    return fx, sd


class _OracleDecoder:
    """Fixed-length decode callbacks (the contract of DistributedGPT3._fixed_len_decoder) over the oracle's fp32 full
    recompute, for `clips` clips of `rows` rows each, all prefilled together at one prompt length; step ignores
    `live`.  The logits of each clip come from its own oracle call over all its rows (the prefill returns each clip's
    first beam), so a search of several clips and a per-clip search see the same bits."""

    def __init__(self, qf, sd, gcfg, ids, rows):
        self.qf, self.sd, self.gcfg, self.ids, self.rows, self.hist = qf, sd, gcfg, ids, rows, None

    def _logits(self):
        r = self.rows
        with torch.no_grad():
            return torch.cat([port.next_token_logits(self.qf[c:c + 1].repeat(r, 1, 1), self.hist[c * r:(c + 1) * r], self.sd, self.gcfg)
                              for c in range(self.qf.shape[0])])

    def prefill(self, group0, group_stride, clips, n):
        assert self.hist is None and (group0, group_stride, list(clips)) == (0, 1, list(range(self.qf.shape[0])))
        self.hist = self.ids[:, :n].repeat_interleave(self.rows, 0)
        return self._logits()[::self.rows]

    def step(self, new_tokens, live):
        self.hist = torch.cat([self.hist, new_tokens], dim=1)
        return self._logits()

    def reorder(self, idx):
        self.hist = self.hist[idx]


def _search(dec, ids, plens, Q, groups, **kw):
    import models.modeling_distributed_gpt3 as M
    return M.run_beam_search(dec.step, dec.prefill, dec.reorder, ids.clone(), plens, Q, groups=groups, **kw)


def _clips(fx, n):
    """n clips: the fixture's two clips, then variants with other prompt tokens (same query features)."""
    g = torch.Generator().manual_seed(7)
    ids, qf = [], []
    for i in range(n):
        row = fx["ids"][i % 2].clone()
        if i >= 2:
            row[1:] = torch.randint(0, fx["gcfg"]["vocab_size"], (row.numel() - 1,), generator=g)
        ids.append(row)
        qf.append(fx["query_features"][i % 2])
    return torch.stack(ids), torch.stack(qf)


@pytest.mark.parametrize("plen", [5, 7])
def test_chunk_groups_equal_per_clip_search(plen):
    fx, sd = _fixture()
    g, eod, Q, beam = fx["gcfg"], fx["eod"], fx["Q"], fx["beam_size"]
    ids, qf = _clips(fx, 4)
    kw = dict(beam_size=beam, num_return_gen=2, stop_token=eod, tokens_to_generate=fx["n_new"],
              max_position_embeddings=g["max_position_embeddings"])
    C = ids.shape[0]
    batched = _search(_OracleDecoder(qf, sd, g, ids, beam), ids, [plen] * C, Q, C, **kw)
    assert len(batched) == C
    for c in range(C):
        one = _OracleDecoder(qf[c:c + 1], sd, g, ids[c:c + 1], beam)
        ref, = _search(one, ids[c:c + 1], [plen], Q, 1, **kw)
        assert torch.equal(batched[c].sequences, ref.sequences), c
        assert torch.equal(batched[c].scores, ref.scores), c
    if plen == int(fx["prompt_length"][0]):   # the fixture's own clip at its own prompt length: the reference's result
        assert torch.equal(batched[0].sequences[:1], fx["beam_sequences"][0])


def test_chunks_group_by_prompt_length_in_input_order():
    import models.modeling_distributed_gpt3 as M
    assert M.beam_search_chunks([7, 5, 7], 5, 64) == [(7, [0, 2]), (5, [1])]
    ch = M.beam_search_chunks([4] * 25, 3, 64)
    assert ch == [(4, list(range(21))), (4, list(range(21, 25)))]
    assert M.beam_search_chunks([9] * 36, 5, 64) == [(9, list(range(s, min(s + 12, 36)))) for s in (0, 12, 24)]
    with pytest.raises(ValueError):
        M.beam_search_chunks([1, 1], 65, 64)


def test_decoder_beam_search_runs_chunks_on_fixed_len_states(monkeypatch):
    """DistributedGPT3.beam_search with B > 1: one search per chunk over a fixed-length decode state of one group per
    clip, each with a wide-step cache of clips x beam rows whose prefill fills every clip's first beam slot; results
    come back in input order."""
    import models.modeling_distributed_gpt3 as M
    from helpers import make_model_dir
    os.environ["YMP_ALLOW_RANDOM_INIT"] = "1"
    gcfg = dict(port.GCFG_TINY)
    dec = M.DistributedGPT3(model_dir=make_model_dir(port.VCFG_TINY, gcfg))
    calls = []

    fixed = M.DistributedGPT3._fixed_len_decoder
    made = []

    def spy(self, *a, **k):
        made.append(fixed(self, *a, **k))
        return made[-1]

    def fake(step, prefill, reorder, tokens, plens, nq, **kw):
        ip = dec.inference_params
        assert (step, prefill, reorder) == made[-1] and len(set(plens)) == 1 and kw["groups"] == tokens.shape[0]
        calls.append((tokens.shape[0], plens[0], nq, ip.max_batch_size, ip.wide_step, ip.prefill_stride, kw["beam_size"]))
        return [M.AttrDict(sequences=tokens[i:i + 1].clone(), scores=torch.tensor([float(plens[i])]))
                for i in range(tokens.shape[0])]
    monkeypatch.setattr(M.DistributedGPT3, "_fixed_len_decoder", spy)
    monkeypatch.setattr(M, "run_beam_search", fake)
    B, beam, Q = 25, 3, 4
    ids = torch.arange(B * 6).view(B, 6)
    plens = torch.tensor([5 if i in (1, 7, 11) else 4 for i in range(B)])
    qe = torch.zeros(B, Q, gcfg["hidden_size"])
    res = dec.beam_search(ids, query_embeds=qe, beam_size=beam, prompt_length=plens)
    assert len(res) == B
    for i in range(B):
        assert torch.equal(res[i].sequences[0], ids[i]) and float(res[i].scores[0]) == float(plens[i])
    assert [c[:2] for c in calls] == [(21, 4), (1, 4), (3, 5)]   # 64 // 3 = 21 clips per chunk
    assert all(c[2] == Q and c[3] == c[0] * beam and c[4] and c[5] == beam and c[6] == beam for c in calls)
    assert len(made) == len(calls)


class _OpCount(TorchDispatchMode):
    """Counts the aten ops issued while no callback runs (callbacks raise `paused`)."""

    def __init__(self):
        super().__init__()
        self.ops, self.paused = [], 0

    def __torch_dispatch__(self, func, types, args=(), kwargs=None):
        if not self.paused:
            self.ops.append(str(func))
        return func(*args, **(kwargs or {}))


# The torch ops of one decoding step of the chunked beam search's own loop, before the chunks ran through
# run_beam_search, counted in this test's setting: 26, three of them tensors built from host lists (aten.lift_fresh: a
# host-to-device copy each on a GPU).
CHUNKED_STEP_OPS, CHUNKED_STEP_HOST_LISTS = 26, 3


@pytest.mark.parametrize("deterministic", [False, True])
def test_all_live_step_issues_no_more_ops_than_the_chunked_loop(deterministic):
    """12 groups of beam 5 at one prompt length whose beams never finish (the stop token's logit is -1e9): every
    decoding step has all groups live and refills nothing.  Its ranking, survivor writes and next tokens issue no more
    torch ops, and no more tensors from host lists, than the chunked loop's step did; all of them also run under
    torch.use_deterministic_algorithms."""
    import models.modeling_distributed_gpt3 as M
    was = torch.are_deterministic_algorithms_enabled()
    G, beam, V, L, plen, stop = 12, 5, 64, 6, 4, 3
    gen = torch.Generator().manual_seed(0)
    mode, marks = _OpCount(), []

    def logits(n):
        mode.paused += 1
        lg = torch.randn(n, V, generator=gen)
        lg[:, stop] = -1e9
        mode.paused -= 1
        return lg

    def step(new_tokens, live):
        assert all(live)
        marks.append(len(mode.ops))
        return logits(G * beam)
    tokens = torch.randint(4, V, (G, L), generator=gen)
    torch.use_deterministic_algorithms(deterministic)
    try:
        with mode:
            res = M.run_beam_search(step, lambda g0, gstride, clips, n: logits(len(clips)), lambda idx: None, tokens,
                                    [plen] * G, 0, groups=G, beam_size=beam, num_return_gen=1, stop_token=stop,
                                    tokens_to_generate=8, max_position_embeddings=100)
    finally:
        torch.use_deterministic_algorithms(was)
    assert len(res) == G and len(marks) == 9   # positions 4 .. 13: the prefill, then 9 steps
    for a, b in zip(marks, marks[1:]):   # from one step's logits to the next step's call
        ops = Counter(mode.ops[a:b])
        assert sum(ops.values()) <= CHUNKED_STEP_OPS, ops
        assert ops["aten.lift_fresh.default"] <= CHUNKED_STEP_HOST_LISTS, ops


def _tool():
    spec = importlib.util.spec_from_file_location("caption_generate", os.path.join(ROOT, "tools", "caption_generate.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_counts_table():
    t = _tool()
    c = t.counts("caption_2.7B")
    h, layers, V = 2560, 32, 51200
    assert c["weight_gb_per_step"] == round((24 * h * h * layers + 2 * V * h) / 1e9, 3)
    assert (c["clips"], c["chunks"], c["rows_per_chunk"], c["kv_positions"]) == (36, 3, 60, 248)
    assert c["passes_per_clip_arm"] == 3600 and c["passes_batched_arm"] == 300   # a 12x cut
    assert abs(c["kv_cache_gb_per_chunk"] - 7.31) < 0.01                          # 32 x 60 x 248 x 3h x 2 bytes
    c = t.counts("caption_1.3B")
    assert (c["clips"], c["chunks"], c["passes_per_clip_arm"], c["passes_batched_arm"]) == (24, 2, 2400, 200)
    assert abs(c["weight_gb_per_step"] - 2.63) < 0.01
