"""CPU: the host logic of the batched beam search (models.modeling_distributed_gpt3.run_beam_search_batched, the
grouping and chunking of DistributedGPT3.beam_search with B > 1) and the counted table of tools/caption_generate.py."""
import importlib.util
import os

import pytest
import torch

from oracle import port

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")


def _fixture():
    fx = torch.load(os.path.join(GOLD, "tiny_generate.pt"), weights_only=False)
    sd = port.generation_state_dict(fx["vcfg"], fx["gcfg"], fx["Q"], fx["wseed"], fx["pos_gain"], fx["ln_gain"])
    return fx, sd


class _OracleDecoder:
    """Decode callbacks over the oracle's fp32 full recompute, for `clips` clips of `rows` rows each.  The logits of
    each clip come from its own oracle call, so a batched run and a per-clip run see the same bits."""

    def __init__(self, qf, sd, gcfg, rows):
        self.qf, self.sd, self.gcfg, self.rows, self.hist = qf, sd, gcfg, rows, None

    def step(self, new_tokens, first):
        self.hist = new_tokens.clone() if first else torch.cat([self.hist, new_tokens], dim=1)
        r = self.rows
        with torch.no_grad():
            return torch.cat([port.next_token_logits(self.qf[c:c + 1].repeat(r, 1, 1), self.hist[c * r:(c + 1) * r], self.sd, self.gcfg)
                              for c in range(self.qf.shape[0])])

    def reorder(self, idx):
        self.hist = self.hist[idx]


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
def test_batched_beam_search_equals_per_clip(plen):
    import models.modeling_distributed_gpt3 as M
    fx, sd = _fixture()
    g, eod, Q, beam = fx["gcfg"], fx["eod"], fx["Q"], fx["beam_size"]
    ids, qf = _clips(fx, 4)
    kw = dict(beam_size=beam, num_return_gen=2, stop_token=eod, tokens_to_generate=fx["n_new"],
              max_position_embeddings=g["max_position_embeddings"])
    dec = _OracleDecoder(qf, sd, g, beam)
    batched = M.run_beam_search_batched(dec.step, dec.reorder, ids.clone(), plen, Q, **kw)
    assert len(batched) == ids.shape[0]
    for c in range(ids.shape[0]):
        one = _OracleDecoder(qf[c:c + 1], sd, g, beam)
        ref = M.run_beam_search(one.step, one.reorder, ids[c:c + 1].clone(), plen, Q, **kw)
        assert torch.equal(batched[c].sequences, ref.sequences), c
        assert torch.equal(batched[c].scores, ref.scores), c
    if plen == int(fx["prompt_length"][0]):   # the fixture's own clip at its own prompt length: the reference's result
        assert torch.equal(batched[0].sequences[:1], fx["beam_sequences"][0])


def test_first_call_may_return_one_row_per_clip():
    """The batched decoder's prefill returns one row per clip: the ranking only reads each clip's first beam."""
    import models.modeling_distributed_gpt3 as M
    fx, sd = _fixture()
    g, beam = fx["gcfg"], fx["beam_size"]
    ids, qf = _clips(fx, 3)
    kw = dict(beam_size=beam, num_return_gen=1, stop_token=fx["eod"], tokens_to_generate=fx["n_new"],
              max_position_embeddings=g["max_position_embeddings"])
    full = _OracleDecoder(qf, sd, g, beam)
    a = M.run_beam_search_batched(full.step, full.reorder, ids.clone(), 5, fx["Q"], **kw)
    thin = _OracleDecoder(qf, sd, g, beam)

    def step(new_tokens, first):
        out = thin.step(new_tokens, first)
        return out.view(ids.shape[0], beam, -1)[:, 0] if first else out
    b = M.run_beam_search_batched(step, thin.reorder, ids.clone(), 5, fx["Q"], **kw)
    assert all(torch.equal(x.sequences, y.sequences) and torch.equal(x.scores, y.scores) for x, y in zip(a, b))


def test_chunks_group_by_prompt_length_in_input_order():
    import models.modeling_distributed_gpt3 as M
    assert M.beam_search_chunks([7, 5, 7], 5, 64) == [(7, [0, 2]), (5, [1])]
    ch = M.beam_search_chunks([4] * 25, 3, 64)
    assert ch == [(4, list(range(21))), (4, list(range(21, 25)))]
    assert M.beam_search_chunks([9] * 36, 5, 64) == [(9, list(range(s, min(s + 12, 36)))) for s in (0, 12, 24)]
    with pytest.raises(ValueError):
        M.beam_search_chunks([1, 1], 65, 64)


def test_decoder_beam_search_routes_chunks_and_returns_input_order(monkeypatch):
    """DistributedGPT3.beam_search with B > 1: one batched search per chunk, each with a wide-step cache of
    clips x beam rows whose prefill fills every clip's first beam slot; results come back in input order."""
    import models.modeling_distributed_gpt3 as M
    from helpers import make_model_dir
    os.environ["YMP_ALLOW_RANDOM_INIT"] = "1"
    gcfg = dict(port.GCFG_TINY)
    dec = M.DistributedGPT3(model_dir=make_model_dir(port.VCFG_TINY, gcfg))
    calls = []

    def fake(step, reorder, tokens, plen, nq, **kw):
        ip = dec.inference_params
        calls.append((tokens.shape[0], plen, nq, ip.max_batch_size, ip.wide_step, ip.prefill_stride, kw["beam_size"]))
        return [M.AttrDict(sequences=tokens[i:i + 1].clone(), scores=torch.tensor([float(plen)])) for i in range(tokens.shape[0])]
    monkeypatch.setattr(M, "run_beam_search_batched", fake)
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
