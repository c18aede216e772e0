"""CPU: the generation host logic of the product (models.modeling_distributed_gpt3.run_sample /
run_beam_search, BeamHypotheses, sample) driven by the ORACLE's fp32 next-token logits must reproduce the
unmodified reference's sequences and scores (tests/golden/tiny_generate.pt, oracle/make_golden.py)."""
import os

import torch

from oracle import port

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


class _OracleDecoder:
    """Decode callbacks over the oracle's fp32 full recompute: run_sample's step(new_tokens, first), and run_beam_search's
    prefill / beam_step / reorder over one clip (ids [1, L]) in `rows` identical beams, with the contract of the model's
    fixed-length decode state (beam_step ignores `live`)."""

    def __init__(self, qf, sd, gcfg, ids=None, rows=1):
        self.qf, self.sd, self.gcfg, self.ids, self.rows, self.hist = qf, sd, gcfg, ids, rows, None

    def step(self, new_tokens, first):
        self.hist = new_tokens.clone() if first else torch.cat([self.hist, new_tokens], dim=1)
        with torch.no_grad():
            return port.next_token_logits(self.qf, self.hist, self.sd, self.gcfg)

    def prefill(self, group0, group_stride, clips, n):
        assert (group0, group_stride, list(clips)) == (0, 1, [0])
        return self.step(self.ids[:, :n].repeat(self.rows, 1), True)[:1]

    def beam_step(self, new_tokens, live):
        return self.step(new_tokens, False)

    def reorder(self, idx):
        self.hist = self.hist[idx]


def _fixture():
    fx = torch.load(os.path.join(GOLD, "tiny_generate.pt"), weights_only=False)
    sd = port.generation_state_dict(fx["vcfg"], fx["gcfg"], fx["Q"], fx["wseed"], fx["pos_gain"], fx["ln_gain"])
    return fx, sd


def test_oracle_generation_matches_reference_fixture():
    fx, sd = _fixture()
    g, eod, qf = fx["gcfg"], fx["eod"], fx["query_features"]
    with torch.no_grad():
        for i in range(fx["B"]):
            seq, sc = port.beam_search_generate(fx["ids"][i:i + 1], sd, g, query_features=qf[i:i + 1], prompt_length=fx["prompt_length"][i],
                                                beam_size=fx["beam_size"], stop_token=eod, tokens_to_generate=fx["n_new"], eod_id=eod)
            assert torch.equal(seq, fx["beam_sequences"][i])
            assert (sc - fx["beam_scores"][i]).abs().max() < 1e-4
        greedy = port.sample_generate(fx["ids"].clone(), sd, g, query_features=qf, prompt_length=fx["prompt_length"].clone(),
                                      tokens_to_generate=fx["n_new"], eod_id=eod, top_k=1, top_p=0.0, termination_id=eod)
    assert torch.equal(greedy, fx["greedy"])


def test_product_loops_with_oracle_logits():
    import models.modeling_distributed_gpt3 as M
    fx, sd = _fixture()
    g, eod, qf, Q = fx["gcfg"], fx["eod"], fx["query_features"], fx["Q"]
    for i in range(fx["B"]):
        dec = _OracleDecoder(qf[i:i + 1].repeat(fx["beam_size"], 1, 1), sd, g, fx["ids"][i:i + 1], fx["beam_size"])
        out, = M.run_beam_search(dec.beam_step, dec.prefill, dec.reorder, fx["ids"][i:i + 1], [int(fx["prompt_length"][i])], Q,
                                 groups=1, beam_size=fx["beam_size"], num_return_gen=1, stop_token=eod,
                                 tokens_to_generate=fx["n_new"], max_position_embeddings=g["max_position_embeddings"])
        assert torch.equal(out.sequences, fx["beam_sequences"][i])
        assert (out.scores.reshape(-1) - fx["beam_scores"][i]).abs().max() < 1e-4
    dec = _OracleDecoder(qf, sd, g)
    toks = M.run_sample(dec.step, fx["ids"].clone(), fx["prompt_length"].clone(), Q, tokens_to_generate=fx["n_new"], eod_id=eod,
                        max_position_embeddings=g["max_position_embeddings"], top_k=1, top_p=0.0, vocab_size=g["vocab_size"],
                        termination_id=eod)
    assert torch.equal(toks, fx["greedy"])


def test_sampling_filters():
    """Top-k / top-p filters and sample() of the product and of the oracle against the reference's own functions
    (outputs stored in the fixture by oracle/make_golden.py)."""
    import models.modeling_distributed_gpt3 as M
    fx, _ = _fixture()
    f = fx["filters"]
    logits = f["logits"]
    a = logits.clone()
    M.modify_logits_for_top_k_filtering(a, 5)
    assert torch.equal(a, f["top_k5"]) and torch.equal(port.filter_top_k(logits, 5), f["top_k5"])
    b = logits.clone()
    M.modify_logits_for_top_p_filtering(b, 0.7)
    assert torch.equal(b, f["top_p07"]) and torch.equal(port.filter_top_p(logits, 0.7), f["top_p07"])
    assert torch.equal(M.sample(logits, top_k=1), f["greedy"])
    torch.manual_seed(3)
    s1 = M.sample(logits, top_k=0, top_p=0.9, temperature=0.7, vocab_size=40)
    torch.manual_seed(3)
    s2 = port.pick_token(logits, top_k=0, top_p=0.9, temperature=0.7, vocab_size=40)
    assert torch.equal(s1, f["sample_seed3_p09_t07_v40"]) and torch.equal(s2, s1) and int(s1.max()) < 40


def test_kv_cache_reorder_is_in_place_and_touches_cached_positions_only():
    """ymp.engine.KVCache host logic (no kernel involved): `reorder` = InferenceParams.swap_key_value_dict
    (modeling_distributed_gpt3.py:1460-1473) on every layer at once, IN PLACE - the captured decoding graph holds the
    buffers' addresses - and only over the positions that hold keys; `reset` forgets the length but keeps the storage."""
    from ymp import engine
    gcfg = dict(port.GCFG_TINY)
    B, ML = 3, 6
    cache = engine.KVCache(gcfg, B, ML, torch.device("cpu"))
    assert len(cache.qkv) == gcfg["num_hidden_layers"] and all(t.shape == (B * ML, 3 * gcfg["hidden_size"]) for t in cache.qkv)
    ptrs = [t.data_ptr() for t in cache.qkv]
    g = torch.Generator().manual_seed(0)
    for t in cache.qkv:
        t.copy_(torch.randn(t.shape, generator=g).to(t.dtype))
    before = [t.clone() for t in cache.qkv]
    cache._set_len(4)
    assert int(cache.len_idx) == 4 and int(cache.len1) == 5 and cache.len == 4
    idx = torch.tensor([2, 0, 0])
    cache.reorder(idx)
    for t, old in zip(cache.qkv, before):
        new3, old3 = t.view(B, ML, -1), old.view(B, ML, -1)
        assert torch.equal(new3[:, :4], old3.index_select(0, idx)[:, :4])      # cached positions follow the beams
        assert torch.equal(new3[:, 4:], old3[:, 4:])                            # rows past the length are left alone
    assert [t.data_ptr() for t in cache.qkv] == ptrs                            # nothing was re-allocated
    cache.reset()
    assert cache.len == 0 and int(cache.len_idx) == 0 and int(cache.len1) == 1
    snapshot = [t.clone() for t in cache.qkv]
    cache.reorder(torch.tensor([1, 2, 0]))                                      # empty cache: nothing to permute
    assert all(torch.equal(a, b) for a, b in zip(cache.qkv, snapshot))
