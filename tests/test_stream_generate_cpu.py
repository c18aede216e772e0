"""CPU: the host logic of the streaming beam search (models.modeling_distributed_gpt3.run_beam_search over a per-row
decode state: a finished clip's slot group takes the next clip), the routing of DistributedGPT3.beam_search with B > 1,
and the per-row table bookkeeping of ymp.engine.KVCache."""
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


def _clips(fx, n):
    """n clips: the fixture's two clips, then variants with other prompt tokens (same query features)."""
    g = torch.Generator().manual_seed(11)
    ids, qf = [], []
    for i in range(n):
        row = fx["ids"][i % 2].clone()
        if i >= 2:
            row[1:] = torch.randint(0, fx["gcfg"]["vocab_size"], (row.numel() - 1,), generator=g)
        ids.append(row)
        qf.append(fx["query_features"][i % 2])
    return torch.stack(ids), torch.stack(qf)


class _OneClip:
    """Fixed-length run_beam_search callbacks of one clip (ids [1, L], groups = 1) over the oracle's fp32 full
    recompute; step ignores `live`."""

    def __init__(self, qf, sd, gcfg, ids, beam):
        self.qf, self.sd, self.gcfg, self.ids, self.beam, self.hist = qf, sd, gcfg, ids, beam, None

    def _logits(self):
        with torch.no_grad():
            return port.next_token_logits(self.qf.repeat(self.beam, 1, 1), self.hist, self.sd, self.gcfg)

    def prefill(self, group0, group_stride, clips, n):
        self.hist = self.ids[:, :n].repeat(self.beam, 1)
        return self._logits()[:1]

    def step(self, new_tokens, live):
        self.hist = torch.cat([self.hist, new_tokens], dim=1)
        return self._logits()

    def reorder(self, idx):
        self.hist = self.hist[idx]


class _StreamDecoder:
    """Per-row run_beam_search callbacks over the oracle: each group keeps its own clip's token history, so a group's
    logits are those of its clip alone.  Records the prefill calls and each group's cache length (prefix + tokens)."""

    def __init__(self, qf, sd, gcfg, ids, groups, beam, max_len):
        self.qf, self.sd, self.gcfg, self.ids, self.G, self.beam, self.max_len = qf, sd, gcfg, ids, groups, beam, max_len
        self.hist = [None] * groups
        self.clip = [None] * groups
        self.lens = [0] * groups
        self.prefills, self.live_log = [], []

    def _logits(self, g):
        with torch.no_grad():
            return port.next_token_logits(self.qf[self.clip[g]:self.clip[g] + 1].repeat(self.hist[g].shape[0], 1, 1),
                                          self.hist[g], self.sd, self.gcfg)

    def prefill(self, group0, group_stride, clips, n):
        self.prefills.append((group0, group_stride, list(clips), n))
        out = []
        for i, c in enumerate(clips):
            g = group0 + i * group_stride
            self.clip[g], self.hist[g] = c, self.ids[c:c + 1, :n].repeat(self.beam, 1)
            self.lens[g] = self.qf.shape[1] + n
            out.append(self._logits(g)[:1])
        return torch.cat(out)

    def step(self, new_tokens, live):
        assert len(live) == self.G
        self.live_log.append(list(live))
        vocab = self.gcfg["vocab_size"]
        out = torch.zeros(self.G * self.beam, vocab)
        for g in range(self.G):
            if not live[g]:
                continue
            r = slice(g * self.beam, (g + 1) * self.beam)
            self.hist[g] = torch.cat([self.hist[g], new_tokens[r]], dim=1)
            assert self.lens[g] + 1 <= self.max_len   # a live group never steps past the cache
            self.lens[g] += 1
            out[r] = self._logits(g)
        return out

    def reorder(self, idx):
        for g in range(self.G):
            base = g * self.beam
            loc = idx[base:base + self.beam] - base
            assert bool(((loc >= 0) & (loc < self.beam)).all()), "rows move only within their group"
            if self.hist[g] is not None:
                self.hist[g] = self.hist[g][loc]


@pytest.mark.parametrize("beam,groups,n_ret", [(3, 2, 2), (5, 3, 1), (3, 4, 3)])
def test_per_row_groups_equal_per_clip_search(beam, groups, n_ret):
    """More clips than groups, mixed prompt lengths: each clip's sequences and scores equal run_beam_search on that clip
    alone, and groups are refilled mid-run."""
    import models.modeling_distributed_gpt3 as M
    fx, sd = _fixture()
    g, eod, Q = fx["gcfg"], fx["eod"], fx["Q"]
    N = 9
    ids, qf = _clips(fx, N)
    plens = [5, 7, 4, 6, 5, 7, 3, 6, 4][:N]
    kw = dict(beam_size=beam, num_return_gen=n_ret, stop_token=eod, tokens_to_generate=fx["n_new"],
              max_position_embeddings=g["max_position_embeddings"])
    final_len = min(ids.shape[1] + fx["n_new"], g["max_position_embeddings"])
    dec = _StreamDecoder(qf, sd, g, ids, groups, beam, final_len + Q)
    res = M.run_beam_search(dec.step, dec.prefill, dec.reorder, ids.clone(), plens, Q, groups=groups, **kw)
    assert len(res) == N
    for c in range(N):
        one = _OneClip(qf[c:c + 1], sd, g, ids[c:c + 1], beam)
        ref, = M.run_beam_search(one.step, one.prefill, one.reorder, ids[c:c + 1].clone(), [plens[c]], Q, groups=1, **kw)
        assert torch.equal(res[c].sequences, ref.sequences), c
        assert torch.equal(res[c].scores, ref.scores), c
    started = [c for _, _, cs, _ in dec.prefills for c in cs]
    assert started == list(range(N))                      # clips start in input order, each once
    assert len(dec.prefills) > 1 and len(dec.live_log) > 0
    # refills mid-run: some prefill happens after the first decoding step
    assert any(not all(live) for live in dec.live_log) or len(dec.prefills) > len({p for *_, p in dec.prefills})


def test_per_row_groups_refill_at_different_steps():
    """Clips whose captions end at different steps: groups are refilled at several distinct steps, and a group with no
    clip left is frozen (not live) for the remaining steps."""
    import models.modeling_distributed_gpt3 as M
    fx, sd = _fixture()
    g, Q, beam, G = fx["gcfg"], fx["Q"], 3, 3
    N = 8
    ids, qf = _clips(fx, N)
    plens = [5, 4, 6, 5, 7, 4, 6, 5]
    final_len = min(ids.shape[1] + fx["n_new"], g["max_position_embeddings"])
    dec = _StreamDecoder(qf, sd, g, ids, G, beam, final_len + Q)
    steps_at = []
    step = dec.step

    def counted(new_tokens, live):
        steps_at.append(len(dec.prefills))
        return step(new_tokens, live)
    M.run_beam_search(counted, dec.prefill, dec.reorder, ids.clone(), plens, Q, beam_size=beam, num_return_gen=1,
                      stop_token=fx["eod"], tokens_to_generate=fx["n_new"],
                      max_position_embeddings=g["max_position_embeddings"], groups=G)
    assert len(set(steps_at)) >= 3           # prefills land between different decoding steps
    assert not all(dec.live_log[-1])         # the tail runs with frozen groups


def test_prefill_runs_share_equal_lengths_and_spacing():
    import models.modeling_distributed_gpt3 as M
    assert M._prefill_runs([0, 1, 2, 3], [5, 5, 5, 5]) == [(5, 0, 1, [0, 1, 2, 3])]
    assert M._prefill_runs([0, 1, 2, 3, 4], [5, 7, 5, 7, 5]) == [(5, 0, 2, [0, 2, 4]), (7, 1, 2, [1, 3])]
    assert M._prefill_runs([1, 2, 5], [4, 4, 4]) == [(4, 1, 1, [1, 2]), (4, 5, 1, [5])]
    assert M._prefill_runs([3], [9]) == [(9, 3, 1, [3])]


def test_streaming_is_chosen_where_it_gains_and_runs():
    """The streaming search runs clips that need more than one batched chunk (more clips than 64 // beam, or several
    prompt lengths), at head_dim 64 / 80 / 96, on a CUDA device; everything else keeps the chunked batched search."""
    import models.modeling_distributed_gpt3 as M
    cuda, cpu = torch.device("cuda", 0), torch.device("cpu")
    assert M.streams_beam_search([4] * 25, 3, 64, cuda)            # 21 clips per chunk: two chunks
    assert M.streams_beam_search([4, 5, 4, 4], 5, 80, cuda)        # two prompt lengths: two chunks
    assert M.streams_beam_search([9] * 36, 5, 96, "cuda")
    assert not M.streams_beam_search([4] * 12, 5, 64, cuda)        # one 60-row chunk: nothing to refill
    assert not M.streams_beam_search([4] * 25, 3, 128, cuda)       # no per-sequence decode attention at 88 / 128
    assert not M.streams_beam_search([4] * 25, 3, 88, cuda)
    assert not M.streams_beam_search([4] * 25, 3, 64, cpu)


def test_decoder_beam_search_streams_on_per_row_state_in_input_order(monkeypatch):
    """DistributedGPT3.beam_search with B > 1 where streams_beam_search says so: one streaming search over a per-row
    decode state of 64 // beam groups (at most B), every clip's own prompt length, results in input order; otherwise
    the chunked search over fixed-length decode states."""
    import models.modeling_distributed_gpt3 as M
    from helpers import make_model_dir
    os.environ["YMP_ALLOW_RANDOM_INIT"] = "1"
    gcfg = dict(port.GCFG_TINY)
    dec = M.DistributedGPT3(model_dir=make_model_dir(port.VCFG_TINY, gcfg))
    calls, chunked, decided, made = [], [], [], {}
    adapters = {k: getattr(M.DistributedGPT3, k) for k in ("_per_row_decoder", "_fixed_len_decoder")}

    def spy(kind):
        def build(self, *a, **k):
            made[kind] = adapters[kind](self, *a, **k)
            return made[kind]
        return build

    def fake(step, prefill, reorder, tokens, plens, nq, **kw):
        if (step, prefill, reorder) == made.pop("_per_row_decoder", None):
            calls.append((tokens.shape[0], list(plens), nq, kw["groups"], kw["beam_size"]))
            return [M.AttrDict(sequences=tokens[i:i + 1].clone(), scores=torch.tensor([float(plens[i])]))
                    for i in range(tokens.shape[0])]
        assert (step, prefill, reorder) == made.pop("_fixed_len_decoder") and len(set(plens)) == 1
        chunked.append((tokens.shape[0], plens[0]))
        return [M.AttrDict(sequences=tokens[i:i + 1].clone(), scores=torch.tensor([0.0])) for i in range(tokens.shape[0])]
    decide = M.streams_beam_search

    def on_device(lengths, beam, hd, device):   # the CPU tensors stand in for CUDA ones
        decided.append((list(lengths), beam, hd, torch.device(device).type))
        return decide(lengths, beam, hd, "cuda")
    for k in adapters:
        monkeypatch.setattr(M.DistributedGPT3, k, spy(k))
    monkeypatch.setattr(M, "run_beam_search", fake)
    monkeypatch.setattr(M, "streams_beam_search", on_device)
    B, beam, Q = 25, 3, 4
    ids = torch.arange(B * 6).view(B, 6)
    plens = [5 if i in (1, 7, 11) else 4 for i in range(B)]
    qe = torch.zeros(B, Q, gcfg["hidden_size"])
    res = dec.beam_search(ids, query_embeds=qe, beam_size=beam, prompt_length=torch.tensor(plens))
    assert len(res) == B
    for i in range(B):
        assert torch.equal(res[i].sequences[0], ids[i]) and float(res[i].scores[0]) == float(plens[i])
    assert calls == [(B, plens, Q, 21, beam)] and not chunked
    assert decided == [(plens, beam, 64, "cpu")]
    # two prompt lengths among 4 clips: two chunks, so the stream with one group per clip
    dec.beam_search(ids[:4], query_embeds=qe[:4], beam_size=5, prompt_length=torch.tensor(plens[:4]))
    assert calls[-1] == (4, plens[:4], Q, 4, 5) and not chunked
    # 12 clips at beam 5 with one prompt length fit one 60-row chunk: the batched search
    res = dec.beam_search(ids[:12], query_embeds=qe[:12], beam_size=5, prompt_length=4)
    assert len(calls) == 2 and chunked == [(12, 4)] and len(res) == 12


def test_kv_cache_per_row_table_after_refill_and_reindex(monkeypatch):
    """Per-row mode on CPU (the layer pass stubbed): a refill resets its group's rows to the identity and points them at
    the group's first slot; reindex_rows gathers each row's own cached columns only, so every column p >= lens[b] stays
    the identity b * max_len + p even when the rows' lengths differ."""
    from ymp import engine
    monkeypatch.setattr(engine, "_decode_layers", lambda W, x, cache, n, off, B, SL, row0=0: x)
    monkeypatch.setattr(engine, "_last_hidden", lambda W, x, g, B, n: torch.zeros(B, g.H))
    gcfg = dict(port.GCFG_TINY)
    beam, G, ML = 3, 4, 16
    c = engine.KVCache(gcfg, G * beam, ML, "cpu")
    c.reset_rows()
    ident = torch.arange(G * beam * ML, dtype=torch.int32).view(G * beam, ML)

    def check():
        lens = c.lens.tolist()
        assert lens == c.lens_host and c.lens1.tolist() == [n + 1 for n in lens]
        for b in range(G * beam):
            assert torch.equal(c.rows[b, lens[b]:], ident[b, lens[b]:]), b
            g0 = b // beam * beam
            # every cached column names a row of the row's own group
            assert bool(((c.rows[b, :lens[b]] // ML >= g0) & (c.rows[b, :lens[b]] // ML < g0 + beam)).all()), b

    c.prefill_groups(None, torch.zeros(2 * 5, gcfg["hidden_size"]), 5, 0, 2, beam)   # groups 0 and 2, 5 positions
    c.prefill_groups(None, torch.zeros(2 * 9, gcfg["hidden_size"]), 9, 1, 2, beam)   # groups 1 and 3, 9 positions
    check()
    assert torch.equal(c.rows[1, :5], ident[0, :5]) and torch.equal(c.rows[4, :9], ident[3, :9])
    gen = torch.Generator().manual_seed(3)
    for t in range(6):
        # a decoding step writes each row's own slot at its length, then the live rows advance
        live = [1, 1, 1, 0] if t >= 3 else [1, 1, 1, 1]
        c.set_live([x for x in live for _ in range(beam)])
        c.lens += c.adv
        c.lens1.copy_(c.lens + 1)
        c.lens_host = [n + a for n, a in zip(c.lens_host, c.adv_host)]
        idx = torch.cat([g * beam + torch.randint(0, beam, (beam,), generator=gen) for g in range(G)])
        c.reindex_rows(idx)
        check()
        if t == 2:   # group 2 finishes; the next clip (7 positions) is prefilled into it mid-run
            c.prefill_groups(None, torch.zeros(7, gcfg["hidden_size"]), 7, 2, 1, beam)
            check()
            assert torch.equal(c.rows[6:9, :7], ident[6, :7].expand(3, 7))
    assert max(c.lens_host) < ML
    assert c.lens_host[9:12] == [9 + 3] * 3   # the frozen group stopped advancing
