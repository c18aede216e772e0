"""GPU: decode attention through a KV row table (ymp_attn_args.kv_rows) and the beam searches that permute their beams
by gathering that table (KVCache.reindex) instead of moving the cached K/V rows.

Kernel: s_q = 1 through a scrambled table over a physical cache (the decode kernel at head_dim 64 / 80 / 96, the
mma.sync tiles at 88 / 128) is bit-identical to the same call on the physically gathered cache, at key counts around
the 128-key prefetch, both as s_kv and as the device-side count; rows that no table entry names hold NaN and must not
reach O.  Engine and model: every decode step and beam search is bit-identical
to the same run with the moving reorder."""
import json
import os

import pytest
import torch

from oracle import port
from oracle.make_golden import make_inputs
from helpers import build_pretrain

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
CFGS = os.path.join(ROOT, "youku-mplug_b200", "configs", "models")

HEADS = 3
KEY_COUNTS = (1, 127, 128, 129, 301)


def _views(buf, hd, m):
    from ymp import ops
    return ops.TView(buf, hd, 3 * hd, m), ops.TView(buf, 2 * hd, 3 * hd, m)


def _setup(dev, hd, n_seq, ld, seed):
    """A physical cache of n_seq * ld + 40 packed [q|k|v] rows (K/V of HEADS heads), a table [n_seq, ld] over a random
    subset of them (repeats allowed, as beams share rows) and the query rows.  Rows no entry names are NaN."""
    g = torch.Generator(device=dev).manual_seed(seed)
    P = n_seq * ld + 40
    buf = torch.randn(P, 3 * HEADS * hd, device=dev, generator=g).bfloat16()
    named = torch.randperm(P, device=dev, generator=g)[:n_seq * ld // 2 + 1]
    table = named[torch.randint(0, named.numel(), (n_seq, ld), device=dev, generator=g)].int()
    unnamed = torch.ones(P, dtype=torch.bool, device=dev)
    unnamed[table.reshape(-1).long()] = False
    buf[unnamed] = float("nan")
    q = torch.randn(n_seq, 3 * HEADS * hd, device=dev, generator=g).bfloat16()
    return buf, table, q


def _call(q, buf, hd, n_seq, s_kv, m_kv, kv_rows=None, s_kv_dev=None):
    from ymp import ops
    o = torch.full((n_seq, HEADS * hd), float("nan"), device=q.device, dtype=torch.bfloat16)
    k, v = _views(buf, hd, m_kv)
    lse = ops.attn_fwd(ops.TView(q, 0, 3 * hd, ops.dense_map(1)), k, v, ops.TView(o, 0, hd, ops.dense_map(1)), n_seq=n_seq,
                       n_heads=HEADS, head_dim=hd, s_q=1, s_kv=s_kv, causal=False, scale=hd ** -0.5, s_kv_dev=s_kv_dev,
                       kv_rows=kv_rows)
    return o, lse


@pytest.mark.parametrize("hd", [64, 80, 88, 96, 128])
def test_decode_through_table_equals_gathered_cache(cuda, hd):
    """head_dim 64 / 80 / 96: the streaming decode kernel.  128 and 88: the mma.sync tiles, which serve every s_q = 1
    call at 128 and, at 88, a table or more than 256 keys (88 takes no device-side count)."""
    from ymp import lib, ops
    n_seq = 5
    path = lib.ATTN_PATH_DECODE if hd in (64, 80, 96) else lib.ATTN_PATH_MMA_SYNC
    for n in KEY_COUNTS if hd != 88 else [k for k in KEY_COUNTS if k > 256]:
        for dev_count in (False, True) if hd != 88 else (False,):
            ld = n + 37 if dev_count else n   # device count: the kernel is launched for s_kv = ld > count keys
            buf, table, q = _setup(cuda, hd, n_seq, ld, seed=hd * 1000 + n * 2 + dev_count)
            if dev_count:   # entries past the count still name rows (the prefetch reads them): make those rows NaN
                buf[table[:, n:].reshape(-1).long()] = float("nan")
                named = table[:, :n].reshape(-1).long()
                buf[named] = torch.randn(named.numel(), buf.shape[1], device=cuda).bfloat16()
            cnt = torch.tensor([n], device=cuda, dtype=torch.int32)
            o, lse = _call(q, buf, hd, n_seq, ld, ops.dense_map(ld), kv_rows=table, s_kv_dev=cnt if dev_count else None)
            assert lib.attn_last_path() == path
            gathered = buf[table[:, :n].reshape(-1).long()].contiguous()
            ro, rlse = _call(q, gathered, hd, n_seq, n, ops.dense_map(n))
            assert lib.attn_last_path() == path
            assert not ro.isnan().any() and not o.isnan().any(), (hd, n, dev_count)
            assert torch.equal(o, ro), (hd, n, dev_count)
            assert torch.equal(lse, rlse), (hd, n, dev_count)


def test_table_wider_than_s_kv_and_ignored_seqmap(cuda):
    """kv_rows_ld > s_kv (the cache's max_len), and a k/v seqmap that would address other rows: the table decides."""
    from ymp import ops
    hd, n_seq, ld, n = 64, 4, 200, 150
    buf, table, q = _setup(cuda, hd, n_seq, ld, seed=3)
    wrong = ops.seqmap(seq_div=1, outer_stride=7, pos_stride=3)
    o, lse = _call(q, buf, hd, n_seq, n, wrong, kv_rows=table)
    gathered = buf[table[:, :n].reshape(-1).long()].contiguous()
    ro, rlse = _call(q, gathered, hd, n_seq, n, ops.dense_map(n))
    assert torch.equal(o, ro) and torch.equal(lse, rlse)


def test_kv_rows_rejected_off_the_decode_kernel(cuda):
    """A table is taken by single-query forward calls only (the decode kernel, and the mma.sync tiles at head_dim
    88 / 128): every other call is an error."""
    from ymp import lib, ops
    hd, n_seq, S = 64, 2, 16
    buf = torch.randn(n_seq * S, 3 * HEADS * hd, device=cuda).bfloat16()
    table = torch.arange(n_seq * S, device=cuda, dtype=torch.int32).view(n_seq, S)
    m = ops.dense_map(S)
    rng = torch.tensor([1, 0], device=cuda, dtype=torch.int64)

    def fwd(s_q, s_kv, causal=False, drop=None, total_rows=0, mask_block=0):
        k, v = _views(buf, hd, m)
        o = torch.empty((n_seq * s_q, HEADS * hd), device=cuda, dtype=torch.bfloat16)
        q = ops.TView(buf, 0, 3 * hd, m)
        return ops.attn_fwd(q, k, v, ops.TView(o, 0, hd, ops.dense_map(s_q)), n_seq=n_seq, n_heads=HEADS,
                            head_dim=hd, s_q=s_q, s_kv=s_kv, causal=causal, scale=0.1, drop=drop,
                            total_rows=total_rows, mask_block=mask_block, kv_rows=table)

    with pytest.raises(lib.YmpError, match="kv_rows"):
        fwd(4, S)                                                  # s_q > 1
    with pytest.raises(lib.YmpError, match="kv_rows"):
        fwd(1, S, causal=True)                                     # a mask (offset causal)
    with pytest.raises(lib.YmpError, match="kv_rows"):
        fwd(1, 1, causal=lib.MASK_BLOCK, mask_block=1)             # a mask (block-diagonal)
    with pytest.raises(lib.YmpError, match="kv_rows"):
        fwd(1, S, drop=ops.Drop(rng, ops.site_attn(0), 0.1))       # dropout
    with pytest.raises(lib.YmpError, match="kv_rows"):
        fwd(1, 1, total_rows=n_seq)                                # total_rows
    # the backward: the same arguments with the table set
    q, k, v = (ops.TView(buf, i * hd, 3 * hd, m) for i in range(3))
    o = torch.zeros((n_seq * S, HEADS * hd), device=cuda, dtype=torch.bfloat16)
    ov = ops.TView(o, 0, hd, m)
    lse = torch.zeros((n_seq, HEADS, S), device=cuda)
    b = lib.AttnBwdArgs()
    b.fwd = ops._attn_args(q, k, v, ov, lse, n_seq, HEADS, hd, S, S, False, 0.1, kv_rows=table)
    delta = torch.empty_like(lse)
    b.delta_ws = delta.data_ptr()
    b.dout, b.dq, b.dk, b.dv = ov.p, ov.p, ov.p, ov.p
    b.lddo = b.lddq = b.lddk = b.lddv = ov.ld
    b.do_head_stride = b.dq_head_stride = b.dk_head_stride = b.dv_head_stride = hd
    b.map_do = b.map_dq = b.map_dkv = m
    with pytest.raises(lib.YmpError, match="kv_rows"):
        lib.call(lib._attn_bwd, b, "ymp_attn_bwd")


# ------------------------------------------------------------------------------------------ engine level
def _gcfg(name, layers=None):
    with open(os.path.join(CFGS, f"config_gpt3_{name}.json")) as f:
        g = json.load(f)
    if layers is not None:
        g["num_hidden_layers"] = layers
    return g


def _tiny(dev):
    fx = torch.load(os.path.join(GOLD, "tiny_generate.pt"), weights_only=False)
    sd = port.generation_state_dict(fx["vcfg"], fx["gcfg"], fx["Q"], fx["wseed"], fx["pos_gain"], fx["ln_gain"])
    model = build_pretrain(fx["vcfg"], fx["gcfg"], fx["Q"], sd=sd, device=dev, dtype=torch.bfloat16,
                           cls_name="DistributedGPT3_Caption", num_frames=fx["vcfg"]["num_frames"]).eval()
    model.text_decoder.config.tokens_to_generate = fx["n_new"]
    return fx, model


def _steps(dec, M, ids, qf, rows, n_steps, moving, wide, stride=1, seed=5):
    """Prefill then n_steps single-token steps, each after a random beam permutation (KVCache.reindex, or the moving
    swap_key_value_dict).  stride > 1: the batched prefill of rows // stride clips into slots c * stride."""
    L = ids.shape[1]
    perm = torch.Generator().manual_seed(seed)
    dec.inference_params = ip = M.InferenceParams(rows, L + n_steps + qf.shape[1])
    ip.wide_step, ip.prefill_stride = wide, stride
    outs = []
    with torch.no_grad():
        out = dec(tokens=ids[::stride, :5], query_embeds=qf[::stride])
        outs.append(out.logits[:, -1].clone())
        logits = out.logits[:, -1].repeat_interleave(stride, 0)
        for t in range(n_steps):
            tok = logits.argmax(-1, keepdim=True)
            idx = torch.randint(0, rows, (rows,), generator=perm).to(ids.device)
            if moving:
                ip.swap_key_value_dict(idx)
            else:
                ip.cache.reindex(idx)
            out = dec(tokens=tok[idx])
            logits = out.logits[:, -1].clone()
            outs.append(logits)
    return torch.cat(outs), ip


@pytest.mark.parametrize("rows,wide,graph", [(5, False, "0"), (5, False, "1"), (60, True, "0"), (60, True, "1"),
                                             (12, False, "1")])
def test_token_steps_reindex_equal_moving_reorder(cuda, monkeypatch, rows, wide, graph):
    """5 and 60 rows through TokenStep (eager and graphed); 12 rows without the wide step take gpt_decode's eager
    single-token branch."""
    import models.modeling_distributed_gpt3 as M
    fx, model = _tiny(cuda)
    dec, Q = model.text_decoder, fx["Q"]
    video, ids, _ = make_inputs(rows, fx["vcfg"], fx["L"], fx["gcfg"]["vocab_size"], 11)
    with torch.no_grad():
        qf = model.visual_prefix(video.to(cuda).bfloat16())[3]
    ids = ids.to(cuda)
    monkeypatch.setenv("YMP_DECODE_GRAPH", graph)
    res = {}
    for moving in (True, False):
        dec.__dict__.pop("_decode_pool", None)
        res[moving], ip = _steps(dec, M, ids, qf, rows, 6, moving, wide)
        if rows <= 8 or wide:
            assert ip.cache.token is not None and (ip.cache.token.graph is not None) == (graph == "1")
        else:
            assert ip.cache.token is None
    assert not bool(torch.equal(ip.cache.rows, torch.arange(ip.cache.rows.numel(), device=cuda, dtype=torch.int32)
                                .view_as(ip.cache.rows)))   # the indexed run did permute through the table
    assert torch.equal(res[True], res[False])


@pytest.mark.parametrize("width", ["tiny", "2.7B"])
def test_seq_stride_prefill_then_steps_equal_moving(cuda, width):
    import models.modeling_distributed_gpt3 as M
    if width == "tiny":
        fx, model = _tiny(cuda)
        vcfg, L, C, beam = fx["vcfg"], fx["L"], 7, 3
    else:
        vcfg, L, C, beam = port.VCFG_TINY, 20, 12, 5
        model = build_pretrain(vcfg, _gcfg(width, layers=2), 128, device=cuda, dtype=torch.bfloat16,
                               cls_name="DistributedGPT3_Caption", num_frames=vcfg["num_frames"]).eval()
    dec = model.text_decoder
    video, ids, _ = make_inputs(C, vcfg, L, dec.config.vocab_size, 13)
    with torch.no_grad():
        qf = model.visual_prefix(video.to(cuda).bfloat16())[3]
    ids = ids.to(cuda).repeat_interleave(beam, 0)
    qf = qf.repeat_interleave(beam, 0)
    res = {}
    for moving in (True, False):
        dec.__dict__.pop("_decode_pool", None)
        res[moving], _ = _steps(dec, M, ids, qf, C * beam, 5, moving, True, stride=beam, seed=9)
    assert torch.equal(res[True], res[False])


# ------------------------------------------------------------------------------------------ model level
def _moving_callbacks(monkeypatch, M):
    """The beam loops' reorder callback as it was: the physical permutation of every cached row."""
    orig = M.DistributedGPT3._decode_callbacks

    def moving(self, query_embeds):
        step, _ = orig(self, query_embeds)
        return step, lambda idx: self.inference_params.cache.reorder(idx)
    monkeypatch.setattr(M.DistributedGPT3, "_decode_callbacks", moving)


def _run_both(monkeypatch, M, model, video, text, beam, per_clip):
    """(indexed, moving): the batched model.generate's beam search results (or, per_clip, one beam_search per clip),
    each with the physical cache rows swap_key_value_dict exposes afterwards."""
    dec = model.text_decoder
    out = {}
    for moving in (False, True):
        with monkeypatch.context() as mp:
            if moving:
                _moving_callbacks(mp, M)
            dec.__dict__.pop("_decode_pool", None)
            with torch.no_grad():
                if per_clip:
                    qf = model.visual_prefix(video)[3]
                    res = [dec.beam_search(text.input_ids[i:i + 1], query_embeds=qf[i:i + 1], beam_size=beam,
                                           stop_token=dec.config.eod_id) for i in range(video.shape[0])]
                else:
                    res = dec._beam_search_batched(text.input_ids, model.visual_prefix(video)[3], beam, 1,
                                                   dec.config.eod_id, text.input_ids.shape[1])
            ip = dec.inference_params
            n = ip.cache.len
            ip.swap_key_value_dict(list(reversed(range(ip.cache.B))))
            kv = torch.stack([t.view(ip.cache.B, ip.cache.max_len, -1)[:, :n] for t in ip.key_value_memory_dict.values()])
            out[moving] = ([(r.sequences.clone(), r.scores.clone()) for r in res], kv.clone())
    return out[False], out[True]


def _check(a, b):
    (res_a, kv_a), (res_b, kv_b) = a, b
    assert len(res_a) == len(res_b)
    for i, ((s0, c0), (s1, c1)) in enumerate(zip(res_a, res_b)):
        assert torch.equal(s0, s1), i
        assert torch.equal(c0, c1), i
    assert torch.equal(kv_a, kv_b)


def _text(M, ids, dev, plen=None):
    att = torch.ones_like(ids)
    if plen is not None:
        att[:, plen + 1:] = 0
    return M.BatchEncoding(dict(input_ids=ids.to(dev), attention_mask=att.to(dev)))


def test_generate_reindex_equals_moving_tiny(cuda, monkeypatch):
    """25 clips at beam 3 (a 21-clip and a 4-clip chunk; the fixture's weights make beams finish early), batched and
    per clip."""
    import models.modeling_distributed_gpt3 as M
    fx, model = _tiny(cuda)
    B = 25
    video, ids, _ = make_inputs(B, fx["vcfg"], fx["L"], fx["gcfg"]["vocab_size"], 17)
    ids[:2] = fx["ids"]
    video = video.to(cuda).bfloat16()
    text = _text(M, ids[:, :6], cuda)
    _check(*_run_both(monkeypatch, M, model, video, text, 3, per_clip=False))
    _check(*_run_both(monkeypatch, M, model, video[:4], _text(M, ids[:4, :6], cuda), 3, per_clip=True))
    # the public entry point, indexed, against the moving loop
    with torch.no_grad():
        res = model.generate(video, text)
    with monkeypatch.context() as mp:
        _moving_callbacks(mp, M)
        with torch.no_grad():
            ref = model.generate(video, text)
    assert all(torch.equal(a, b) for a, b in zip(res, ref)) and len(res) == len(ref) == B


@pytest.mark.parametrize("width", ["1.3B", "2.7B"])
def test_generate_reindex_equals_moving_wide(cuda, monkeypatch, width):
    """2-layer decoders at the 1.3B / 2.7B widths, 13 clips at beam 5 (a 60-row chunk and a 5-row one), and the
    per-clip beam search on three of them."""
    import models.modeling_distributed_gpt3 as M
    vcfg, Q, L, B = port.VCFG_TINY, 128, 20, 13
    model = build_pretrain(vcfg, _gcfg(width, layers=2), Q, device=cuda, dtype=torch.bfloat16,
                           cls_name="DistributedGPT3_Caption", num_frames=vcfg["num_frames"]).eval()
    model.text_decoder.config.tokens_to_generate = 12
    video, ids, _ = make_inputs(B, vcfg, L, model.text_decoder.config.vocab_size, 19)
    video = video.to(cuda).bfloat16()
    _check(*_run_both(monkeypatch, M, model, video, _text(M, ids, cuda), 5, per_clip=False))
    _check(*_run_both(monkeypatch, M, model, video[:3], _text(M, ids[:3], cuda), 5, per_clip=True))


def test_head_dim_128_decoder_reindex_equals_moving(cuda, monkeypatch):
    """A 2-layer decoder at head_dim 128 (hidden 256, 2 heads): its single-token steps attend through the row table on
    the mma.sync tiles; batched and per-clip beam searches are bit-equal to the moving reorder."""
    import models.modeling_distributed_gpt3 as M
    vcfg, Q, L, B = port.VCFG_TINY, 8, 8, 7
    gcfg = dict(port.GCFG_TINY, hidden_size=256, ffn_hidden_size=1024, num_attention_heads=2)
    model = build_pretrain(vcfg, gcfg, Q, device=cuda, dtype=torch.bfloat16, cls_name="DistributedGPT3_Caption",
                           num_frames=vcfg["num_frames"]).eval()
    model.text_decoder.config.tokens_to_generate = 8
    video, ids, _ = make_inputs(B, vcfg, L, gcfg["vocab_size"], 29)
    video = video.to(cuda).bfloat16()
    _check(*_run_both(monkeypatch, M, model, video, _text(M, ids, cuda), 3, per_clip=False))
    _check(*_run_both(monkeypatch, M, model, video[:2], _text(M, ids[:2], cuda), 3, per_clip=True))
