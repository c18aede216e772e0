"""GPU: batched caption generation.  The wide skinny GEMM (9..64 rows) against the M <= 8 one (bit for bit, row by
row) and an fp32 reference; the 60-row captured decode step; the batched prefill into each clip's first beam slot;
DistributedGPT3_Caption.generate against the per-clip beam-search loop (sequences and scores bit for bit); and the
visual prefix under torch.no_grad() (no kept block activations)."""
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


def _gcfg(name, layers=None):
    with open(os.path.join(CFGS, f"config_gpt3_{name}.json")) as f:
        g = json.load(f)
    if layers is not None:
        g["num_hidden_layers"] = layers
    return g


def _linear_shapes():
    """(N, K) of every skinny GEMM of the 1.3B and 2.7B decoding step: QKV, dense, h->4h, 4h->h, LM head."""
    out = []
    for name in ("1.3B", "2.7B"):
        g = _gcfg(name)
        h, V = g["hidden_size"], g["vocab_size"]
        out += [(3 * h, h), (h, h), (4 * h, h), (h, 4 * h), (V, h)]
    return out


# (bias, act, residual dtype, out dtype, y2): every epilogue the decoding step uses, and the other combinations
EPILOGUES = [
    (False, 0, None, torch.bfloat16, False),
    (True, 2, None, torch.bfloat16, False),              # h -> 4h: bias + tanh GELU
    (True, 1, torch.bfloat16, torch.float32, False),     # erf GELU, bf16 residual, fp32 out
    (True, 0, torch.float32, torch.float32, False),      # dense / 4h -> h: bias + fp32 residual stream
    (False, 0, torch.float32, torch.bfloat16, False),
    (True, 0, None, torch.bfloat16, True),               # QKV: bias + the KV-cache copy at the device offset
]
WIDE_M = (5, 9, 16, 17, 40, 60, 64)   # 5: the wide entry point's M <= 8 launch


def _skinny(x, w, bias, act, residual, out_dtype, y2, wide=True):
    """ops.gemm_skinny_wide (or, with wide=False, ops.gemm_skinny: at most 8 rows)."""
    from ymp import ops
    fn = ops.gemm_skinny_wide if wide else ops.gemm_skinny
    if not y2:
        return fn(x, w, bias=bias, act=act, residual=residual, out_dtype=out_dtype), None
    M, N = x.shape[0], w.shape[0]
    stride, off = 3, torch.tensor([2], device=x.device, dtype=torch.int64)
    buf = torch.zeros((M * stride, N), device=x.device, dtype=torch.bfloat16)
    y = fn(x, w, bias=bias, act=act, residual=residual, out_dtype=out_dtype, out2=buf, out2_row_stride=stride, out2_off=off)
    assert torch.equal(buf.view(M, stride, N)[:, 2], y)                       # row m at m * stride + *off
    assert not buf.view(M, stride, N)[:, :2].any()                            # nothing else written
    return y, buf


@pytest.mark.parametrize("N,K", _linear_shapes())
def test_wide_skinny_rows_equal_narrow_rows(cuda, N, K):
    g = torch.Generator(device=cuda).manual_seed(N * 7 + K)
    w = (torch.randn(N, K, device=cuda, generator=g) * K ** -0.5).bfloat16()
    x = torch.randn(64, K, device=cuda, generator=g).bfloat16()
    bias = (torch.randn(N, device=cuda, generator=g) * 0.5).bfloat16()
    for has_bias, act, rdt, odt, y2 in EPILOGUES:
        b = bias if has_bias else None
        res = None if rdt is None else torch.randn(64, N, device=cuda, generator=g).to(rdt)
        narrow = torch.cat([_skinny(x[r:r + 8], w, b, act, None if res is None else res[r:r + 8], odt, y2, wide=False)[0]
                            for r in range(0, 64, 8)])
        ref = x.float() @ w.float().t()
        if has_bias:
            ref += bias.float()
        if act == 2:
            ref = torch.nn.functional.gelu(ref, approximate="tanh")
        elif act == 1:
            ref = torch.nn.functional.gelu(ref)
        if res is not None:
            ref += res.float()
        err = (narrow.float() - ref).abs().max().item()
        assert err <= 2e-2 * ref.abs().max().item() + 1e-3, (N, K, act, rdt, odt, err)
        for M in WIDE_M:
            y, _ = _skinny(x[:M], w, b, act, None if res is None else res[:M].contiguous(), odt, y2)
            assert y.dtype == odt and y.shape == (M, N)
            assert torch.equal(y, narrow[:M]), (N, K, M, has_bias, act, rdt, odt, y2)


def test_wide_skinny_rejects(cuda):
    from ymp import ops, lib
    w = torch.randn(256, 512, device=cuda).bfloat16()
    with pytest.raises(lib.YmpError, match="M <= 64"):
        ops.gemm_skinny_wide(torch.randn(65, 512, device=cuda).bfloat16(), w)
    x8 = torch.randn(8, 512, device=cuda).bfloat16()
    y = ops.gemm_skinny_wide(x8, w, out_dtype=torch.float32)   # M <= 8: gemm_skinny's launch
    y0 = ops.gemm_skinny(x8, w, out_dtype=torch.float32)
    assert torch.equal(y, y0)
    with pytest.raises(AssertionError):   # ymp_gemm_skinny keeps its 8-row limit
        ops.gemm_skinny(torch.randn(9, 512, device=cuda).bfloat16(), w)


# ------------------------------------------------------------------------------------------ tiny fixture model
def _tiny(dev):
    fx = torch.load(os.path.join(GOLD, "tiny_generate.pt"), weights_only=False)
    sd = port.generation_state_dict(fx["vcfg"], fx["gcfg"], fx["Q"], fx["wseed"], fx["pos_gain"], fx["ln_gain"])
    model = build_pretrain(fx["vcfg"], fx["gcfg"], fx["Q"], sd=sd, device=dev, dtype=torch.bfloat16,
                           cls_name="DistributedGPT3_Caption", num_frames=fx["vcfg"]["num_frames"]).eval()
    model.text_decoder.config.tokens_to_generate = fx["n_new"]
    return fx, model


def test_token_step_60_rows_graph_equals_eager(cuda, monkeypatch):
    """The captured single-token step at 60 rows (the 9..64-row skinny kernel) against the same kernels enqueued
    eagerly, bit for bit, through cache reorders."""
    import models.modeling_distributed_gpt3 as M
    fx, model = _tiny(cuda)
    dec, Q, rows = model.text_decoder, fx["Q"], 60
    video, ids, _ = make_inputs(rows, fx["vcfg"], fx["L"], fx["gcfg"]["vocab_size"], 11)
    with torch.no_grad():
        qf = model.visual_prefix(video.to(cuda).bfloat16())[3]
    ids = ids.to(cuda)
    perm = torch.Generator().manual_seed(5)

    def run(n_steps):
        dec.inference_params = ip = M.InferenceParams(rows, fx["L"] + n_steps + Q)
        ip.wide_step = True
        outs = []
        with torch.no_grad():
            out = dec(tokens=ids[:, :5], query_embeds=qf)
            outs.append(out.logits[:, -1].clone())
            for t in range(n_steps):
                tok = out.logits[:, -1].argmax(-1, keepdim=True)
                ip.swap_key_value_dict(torch.randperm(rows, generator=perm).to(cuda))
                out = dec(tokens=tok)
                outs.append(out.logits[:, -1].clone())
        assert ip.cache.token is not None and ip.cache.B == rows
        return torch.stack(outs)

    monkeypatch.setenv("YMP_DECODE_GRAPH", "0")
    perm.manual_seed(5)
    eager = run(6)
    monkeypatch.setenv("YMP_DECODE_GRAPH", "1")
    dec.__dict__.pop("_decode_pool", None)
    perm.manual_seed(5)
    graphed = run(6)
    assert dec.inference_params.cache.token.graph is not None
    assert torch.equal(eager, graphed)


def _prefill(dec, M, ids, qf, beam, plen, Q, batched):
    """Cache rows and first-step logits of the prefill: per clip (beam identical rows) or batched (one row per clip into
    slot c * beam).  Returns ([clips, layers, plen + Q, 3H] cache rows of each clip's first slot, [clips, V] logits)."""
    C = ids.shape[0]
    ML = plen + Q + 2
    rows, logits = [], []
    with torch.no_grad():
        if batched:
            ip = dec.inference_params = M.InferenceParams(C * beam, ML)
            ip.wide_step, ip.prefill_stride = True, beam
            out = dec(tokens=ids[:, :plen], query_embeds=qf)
            st = ip.cache.store.view(ip.cache.g.layers, C, beam, ML, -1)
            return st[:, :, 0, :plen + Q].transpose(0, 1).clone(), out.logits[:, -1].clone()
        for c in range(C):
            ip = dec.inference_params = M.InferenceParams(beam, ML)
            out = dec(tokens=ids[c:c + 1, :plen].repeat(beam, 1), query_embeds=qf[c:c + 1].repeat(beam, 1, 1))
            st = ip.cache.store.view(ip.cache.g.layers, beam, ML, -1)
            assert all(torch.equal(st[:, b, :plen + Q], st[:, 0, :plen + Q]) for b in range(beam))
            rows.append(st[:, 0, :plen + Q].clone())
            logits.append(out.logits[0, -1].clone())
    return torch.stack(rows), torch.stack(logits)


@pytest.mark.parametrize("width", ["tiny", "1.3B", "2.7B"])
def test_batched_prefill_rows_equal_per_clip(cuda, width):
    import models.modeling_distributed_gpt3 as M
    if width == "tiny":
        fx, model = _tiny(cuda)
        vcfg, Q, L, C, beam = fx["vcfg"], fx["Q"], fx["L"], 7, 3
    else:
        vcfg, Q, L, C, beam = port.VCFG_TINY, 128, 20, 12, 5
        model = build_pretrain(vcfg, _gcfg(width, layers=2), Q, device=cuda, dtype=torch.bfloat16,
                               cls_name="DistributedGPT3_Caption", num_frames=vcfg["num_frames"]).eval()
    dec = model.text_decoder
    video, ids, _ = make_inputs(C, vcfg, L, dec.config.vocab_size, 13)
    with torch.no_grad():
        qf = model.visual_prefix(video.to(cuda).bfloat16())[3]
    ids = ids.to(cuda)
    plen = L - 1
    ref_rows, ref_logits = _prefill(dec, M, ids, qf, beam, plen, Q, batched=False)
    rows, logits = _prefill(dec, M, ids, qf, beam, plen, Q, batched=True)
    assert torch.equal(rows, ref_rows)
    assert torch.equal(logits, ref_logits)


# ------------------------------------------------------------------------------------------ model level
def _generate_both(model, video, text, beam):
    """(batched model.generate's list, the per-clip beam searches' AttrDicts, the batched beam searches' AttrDicts,
    the largest row count a decode step ran at)."""
    from ymp import engine
    dec = model.text_decoder
    orig = dec.beam_search
    got = []

    def beam_search(*a, **k):
        out = orig(*a, **dict(k, beam_size=beam))
        got.extend(out if isinstance(out, list) else [out])
        return out
    dec.beam_search = beam_search
    step_rows = []
    run = engine.TokenStep.run

    def counted(self, emb):
        step_rows.append(self.cache.B)
        return run(self, emb)
    engine.TokenStep.run = counted
    try:
        res = model.generate(video, text)
        batched = list(got)
        got.clear()
        eos = dec.config.eod_id
        with torch.no_grad():
            qf = model.visual_prefix(video)[3]
            for i in range(text.input_ids.shape[0]):
                dec.generate(text.input_ids[i:i + 1], query_embeds=qf[i:i + 1], termination_id=eos, do_sample=False,
                             prompt_length=text.attention_mask.sum(-1)[i] - 1)
    finally:
        engine.TokenStep.run = run
        del dec.beam_search
    return res, got, batched, max(step_rows)


def _check(res, per, batched, B):
    assert len(res) == len(per) == len(batched) == B
    for i in range(B):
        assert torch.equal(batched[i].sequences, per[i].sequences), i
        assert torch.equal(batched[i].scores, per[i].scores), i
        assert res[i].device.type == "cpu" and torch.equal(res[i], per[i].sequences.cpu())


def test_caption_generate_equals_per_clip_tiny(cuda):
    """25 clips at beam 3: chunks of 21 and 4 clips; the fixture's weights make beams finish early."""
    import models.modeling_distributed_gpt3 as M
    fx, model = _tiny(cuda)
    B = 25
    video, ids, _ = make_inputs(B, fx["vcfg"], fx["L"], fx["gcfg"]["vocab_size"], 17)
    ids[:2] = fx["ids"]
    att = torch.ones_like(ids)
    att[:, 6:] = 0   # one prompt length (5) for every clip
    text = M.BatchEncoding(dict(input_ids=ids.to(cuda), attention_mask=att.to(cuda)))
    res, per, batched, rows = _generate_both(model, video.to(cuda).bfloat16(), text, 3)
    _check(res, per, batched, B)
    assert rows == 63
    assert any((s.sequences == fx["eod"]).any() for s in per)


@pytest.mark.parametrize("width", ["1.3B", "2.7B"])
def test_caption_generate_equals_per_clip_wide(cuda, width):
    """2-layer decoders at the 1.3B / 2.7B widths, 13 clips at beam 5: a 60-row chunk and a 5-row one."""
    import models.modeling_distributed_gpt3 as M
    vcfg, Q, L, B = port.VCFG_TINY, 128, 20, 13
    model = build_pretrain(vcfg, _gcfg(width, layers=2), Q, device=cuda, dtype=torch.bfloat16,
                           cls_name="DistributedGPT3_Caption", num_frames=vcfg["num_frames"]).eval()
    model.text_decoder.config.tokens_to_generate = 12
    video, ids, _ = make_inputs(B, vcfg, L, model.text_decoder.config.vocab_size, 19)
    text = M.BatchEncoding(dict(input_ids=ids.to(cuda), attention_mask=torch.ones_like(ids).to(cuda)))
    res, per, batched, rows = _generate_both(model, video.to(cuda).bfloat16(), text, 5)
    _check(res, per, batched, B)
    assert rows == 60


# ------------------------------------------------------------------------------------------ no-grad visual prefix
def test_visual_prefix_no_grad_keeps_no_activations(cuda):
    """ViT-B width (12 blocks, 768), 4 clips x 8 frames: under torch.no_grad() the outputs equal the grad-mode forward
    bit for bit, and the peak grows by less than two blocks' counted activations (52 D bytes per token row)."""
    vcfg = dict(port.VCFG_CLIP_B16, num_frames=8)
    model = build_pretrain(vcfg, port.GCFG_TINY, 8, device=cuda, dtype=torch.bfloat16, cls_name="DistributedGPT3_Caption",
                           num_frames=8).eval()
    video, _, _ = make_inputs(4, vcfg, 8, port.GCFG_TINY["vocab_size"], 23)
    video = video.to(cuda).bfloat16()
    with torch.enable_grad():
        ref = [t.detach().clone() if torch.is_tensor(t) else t for t in model.visual_prefix(video)]
    with torch.no_grad():
        model.visual_prefix(video)   # warm-up: lazily built tables are not activations
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        out = model.visual_prefix(video)
        torch.cuda.synchronize()
        growth = torch.cuda.max_memory_allocated() - base
    for a, b in zip(ref, out):
        if torch.is_tensor(a):
            assert torch.equal(a, b)
    D = vcfg["embed_dim"]
    rows = 4 * (vcfg["num_frames"] * (vcfg["img_size"] // vcfg["patch_size"]) ** 2 + 1)
    block = 52 * D * rows
    print("no-grad visual prefix peak growth", growth, "one block's activations", block)
    assert growth < 2 * block, (growth, block)
