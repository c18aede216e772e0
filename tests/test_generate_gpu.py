"""GPU: KV-cache decoding and generation (SURVEY.md 8f N2) on the H100 kernels against the reference's golden
sequences (tests/golden/tiny_generate.pt) and the oracle's teacher-forced log-probabilities."""
import os

import pytest
import torch

from oracle import port
from oracle.make_golden import make_inputs
from helpers import build_pretrain

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _setup(dev):
    fx = torch.load(os.path.join(GOLD, "tiny_generate.pt"), weights_only=False)
    sd = port.generation_state_dict(fx["vcfg"], fx["gcfg"], fx["Q"], fx["wseed"], fx["pos_gain"], fx["ln_gain"])
    model = build_pretrain(fx["vcfg"], fx["gcfg"], fx["Q"], sd=sd, device=dev, dtype=torch.bfloat16,
                           cls_name="DistributedGPT3_Caption", num_frames=fx["vcfg"]["num_frames"]).eval()
    video, _, _ = make_inputs(fx["B"], fx["vcfg"], fx["L"], fx["gcfg"]["vocab_size"], fx["iseed"])
    assert abs(float(video.double().abs().sum()) - fx["video_checksum"]) < 1e-6 * fx["video_checksum"]
    rsd = {k: v.bfloat16().float() for k, v in sd.items()}  # oracle on the bf16-rounded weights
    return fx, model, video, rsd


def test_kv_cache_logits_match_oracle_teacher_forced(cuda):
    """Prefill [prefix | prompt] then one golden token at a time: every step's next-token log-probs against the
    oracle's full recompute (fp32, same bf16-rounded weights)."""
    import models.modeling_distributed_gpt3 as M
    fx, model, video, rsd = _setup(cuda)
    dec, Q = model.text_decoder, fx["Q"]
    with torch.no_grad():
        qf = model.visual_prefix(video.to(cuda).bfloat16())[3]
        qf_ref = port.visual_prefix(video.bfloat16().float(), rsd, fx["vcfg"])[3]
        worst = 0.0
        for i in range(fx["B"]):
            seq, plen = fx["greedy"][i], int(fx["prompt_length"][i])
            dec.inference_params = M.InferenceParams(1, seq.numel() + Q)
            prev = 0
            for t in range(plen, seq.numel()):
                out = dec(tokens=seq[None, prev:t].to(cuda), query_embeds=qf[i:i + 1] if prev == 0 else None)
                lp = torch.log_softmax(out.logits[0, -1].float(), -1).cpu()
                ref = torch.log_softmax(port.next_token_logits(qf_ref[i:i + 1], seq[None, :t], rsd, fx["gcfg"])[0], -1)
                err = ((lp - ref).norm() / ref.norm()).item()
                worst = max(worst, err)
                assert err < 3e-2, (i, t, err)
                prev = t
            assert dec.inference_params.sequence_len_offset == seq.numel() - 1 + Q
    print("worst rel-L2 log-prob error", worst)


def _oracle_score(seq, plen, qf_ref, rsd, gcfg, eod):
    """sum of teacher-forced log-probs of the generated tokens up to and including the first stop token,
    divided by the (padded) row length - the quantity BeamHypotheses ranks by."""
    total = 0.0
    for t in range(plen, seq.numel()):
        lp = torch.log_softmax(port.next_token_logits(qf_ref, seq[None, :t], rsd, gcfg)[0], -1)
        total += float(lp[seq[t]])
        if int(seq[t]) == eod:
            break
    return total / seq.numel()


def test_caption_generate_beam_search(cuda):
    import models.modeling_distributed_gpt3 as M
    fx, model, video, rsd = _setup(cuda)
    model.text_decoder.config.tokens_to_generate = fx["n_new"]

    class _Tok:  # generate() reads tokenizer.tokenizer.eos
        class tokenizer:
            eos = fx["eod"]
    model.tokenizer = _Tok()
    text = M.BatchEncoding(dict(input_ids=fx["ids"].to(cuda), attention_mask=fx["att"].to(cuda)))
    beam = fx["beam_size"]
    orig = model.text_decoder.beam_search
    model.text_decoder.beam_search = lambda *a, **k: orig(*a, **dict(k, beam_size=beam))
    res = model.generate(video.to(cuda).bfloat16(), text)
    with torch.no_grad():
        qf_ref = port.visual_prefix(video.bfloat16().float(), rsd, fx["vcfg"])[3]
    for i in range(fx["B"]):
        seq = res[i][0]
        assert seq.shape == fx["beam_sequences"][i][0].shape
        if torch.equal(seq, fx["beam_sequences"][i][0]):
            continue
        # a bf16 run may pick another hypothesis when two are nearly tied: it must be (almost) as good
        got = _oracle_score(seq, int(fx["prompt_length"][i]), qf_ref[i:i + 1], rsd, fx["gcfg"], fx["eod"])
        assert got > float(fx["beam_scores"][i][0]) - 0.03, (i, seq.tolist(), got, fx["beam_scores"][i])


def test_greedy_sampling_matches_reference(cuda):
    fx, model, video, rsd = _setup(cuda)
    dec = model.text_decoder
    with torch.no_grad():
        qf = model.visual_prefix(video.to(cuda).bfloat16())[3]
        out = dec.generate(fx["ids"].to(cuda), query_embeds=qf, termination_id=fx["eod"], do_sample=True,
                           prompt_length=fx["prompt_length"].to(cuda)).cpu()
    ref = fx["greedy"]
    margins = {(s["sample"], s["pos"]): s["margin"] for s in fx["steps"]}
    for i in range(fx["B"]):
        n = min(out.shape[1], ref.shape[1])
        diff = (out[i, :n] != ref[i, :n]).nonzero()
        if diff.numel():
            t = int(diff[0])
            assert margins.get((i, t), 0.0) < 0.1, (i, t, out[i].tolist(), ref[i].tolist(), margins.get((i, t)))
    assert out.shape == ref.shape


def test_token_step_graph_equals_eager_and_survives_reuse(cuda, monkeypatch):
    """The captured single-token step (skinny GEMMs, device-side cache length) against the same kernels enqueued
    eagerly, bit for bit, over a beam-shaped decode with cache reordering; then a second generate-style call that
    reuses the pooled cache and its graph."""
    import models.modeling_distributed_gpt3 as M
    from ymp import lib
    fx, model, video, _ = _setup(cuda)
    dec, Q, beam = model.text_decoder, fx["Q"], 3
    with torch.no_grad():
        qf = model.visual_prefix(video.to(cuda).bfloat16())[3]

    def run(sample, n_steps):
        seq, plen = fx["greedy"][sample], int(fx["prompt_length"][sample])
        dec.inference_params = M.InferenceParams(beam, plen + n_steps + 1 + Q)
        outs = []
        with torch.no_grad():
            out = dec(tokens=seq[None, :plen].repeat(beam, 1).to(cuda), query_embeds=qf[sample:sample + 1].repeat(beam, 1, 1))
            outs.append(out.logits[:, -1].clone())
            for t in range(n_steps):
                tok = out.logits[:, -1].argmax(-1, keepdim=True)
                tok[1] = (tok[1] + 1 + t) % fx["gcfg"]["vocab_size"]   # make the beams differ
                dec.inference_params.swap_key_value_dict([1, 0, 2] if t % 2 else [0, 2, 1])
                out = dec(tokens=tok)
                outs.append(out.logits[:, -1].clone())
        return torch.stack(outs)

    monkeypatch.setenv("YMP_DECODE_GRAPH", "0")
    eager = run(0, 6)
    monkeypatch.setenv("YMP_DECODE_GRAPH", "1")
    dec.__dict__.pop("_decode_pool", None)
    n0 = lib.launch_count()
    graphed = run(0, 6)
    assert torch.equal(eager, graphed)
    ts = dec.inference_params.cache.token
    assert ts is not None and ts.graph is not None
    cache = dec.inference_params.cache
    again = run(0, 6)                      # pooled cache + graph reused after reset()
    assert dec.inference_params.cache is cache and cache.token is ts
    assert torch.equal(eager, again)
    assert lib.launch_count() > n0
