"""GPU: the downstream task models (SURVEY.md section 8a rows a20-a23) on the H100 kernels against the
oracle composed from the same reference-pinned primitives (oracle/port.py)."""
import os

import pytest
import torch

from oracle import port
from oracle.make_golden import make_inputs
from helpers import build_pretrain

pytestmark = pytest.mark.gpu
VC, GC, Q = port.VCFG_TINY, port.GCFG_TINY, 8
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _rel(a, b):
    return ((a.float().cpu() - b.float().cpu()).abs().max() / (b.float().abs().max() + 1e-12)).item()


def _enc(dev, **kw):
    import models.modeling_distributed_gpt3 as G
    return G.BatchEncoding({k: v.to(dev) for k, v in kw.items()})


def _sd(extra=None, seed=21):
    sd = port.init_state_dict(VC, GC, Q, seed=seed, randomize=True)
    g = torch.Generator().manual_seed(seed + 1)
    for k, shape in (extra or {}).items():
        sd[k] = 0.05 * torch.randn(shape, generator=g)
    return sd


def test_cls_train_and_eval(cuda):
    sd = _sd({"cls_head.0.weight": (128, 128), "cls_head.0.bias": (128,), "cls_head.2.weight": (5, 128), "cls_head.2.bias": (5,)})
    m = build_pretrain(VC, GC, Q, sd=sd, device=cuda, dtype=torch.bfloat16, cls_name="DistributedGPT3_Cls",
                       num_frames=VC["num_frames"], use_cls=True, num_classes=5)
    B, L, ncls = 2, 8, 3
    video, ids, att = make_inputs(B, VC, L, GC["vocab_size"], 31)
    pl = torch.tensor([2, 3])
    rsd = {k: v.bfloat16().float() for k, v in sd.items()}
    _, _, _, qf = port.visual_prefix(video.bfloat16().float(), rsd, VC)
    # ---- training branch: generation loss with the prompt masked + cls_head CE on the prompt pass
    _, pids, patt = make_inputs(B, VC, L, GC["vocab_size"], 32)
    labels = torch.tensor([1, 4])
    loss_cap, loss_cls = m(video.to(cuda).bfloat16(), _enc(cuda, input_ids=ids, attention_mask=att, prompt_lengths=pl),
                           _enc(cuda, input_ids=pids, attention_mask=patt), labels.to(cuda), train=True)
    ref = port.prefix_decoder_pass(qf, ids, att, pl, rsd, GC)
    assert abs(loss_cap.item() - ref["loss"].item()) < 1e-2 * ref["loss"].item()
    refp = port.prefix_decoder_pass(qf, pids, patt, None, rsd, GC)
    pooled = refp["hidden"][torch.arange(B), Q + patt.sum(-1) - 1]
    h = torch.relu(torch.nn.functional.linear(pooled, rsd["cls_head.0.weight"], rsd["cls_head.0.bias"]))
    ref_cls = torch.nn.functional.cross_entropy(torch.nn.functional.linear(h, rsd["cls_head.2.weight"], rsd["cls_head.2.bias"]), labels)
    assert abs(loss_cls.item() - ref_cls.item()) < 3e-2 * ref_cls.item()
    (loss_cap + loss_cls).backward()
    assert m.cls_head[0].weight.grad is not None and m.visual_fc.weight.grad is not None
    # ---- eval branch: num_cls prompts per video
    _, cids, catt = make_inputs(B * ncls, VC, L, GC["vocab_size"], 33)
    cpl = torch.randint(1, 4, (B * ncls,), generator=torch.Generator().manual_seed(5))
    with torch.no_grad():
        gen, cls_logits = m(video.to(cuda).bfloat16(), _enc(cuda, input_ids=cids, attention_mask=catt, prompt_lengths=cpl),
                            _enc(cuda, input_ids=pids, attention_mask=patt), train=False)
    ref_gen = port.cls_eval_scores(qf, cids, catt, cpl, rsd, GC, ncls)
    assert gen.shape == (B, ncls) and cls_logits.shape == (B, 5)
    assert _rel(gen, ref_gen) < 3e-2


def test_retrieval_features_and_loss(cuda):
    sd = _sd({"vision_proj.weight": (32, 192), "vision_proj.bias": (32,), "text_proj.weight": (32, 128),
              "text_proj.bias": (32,)})
    sd["temp"] = torch.tensor(0.07)
    m = build_pretrain(VC, GC, Q, sd=sd, device=cuda, dtype=torch.bfloat16, cls_name="DistributedGPT3_Retrieval",
                       num_frames=VC["num_frames"], contrastive_embed_dim=32)
    B, L = 3, 8
    video, ids, att = make_inputs(B, VC, L, GC["vocab_size"], 41)
    idx = torch.tensor([7, 9, 7])
    rsd = {k: v.bfloat16().float() for k, v in sd.items()}
    rv, rt = port.retrieval_features(video.bfloat16().float(), ids, att, rsd, VC, GC)
    text = _enc(cuda, input_ids=ids, attention_mask=att)
    with torch.no_grad():
        v = m.extract_vision_feature(video.to(cuda).bfloat16())
        t = m.extract_text_feature(text)
    assert _rel(v, rv) < 2e-2 and _rel(t, rt) < 2e-2
    loss = m(video.to(cuda).bfloat16(), text, idx.to(cuda))
    ref = port.retrieval_loss(rv, rt, idx, 0.07)
    assert abs(loss.item() - ref.item()) < 3e-2 * abs(ref.item())
    loss.backward()
    assert m.vision_proj.weight.grad is not None and m.visual_encoder.cls_token.grad is not None
    assert all(p.grad is None for p in m.text_decoder.parameters())


def test_retrieval_cls_shapes_and_negatives(cuda):
    sd = _sd({"cls_head.0.weight": (128, 128), "cls_head.0.bias": (128,), "cls_head.2.weight": (2, 128), "cls_head.2.bias": (2,)})
    m = build_pretrain(VC, GC, Q, sd=sd, device=cuda, dtype=torch.bfloat16, cls_name="DistributedGPT3_Retrieval_Cls",
                       num_frames=VC["num_frames"], use_cls=True)
    B, L = 2, 8
    video, _, _ = make_inputs(B, VC, L, GC["vocab_size"], 51)
    _, ids, att = make_inputs(2 * B, VC, L, GC["vocab_size"], 52)       # positives then negatives
    pl = torch.tensor([2, 2, 3, 1])
    neg = torch.tensor([1, 0])
    labels = torch.tensor([1, 1, 0, 0])
    text = _enc(cuda, input_ids=ids, attention_mask=att, prompt_lengths=pl)
    prompt = _enc(cuda, input_ids=ids, attention_mask=att)
    lc, lcls = m(video.to(cuda).bfloat16(), text, prompt, neg.to(cuda), labels.to(cuda), train=True)
    rsd = {k: v.bfloat16().float() for k, v in sd.items()}
    _, _, _, qf = port.visual_prefix(video.bfloat16().float(), rsd, VC)
    ref = port.prefix_decoder_pass(torch.cat([qf, qf[neg]], 0), ids, att, pl, rsd, GC)
    assert abs(lc.item() - ref["loss"].item()) < 1e-2 * ref["loss"].item()
    assert torch.isfinite(lcls)
    with torch.no_grad():
        gen, cls = m(video.to(cuda).bfloat16(), text, prompt, train=False)
    assert gen.shape == (B, 2) and cls.shape == (B, 2)
    ref_eval = port.prefix_decoder_pass(qf.repeat_interleave(2, 0), ids, att, pl, rsd, GC)
    ref_gen = (-(ref_eval["losses"] * ref_eval["loss_mask"]).sum(-1)).view(B, 2)
    assert _rel(gen, ref_gen) < 2e-2


def test_downstream_models_match_reference_fixture(cuda):
    """The four downstream task models on the H100 kernels against the UNMODIFIED reference's outputs
    (tests/golden/tiny_downstream.pt: same seeded weights and inputs, reference run in fp32 on CPU)."""
    import os
    fx = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "tiny_downstream.pt"), weights_only=False)
    assert fx["Q"] == Q and fx["vcfg"] == VC and fx["gcfg"] == GC
    V = GC["vocab_size"]

    def model(cls_name, extra, **cfg):
        sd = port.init_state_dict(VC, GC, Q, seed=fx["wseed"], randomize=True)
        sd.update(extra)
        return build_pretrain(VC, GC, Q, sd=sd, device=cuda, dtype=torch.bfloat16, cls_name=cls_name, num_frames=VC["num_frames"], **cfg)

    def close(a, b, tol):
        b = torch.as_tensor(b)
        return ((a.detach().float().cpu() - b.float()).abs().max() <= tol * (b.float().abs().max() + 1e-12)).item()

    with torch.no_grad():
        c = fx["cls"]
        m = model("DistributedGPT3_Cls", c["head"], use_cls=True, num_classes=5)
        video, ids, att = make_inputs(2, VC, 8, V, c["seeds"][0])
        _, pids, patt = make_inputs(2, VC, 8, V, c["seeds"][1])
        vd = video.to(cuda).bfloat16()
        lc, lk = m(vd, _enc(cuda, input_ids=ids, attention_mask=att, prompt_lengths=c["prompt_lengths"]),
                   _enc(cuda, input_ids=pids, attention_mask=patt), c["labels"].to(cuda), train=True)
        assert close(lc, c["loss_caption"], 1e-2) and close(lk, c["loss_cls"], 3e-2)
        _, cids, catt = make_inputs(2 * c["ncls"], VC, 8, V, c["seeds"][2])
        gen, cl = m(vd, _enc(cuda, input_ids=cids, attention_mask=catt, prompt_lengths=c["eval_prompt_lengths"]),
                    _enc(cuda, input_ids=pids, attention_mask=patt), train=False)
        assert close(gen, c["eval_generation"], 3e-2) and close(cl, c["eval_cls_logits"], 3e-2)
        m = model("DistributedGPT3_Caption", {})
        loss = m(vd, _enc(cuda, input_ids=ids, attention_mask=att, prompt_lengths=fx["caption"]["prompt_lengths"]))
        assert close(loss, fx["caption"]["loss"], 1e-2)
        r = fx["retrieval"]
        m = model("DistributedGPT3_Retrieval", dict(r["proj"], temp=torch.tensor(0.07)), contrastive_embed_dim=32)
        video3, ids3, att3 = make_inputs(3, VC, 8, V, r["seed"])
        text3 = _enc(cuda, input_ids=ids3, attention_mask=att3)
        assert close(m.extract_vision_feature(video3.to(cuda).bfloat16()), r["vision_feats"], 2e-2)
        assert close(m.extract_text_feature(text3), r["text_feats"], 2e-2)
        assert close(m(video3.to(cuda).bfloat16(), text3, r["idx"].to(cuda)), r["loss"], 3e-2)
        rc = fx["retrieval_cls"]
        m = model("DistributedGPT3_Retrieval_Cls", rc["head"], use_cls=True, num_classes=2)
        videoB, _, _ = make_inputs(2, VC, 8, V, rc["seeds"][0])
        _, ids4, att4 = make_inputs(4, VC, 8, V, rc["seeds"][1])
        text4 = _enc(cuda, input_ids=ids4, attention_mask=att4, prompt_lengths=rc["prompt_lengths"])
        prompt4 = _enc(cuda, input_ids=ids4, attention_mask=att4)
        lc4, lk4 = m(videoB.to(cuda).bfloat16(), text4, prompt4, rc["negative_indices"].to(cuda), rc["labels"].to(cuda), train=True)
        assert close(lc4, rc["loss_caption"], 1e-2) and close(lk4, rc["loss_cls"], 3e-2)
        gen4, cls4 = m(videoB.to(cuda).bfloat16(), text4, prompt4, train=False)
        assert close(gen4, rc["eval_generation"], 2e-2) and close(cls4, rc["eval_cls"], 3e-2)
        pc = fx["pretrain_contrastive"]
        m = model("DistributedGPT3_Pretrain", dict(pc["proj"], temp=torch.tensor(0.07)), use_contrastive=True, contrastive_embed_dim=32)
        lcap, lcon = m(video3.to(cuda).bfloat16(), text3)
        assert close(lcap, pc["loss_caption"], 1e-2) and close(lcon, pc["loss_contrastive"], 3e-2)


@pytest.mark.skipif(os.environ.get("YMP_SKIP_FULL", "0") == "1", reason="full-size parity disabled")
def test_full_2p7b_caption_matches_reference_fixture(cuda):
    """BASELINE config-4 at its real dims (GPT-3 2.7B: 32 layers x 2560, 32 heads x 80; 16 frames; text 256 ->
    S = 384; B = 1): DistributedGPT3_Caption forward + backward against the UNMODIFIED reference's fp32 outputs
    (tests/golden/full_2p7b_caption_T16_B1.pt, oracle/make_golden.py --caption27b).  Exercises head_dim 80,
    key ranges > 256 and T = 16 through the model."""
    from oracle.make_golden import make_inputs
    fx = torch.load(os.path.join(GOLD, "full_2p7b_caption_T16_B1.pt"), weights_only=False)
    torch.set_num_threads(os.cpu_count())
    sd = port.init_state_dict(fx["vcfg"], fx["gcfg"], fx["Q"], seed=fx["wseed"], randomize=False)
    cs = float(sum(v.double().abs().sum() for v in sd.values()))
    assert abs(cs - fx["sd_checksum"]) <= 1e-9 * fx["sd_checksum"]
    model = build_pretrain(fx["vcfg"], fx["gcfg"], fx["Q"], sd=sd, device=cuda, dtype=torch.bfloat16,
                           cls_name="DistributedGPT3_Caption", num_frames=fx["vcfg"]["num_frames"])
    del sd
    video, ids, att = make_inputs(fx["B"], fx["vcfg"], fx["L"], fx["gcfg"]["vocab_size"], fx["iseed"])
    v = video.to(cuda).bfloat16()
    import models.modeling_distributed_gpt3 as G
    import models.distributed_gpt3 as D
    text = G.BatchEncoding(dict(input_ids=ids.to(cuda), attention_mask=att.to(cuda), prompt_lengths=fx["prompt_lengths"].to(cuda)))
    with torch.no_grad():
        _, image_embeds, _, qf = model.visual_prefix(v)
        tla = text.attention_mask[:, 1:].clone()
        for i, ln in enumerate(fx["prompt_lengths"].tolist()):
            tla[i, :ln] = 0
        targets, loss_mask = D.build_targets(text.input_ids, tla, fx["Q"])
        emb = model.text_decoder.dist_model.language_model.embedding.word_embeddings(text.input_ids)
        out = model.text_decoder(input_embeds=torch.cat([qf, emb.to(qf.dtype)], 1), loss_mask=loss_mask, labels=targets)
    idx = fx["logit_idx"]
    got = out.logits[idx[:, 0], idx[:, 1], idx[:, 2]].float().cpu()
    ref_vals = fx["logit_vals"]
    err_l2 = ((got - ref_vals).norm() / ref_vals.norm()).item()
    err_max = (got - ref_vals).abs().max().item() / fx["logits_absmax"].item()
    print("2.7B caption sampled logits: rel L2 err", err_l2, "max err / max|logit|", err_max, "loss", out.loss.item(),
          "ref", fx["loss"].item())
    assert err_l2 < 1e-2 and err_max < 2e-2
    assert abs(out.loss.item() - fx["loss"].item()) < 5e-3 * fx["loss"].item()
    assert _rel(out.losses, fx["losses"]) < 2e-2
    assert _rel(image_embeds.float().norm(dim=-1), fx["image_embeds_norm"]) < 1e-2
    assert _rel(out.last_hidden_state.float().norm(dim=-1), fx["hidden_norm"]) < 1e-2
    del out
    loss = model(v, text)
    loss.backward()
    assert abs(loss.item() - fx["loss"].item()) < 5e-3 * fx["loss"].item()
    params = dict(model.named_parameters())
    for k, (stride, vals) in fx["grads"].items():
        g = params[k].grad.float().cpu().flatten()[::stride]
        if vals.abs().max() > 1e-9:
            assert _rel(g, vals) < 0.1, k
    bad = []
    for k, n in fx["grad_norms"].items():
        gn = params[k].grad.float().norm().item()
        if n.item() > 1e-9 and abs(gn - n.item()) > 0.1 * n.item():
            bad.append((k, gn, n.item()))
    assert not bad, bad[:5]


def test_pretrain_image_eva_matches_reference_fixture(cuda):
    """SURVEY 8f N3: DistributedGPT3_Pretrain_Image with the EVA encoder (head_dim 88, 14 x 14 patches, conv bias)
    forward + backward against the unmodified reference's fp32 outputs (tests/golden/tiny_pretrain_image.pt)."""
    from helpers import build_pretrain_image
    fx = torch.load(os.path.join(GOLD, "tiny_pretrain_image.pt"), weights_only=False)
    sd = port.eva_state_dict(fx["ecfg"], fx["gcfg"], fx["Q"], seed=fx["wseed"])
    m = build_pretrain_image(fx["ecfg"], fx["gcfg"], fx["Q"], sd=sd, device=cuda, dtype=torch.bfloat16)
    img = fx["image"].to(cuda).bfloat16()
    with torch.no_grad():
        _, emb = m.visual_encoder(img)
    assert _rel(emb, fx["image_embeds"]) < 2e-2
    loss, zero = m(img, _enc(cuda, input_ids=fx["ids"], attention_mask=fx["att"]))
    assert float(zero) == 0.0
    assert abs(loss.item() - fx["loss"].item()) < 1e-2 * abs(fx["loss"].item())
    loss.backward()
    params = dict(m.named_parameters())
    for k, (stride, vals) in fx["grads"].items():
        g = params[k].grad.float().cpu().flatten()[::stride]
        if vals.abs().max() > 1e-7:
            assert _rel(g, vals) < 8e-2, k
    bad = [(k, params[k].grad.float().norm().item(), n.item()) for k, n in fx["grad_norms"].items()
           if n.item() > 1e-7 and abs(params[k].grad.float().norm().item() - n.item()) > 0.1 * n.item()]
    assert not bad, bad[:5]
    assert all(p.grad is None for k, p in params.items() if k.startswith("text_decoder."))
