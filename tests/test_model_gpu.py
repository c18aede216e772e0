"""GPU parity of the whole hot path: the drop-in models (bf16, H100 kernels) against
(a) the golden fixtures = outputs of the UNMODIFIED reference (fp32), and
(b) the oracle (oracle/port.py, fp32 on CPU) fed the same bf16-rounded weights.
Tolerance: north_star asks forward logits within 1e-2 rel of the reference; measured against the
max-magnitude of each tensor (bf16 has 8 mantissa bits; everything else is fp32-accumulated)."""
import os

import pytest
import torch

from oracle import port
from oracle.make_golden import make_inputs
from helpers import build_pretrain

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _rel(a, b):
    return ((a.float().cpu() - b.float().cpu()).abs().max() / (b.float().abs().max() + 1e-12)).item()


def _text(ids, att, dev):
    import models.modeling_distributed_gpt3 as G
    return G.BatchEncoding(dict(input_ids=ids.to(dev), attention_mask=att.to(dev)))


def _run_fused(fx, dev):
    sd = port.init_state_dict(fx["vcfg"], fx["gcfg"], fx["Q"], seed=fx["wseed"], randomize=fx["randomize"])
    model = build_pretrain(fx["vcfg"], fx["gcfg"], fx["Q"], sd=sd, device=dev, dtype=torch.bfloat16)
    video, ids, att = make_inputs(fx["B"], fx["vcfg"], fx["L"], fx["gcfg"]["vocab_size"], fx["iseed"])
    loss, lc = model(video.to(dev).bfloat16(), _text(ids, att, dev))
    loss.backward()
    return model, sd, (video, ids, att), loss


@pytest.mark.parametrize("name", ["tiny_pretrain", "tiny_pretrain_refinit"])
def test_fused_pretrain_matches_reference_fixture(cuda, name):
    fx = torch.load(os.path.join(GOLD, name + ".pt"), weights_only=False)
    model, sd, (video, ids, att), loss = _run_fused(fx, cuda)
    assert abs(loss.item() - fx["loss"].item()) < 1e-2 * abs(fx["loss"].item())
    Q = fx["Q"]  # losses of the visual-prefix positions are never used (loss_mask == 0 there) and not computed
    assert _rel(model.last_losses[:, Q:-1], fx["losses"][:, Q:]) < 2e-2
    assert float(model.last_losses[:, :Q].abs().max()) == 0.0
    # oracle on the bf16-rounded weights/inputs (isolates kernel error from weight rounding)
    train = set(port.trainable_keys(sd))
    psd = {k: v.bfloat16().float().requires_grad_(k in train) for k, v in sd.items()}
    res = port.pretrain_forward(video.bfloat16().float(), ids, att, psd, fx["vcfg"], fx["gcfg"], return_all=True)
    res["loss"].backward()
    assert abs(loss.item() - res["loss"].item()) < 5e-3 * abs(res["loss"].item())
    assert _rel(model.last_losses[:, Q:], res["losses"][:, Q:]) < 2e-2
    worst = 0.0
    for k, p in model.named_parameters():
        if k.startswith("text_decoder."):
            assert p.grad is None, k          # frozen decoder: no grads (distributed_gpt3.py:91-93)
            continue
        assert p.grad is not None, k
        g_ref = psd[k].grad
        denom = g_ref.abs().max().item()
        if denom < 1e-7:
            continue
        err = _rel(p.grad, g_ref)
        worst = max(worst, err)
        assert err < 6e-2, (k, err)
    # sampled grads of the fp32 reference itself
    for k, (stride, vals) in fx["grads"].items():
        g = dict(model.named_parameters())[k].grad.float().cpu().flatten()[::stride]
        if vals.abs().max() > 1e-7:
            assert _rel(g, vals) < 8e-2, k
    print(f"[{name}] worst grad rel err vs oracle: {worst:.3e}")


def test_component_path_equals_fused_path(cuda):
    """DistributedGPT3_Caption.forward (VitFn + AttnPoolFn + LinearFn + GptFn through torch autograd)
    must give the same loss and grads as the fused PretrainFn."""
    fx = torch.load(os.path.join(GOLD, "tiny_pretrain.pt"), weights_only=False)
    model, sd, (video, ids, att), loss = _run_fused(fx, cuda)
    cap = build_pretrain(fx["vcfg"], fx["gcfg"], fx["Q"], sd=sd, device=cuda, dtype=torch.bfloat16,
                         cls_name="DistributedGPT3_Caption", num_frames=fx["vcfg"]["num_frames"])
    loss2 = cap(video.to(cuda).bfloat16(), _text(ids, att, cuda))
    loss2.backward()
    assert abs(loss.item() - loss2.item()) < 2e-3 * abs(loss.item())
    pf = dict(model.named_parameters())
    for k, p in cap.named_parameters():
        if p.grad is None:
            assert pf[k].grad is None, k
            continue
        if pf[k].grad.abs().max() > 1e-7:
            assert _rel(p.grad, pf[k].grad) < 3e-2, k


def test_decoder_api_outputs(cuda):
    """DistributedGPT3.forward contract: logits [B,S,V], losses [B,S-1], last_hidden_state [B,S,H]."""
    fx = torch.load(os.path.join(GOLD, "tiny_pretrain.pt"), weights_only=False)
    sd = port.init_state_dict(fx["vcfg"], fx["gcfg"], fx["Q"], seed=fx["wseed"], randomize=True)
    model = build_pretrain(fx["vcfg"], fx["gcfg"], fx["Q"], sd=sd, device=cuda, dtype=torch.bfloat16)
    video, ids, att = make_inputs(fx["B"], fx["vcfg"], fx["L"], fx["gcfg"]["vocab_size"], fx["iseed"])
    with torch.no_grad():
        _, image_embeds, image_query, qf = model.visual_prefix(video.to(cuda).bfloat16())
        emb = model.text_decoder.dist_model.language_model.embedding.word_embeddings(ids.to(cuda))
        out = model.text_decoder(input_embeds=torch.cat([qf, emb], 1), loss_mask=fx["loss_mask"].to(cuda),
                                 labels=fx["targets"].to(cuda))
    assert _rel(image_embeds, fx["image_embeds"]) < 2e-2
    assert _rel(qf, fx["query_features"]) < 2e-2
    assert _rel(out.logits, fx["logits"]) < 1e-2          # north_star: forward logits within 1e-2 rel
    assert _rel(out.losses, fx["losses"]) < 2e-2
    assert _rel(out.last_hidden_state, fx["hidden"]) < 2e-2
    assert abs(out.loss.item() - fx["loss"].item()) < 1e-2 * fx["loss"].item()


@pytest.mark.skipif(os.environ.get("YMP_SKIP_FULL", "0") == "1", reason="full-size parity disabled")
def test_full_1p3b_forward_backward_vs_reference_fixture(cuda):
    """Real config (1.3B, T=8, Q=128, L=128, B=1): loss, sampled logits, hidden/embedding norms and a
    few gradients against the reference's fp32 outputs."""
    fx = torch.load(os.path.join(GOLD, "full_1p3b_T8_B1.pt"), weights_only=False)
    torch.set_num_threads(os.cpu_count())
    sd = port.init_state_dict(fx["vcfg"], fx["gcfg"], fx["Q"], seed=fx["wseed"], randomize=False)
    cs = float(sum(v.double().abs().sum() for v in sd.values()))
    assert abs(cs - fx["sd_checksum"]) <= 1e-9 * fx["sd_checksum"]
    model = build_pretrain(fx["vcfg"], fx["gcfg"], fx["Q"], sd=sd, device=cuda, dtype=torch.bfloat16)
    del sd
    video, ids, att = make_inputs(fx["B"], fx["vcfg"], fx["L"], fx["gcfg"]["vocab_size"], fx["iseed"])
    v = video.to(cuda).bfloat16()
    with torch.no_grad():
        _, image_embeds, _, qf = model.visual_prefix(v)
        emb = model.text_decoder.dist_model.language_model.embedding.word_embeddings(ids.to(cuda))
        out = model.text_decoder(input_embeds=torch.cat([qf, emb], 1), loss_mask=fx["loss_mask"].to(cuda),
                                 labels=fx["targets"].to(cuda))
    idx = fx["logit_idx"]
    got = out.logits[idx[:, 0], idx[:, 1], idx[:, 2]].float().cpu()
    ref_vals = fx["logit_vals"]
    err_max = (got - ref_vals).abs().max().item() / fx["logits_absmax"].item()
    err_l2 = ((got - ref_vals).norm() / ref_vals.norm()).item()
    print("full-config sampled logits: rel L2 err", err_l2, "max err / max|logit|", err_max,
          "loss", out.loss.item(), "ref", fx["loss"].item())
    # north_star: forward logits within 1e-2 rel of the reference.  Relative error is taken in the L2
    # norm over 2048 sampled logits; the worst single logit (bf16 storage: 8 mantissa bits, 24 layers)
    # is additionally bounded at 2e-2 of the largest logit.
    assert err_l2 < 1e-2
    assert err_max < 2e-2
    assert abs(out.loss.item() - fx["loss"].item()) < 5e-3 * fx["loss"].item()
    assert _rel(image_embeds.float().norm(dim=-1), fx["image_embeds_norm"]) < 1e-2
    assert _rel(out.last_hidden_state.float().norm(dim=-1), fx["hidden_norm"]) < 1e-2
    del out
    loss, _ = model(v, _text(ids, att, cuda))
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
