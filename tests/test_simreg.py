"""Similarity regularisation (sim_reg_loss_weight > 0, reference x_clip/x_clip.py:771-784, :870-873) on
the CPU: the oracle plus tests/simreg_oracle.py against the reference's fixtures
(tests/golden/*simreg*.json, written by tests/golden/make_golden_simreg.py), and the combinations the
reference itself cannot run still raising Unsupported."""
import json
import math
from pathlib import Path

import pytest
import torch

import simreg_oracle as SR
import x_clip_b200
from oracle import clip_oracle as O

GOLD = Path(__file__).parent / "golden"
SIMREG_CASES = ["tiny_simreg_extra", "tiny_simreg_dcl_extra", "vitb16_shaped_simreg_extra"]
TINY = dict(dim_text=256, dim_image=256, dim_latent=256, num_text_tokens=128, text_enc_depth=2,
            text_seq_len=16, text_heads=4, visual_enc_depth=2, visual_heads=4,
            visual_image_size=64, visual_patch_size=16)


@pytest.mark.parametrize("case", SIMREG_CASES)
def test_oracle_reproduces_simreg_goldens(case):
    gold = json.loads((GOLD / f"{case}.json").read_text())
    cfg = O.ClipConfig(**gold["cfg"])
    w = gold["sim_reg_loss_weight"]
    state = O.protocol_state_dict(cfg, gold["weight_seed"])
    text, image = O.protocol_inputs(cfg, gold["batch"], gold["input_seed"], gold["pad_fraction"])
    p = {k: v.clone().requires_grad_(True) for k, v in state.items()}
    loss = SR.clip_forward(p, text, image, cfg, w)
    loss.backward()
    assert abs(loss.item() - gold["loss"]) <= 1e-5 * abs(gold["loss"]), (loss.item(), gold["loss"])
    with torch.no_grad():
        loss0 = O.clip_forward(state, text, image, cfg)
    assert abs(loss0.item() - gold["loss_without_sim_reg"]) <= 1e-5 * abs(gold["loss_without_sim_reg"])
    assert gold["loss"] - gold["loss_without_sim_reg"] >= gold["loss_without_sim_reg"]   # the term is visible
    assert abs(p["temperature"].grad.item() - gold["dtemperature"]) <= 2e-6
    total = 0.0
    for k, n in gold["grad_norms"].items():
        gn = p[k].grad.double().norm().item()
        total += gn * gn
        assert abs(gn - n) <= 3e-4 * max(n, 1e-5) + 1e-8, (k, gn, n)
    assert abs(math.sqrt(total) - gold["grad_norm"]) <= 1e-4 * gold["grad_norm"]


def test_oracle_simreg_sharded_contract():
    """Two gloo ranks of the reference: every rank returns the global loss, its gradients are those
    of its own shard, and they add up to the single-process gradients."""
    gold = json.loads((GOLD / "sharded_simreg_extra.json").read_text())
    cfg = O.ClipConfig(**gold["cfg"])
    w = gold["sim_reg_loss_weight"]
    state = O.protocol_state_dict(cfg, gold["weight_seed"])
    world = gold["world"]
    text, image = O.protocol_inputs(cfg, world * gold["per_rank"], gold["input_seed"], gold["pad_fraction"])
    texts, images = list(text.chunk(world)), list(image.chunk(world))
    full = {k: v.clone().requires_grad_(True) for k, v in state.items()}
    full_loss = SR.clip_forward(full, text, image, cfg, w)
    full_loss.backward()
    acc = {}
    for r in gold["ranks"]:
        p = {k: v.clone().requires_grad_(True) for k, v in state.items()}
        loss = SR.clip_forward_sharded(p, texts, images, cfg, r["rank"], w)
        loss.backward()
        assert abs(loss.item() - r["loss"]) <= 1e-5 * abs(r["loss"])
        assert abs(loss.item() - full_loss.item()) <= 1e-5 * abs(r["loss"])
        assert abs(p["temperature"].grad.item() - r["dtemperature"]) <= 2e-6
        for k, n in r["grad_norms"].items():
            gn = 0.0 if p[k].grad is None else p[k].grad.double().norm().item()
            assert abs(gn - n) <= 3e-4 * max(n, 1e-5) + 1e-8, (k, gn, n)
        for k, v in p.items():
            if v.grad is not None and k != "temperature":
                acc[k] = acc.get(k, 0) + v.grad
    for k, g in acc.items():
        assert torch.allclose(g, full[k].grad, atol=1e-4, rtol=1e-3), k


def test_oracle_simreg_batch_one_is_nan_without_gradient():
    """The reference's mean over zero off-diagonal entries: NaN, and nothing flows back from it."""
    z = [torch.nn.functional.normalize(torch.randn(1, 8), dim=-1).requires_grad_(True) for _ in range(4)]
    loss = SR.sim_reg_loss(*z)
    assert math.isnan(loss.item())
    loss.backward()
    for t in z:
        assert t.grad is None or not t.grad.any()


def test_simreg_construction_and_flag():
    clip = x_clip_b200.CLIP(**TINY, extra_latent_projection=True, sim_reg_loss_weight=0.1)
    assert clip.has_sim_reg_loss and clip.sim_reg_loss_weight == 0.1
    assert not x_clip_b200.CLIP(**TINY, extra_latent_projection=True).has_sim_reg_loss
    ref_keys = set(x_clip_b200.CLIP(**TINY, extra_latent_projection=True).state_dict())
    assert set(clip.state_dict()) == ref_keys                 # no new parameters or buffers


@pytest.mark.parametrize("kw", [dict(), dict(use_all_token_embeds=True, extra_latent_projection=True),
                                dict(use_all_token_embeds=True)])
def test_simreg_without_extra_or_with_filip_raises(kw):
    with pytest.raises(x_clip_b200.Unsupported, match="779"):
        x_clip_b200.CLIP(**TINY, sim_reg_loss_weight=0.1, **kw)


@pytest.mark.parametrize("views", [dict(aug_text=True), dict(aug_image=True), dict(aug_text=True, aug_image=True)])
def test_simreg_multiview_raises_before_encoding(views):
    clip = x_clip_b200.CLIP(**TINY, extra_latent_projection=True, sim_reg_loss_weight=0.1)
    clip.train()
    text = torch.randint(1, 128, (4, 16))
    image = torch.randn(4, 3, 64, 64)
    aug = dict(aug_text=text.clone() if "aug_text" in views else None,
               aug_image=image.clone() if "aug_image" in views else None)
    with pytest.raises(x_clip_b200.Unsupported, match="aug_text"):
        clip(text, image, return_loss=True, **aug)
