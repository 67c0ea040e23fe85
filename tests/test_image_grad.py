"""d loss / d image: the CPU oracle against the reference's gradients pinned in tests/golden/imggrad_*.json
(written by tests/golden/make_golden_image_grad.py), without a GPU.  The GPU side is
tests/test_gpu_image_grad.py, which compares x_clip_b200 with this oracle."""
import json
from pathlib import Path

import pytest
import torch

from oracle import clip_oracle as O

GOLD = Path(__file__).parent / "golden"
CASES = ["imggrad_tiny", "imggrad_tiny_drop", "imggrad_vitb16_drop", "imggrad_tiny_filip_dcl_extra",
         "imggrad_tiny_multiview", "imggrad_tiny_guidance"]


def load(case):
    return json.loads((GOLD / f"{case}.json").read_text())


def oracle_image_grads(gold):
    """(objective, [d objective / d image per view], keep) by the oracle in fp32 on the CPU"""
    cfg = O.ClipConfig(**gold["cfg"])
    state = O.protocol_state_dict(cfg, gold["weight_seed"])
    B = gold["batch"]
    text, image = O.protocol_inputs(cfg, B, gold["input_seed"], gold["pad_fraction"])
    images = [image]
    if gold["kind"] == "multiview":
        images += [O.protocol_inputs(cfg, B, gold["input_seed"] + gold["aug_seed_stride"] * (v + 1), 0.2)[1]
                   for v in range(len(gold["images"]) - 1)]
    keep = None if gold["keep"] is None else torch.tensor(gold["keep"])
    p = {k: v.clone().requires_grad_(True) for k, v in state.items()}
    ims = [im.clone().requires_grad_(True) for im in images]
    if gold["kind"] == "loss":
        obj = O.clip_forward(p, text, ims[0], cfg, keep=keep)
    elif gold["kind"] == "multiview":
        obj = O.clip_forward_multiview(p, [text], ims, cfg, gold["multiview_loss_weight"])
    else:
        mask = text != cfg.text_pad_id
        _, zi, _, _ = O.project_latents(O.encode_text(text, mask, p, cfg), O.encode_image(ims[0], p, cfg), p, cfg)
        target = torch.randn(B, cfg.dim_latent, generator=torch.Generator().manual_seed(gold["target_seed"]))
        obj = (zi * target).sum()
    obj.backward()
    return obj.item(), [im.grad for im in ims], keep, p


def patch_norms(g, patch):
    return O.patchify(g.double(), patch).norm(dim=-1)


def sample_positions(numel, n, seed):
    return [(seed * 7919 + j * 1000003) % numel for j in range(min(n, numel))]


@pytest.mark.parametrize("case", CASES)
def test_oracle_reproduces_reference_image_gradient(case):
    gold = load(case)
    patch = gold["cfg"]["visual_patch_size"]
    obj, grads, keep, p = oracle_image_grads(gold)
    assert abs(obj - gold["loss"]) <= 3e-6 * max(1.0, abs(gold["loss"])), (obj, gold["loss"])
    assert len(grads) == len(gold["images"])
    for g, rec in zip(grads, gold["images"]):
        assert list(g.shape) == rec["summ"]["shape"]
        sn = g.double().flatten(1).norm(dim=1)
        ref_sn = torch.tensor(rec["sample_norms"], dtype=torch.float64)
        assert ((sn - ref_sn).abs() <= 1e-4 * ref_sn).all(), (sn, ref_sn)
        pn = patch_norms(g, patch)
        ref_pn = torch.tensor(rec["patch_norms"], dtype=torch.float64)
        kept = ref_pn > 0
        assert ((pn - ref_pn).abs()[kept] <= 1e-4 * ref_pn[kept]).all()
        assert (pn[~kept] == 0).all()                                       # dropped patches: exactly 0
        d = g.flatten()
        pos = sample_positions(d.numel(), len(rec["samples"]), 3)
        got, ref = d[pos].double(), torch.tensor(rec["samples"], dtype=torch.float64)
        assert ((got - ref).abs() <= 1e-3 * ref.abs() + 1e-4 * ref.abs().max()).all()
    for k, v in gold["grad_norms"].items():
        assert abs(p[k].grad.double().norm().item() - v) <= 2e-4 * v + 1e-9, k


@pytest.mark.parametrize("case", ["imggrad_tiny_drop", "imggrad_vitb16_drop"])
def test_patch_dropout_cases_have_distinct_kept_rows_and_zero_dropped_patches(case):
    gold = load(case)
    keep = torch.tensor(gold["keep"])
    n = (gold["cfg"]["visual_image_size"] // gold["cfg"]["visual_patch_size"]) ** 2
    B, k = keep.shape
    assert k == max(1, int(n * (1 - gold["patch_dropout"])))
    for row in keep:
        assert len(set(row.tolist())) == k and int(row.min()) >= 0 and int(row.max()) < n
    pn = torch.tensor(gold["images"][0]["patch_norms"])
    dropped = torch.ones(B, n, dtype=torch.bool).scatter_(1, keep, False)
    assert (pn[dropped] == 0).all() and (pn[~dropped] > 0).all()


def test_reference_gives_no_image_gradient_with_a_frozen_image_encoder():
    """freeze_image_encoder=True: the reference encodes under no_grad and detaches, so image.grad stays
    None; tests/test_gpu_image_grad.py holds x_clip_b200 to the same."""
    assert load("imggrad_freeze")["image_grad_is_none"] is True


def test_every_multiview_view_gets_a_gradient():
    gold = load("imggrad_tiny_multiview")
    assert len(gold["images"]) == 3
    assert all(min(im["sample_norms"]) > 0 for im in gold["images"])
