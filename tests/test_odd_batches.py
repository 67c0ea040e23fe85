"""Whole models at odd global batches.  In ContrastiveLossFn the image-direction log-denominators of an
odd batch B sit 8 B bytes into the gathered [4, B] statistics, an address the backward's 16-byte loads
cannot take as it is, and from B = 33 on every row of the InfoNCE backward has 32-column chunks on the
vectorised interior path.  Goldens: tests/golden/{tiny_b65, tiny_b33_dcl_extra}.json, written by
tests/golden/make_golden_odd.py."""
import json
from pathlib import Path

import pytest
import torch

import test_gpu_clip_parity
import test_oracle_golden

GOLD = Path(__file__).parent / "golden"
ODD_CASES = ["tiny_b65", "tiny_b33_dcl_extra"]


@pytest.mark.parametrize("case", ODD_CASES)
def test_oracle_reproduces_odd_batch_goldens(case):
    test_oracle_golden.test_oracle_reproduces_reference(case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", ODD_CASES)
def test_odd_batch_clip_matches_reference(cuda_device, case):
    """Loss, latent summaries (shape, abs sum, first values), d temperature, gradient norm and
    per-parameter gradients against the reference, with the gates of test_gpu_clip_parity."""
    test_gpu_clip_parity.test_clip_matches_reference(cuda_device, case)


@pytest.mark.gpu
def test_microbatched_odd_batch_equals_single_pass(cuda_device):
    """B = 65 in micro-batches of 32 (chunks of 32, 32 and 1, concatenated before the loss) is the same
    step as the single pass: loss within 1e-5, every gradient within 2e-2 of its norm (the gates of
    test_microbatched_step_equals_single_pass)."""
    from oracle import clip_oracle as O
    import x_clip_b200
    gold = json.loads((GOLD / "tiny_b65.json").read_text())
    cfg = O.ClipConfig(**gold["cfg"])
    state = O.protocol_state_dict(cfg, gold["weight_seed"])
    text, image = O.protocol_inputs(cfg, gold["batch"], gold["input_seed"], gold["pad_fraction"])
    text, image = text.to(cuda_device), image.to(cuda_device)
    res = []
    for mb in (None, 32):
        clip = x_clip_b200.CLIP(**gold["cfg"], visual_patch_dropout=0., microbatch=mb).to(cuda_device)
        clip.load_state_dict(state)
        clip.train()
        loss = clip(text, image, return_loss=True)
        loss.backward()
        if mb is not None:
            assert clip.last_step_plan["chunks"] == 3, clip.last_step_plan
        res.append((loss.item(), {k: p.grad.clone() for k, p in clip.named_parameters() if p.grad is not None}))
    (loss0, grads0), (loss1, grads1) = res
    assert abs(loss0 - gold["loss"]) <= 1e-3 * abs(gold["loss"])
    assert abs(loss1 - loss0) < 1e-5, (loss1, loss0)
    assert grads1.keys() == grads0.keys()
    for k, g in grads1.items():
        ref = grads0[k]
        assert (g - ref).norm().item() <= 2e-2 * ref.norm().item() + 1e-6, k
