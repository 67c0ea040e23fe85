"""Models whose attention runs on sequences longer than 320 tokens: a 400-token text tower (401 with
CLS, also with rotary embedding), a 400 px / patch 16 image tower (625 tokens) and ViT-B/16 at 384 px
(576 tokens).  Goldens: tests/golden/{long_t401_i625, long_rotary_t401, vitb16_384_shaped}.json, written
by tests/golden/make_golden_long.py."""
import json
from pathlib import Path

import pytest
import torch

import test_gpu_clip_parity
import test_oracle_golden
from oracle import clip_oracle as O

GOLD = Path(__file__).parent / "golden"
LONG_CASES = ["long_t401_i625", "long_rotary_t401", "vitb16_384_shaped"]


def _gold(case):
    return json.loads((GOLD / f"{case}.json").read_text())


@pytest.mark.parametrize("case", LONG_CASES)
def test_long_models_construct_with_the_reference_parameter_tree(case):
    import x_clip_b200
    gold = _gold(case)
    clip = x_clip_b200.CLIP(**gold["cfg"], visual_patch_dropout=gold["patch_dropout"])
    want = O.param_shapes(O.ClipConfig(**gold["cfg"]))
    got = {k: tuple(v.shape) for k, v in clip.state_dict().items()}
    # (the rotary tower also keeps the reference's inv_freq buffer, which is not a parameter)
    assert set(got) - set(want) <= {"text_transformer.rotary_pos_emb.inv_freq"} and not set(want) - set(got)
    assert all(got[k] == want[k] for k in want)


@pytest.mark.parametrize("case", LONG_CASES)
def test_oracle_reproduces_long_goldens(case):
    test_oracle_golden.test_oracle_reproduces_reference(case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", LONG_CASES)
def test_long_clip_matches_reference(cuda_device, case):
    """Loss, latents, d temperature, gradient norm and per-parameter gradients against the reference,
    with the gates of test_gpu_clip_parity."""
    test_gpu_clip_parity.test_clip_matches_reference(cuda_device, case)


@pytest.mark.gpu
def test_long_microbatched_step_equals_single_pass(cuda_device):
    import x_clip_b200
    gold = _gold("long_t401_i625")
    cfg = O.ClipConfig(**gold["cfg"])
    state = O.protocol_state_dict(cfg, gold["weight_seed"])
    text, image = O.protocol_inputs(cfg, gold["batch"], gold["input_seed"], gold["pad_fraction"])
    text, image = text.to(cuda_device), image.to(cuda_device)
    res = []
    for mb in (None, 2):
        clip = x_clip_b200.CLIP(**gold["cfg"], visual_patch_dropout=0., microbatch=mb).to(cuda_device)
        clip.load_state_dict(state)
        clip.train()
        loss = clip(text, image, return_loss=True)
        loss.backward()
        if mb is not None:
            assert clip.last_step_plan["chunks"] == 2, clip.last_step_plan
        res.append((loss.item(), {k: p.grad.clone() for k, p in clip.named_parameters() if p.grad is not None}))
    (loss0, g0), (loss1, g1) = res
    assert abs(loss1 - loss0) < 1e-5
    assert g1.keys() == g0.keys()
    for k, g in g1.items():
        assert (g - g0[k]).norm().item() <= 2e-2 * g0[k].norm().item() + 1e-6, k


@pytest.mark.gpu
def test_vitb16_384_return_latents_in_eval(cuda_device):
    """Evaluation sees all 576 image tokens whatever the training patch dropout."""
    import x_clip_b200
    gold = _gold("vitb16_384_shaped")
    cfg = O.ClipConfig(**gold["cfg"])
    text, image = O.protocol_inputs(cfg, gold["batch"], gold["input_seed"], gold["pad_fraction"])
    clip = x_clip_b200.CLIP(**gold["cfg"]).to(cuda_device)      # default patch dropout 0.5
    clip.load_state_dict(O.protocol_state_dict(cfg, gold["weight_seed"]))
    clip.eval()
    with torch.no_grad():
        zt, zi = clip(text.to(cuda_device), image.to(cuda_device), return_latents=True)
    for z, ref, name in ((zt, gold["text_latents"], "text"), (zi, gold["image_latents"], "image")):
        cos = torch.nn.functional.cosine_similarity(z.float().cpu(), torch.tensor(ref), dim=-1).min().item()
        assert cos >= 0.999, f"{name} latents cosine {cos}"
