"""Patch sizes whose rows are not a multiple of 8 values, without a GPU: the CPU oracle against the
reference goldens of tests/golden/make_golden_patch14.py, the ViT-L/14 and patch-7 towers build, their
parameter tree is the reference's, and a protocol state dict loads strictly.  The GPU side is
tests/test_gpu_patch14.py."""
import json
from pathlib import Path

import pytest
import torch

from oracle import clip_oracle as O

GOLD = Path(__file__).parent / "golden"
CLIP_CASES = ["tiny_p14", "tiny_p14_drop", "tiny_p14_c1", "tiny_p7", "vitl14_shaped", "vitl14_336_filip"]


@pytest.mark.parametrize("case", CLIP_CASES)
def test_oracle_reproduces_reference_at_any_patch_size(case):
    import test_oracle_golden as OG
    OG.test_oracle_reproduces_reference(case)


def test_oracle_reproduces_reference_image_gradient_at_patch_14():
    import test_image_grad as IG
    IG.test_oracle_reproduces_reference_image_gradient("imggrad_p14")


def test_goldens_cover_the_patch_sizes_they_name():
    def cfg(case):
        return json.loads((GOLD / f"{case}.json").read_text())["cfg"]
    pd = {c: cfg(c).get("channels", 3) * cfg(c)["visual_patch_size"] ** 2 for c in CLIP_CASES + ["imggrad_p14"]}
    assert pd["tiny_p14"] == pd["vitl14_shaped"] == pd["imggrad_p14"] == 588
    assert pd["tiny_p14_c1"] == 196 and pd["tiny_p7"] == 147
    assert all(v % 8 != 0 for v in pd.values())
    vl = cfg("vitl14_shaped")
    assert (vl["dim_image"], vl["visual_heads"], vl["visual_image_size"], vl["text_seq_len"]) == (1024, 16, 224, 77)
    assert vl["text_causal_mask"] and cfg("vitl14_336_filip")["visual_image_size"] == 336
    assert cfg("vitl14_336_filip")["use_all_token_embeds"]


VITL14 = dict(dim_text=768, dim_image=1024, dim_latent=768, num_text_tokens=49408, text_enc_depth=12,
              text_seq_len=77, text_heads=12, visual_enc_depth=24, visual_heads=16,
              visual_image_size=224, visual_patch_size=14, text_causal_mask=True, text_eos_id=49407)


@pytest.mark.parametrize("kw", [
    dict(VITL14),
    dict(VITL14, visual_image_size=336),
    dict(dim_text=256, dim_image=256, dim_latent=256, num_text_tokens=128, text_enc_depth=1, text_seq_len=16,
         text_heads=4, visual_enc_depth=1, visual_heads=4, visual_image_size=28, visual_patch_size=7),
    dict(dim_text=256, dim_image=256, dim_latent=256, num_text_tokens=128, text_enc_depth=1, text_seq_len=16,
         text_heads=4, visual_enc_depth=1, visual_heads=4, visual_image_size=56, visual_patch_size=14, channels=1),
])
def test_any_patch_size_builds_with_the_reference_parameter_tree(kw):
    import x_clip_b200
    clip = x_clip_b200.CLIP(**kw, visual_patch_dropout=0.5)
    cfg = O.ClipConfig(**kw)
    shapes = O.param_shapes(cfg)
    sd = clip.state_dict()
    assert set(sd) == set(shapes)
    for k, v in sd.items():
        assert tuple(v.shape) == shapes[k], k
    p = kw["visual_patch_size"]
    assert tuple(sd["visual_transformer.to_tokens.1.weight"].shape) == (kw["dim_image"], kw.get("channels", 3) * p * p)
    if kw["dim_image"] <= 256:              # (the full ViT-L/14 protocol state dict is slow to draw)
        clip.load_state_dict(O.protocol_state_dict(cfg, 1234), strict=True)
