"""FILIP models at token counts other than 16, 32, 64 and 256: 48 text tokens against 144 image tokens
(192 px / patch 16), so the segment-max GEMMs run with seg_len 144 and seg_len 48: neither divides
the 256-column tile, so segments are cut by tile edges and restart inside a 128-column staging pass.
Goldens:
tests/golden/{filip_t48_i144, filip_t48_i144_dcl_extra}.json, written by
tests/golden/make_golden_filip.py."""
import json
import math
from pathlib import Path

import pytest
import torch

import test_gpu_clip_parity
import test_gpu_filip
import test_oracle_golden
from oracle import clip_oracle as O

GOLD = Path(__file__).parent / "golden"
FILIP_CASES = ["filip_t48_i144", "filip_t48_i144_dcl_extra"]


@pytest.mark.parametrize("case", FILIP_CASES)
def test_filip_models_construct_with_the_reference_parameter_tree(case):
    import x_clip_b200
    gold = json.loads((GOLD / f"{case}.json").read_text())
    clip = x_clip_b200.CLIP(**gold["cfg"], visual_patch_dropout=gold["patch_dropout"])
    want = O.param_shapes(O.ClipConfig(**gold["cfg"]))
    got = {k: tuple(v.shape) for k, v in clip.state_dict().items()}
    assert got == want


@pytest.mark.parametrize("case", FILIP_CASES)
def test_oracle_reproduces_filip_goldens(case):
    test_oracle_golden.test_oracle_reproduces_reference(case)


@pytest.mark.gpu
@pytest.mark.parametrize("case", FILIP_CASES)
def test_filip_clip_matches_reference(cuda_device, case):
    """Loss, latent checksums, d temperature, gradient norm and per-parameter gradients against the
    reference, with the gates of test_gpu_clip_parity."""
    test_gpu_clip_parity.test_clip_matches_reference(cuda_device, case)


@pytest.mark.parametrize("dcl,extra", [(False, False), (True, True)])
def test_chunked_fp64_reference_equals_the_oracle(dcl, extra):
    """The text-block restatement that checks cfg4-sized batches on the GPU (test_gpu_filip) is the
    oracle's contrastive_loss: same loss, d temperature and latent gradients, empty caption included."""
    dev = torch.device("cpu")
    lat, mask = test_gpu_filip._filip_inputs(dev, 7, 32, 16, 24, extra, seed=3, empty=(2,))
    ref = test_gpu_filip._oracle_filip(lat, mask, math.log(10.0), dcl)
    got = test_gpu_filip.oracle_filip_chunked(lat, mask, math.log(10.0), dcl, block=3)
    assert abs(got[0] - ref[0]) <= 1e-12 * abs(ref[0])
    assert abs(got[1] - ref[1]) <= 1e-12 * abs(ref[1]) + 1e-15
    for g, r in zip(got[2], ref[2]):
        assert torch.allclose(g, r, rtol=1e-10, atol=1e-15)
