"""Model and latent widths that are odd multiples of 128 (128, 384, 640, 896) on the GPU, with the gates of
the existing kernel and parity tests:
- the row-wise kernels (LayerNorm forward, chain and backward; l2norm; ff_bwd_prep), whose rows end in a
  128-column half vector held by lanes 0-15;
- the fused feed-forward stages and their backward;
- the encoder (engine.TransformerFn) against fp64, including an attention width heads * 64 != d;
- the C-ABI refusals of widths outside 128 * {1..8};
- CLIP end to end on the reference's fixtures (tests/golden/make_golden_widths.py), and a micro-batched
  ViT-S-shaped step against the single pass.
"""
import json
from pathlib import Path
from unittest import mock

import pytest
import torch

import block_oracle as BO
import test_gpu_clip_parity
import test_gpu_ff
import test_gpu_rowwise
import test_gpu_simreg
import test_gpu_transformer_fp64

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).parent / "golden"
NEW_WIDTHS = (128, 384, 640, 896)

# rows: one, a few, many, and past both LayerNorm grid caps (a warp then gets a second row)
LN_CASES = [(rows, d) for d in NEW_WIDTHS
            for rows in (1, 7, 1003, test_gpu_rowwise.LN_BWD_CAP + 37, test_gpu_rowwise.LN_FWD_CAP + 37)]


@pytest.mark.parametrize("rows,d", LN_CASES)
def test_layernorm_fp64_at_new_widths(cuda_device, rows, d):
    """out = LN(x) g + res, the chained out2 = LN(bf16 out) g2, both statistics, dx + add and dg against
    fp64 (test_gpu_rowwise._check_ln)."""
    test_gpu_rowwise.test_layernorm_fp64(cuda_device, rows, d)


@pytest.mark.parametrize("d", NEW_WIDTHS)
def test_layernorm_strided_at_new_widths(cuda_device, d):
    test_gpu_rowwise.test_layernorm_strided(cuda_device, d)


@pytest.mark.parametrize("d", NEW_WIDTHS)
def test_layernorm_grid_knobs_at_new_widths(cuda_device, d):
    """Grid capped at one block per SM: bit-identical outputs (dg within its fp64 gate)."""
    test_gpu_rowwise.test_layernorm_rows_per_warp_knobs(cuda_device, d)


@pytest.mark.parametrize("rows,d", [(1, 128), (7, 384), (1003, 640), (9000, 896)])
def test_l2norm_at_new_widths(cuda_device, rows, d):
    """Forward and backward against fp32 autograd, and the split-bf16 operands exactly:
    zrow = [hi | lo | hi], zcol = [hi | hi | lo] with hi = bf16(z), lo = bf16(z - hi)."""
    from x_clip_b200 import kernels as K
    test_gpu_rowwise.test_l2norm(cuda_device, rows, d)
    torch.manual_seed(4)
    p = torch.randn(rows, d, device=cuda_device) * 3
    z, zrow, zcol, inv = K.l2norm_fwd(p)
    torch.cuda.synchronize()
    hi = z.bfloat16()
    lo = (z - hi.float()).bfloat16()
    assert torch.equal(zrow, torch.cat([hi, lo, hi], 1))
    assert torch.equal(zcol, torch.cat([hi, hi, lo], 1))
    n64 = p.double().norm(dim=1)
    assert ((inv.double() - 1 / n64).abs() <= 1e-6 / n64).all()


FF_CASES = [(M, d) for d in NEW_WIDTHS for M in (1, 127, 128, 129)] + [
    (8577, 128), (8577, 384), (3000, 640), (1413, 896)]


@pytest.mark.parametrize("M,d", FF_CASES)
def test_ff_stages_fp64_at_new_widths(cuda_device, M, d):
    """Up-projection (u, hp, rowsum), down-projection (stats, x2, acc), ff_bwd_prep (dxs exact, vsum, a,
    b), the fused backward (du) and ff_w2_grad_post (dW2 exact, dg4) against fp64 (test_gpu_ff).  M =
    8577 passes ff_bwd_prep's 8448-row grid cap; 4d = 512 / 1536 / 2560 / 3584 hidden columns."""
    test_gpu_ff.test_ff_stages_fp64(cuda_device, M, d)


WIDTH_BLOCK_CASES = {
    # name: (B, n, d, heads, masked, causal, rotary), as block_oracle.BLOCK_CASES
    "d384_h6_n197": (4, 197, 384, 6, False, False, False),
    "d384_h8_mask": (6, 78, 384, 8, True, False, False),        # attention width 512 != d
    "d640_h10_rotary": (6, 33, 640, 10, True, False, True),
    "d128_h2_causal": (6, 78, 128, 2, True, True, False),
}


@pytest.mark.parametrize("name", list(WIDTH_BLOCK_CASES))
def test_transformer_fp64_at_new_widths(cuda_device, name):
    """engine.TransformerFn (depth 2) forward and backward against fp64 with BLOCK_GATES."""
    with mock.patch.dict(BO.BLOCK_CASES, {name: WIDTH_BLOCK_CASES[name]}):
        test_gpu_transformer_fp64.test_transformer_fp64(cuda_device, name)


@pytest.mark.parametrize("d", [64, 192, 320, 1152])
def test_row_entries_refuse_other_widths_without_launching(cuda_device, d):
    from x_clip_b200 import _lib
    lib = _lib.load()
    rows, ld = 4, 1152
    bf = torch.zeros(rows, 3 * ld, device=cuda_device, dtype=torch.bfloat16)
    f = torch.zeros(rows, 3 * ld, device=cuda_device)
    b2 = torch.zeros(rows, 3 * ld, device=cuda_device, dtype=torch.bfloat16)
    st = torch.zeros(rows, 2, device=cuda_device)
    vec = torch.zeros(4 * ld, device=cuda_device)
    torch.cuda.synchronize()
    n0 = lib.xclip_launch_count()
    P = lambda t: t.data_ptr()   # noqa: E731
    calls = [
        ("xclip_layernorm_fwd", (P(bf), ld, P(vec), None, 0, P(b2), ld, P(st), None, None, 0, None, rows, d, 1e-5)),
        ("xclip_layernorm_fwd", (P(bf), ld, P(vec), P(bf), ld, P(b2), ld, P(st), P(vec), P(b2), ld, P(st), rows, d,
                                 1e-5)),
        ("xclip_layernorm_bwd", (P(bf), ld, P(bf), ld, P(st), P(vec), None, 0, P(b2), ld, P(vec), rows, d)),
        ("xclip_l2norm_fwd", (P(f), ld, P(f), P(bf), P(b2), P(vec), rows, d)),
        ("xclip_l2norm_bwd", (P(f), P(f), P(vec), P(bf), rows, d)),
        ("xclip_ff_bwd_prep", (P(bf), ld, P(st), P(bf), ld, P(vec), P(b2), P(vec), P(st), rows, d)),
    ]
    for name, args in calls:
        assert getattr(lib, name)(*args, None) != 0, (name, d)
        assert str(d).encode() in lib.xclip_last_error(), (name, lib.xclip_last_error())
    assert lib.xclip_launch_count() == n0
    if d in (64, 192, 320):         # not a multiple of 128: the feed-forward entries refuse too
        from x_clip_b200 import kernels as K
        with pytest.raises(_lib.XClipB200Error):
            K.ff_weights(torch.zeros(8 * d, d, device=cuda_device), torch.zeros(d, 4 * d, device=cuda_device),
                         torch.ones(4 * d, device=cuda_device))
        assert lib.xclip_launch_count() == n0


WIDTH_CASES = ["tiny128_h2", "vits16_shaped", "vits16_shaped_drop", "w384_h8", "b16plus_shaped_dcl_extra",
               "vits16_filip", "vits16_text_causal"]


@pytest.mark.parametrize("case", WIDTH_CASES)
def test_clip_matches_reference_at_new_widths(cuda_device, case):
    """Loss, latents, d temperature, gradient norm and per-parameter gradients against the reference,
    with the gates of test_gpu_clip_parity."""
    test_gpu_clip_parity.test_clip_matches_reference(cuda_device, case)


def test_clip_with_simreg_matches_reference_at_latent_384(cuda_device):
    test_gpu_simreg.test_clip_with_simreg_matches_reference(cuda_device, "vits16_simreg_extra")


def test_microbatched_vits_step_equals_single_pass(cuda_device):
    """A ViT-S/16-shaped step (width 384, 6 heads) in micro-batches of 2 equals the single pass: loss
    within 1e-5, every gradient within 2e-2 of its norm (the gates of test_odd_batches)."""
    from oracle import clip_oracle as O
    import x_clip_b200
    gold = json.loads((GOLD / "vits16_shaped.json").read_text())
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
    (loss0, grads0), (loss1, grads1) = res
    assert abs(loss0 - gold["loss"]) <= 1e-3 * abs(gold["loss"])
    assert abs(loss1 - loss0) < 1e-5, (loss1, loss0)
    assert grads1.keys() == grads0.keys()
    for k, g in grads1.items():
        ref = grads0[k]
        assert (g - ref).norm().item() <= 2e-2 * ref.norm().item() + 1e-6, k
