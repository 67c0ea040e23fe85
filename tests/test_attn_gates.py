"""CPU checks of the attention tests' reference, gates and input recipes (no GPU).

- The kernels' online softmax restated block by block in fp64 agrees with the direct reference.
- The recipes make the terms they exist for large: peaked scores, late row maxima, rows with no
  visible key.
- Each gate of the GPU attention tests is at most a quarter of the effect of the defect it exists to
  catch, on the inputs those tests build from the same seeds (`bite` >= 4, as in
  test_block_gates.py).  Loosening an attention gate 4x fails here.
"""
import math

import pytest
import torch

import attn_oracle as AO
import block_oracle as BO

BITE = 4.0
B, N, H = 3, 257, 2          # the recipe shape of test_gpu_attention.py: 4 full blocks + a one-key tail
SCALE = 64 ** -0.5


def _case(recipe, causal):
    c = AO.attn_case(recipe, B, N, H, causal=causal)
    ref = AO.attn_ref64(c["qkv"], c["mask"], B, N, H, SCALE, causal, d_o=c["d_o"])
    return c, ref


def _grads(ref, dqkv):
    inner = H * 64
    return [(name, dqkv[:, sl] - ref["dqkv"][:, sl], ref["g_dqkv"][:, sl])
            for name, sl in (("dq", slice(0, inner)), ("dk", slice(inner, 2 * inner)),
                             ("dv", slice(2 * inner, 3 * inner)))]


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("recipe", ["flat", "late_max", "block_masked", "no_visible"])
def test_block_emulation_matches_reference(recipe, causal):
    c = AO.attn_case(recipe, B, N, H, causal=causal)
    ref = AO.attn_ref64(c["qkv"], c["mask"], B, N, H, SCALE, causal)
    o, lse = AO.attn_fwd_blocks64(c["qkv"], c["mask"], B, N, H, SCALE, causal)
    assert (o - ref["o"]).abs().max().item() <= 1e-12 * ref["o"].abs().max().item()
    assert torch.equal(lse == -AO.FLT_MAX, ref["lse"] == -AO.FLT_MAX)
    assert (lse - ref["lse"]).abs().max().item() <= 1e-9


@pytest.mark.parametrize("causal", [False, True])
def test_recipes_make_their_terms_large(causal):
    q, k, _ = AO.split_heads(AO.attn_case("peaked", B, N, H, causal=causal)["qkv"], B, N, H, 3)
    assert 4.0 <= (SCALE * q @ k.transpose(-1, -2)).std().item() <= 8.0
    c = AO.attn_case("late_max", B, N, H, causal=causal)
    q, k, _ = AO.split_heads(c["qkv"], B, N, H, 3)
    vis = AO.visible(c["mask"], B, N, causal, "cpu")
    s = (q @ k.transpose(-1, -2)).masked_fill(~vis, -math.inf)
    top2 = s.topk(2, dim=-1)
    i = torch.arange(N)
    late = top2.indices[..., 0] // 64 == (i if causal else torch.full_like(i, N - 1)) // 64
    wide = (top2.values[..., 0] - top2.values[..., 1]) * SCALE >= 1.0
    assert (late & wide)[..., 64:].float().mean().item() >= 0.8    # rows past block 0
    m = AO.attn_case("no_visible", B, N, H, causal=causal)["mask"]
    empty = ~AO.visible(m, B, N, causal, "cpu").any(-1)
    assert empty[1].all() and empty[0].any() == causal and not empty[2].any()


@pytest.mark.parametrize("causal", [False, True])
def test_attn_gates_bite(causal):
    # ds without - delta: dq and dk
    c, ref = _case("flat", causal)
    bad = AO.attn_ref64(c["qkv"], c["mask"], B, N, H, SCALE, causal, d_o=c["d_o"], defect="no_delta")
    for name, eff, gate in _grads(ref, bad["dqkv"])[:2]:
        assert BO.bite(eff, gate) >= BITE, name
    # lse in natural log; lse without block 0's share of l
    finite = ref["lse"] != -AO.FLT_MAX
    assert BO.bite((ref["lse"] * AO.LN2 - ref["lse"])[finite], ref["g_lse"][finite]) >= BITE
    _, lse_skip = AO.attn_fwd_blocks64(c["qkv"], c["mask"], B, N, H, SCALE, causal, lse_skip_block0=True)
    assert BO.bite((lse_skip - ref["lse"])[finite], ref["g_lse"][finite]) >= BITE
    # the key mask shifted by one key
    bad = AO.attn_ref64(c["qkv"], c["mask"], B, N, H, SCALE, causal, defect="mask_shift")
    assert BO.bite(bad["o"] - ref["o"], ref["g_o"]) >= BITE
    # the causal diagonal hidden (j >= i instead of j > i)
    if causal:
        bad = AO.attn_ref64(c["qkv"], c["mask"], B, N, H, SCALE, causal, defect="causal_no_diag")
        assert BO.bite(bad["o"] - ref["o"], ref["g_o"]) >= BITE
    # an online softmax that does not rescale l, or oacc, when the row maximum grows
    c, ref = _case("late_max", causal)
    for kw in ("rescale_l", "rescale_o"):
        o, lse = AO.attn_fwd_blocks64(c["qkv"], c["mask"], B, N, H, SCALE, causal, **{kw: False})
        assert BO.bite(o - ref["o"], ref["g_o"]) >= BITE, kw
    # gradient let through hidden scores, p = 1 on rows with no visible key (the backward before the
    # fix of such rows): every gradient moves
    c, ref = _case("no_visible", causal)
    bad = AO.attn_ref64(c["qkv"], c["mask"], B, N, H, SCALE, causal, d_o=c["d_o"], defect="masked_grad")
    for name, eff, gate in _grads(ref, bad["dqkv"]):
        assert BO.bite(eff, gate) >= BITE, name


def test_gates_at_one_key():
    """n = 1: dS is exactly 0, so only the cancellation term gates dq and dk; it must be non-zero and
    at least the size of one fp32 rounding of dp."""
    c = AO.attn_case("flat", 4, 1, 3, masked=False)
    ref = AO.attn_ref64(c["qkv"], None, 4, 1, 3, SCALE, False, d_o=c["d_o"])
    inner = 3 * 64
    assert ref["dqkv"][:, :2 * inner].abs().max().item() <= 1e-12
    (do,) = AO.split_heads(c["d_o"], 4, 1, 3, 1)
    _, _, v = AO.split_heads(c["qkv"], 4, 1, 3, 3)
    dp_ulp = 2.0 ** -24 * (do.abs() * v.abs()).sum(-1)
    _, k, _ = AO.split_heads(c["qkv"], 4, 1, 3, 3)
    floor = SCALE * dp_ulp[..., None] * k.abs()
    assert (AO.merge_heads(floor) <= ref["g_dqkv"][:, :inner]).all()
