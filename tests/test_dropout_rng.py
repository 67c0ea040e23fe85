"""Attention dropout on the CPU: the numpy Philox restatement against the Random123 known-answer
vectors, the properties of the documented counter layout, and how the modules take `attn_dropout` /
`ff_dropout` (as the reference's nn.Dropout / Transformer do)."""
import numpy as np
import pytest
import torch

import dropout_oracle as DO


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
    ((0xffffffff,) * 4, (0xffffffff,) * 2, (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
    ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0),
     (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1)),
])
def test_philox_known_answers(ctr, key, want):
    got = DO.philox4x32_10(np.array(ctr, dtype=np.uint32), key)
    assert tuple(int(w) for w in got) == want


def test_mask_is_a_function_of_the_element():
    """A row's mask does not depend on n (so not on the padding to 64-key blocks or on the schedule),
    and differs between layers, seeds, heads and batch items."""
    seed, p = -1234567890123, 0.3
    short = DO.attn_keep(seed, 2, 3, 77, 0, p)
    long = DO.attn_keep(seed, 2, 3, 577, 0, p)
    assert np.array_equal(short, long[:, :, :77, :77])
    assert np.array_equal(DO.attn_keep(seed, 2, 3, 577, 0, p, rows=[5, 300]), long[:, :, [5, 300]])
    for other in (DO.attn_keep(seed, 2, 3, 77, 1, p), DO.attn_keep(seed + 1, 2, 3, 77, 0, p)):
        assert (other != short).mean() > 0.3
    assert (short[0, 0] != short[0, 1]).mean() > 0.3 and (short[0, 0] != short[1, 0]).mean() > 0.3


@pytest.mark.parametrize("p", [0.0, 2.0 ** -40, 0.1, 0.5, 0.9, 1.0])
def test_keep_threshold(p):
    """keep iff word < round((1 - p) 2^32): p = 0 (and p below 2^-33) keeps everything, p = 1 nothing."""
    thr = DO.keep_threshold(p)
    assert thr == round((1 - float(np.float32(p))) * 2 ** 32)
    keep = DO.attn_keep(7, 4, 4, 128, 0, p)
    if p < 2.0 ** -33:
        assert keep.all()
    elif p == 1.0:
        assert not keep.any()
    else:
        sd = (p * (1 - p) / keep.size) ** 0.5
        assert abs(keep.mean() - (1 - p)) < 5 * sd


def test_modules_take_dropout_like_the_reference():
    """attn_dropout in [0, 1] is accepted and out-of-range values raise ValueError (nn.Dropout's
    check); the parameter tree and state_dict are those of the model without dropout; ff_dropout is
    accepted and not applied, as in the reference's Transformer."""
    import x_clip_b200
    from x_clip_b200 import clip as C

    kw = dict(dim=256, num_tokens=100, max_seq_len=16, dim_head=64, depth=2, heads=4)
    for p in (0.0, 0.1, 1.0):
        C.Attention(256, dropout=p)
    for bad in (-0.1, 1.5):
        with pytest.raises(ValueError):
            C.Attention(256, dropout=bad)
        with pytest.raises(ValueError):
            x_clip_b200.TextTransformer(**kw, attn_dropout=bad)
    torch.manual_seed(0)
    plain = x_clip_b200.TextTransformer(**kw)
    torch.manual_seed(0)
    drop = x_clip_b200.TextTransformer(**kw, attn_dropout=0.1, ff_dropout=0.1)
    a, b = plain.state_dict(), drop.state_dict()
    assert list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)
    assert [n for n, _ in plain.named_parameters()] == [n for n, _ in drop.named_parameters()]
    attn = drop.transformer.layers[0][0].fn
    assert isinstance(attn.dropout, torch.nn.Dropout) and attn.dropout.p == 0.1
    drop.eval()
    assert not attn.dropout.training
    vit = x_clip_b200.VisionTransformer(256, image_size=32, patch_size=16, channels=3, depth=1, heads=4,
                                        attn_dropout=0.2, ff_dropout=0.3)
    assert vit.transformer.layers[0][0].fn.dropout.p == 0.2
    assert vit.transformer.forced_dropout_seed is None


@pytest.mark.parametrize("causal", [False, True])
def test_dropout_references_restate_the_plain_ones(causal):
    """With every element kept at scale 1 the fp64 references with dropout are attn_oracle.attn_ref64 and
    block_oracle.transformer_stack; with a real mask they differ from them."""
    import attn_oracle as AO
    import block_oracle as BO
    B, n, H = 3, 70, 2
    case = AO.attn_case("no_visible", B, n, H, causal=causal, seed=3)
    o = AO.attn_ref64(case["qkv"], case["mask"], B, n, H, 0.125, causal)["o"].bfloat16()
    want = AO.attn_ref64(case["qkv"], case["mask"], B, n, H, 0.125, causal, o=o, d_o=case["d_o"])
    ones = torch.ones(B, H, n, n, dtype=torch.float64)
    got = DO.attn_dropout_ref64(case["qkv"], case["mask"], B, n, H, 0.125, causal, ones, o, case["d_o"])
    for k in ("o", "lse", "g_o", "g_lse", "dqkv", "g_dqkv"):
        assert torch.allclose(got[k], want[k], rtol=1e-12, atol=0), k
    drop = DO.attn_drop_mul(5, B, H, n, 0, 0.3)
    dropped = DO.attn_dropout_ref64(case["qkv"], case["mask"], B, n, H, 0.125, causal, drop, o, case["d_o"])
    assert not torch.allclose(dropped["o"], want["o"])

    blk = BO.block_case("d256_rotary" if not causal else "d512_mask_causal")
    Bb, nb, _ = blk["x"].shape
    args = (blk["x"].double(), [w.double() for w in blk["weights"]], BO.BLOCK_DEPTH, blk["heads"], blk["mask"],
            blk["causal"], blk["rot"])
    plain = BO.transformer_stack(*args)
    keep_all = [torch.ones(Bb, blk["heads"], nb, nb, dtype=torch.float64)] * BO.BLOCK_DEPTH
    assert torch.allclose(DO.transformer_stack_dropout(*args, keep_all), plain, rtol=1e-12, atol=1e-12)
