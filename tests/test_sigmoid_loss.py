"""The pairwise sigmoid loss without a GPU: sigmoid_oracle against a restatement with F.logsigmoid in fp64
autograd, the rank shares, CLIP(sigmoid_loss=True)'s parameters and the combinations it refuses."""
import math

import pytest
import torch
import torch.nn.functional as F

import sigmoid_oracle as SG

TINY = dict(dim_text=128, dim_image=128, dim_latent=128, num_text_tokens=64, text_enc_depth=1, text_seq_len=8,
            text_heads=2, visual_enc_depth=1, visual_heads=2, visual_image_size=32, visual_patch_size=16)


def _latents(B, D, seed):
    g = torch.Generator().manual_seed(seed)
    zt = F.normalize(torch.randn(B, D, generator=g, dtype=torch.float64), dim=-1)
    zi = F.normalize(torch.randn(B, D, generator=g, dtype=torch.float64) + 0.5 * zt, dim=-1)
    return zt.requires_grad_(True), zi.requires_grad_(True)


@pytest.mark.parametrize("B,temp,bias", [(1, math.log(10.0), -10.0), (5, math.log(10.0), -10.0),
                                         (33, math.log(100.0), 0.0), (64, 0.3, 2.5)])
def test_oracle_matches_logsigmoid(B, temp, bias):
    """Loss, d latents, d temperature and d logit_bias of the oracle against -(1/B) sum log sigmoid(z l),
    and d loss / d logit = (sigmoid(l) - [i == j]) / B."""
    zt, zi = _latents(B, 24, B)
    t = torch.tensor(temp, dtype=torch.float64, requires_grad=True)
    lb = torch.tensor(bias, dtype=torch.float64, requires_grad=True)
    loss = SG.sigmoid_loss(zt, zi, t, lb)
    got = torch.autograd.grad(loss, (zt, zi, t, lb))

    lg = t.exp() * zt @ zi.t() + lb
    z = 2.0 * torch.eye(B, dtype=torch.float64) - 1.0
    ref = -F.logsigmoid(z * lg).sum() / B
    want = torch.autograd.grad(ref, (zt, zi, t, lb), retain_graph=True)
    assert torch.allclose(loss, ref, rtol=1e-12, atol=0)
    for a, b in zip(got, want):
        assert torch.allclose(a, b, rtol=1e-11, atol=1e-14)

    lgd = lg.detach().requires_grad_(True)
    (dl,) = torch.autograd.grad(SG.softplus(-z * lgd).sum() / B, lgd)
    assert torch.allclose(dl, (torch.sigmoid(lgd) - torch.eye(B, dtype=torch.float64)) / B, rtol=1e-12, atol=1e-16)


@pytest.mark.parametrize("world,b", [(2, 3), (3, 5), (4, 1)])
def test_rank_shares_sum_to_the_loss(world, b):
    zt, zi = _latents(world * b, 16, 7 * world + b)
    t = torch.tensor(math.log(10.0), dtype=torch.float64)
    lb = torch.tensor(-10.0, dtype=torch.float64)
    shares = [SG.rank_share(zt, zi, t, lb, world, r) for r in range(world)]
    full = SG.sigmoid_loss(zt, zi, t, lb)
    assert torch.allclose(sum(shares), full, rtol=1e-14, atol=0)
    assert all(s > 0 for s in shares)


def test_clip_parameters():
    import x_clip_b200
    plain = x_clip_b200.CLIP(**TINY)
    sig = x_clip_b200.CLIP(**TINY, sigmoid_loss=True)
    assert "logit_bias" not in dict(plain.named_parameters())
    assert plain.temperature.item() == 1.0
    assert set(sig.state_dict()) - set(plain.state_dict()) == {"logit_bias"}
    assert set(plain.state_dict()) <= set(sig.state_dict())
    assert sig.logit_bias.shape == () and sig.logit_bias.item() == -10.0 and sig.logit_bias.requires_grad
    assert sig.temperature.item() == pytest.approx(math.log(10.0), rel=1e-7)


@pytest.mark.parametrize("extra", [dict(use_all_token_embeds=True), dict(decoupled_contrastive_learning=True),
                                   dict(extra_latent_projection=True),
                                   dict(extra_latent_projection=True, sim_reg_loss_weight=1.0)],
                         ids=["filip", "dcl", "extra", "simreg"])
def test_refused_combinations(extra):
    import x_clip_b200
    from x_clip_b200.clip import Unsupported
    with pytest.raises(Unsupported):
        x_clip_b200.CLIP(**TINY, sigmoid_loss=True, **extra)
    x_clip_b200.CLIP(**TINY, **extra)          # each is fine with the default loss
