"""CLIP.forward's training loss on the CPU: which loss Function runs for each configuration, with which
views, weights and similarity-regularisation arguments, and how its value is weighted with the MLM and
multiview terms (x_clip.py:851-873).  The towers are pluggable CPU encoders, the projection is the
identity, and the loss Functions are recorders that return constants."""
import pytest
import torch

import x_clip_b200
from x_clip_b200 import engine as E
from x_clip_b200 import filip as F

TINY = dict(dim_text=256, dim_image=256, dim_latent=256, num_text_tokens=128, text_enc_depth=1,
            text_seq_len=16, text_heads=4, visual_enc_depth=1, visual_heads=4, visual_image_size=64,
            visual_patch_size=16, visual_patch_dropout=0.0)
FILIP = dict(use_all_token_embeds=True)
EXTRA = dict(extra_latent_projection=True)
SIM_REG = dict(extra_latent_projection=True, sim_reg_loss_weight=0.3)
MLM = dict(use_mlm=True)

# name: (CLIP keywords, text views m, image views n)
CASES = {
    "plain": ({}, 1, 1),
    "dcl_extra": (dict(decoupled_contrastive_learning=True, **EXTRA), 1, 1),
    "sim_reg": (SIM_REG, 1, 1),
    "sim_reg_mlm": (dict(**SIM_REG, **MLM), 1, 1),
    "sigmoid": (dict(sigmoid_loss=True), 1, 1),
    "sigmoid_views": (dict(sigmoid_loss=True), 2, 2),
    "cls_views": ({}, 2, 3),
    "cls_views_extra_mlm": (dict(**EXTRA, **MLM), 1, 2),
    "filip": (FILIP, 1, 1),
    "filip_mlm": (dict(**FILIP, **MLM), 1, 1),
    "filip_extra": (dict(**FILIP, **EXTRA), 1, 1),
    "filip_views_1x2": (FILIP, 1, 2),
    "filip_views_2x1": (FILIP, 2, 1),
    "filip_views_3x2": (FILIP, 3, 2),
    "filip_views_mlm": (dict(**FILIP, **MLM), 2, 2),
}


class _Enc(torch.nn.Module):
    """A pluggable tower: [b, ...] -> [b, 1 + tokens, dim] that depends on the input."""

    def __init__(self, tokens, dim):
        super().__init__()
        self.tokens, self.dim = tokens, dim

    def forward(self, x, mask=None):
        seed = x.reshape(x.shape[0], -1).float().sum(dim=1)
        return seed[:, None, None] + torch.zeros(x.shape[0], 1 + self.tokens, self.dim)


class _Recorder:
    """Stands in for a Function's apply: keeps the arguments of every call and returns base + k / 16 for
    the k-th call, so that every Function and every view pair gives a value of its own."""

    def __init__(self, base):
        self.base, self.calls = base, []

    def __call__(self, *args):
        self.calls.append(args)
        return torch.tensor(self.base + (len(self.calls) - 1) / 16.0)

    def values(self):
        return [self.base + k / 16.0 for k in range(len(self.calls))]


def _run(monkeypatch, kw, m, n):
    import x_clip_b200.clip as C
    real = C._require
    monkeypatch.setattr(C, "_require", lambda cond, msg: None if "CUDA" in msg else real(cond, msg))
    # the identity projection; its operands are plain tensors, as the view pairs slice them
    monkeypatch.setattr(C.CLIP, "_project", lambda self, e, lin: (e.float(), (e.float(), e.float() + 1.0)))
    rec = dict(contrastive=_Recorder(1.25), sigmoid=_Recorder(2.5), filip=_Recorder(3.75), mlm=_Recorder(5.5))
    monkeypatch.setattr(E.ContrastiveLossFn, "apply", rec["contrastive"])
    monkeypatch.setattr(E.SigmoidLossFn, "apply", rec["sigmoid"])
    monkeypatch.setattr(F.FilipLossFn, "apply", rec["filip"])
    monkeypatch.setattr(E.VocabCrossEntropyFn, "apply", rec["mlm"])
    clip = x_clip_b200.CLIP(**TINY, **kw, text_encoder=_Enc(16, 256), image_encoder=_Enc(16, 256))
    clip.train()
    b = 3
    torch.manual_seed(0)
    text = torch.randint(1, 128, (b, 16))
    image = torch.randn(b, 3, 64, 64)
    aug_t = [text.clone().masked_fill(torch.rand(b, 16) < 0.5, 0) for _ in range(m - 1)]
    aug_i = [torch.randn(b, 3, 64, 64) for _ in range(n - 1)]
    loss = clip(text, image, return_loss=True, aug_text=tuple(aug_t) or None, aug_image=tuple(aug_i) or None)
    return clip, rec, loss, [text] + aug_t, [image] + aug_i


@pytest.mark.parametrize("case", list(CASES))
def test_loss_head(monkeypatch, case):
    kw, m, n = CASES[case]
    clip, rec, loss, texts, images = _run(monkeypatch, kw, m, n)
    b = texts[0].shape[0]
    filip = clip.use_all_token_embeds
    extra = clip.extra_latent_projection
    main = "filip" if filip else "sigmoid" if clip.sigmoid_loss else "contrastive"
    assert {k for k, r in rec.items() if r.calls} == {main} | ({"mlm"} if clip.use_mlm else set())

    tw, iw = clip.text_ssl_loss_weight, clip.image_ssl_loss_weight
    mv_w = clip.multiview_loss_weight if m * n > 1 else 0
    cl_w = 1 - (tw + iw + mv_w)
    calls = rec[main].calls
    if filip:
        # every (text view, image view) pair in one call, weighted inside the loss when there are views
        assert len(calls) == 1
        zt, zi, zt_x, zi_x, temperature, ops, mask = calls[0][:7]
        views = calls[0][10] if len(calls[0]) > 10 else (1, 1)
        assert views == (m, n)
        if m * n > 1:
            assert calls[0][11] == pytest.approx((cl_w, mv_w))
        assert zt.shape[0] == m * b and zi.shape[0] == n * b
        assert torch.equal(mask, torch.cat(texts) != 0)
        assert temperature is clip.temperature
        assert (zt_x is None, zi_x is None) == (not extra, not extra)
        assert len(ops) == (4 if extra else 2)
        weighted_inside = m * n > 1
    else:
        # one call per (text view i, image view j) pair, in the order i * n + j
        assert len(calls) == m * n
        lat = lambda enc, x: enc(x)[:, 0].float()
        for k, args in enumerate(calls):
            i, j = divmod(k, n)
            assert torch.equal(args[0], lat(clip.text_transformer, texts[i]))
            assert torch.equal(args[1], lat(clip.visual_transformer, images[j]))
            if clip.sigmoid_loss:
                temperature, logit_bias, ops = args[2], args[3], args[4]
                assert logit_bias is clip.logit_bias
            else:
                zt_x, zi_x, temperature, ops, dcl = args[2], args[3], args[4], args[5], args[6]
                assert dcl == clip.decoupled_contrastive_learning
                assert (zt_x is None, zi_x is None) == (not extra, not extra)
                if extra:
                    assert torch.equal(zt_x, args[0]) and torch.equal(zi_x, args[1])
                # the similarity regularisation weighs its contrastive term itself: (w, cl_w)
                if clip.has_sim_reg_loss:
                    assert args[8:] == pytest.approx((clip.sim_reg_loss_weight, cl_w))
                else:
                    assert args[8:] == ()
            assert temperature is clip.temperature
            assert len(ops) == (4 if extra else 2)
            for o, z in zip(ops, (args[0], args[1]) * 2):
                assert torch.equal(o[0], z) and torch.equal(o[1], z + 1.0)
        weighted_inside = clip.has_sim_reg_loss

    if clip.use_mlm:
        assert len(rec["mlm"].calls) == 1
        rows, weight, bias, labels = rec["mlm"].calls[0]
        assert weight is clip.mlm.to_logits.weight and bias is clip.mlm.to_logits.bias
        assert rows.shape[0] == labels.shape[0] > 0
    values = rec[main].values()
    mlm = rec["mlm"].values()[0] if clip.use_mlm else 0.0
    if weighted_inside:
        want = values[0] + mlm * tw
    else:
        others = values[1:]
        want = values[0] * cl_w + mlm * tw + (sum(others) / len(others) * mv_w if others else 0.0)
    assert loss.item() == pytest.approx(want, rel=1e-6)

