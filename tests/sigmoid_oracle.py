"""fp64 reference of the pairwise sigmoid loss (SigLIP) and of CLIP(sigmoid_loss=True)'s training step.
TEST INFRASTRUCTURE ONLY.

    l_ij = exp(temperature) <t_i, v_j> + logit_bias,   z_ij = +1 if i == j else -1
    L = (1/B) sum_ij softplus(-z_ij l_ij)

The step restates step_oracle.step_loss with this loss in place of InfoNCE, on step_oracle's encoders and
oracle.clip_oracle.project_latents; the MLM and SimCLR terms and the multiview weights are step_oracle's.
Used by test_sigmoid_loss.py (CPU) and test_gpu_sigmoid_loss.py (H100).
"""
from __future__ import annotations

import math
from typing import Sequence
from unittest import mock

import torch

import multirank_oracle as MR
import step_oracle as SO
from oracle import clip_oracle as O

INIT_TEMPERATURE = math.log(10.0)
INIT_LOGIT_BIAS = -10.0


def logits(zt, zi, temperature, logit_bias):
    return temperature.exp() * (zt @ zi.t()) + logit_bias


def labels(rows: int, cols: int, diag_offset: int = 0, like=None):
    """z [rows, cols]: +1 at (r, r + diag_offset), -1 elsewhere."""
    z = -torch.ones((rows, cols), dtype=like.dtype if like is not None else torch.float64,
                    device=like.device if like is not None else None)
    r = torch.arange(rows, device=z.device)
    z[r, r + diag_offset] = 1.0
    return z


def softplus(x):
    """log(1 + e^x) without F.softplus's linear branch above x = 20 (an error of e^-20 per term)."""
    return x.clamp_min(0.0) + torch.log1p(torch.exp(-x.abs()))


def sigmoid_loss(zt, zi, temperature, logit_bias):
    """The loss of the global batch: zt, zi [B, D] unit rows."""
    lg = logits(zt, zi, temperature, logit_bias)
    return softplus(-labels(*lg.shape, like=lg) * lg).sum() / zt.shape[0]


def rank_share(zt, zi, temperature, logit_bias, world: int, rank: int):
    """Rank `rank`'s part of the loss: its b = B / world texts against all B images, over the global B.
    The shares of all ranks sum to sigmoid_loss."""
    B = zt.shape[0]
    b = B // world
    lg = logits(zt[rank * b:(rank + 1) * b], zi, temperature, logit_bias)
    return softplus(-labels(b, B, rank * b, like=lg) * lg).sum() / B


# --------------------------------------------------------------------------- whole step

def make_case(name: str, spec: dict, world: int = 1, b: int = None) -> dict:
    """step_oracle.make_case of `spec` with sigmoid_loss=True (at the global batch world * b when b is
    given), temperature and logit_bias at SigLIP's initial values.  Build it after init_process_group
    when world > 1."""
    spec = dict(spec, kw=dict(spec.get("kw", {}), sigmoid_loss=True))
    if b is not None:
        spec["batch"] = world * b
    key = f"sigmoid_{name}_w{world}"
    with mock.patch.dict(SO.CASES, {key: spec}):
        c = SO.make_case(key)
    clip = c["model"]
    with torch.no_grad():
        clip.temperature.fill_(INIT_TEMPERATURE)
        clip.logit_bias.fill_(INIT_LOGIT_BIAS)
    c["params"]["temperature"] = clip.temperature.detach().clone()
    c["params"]["logit_bias"] = clip.logit_bias.detach().clone()
    c.update(world=world, b=b)
    return c


def step_loss(p, c, texts: Sequence[torch.Tensor], images: Sequence[torch.Tensor], keep=None):
    """CLIP(sigmoid_loss=True).forward(texts[0], images[0], return_loss=True, aug_text=texts[1:],
    aug_image=images[1:]): every (text view, image view) pair is a sigmoid loss of its own, weighted
    as step_oracle.step_loss weighs the InfoNCE pairs."""
    cfg, kw = c["cfg"], c["kw"]
    pad = cfg.text_pad_id
    text_ssl_w = kw.get("text_ssl_loss_weight", 0.05) if kw.get("use_mlm") else 0.0
    image_ssl_w = kw.get("image_ssl_loss_weight", 0.05) if kw.get("use_visual_ssl") else 0.0
    multiview = len(texts) > 1 or len(images) > 1
    mv_w = kw.get("multiview_loss_weight", 0.1) if multiview else 0.0
    enc_t = [SO.encode_text(p, t, cfg, None if kw.get("text_encode_without_mask") else t != pad) for t in texts]
    enc_i = [SO.encode_image(p, im, cfg, keep if v == 0 else None) for v, im in enumerate(images)]
    losses = []
    for et in enc_t:
        for ei in enc_i:
            zt, zi, _, _ = O.project_latents(et, ei, p, cfg)
            losses.append(sigmoid_loss(zt, zi, p["temperature"], p["logit_bias"]))
    loss = (1.0 - (text_ssl_w + image_ssl_w + mv_w)) * losses[0]
    if multiview:
        loss = loss + mv_w * torch.stack(losses[1:]).mean()
    if text_ssl_w:
        masked, lab = (t.to(texts[0].device) for t in c["mlm"])
        loss = loss + text_ssl_w * SO.mlm_loss(p, cfg, masked, lab, texts[0] != pad, pad)
    if image_ssl_w:
        loss = loss + image_ssl_w * SO.simclr_loss(p, images[0], cfg, kw.get("simclr_temperature", 0.1))
    return loss


def reference(c, device, keep=None) -> dict:
    """fp64 loss and gradients of one step of case `c`: dict(loss, grads {name: tensor or None},
    image_grads [per view, or None]), as step_oracle.reference."""
    p = {k: v.to(device).double().requires_grad_(not c["frozen"]) for k, v in c["params"].items()}
    text, image = c["batches"][0]
    texts = [t.to(device) for t in [text] + c["aug_text"]]
    images = [im.to(device).double().requires_grad_(c["image_grad"]) for im in [image] + c["aug_image"]]
    if keep is None and c["keep"] is not None:
        keep = c["keep"]
    keep = None if keep is None else keep.to(device)
    with SO.pinned():
        loss = step_loss(p, c, texts, images, keep)
        loss.backward()
    return dict(loss=loss.item(), grads={k: v.grad for k, v in p.items()},
                image_grads=[im.grad for im in images] if c["image_grad"] else None)


def rank_reference(c, device, world: int, rank: int, keep=None) -> dict:
    """What rank `rank` of `world` must compute: the global batch's step with gradients through rank
    `rank`'s latents only (multirank_oracle's contract; the other ranks' latents are constants)."""
    with MR._only_rank_rows("unit_rows", world, rank):
        return reference(c, device, keep)
