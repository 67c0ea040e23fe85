"""CPU restatement of the similarity-regularisation term (arXiv 2309.08773; reference
x_clip/x_clip.py:771-784, :870-873) on top of oracle/clip_oracle.py.  TEST INFRASTRUCTURE ONLY.

    L_sim = ( mse(T T^T, V V^T) + mse(T' T'^T, V' V'^T) ) / 2     over the off-diagonal entries
    loss  = contrastive loss + sim_reg_loss_weight * L_sim

T, V are the unit-norm text / image latents of the GLOBAL batch, T', V' the *_extra pair.  The
reference runs the term only with extra_latent_projection=True, without FILIP and with one view;
at a global batch of 1 the means are over nothing and the term is NaN."""
from __future__ import annotations

from typing import Sequence

import torch

from oracle import clip_oracle as O

# Gates of the kernels xclip_simreg_fwd / _bwd against fp64 E = a b^T of their exact bf16 operands (shared
# by test_gpu_simreg.py and the per-call checks of bench_call_oracle.py; measured maxima from an H100 80GB
# HBM3 at a 700 W power limit).  E's own error is the tensor cores' fp32 accumulation over K = 6 D terms
# whose partial sums reach the size of <t_r, t_c>, not of E: measured at most 6.2e-7 absolute (an aligned
# case, |E| ~ 1e-4).  A row sum of E^2 may therefore miss 2 |E| E_ABS per entry on top of its relative
# error (measured 1.6e-5 where E is not small); g = bf16(gscale * E) one bf16 rounding (2^-9) plus
# gscale * E_ABS.
E_ABS = 1.5e-6
ROWSUM_REL = 5e-5
LOSS_REL = 1e-4        # loss_accum against fp64 (measured at most 4.3e-5); g measured at most 1.45e-6 beyond
G_REL = 2 ** -8        #   its bf16 rounding (gate 2.55e-6); row sums at most 0.16 of their gate


def sim_reg_loss(zt, zi, zt_x, zi_x):
    """(:777-784) F.mse_loss of the off-diagonal similarities, averaged over the two latent pairs."""
    off = ~torch.eye(zt.shape[0], dtype=torch.bool, device=zt.device)

    def mse(a, b):
        return ((a @ a.t())[off] - (b @ b.t())[off]).pow(2).mean()

    return (mse(zt, zi) + mse(zt_x, zi_x)) / 2


def clip_forward(p, text, image, cfg, sim_reg_loss_weight, keep=None, return_parts=False):
    """oracle.clip_forward plus sim_reg_loss_weight * L_sim (:870-873)."""
    loss, parts = O.clip_forward(p, text, image, cfg, keep=keep, return_parts=True)
    loss = loss + sim_reg_loss_weight * sim_reg_loss(
        parts["text_latents"], parts["image_latents"], parts["text_latents_extra"], parts["image_latents_extra"])
    return (loss, parts) if return_parts else loss


def clip_forward_sharded(p, texts: Sequence, images: Sequence, cfg, rank: int, sim_reg_loss_weight):
    """oracle.clip_forward_sharded with the term: every rank evaluates it on the gathered latents,
    the latents of the other ranks are constants (AllGather.backward, x_clip/distributed.py:50-54)."""
    lat = []
    for r, (t, im) in enumerate(zip(texts, images)):
        ctx = torch.enable_grad() if r == rank else torch.no_grad()
        with ctx:
            m = t != cfg.text_pad_id
            et = O.encode_text(t, m, p, cfg)
            if cfg.text_causal_mask:
                et = O.eos_to_front(et, t, cfg.text_eos_id)
            lat.append(O.project_latents(et, O.encode_image(im, p, cfg), p, cfg))
    cat = [torch.cat([z[j] for z in lat], dim=0) for j in range(4)]
    return O.contrastive_loss(cat[0], cat[1], cat[2], cat[3], p["temperature"], cfg) \
        + sim_reg_loss_weight * sim_reg_loss(*cat)
