"""FILIP with augmented views (x_clip.py:625-650, :797-811, :821-868) restated on the oracle's pieces.

oracle.clip_oracle.clip_forward_multiview covers the CLS loss only, and step_oracle.filip_loss is called
with the original text's mask for every view.  Here every text view is masked by its own pad pattern:
t2i[i, j] takes the masked mean over text view i's valid tokens, i2t[i, j] fills text view i's padded
tokens with -max.  The image views go through one encoder call over the concatenated batch, as in
the reference.  Loss: (1 - w) * L[0, 0] + w * mean(the other m n - 1 pairs), where L[i, j] is
oracle.contrastive_loss of text view i against image view j."""
from __future__ import annotations

from typing import Optional, Sequence

import torch

from oracle import clip_oracle as O


def view_losses(zts, zis, temperature, cfg, masks):
    """[L[i, j] for i over text views for j over image views]; zts / zis: lists of (z, z_extra)."""
    out = []
    for (zt, ztx), mask in zip(zts, masks):
        for (zi, zix) in zis:
            out.append(O.contrastive_loss(zt, zi, ztx, zix, temperature, cfg, mask))
    return out


def combine(losses, multiview_loss_weight: float):
    w = multiview_loss_weight
    return losses[0] * (1 - w) + torch.stack(losses[1:]).mean() * w


def latents(p, texts: Sequence[torch.Tensor], images: Sequence[torch.Tensor], cfg: O.ClipConfig,
            keep: Optional[torch.Tensor] = None):
    """-> (zts, zis, masks): per text view (zt, zt_x) [b, T, D], per image view (zi, zi_x) [b, I, D]."""
    b = texts[0].shape[0]
    text = torch.cat(list(texts))
    mask = text != cfg.text_pad_id
    et = O.encode_text(text, mask, p, cfg)
    ei = O.encode_image(torch.cat(list(images)), p, cfg, keep)
    zt, zi, zt_x, zi_x = O.project_latents(et, ei, p, cfg)
    zts = [(zt[v * b:(v + 1) * b], zt_x[v * b:(v + 1) * b]) for v in range(len(texts))]
    zis = [(zi[v * b:(v + 1) * b], zi_x[v * b:(v + 1) * b]) for v in range(len(images))]
    masks = [mask[v * b:(v + 1) * b] for v in range(len(texts))]
    return zts, zis, masks


def clip_forward_filip_multiview(p, texts, images, cfg: O.ClipConfig, multiview_loss_weight: float = 0.1,
                                 keep: Optional[torch.Tensor] = None):
    """CLIP(use_all_token_embeds=True)(texts[0], images[0], return_loss=True, aug_text=texts[1:],
    aug_image=images[1:]); keep: PatchDropout's kept indices over the concatenated image batch."""
    assert cfg.use_all_token_embeds and len(texts) * len(images) > 1
    zts, zis, masks = latents(p, texts, images, cfg, keep)
    return combine(view_losses(zts, zis, p["temperature"], cfg, masks), multiview_loss_weight)
