"""Auxiliary self-supervised losses of x-clip run THROUGH the fast encoders (SURVEY.md 8f rank 4).

The reference wraps its encoders in generic torch modules: `MLM` (x_clip/mlm.py:40-107, masked
language modelling on the text transformer), `SimSiam` / `SimCLR` (x_clip/visual_ssl.py, a
BYOL-style wrapper around the vision transformer) and mixes their losses into the contrastive
loss (x_clip/x_clip.py:611-621, :851-868).  Here the same objectives are written against the
H100 encoders of this package: the expensive part - every encoder pass - runs on the CUDA kernels
(engine.TransformerFn), the vocabulary projection of the MLM head runs on the wgmma GEMM over the
MASKED positions only (engine.LinearFn), and the small heads (cross entropy over the selected
rows, BatchNorm MLPs, cosine / NT-Xent losses, torchvision augmentations) stay ordinary torch
modules, exactly as in the reference - they are not on the north-star path.

Parameter names follow the reference (`mlm.to_logits.*`, `visual_ssl.online_encoder.*`) where the
reference has parameters; masks and augmentations are random in both implementations, so parity is
checked on the deterministic parts (tests/test_gpu_aux.py: a fixed masking, identity augmentation).
"""
from __future__ import annotations

import math
from typing import Optional, Sequence

import torch
import torch.nn.functional as F
from torch import nn

from . import engine as E

BF16 = torch.bfloat16


# ----------------------------------------------------------------------------- MLM

class MLM(nn.Module):
    """Masked language modelling head on the text transformer (reference mlm.py:40-107).

    forward(seq, mask=...) -> scalar loss: choose ceil(mask_prob * n) of the maskable tokens per
    row, replace `replace_prob` of them by the [MASK] id (optionally some by random tokens), encode
    the corrupted sequence with the FAST text transformer, project the encodings of the chosen
    positions onto the vocabulary and take the cross entropy against the original tokens."""

    def __init__(self, transformer: nn.Module, *, dim: int, num_tokens: int, mask_prob: float = 0.15,
                 replace_prob: float = 0.9, random_token_prob: float = 0., mask_token_id: int = 2,
                 pad_token_id: int = 0, mask_ignore_token_ids: Sequence[int] = ()):
        super().__init__()
        self.transformer = transformer
        self.mask_prob, self.replace_prob = mask_prob, replace_prob
        self.num_tokens, self.random_token_prob = num_tokens, random_token_prob
        self.pad_token_id, self.mask_token_id = pad_token_id, mask_token_id
        self.mask_ignore_token_ids = set([*mask_ignore_token_ids, pad_token_id])
        self.to_logits = nn.Linear(dim, num_tokens)

    def _excluded(self, t: torch.Tensor) -> torch.Tensor:
        out = torch.zeros_like(t, dtype=torch.bool)
        for tok in self.mask_ignore_token_ids:
            out |= t == tok
        return out

    def corrupt(self, seq: torch.Tensor):
        """-> (masked_seq, labels): labels hold the original token at the chosen positions and the
        pad id elsewhere (ignored by the loss), reference mlm.py:69-95."""
        b, n = seq.shape
        can = ~self._excluded(seq)
        # ceil(prob * #maskable) positions per row, uniformly among the maskable ones
        quota = (can.sum(dim=-1, keepdim=True) * self.mask_prob).ceil()
        score = torch.rand((b, n), device=seq.device).masked_fill(~can, -1.)
        rank = score.argsort(dim=-1, descending=True).argsort(dim=-1)        # 0 = highest score
        chosen = (rank < quota) & can
        labels = seq.masked_fill(~chosen, self.pad_token_id)
        masked = seq.clone()
        if self.random_token_prob > 0:
            rnd_where = (torch.rand((b, n), device=seq.device) < self.random_token_prob)
            rnd_tok = torch.randint(0, self.num_tokens, (b, n), device=seq.device)
            rnd_where &= ~self._excluded(rnd_tok)
            masked = torch.where(rnd_where, rnd_tok, masked)
            chosen = chosen & ~rnd_where
        replace = torch.rand((b, n), device=seq.device) < self.replace_prob
        masked = masked.masked_fill(chosen & replace, self.mask_token_id)
        return masked, labels

    def loss_from(self, masked_seq: torch.Tensor, labels: torch.Tensor, **kwargs) -> torch.Tensor:
        enc = self.transformer(masked_seq, **kwargs)[:, 1:]                  # drop CLS (mlm.py:98-99)
        sel = labels != self.pad_token_id                                     # ignore_index rows
        rows = enc[sel]                                                       # [n_sel, dim] bf16
        if rows.shape[0] == 0:
            return enc.sum() * 0.
        if rows.is_cuda and rows.dtype == BF16 and self.num_tokens % 8 == 0:
            logits = E.LinearFn.apply(rows.contiguous(), self.to_logits.weight, self.to_logits.bias, None)
        else:                           # vocabulary not a multiple of 8 (e.g. 10000 + [MASK]): torch matmul
            logits = F.linear(rows.float(), self.to_logits.weight, self.to_logits.bias)
        # mean over the selected positions == F.cross_entropy(..., ignore_index=pad) of the reference
        return F.cross_entropy(logits.float(), labels[sel])

    def forward(self, seq: torch.Tensor, **kwargs) -> torch.Tensor:
        masked, labels = self.corrupt(seq)
        return self.loss_from(masked, labels, **kwargs)


# ----------------------------------------------------------------------------- visual SSL

def default_augmentation(image_size: int, channels: int = 3) -> nn.Module:
    """The SimCLR-style pipeline the reference builds (visual_ssl.py:59-88) from torchvision."""
    from torchvision import transforms as T

    class RandomApply(nn.Module):
        def __init__(self, fn, p):
            super().__init__()
            self.fn, self.p = fn, p

        def forward(self, x):
            return x if torch.rand(()) > self.p else self.fn(x)

    is_rgb = channels == 3
    is_gt1 = channels > 1
    return nn.Sequential(
        RandomApply(T.ColorJitter(0.8, 0.8, 0.8, 0.2), p=0.3) if is_rgb else nn.Identity(),
        T.RandomGrayscale(p=0.2) if is_rgb else nn.Identity(),
        T.RandomHorizontalFlip(),
        RandomApply(T.GaussianBlur((3, 3), (1.0, 2.0)), p=0.2) if is_gt1 else nn.Identity(),
        T.RandomResizedCrop((image_size, image_size)),
        T.Normalize(mean=torch.tensor([0.485, 0.456, 0.406]), std=torch.tensor([0.229, 0.224, 0.225]))
        if is_rgb else nn.Identity(),
    )


def _mlp(dim: int, out: int, hidden: int) -> nn.Sequential:
    return nn.Sequential(nn.Linear(dim, hidden), nn.BatchNorm1d(hidden), nn.ReLU(inplace=True),
                         nn.Linear(hidden, out))


class _Projected(nn.Module):
    """representation = CLS token of the fast vision transformer (the reference hooks the LAST child
    of the net, `to_cls_tokens`, visual_ssl.py:105-150 with hidden_layer=-1) -> projector MLP."""

    def __init__(self, net: nn.Module, rep_dim: int, projection_size: int, hidden: int):
        super().__init__()
        self.net = net
        self.projector = _mlp(rep_dim, projection_size, hidden)

    def forward(self, x):
        rep = self.net(x)
        rep = rep[:, 0] if rep.ndim == 3 else rep
        rep = rep.float()
        return self.projector(rep), rep


class SimSiam(nn.Module):
    """Negative-cosine SimSiam objective (reference visual_ssl.py:207-259) on two augmented views."""

    def __init__(self, net: nn.Module, image_size: int, channels: int = 3, rep_dim: Optional[int] = None,
                 projection_size: int = 256, projection_hidden_size: int = 4096, augment_fn=None,
                 augment_fn2=None):
        super().__init__()
        rep_dim = rep_dim or getattr(getattr(net, "transformer", None), "dim", None)
        assert rep_dim, "SimSiam: pass rep_dim (width of the encoder's CLS representation)"
        self.augment1 = augment_fn if augment_fn is not None else default_augmentation(image_size, channels)
        self.augment2 = augment_fn2 if augment_fn2 is not None else self.augment1
        self.online_encoder = _Projected(net, rep_dim, projection_size, projection_hidden_size)
        self.online_predictor = _mlp(projection_size, projection_size, projection_hidden_size)

    @staticmethod
    def _neg_cos(p, z):
        return 2 - 2 * (F.normalize(p, dim=-1) * F.normalize(z, dim=-1)).sum(dim=-1)

    def forward(self, x):
        assert not (self.training and x.shape[0] == 1), \
            'you must have greater than 1 sample when training, due to the batchnorm in the projection layer'
        one, two = self.augment1(x), self.augment2(x)
        p1, _ = self.online_encoder(one)
        p2, _ = self.online_encoder(two)
        q1, q2 = self.online_predictor(p1), self.online_predictor(p2)
        with torch.no_grad():
            t1, _ = self.online_encoder(one)
            t2, _ = self.online_encoder(two)
        return (self._neg_cos(q1, t2.detach()) + self._neg_cos(q2, t1.detach())).mean()


class SimCLR(nn.Module):
    """NT-Xent over two augmented views (reference visual_ssl.py:263-end)."""

    def __init__(self, net: nn.Module, image_size: int, channels: int = 3, rep_dim: Optional[int] = None,
                 project_hidden: bool = True, project_dim: int = 128, temperature: float = 0.1,
                 augment_fn=None, augment_fn2=None, **_):
        super().__init__()
        rep_dim = rep_dim or getattr(getattr(net, "transformer", None), "dim", None)
        assert rep_dim, "SimCLR: pass rep_dim (width of the encoder's CLS representation)"
        self.net = _Projected(net, rep_dim, project_dim, 4096 if project_hidden else project_dim)
        self.temperature = temperature
        self.augment1 = augment_fn if augment_fn is not None else default_augmentation(image_size, channels)
        self.augment2 = augment_fn2 if augment_fn2 is not None else self.augment1

    def forward(self, x):
        b = x.shape[0]
        q, _ = self.net(self.augment1(x))
        k, _ = self.net(self.augment2(x))
        z = torch.cat((q, k), dim=0)                 # (not normalised, as in the reference's nt_xent_loss)
        logits = z @ z.t() / self.temperature
        logits = logits.masked_fill(torch.eye(2 * b, dtype=torch.bool, device=x.device), -torch.finfo(logits.dtype).max)
        target = torch.cat((torch.arange(b, 2 * b), torch.arange(0, b))).to(x.device)
        return F.cross_entropy(logits, target)
