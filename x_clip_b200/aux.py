"""Auxiliary self-supervised losses of x-clip run THROUGH the fast encoders (SURVEY.md 8f rank 4).

The reference wraps its encoders in generic torch modules: `MLM` (x_clip/mlm.py:40-107, masked
language modelling on the text transformer), `SimSiam` / `SimCLR` (x_clip/visual_ssl.py, a
BYOL-style wrapper around the vision transformer) and mixes their losses into the contrastive
loss (x_clip/x_clip.py:611-621, :851-868).  Here the same objectives are written against the
H100 encoders of this package: the expensive part - every encoder pass - runs on the CUDA kernels
(engine.TransformerFn), the MLM head's vocabulary projection and its cross entropy run as one
wgmma GEMM with the softmax in its epilogue over the MASKED positions only
(engine.VocabCrossEntropyFn: no [n_sel, V] logits, any vocabulary size), and the SimCLR augmentation
of the two views runs as two CUDA kernels with torchvision's draws and arithmetic (SimCLRAugmentation:
the torchvision pipeline's own temporaries do not fit at thousands of images per GPU).  The small
heads (BatchNorm MLPs, cosine / NT-Xent losses) stay ordinary torch modules, exactly as in the
reference - they are not on the north-star path.

Parameter names follow the reference (`mlm.to_logits.*`, `visual_ssl.online_encoder.*`) where the
reference has parameters; masks and augmentations are random in both implementations, so parity is
checked on the deterministic parts (tests/test_gpu_aux.py: a fixed masking, identity augmentation).
"""
from __future__ import annotations

import math
from typing import NamedTuple, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F
from torch import nn

from . import engine as E


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
        return self.loss_from_rows(enc[sel], labels[sel])

    def loss_from_rows(self, rows: torch.Tensor, labels: torch.Tensor) -> torch.Tensor:
        """The head on the encodings of the selected positions, rows [n_sel, dim], against their tokens:
        the mean over the selected positions == F.cross_entropy(..., ignore_index=pad) of the reference,
        fused into the vocabulary GEMM for any vocabulary size (no [n_sel, V] logits are written).  No
        selected position gives 0, still connected to the encoder."""
        if rows.shape[0] == 0:
            return rows.sum() * 0.
        return E.VocabCrossEntropyFn.apply(rows, self.to_logits.weight, self.to_logits.bias, labels)

    def forward(self, seq: torch.Tensor, **kwargs) -> torch.Tensor:
        masked, labels = self.corrupt(seq)
        return self.loss_from(masked, labels, **kwargs)


# ----------------------------------------------------------------------------- visual SSL

class AugmentParams(NamedTuple):
    """The draws of one call of the SimCLR augmentation (SimCLRAugmentation.draw), for the whole batch.
    order: the colour-jitter op ids (0 brightness, 1 contrast, 2 saturation, 3 hue) in the drawn order,
    () when the jitter does not apply; factors: the four jitter factors indexed by op id (None skips an
    op); sigma: the blur's sigma, None when the blur does not apply; crop: (top, left, height, width)."""
    order: Tuple[int, ...]
    factors: Tuple[Optional[float], ...]
    grayscale: bool
    flip: bool
    sigma: Optional[float]
    crop: Tuple[int, int, int, int]


class SimCLRAugmentation(nn.Module):
    """The SimCLR-style pipeline the reference builds (visual_ssl.py:59-88) from torchvision:

        RandomApply(ColorJitter(0.8, 0.8, 0.8, 0.2), p=0.3)      (RGB only)
        RandomGrayscale(p=0.2)                                    (RGB only)
        RandomHorizontalFlip()
        RandomApply(GaussianBlur((3, 3), (1.0, 2.0)), p=0.2)     (channels > 1)
        RandomResizedCrop((image_size, image_size))
        Normalize(ImageNet mean / std)                            (RGB only)

    as one decision per call for the whole batch.  `draw(shape)` takes every parameter from
    torchvision's own get_params / torch.rand calls in the Sequential's order (CPU generator only, from
    the shape alone: no host synchronisation); `apply(x, params)` applies them.  A CUDA input that does
    not take part in autograd runs the CUDA kernels (kernels.augment: one HBM read of the input, one
    more when contrast needs its per-image mean, one write of the view), which is what lets SimSiam /
    SimCLR augment thousands of images per GPU at once; an input that requires grad (or a CPU input)
    takes torchvision's functional ops with the same parameters, so the image still gets a gradient.
    Registers no parameters or buffers."""

    BLUR_P, JITTER_P, GRAY_P = 0.2, 0.3, 0.2
    MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)

    def __init__(self, image_size: int, channels: int = 3):
        super().__init__()
        from torchvision import transforms as T
        self.image_size, self.channels = int(image_size), int(channels)
        self.rgb, self.blurs = channels == 3, channels > 1
        jitter = T.ColorJitter(0.8, 0.8, 0.8, 0.2)
        self._jitter = (jitter.brightness, jitter.contrast, jitter.saturation, jitter.hue)
        crop = T.RandomResizedCrop((self.image_size, self.image_size))
        self._scale, self._ratio = crop.scale, crop.ratio
        self._blur_sigma = T.GaussianBlur((3, 3), (1.0, 2.0)).sigma

    def draw(self, shape) -> AugmentParams:
        from torchvision import transforms as T
        order, factors, gray = (), (None,) * 4, False
        if self.rgb:
            if not torch.rand(()) > self.JITTER_P:                # the reference's RandomApply
                fn_idx, *factors = T.ColorJitter.get_params(*self._jitter)
                order, factors = tuple(int(i) for i in fn_idx), tuple(factors)
            gray = bool(torch.rand(1) < self.GRAY_P)
        flip = bool(torch.rand(1) < 0.5)
        sigma = None
        if self.blurs and not torch.rand(()) > self.BLUR_P:
            sigma = T.GaussianBlur.get_params(*self._blur_sigma)
        crop = T.RandomResizedCrop.get_params(torch.empty(tuple(shape), device="meta"), self._scale, self._ratio)
        return AugmentParams(order, factors, gray, flip, sigma, tuple(int(v) for v in crop))

    def apply(self, x: torch.Tensor, params: AugmentParams) -> torch.Tensor:
        if x.is_cuda and not (x.requires_grad and torch.is_grad_enabled()):
            return self._apply_kernels(x, params)
        return self.apply_torchvision(x, params)

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        return self.apply(x, self.draw(x.shape))

    def apply_torchvision(self, x: torch.Tensor, params: AugmentParams) -> torch.Tensor:
        """The same parameters through torchvision's functional ops (any device, dtype and autograd)."""
        from torchvision.transforms import functional as TF
        jitter = (TF.adjust_brightness, TF.adjust_contrast, TF.adjust_saturation, TF.adjust_hue)
        for op in params.order:
            if params.factors[op] is not None:
                x = jitter[op](x, params.factors[op])
        if params.grayscale:
            x = TF.rgb_to_grayscale(x, num_output_channels=x.shape[-3])
        if params.flip:
            x = TF.hflip(x)
        if params.sigma is not None:
            x = TF.gaussian_blur(x, [3, 3], [params.sigma, params.sigma])
        x = TF.resized_crop(x, *params.crop, [self.image_size, self.image_size],
                            TF.InterpolationMode.BILINEAR, antialias=True)
        if self.rgb:
            x = TF.normalize(x, torch.tensor(self.MEAN), torch.tensor(self.STD))
        return x

    def _apply_kernels(self, x: torch.Tensor, params: AugmentParams) -> torch.Tensor:
        from . import kernels as K
        ops = [op for op in params.order if params.factors[op] is not None]
        factor = [0.0 if f is None else float(f) for f in params.factors]
        # _blend's (1.0 - ratio) is a double rounded to fp32 when it scales the fp32 image
        one_minus = [1.0 - f for f in factor]
        blur = None
        if params.sigma is not None:
            from torchvision.transforms._functional_tensor import _get_gaussian_kernel2d
            blur = _get_gaussian_kernel2d([3, 3], [params.sigma, params.sigma], torch.float32,
                                          torch.device("cpu")).flatten().tolist()
        squeeze = x.dim() == 3
        out = K.augment(x.unsqueeze(0) if squeeze else x, ops=ops, factor=factor, one_minus=one_minus,
                        grayscale=params.grayscale, flip=params.flip, blur_kernel=blur,
                        normalize=(self.MEAN, self.STD) if self.rgb else None, crop=params.crop,
                        out_size=(self.image_size, self.image_size))
        return out[0] if squeeze else out


def default_augmentation(image_size: int, channels: int = 3) -> nn.Module:
    """The SimCLR-style pipeline the reference builds (visual_ssl.py:59-88): SimCLRAugmentation."""
    return SimCLRAugmentation(image_size, channels)


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

    def rep(self, x):
        rep = self.net(x)
        rep = rep[:, 0] if rep.ndim == 3 else rep
        return rep.float()

    def forward(self, x):
        rep = self.rep(x)
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
        enc = self.online_encoder
        r1, r2 = enc.rep(one), enc.rep(two)
        with torch.no_grad():
            t1, t2 = enc.rep(one), enc.rep(two)
        return self.loss_from_reps(r1, r2, t1, t2)

    def loss_from_reps(self, r1, r2, t1, t2):
        """The head on the encoders' CLS representations: r1 / r2 of the two views (with gradient),
        t1 / t2 the same views encoded again without gradient (their own patch-dropout draws).  The
        BatchNorm layers run in the order of the reference's forward: projector on r1, r2, predictor on
        both, projector on t1, t2 - so their running statistics end as they would there."""
        proj = self.online_encoder.projector
        p1, p2 = proj(r1), proj(r2)
        q1, q2 = self.online_predictor(p1), self.online_predictor(p2)
        with torch.no_grad():
            z1, z2 = proj(t1), proj(t2)
        return (self._neg_cos(q1, z2.detach()) + self._neg_cos(q2, z1.detach())).mean()


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
        return self.loss_from_reps(self.net.rep(self.augment1(x)), self.net.rep(self.augment2(x)))

    def loss_from_reps(self, r1, r2):
        """NT-Xent on the encoders' CLS representations of the two views."""
        b = r1.shape[0]
        q, k = self.net.projector(r1), self.net.projector(r2)
        z = torch.cat((q, k), dim=0)                 # (not normalised, as in the reference's nt_xent_loss)
        logits = z @ z.t() / self.temperature
        logits = logits.masked_fill(torch.eye(2 * b, dtype=torch.bool, device=z.device), -torch.finfo(logits.dtype).max)
        target = torch.cat((torch.arange(b, 2 * b), torch.arange(0, b))).to(z.device)
        return F.cross_entropy(logits, target)
