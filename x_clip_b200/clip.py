"""Drop-in `CLIP` / `TextTransformer` / `VisionTransformer` for lucidrains/x-clip, H100 path.

The constructor keywords, forward signature, early returns, assertions and - crucially -
the parameter tree (`state_dict` keys and shapes, SURVEY.md 8b) mirror the reference
(x_clip/x_clip.py:295-390 and :412-875) so existing checkpoints and user code keep
working.  The modules here are parameter CONTAINERS: all arithmetic on the hot path is
done by the CUDA kernels behind include/xclip_b200.h, scheduled by x_clip_b200.engine.

Sequence length is not limited by the non-causal attention: image towers such as ViT-B/16 at 384 px
(576 patches) and long text towers run on the same kernels (streamed through shared memory above
320 tokens).  The FILIP loss (`use_all_token_embeds=True`) takes any number of text and image
tokens: cfg3's 77 x 196 (98 under patch dropout), 576-patch towers and grids smaller than 16 tokens
run on the same segment-max kernels.  Model and latent widths may be any multiple of 128 from 128 to
1024 (ViT-S at 384, B/16-plus at 640 / 896, tiny 128-wide ablations), with any head count: the
attention width heads * 64 need not equal the model width.  Any patch size works, ViT-L/14's 588
values per patch included: the patch embedding pads rows of channels * patch^2 values to a multiple of
8 with zero columns (engine.patch_rows), which adds exact zeros to its sums.  Feature combinations the kernels do not
cover raise at construction (never a silent CPU or eager fallback): dim_head != 64, model or latent
widths that are not 128 * {1..8}, a causal text tower longer than
128 tokens, rotary + causal together (broken in the reference itself: n+1 angles for n tokens,
x_clip.py:328) and conv-downsampled image latents.  Attention dropout (`attn_dropout`, 0 <= p <= 1)
runs inside the attention kernels, with a counter-based mask that a re-encode regenerates exactly
(engine.TransformerFn); `ff_dropout` is accepted and, as in the reference's Transformer
(x_clip.py:268), not applied.  MLM, SimSiam / SimCLR and the multiview term run through the fast encoders (aux.py);
with FILIP, the augmented views (`aug_text` / `aug_image`) run every (text view, image view) pair in one
pair of segment-max passes (filip.FilipLossFn), each text view masked by its own pad pattern.  The similarity-regularisation term
(`sim_reg_loss_weight > 0`) runs fused with the contrastive loss (engine.ContrastiveLossFn) where the
reference itself runs it: with `extra_latent_projection=True`, without FILIP and with a single view;
the other combinations fail inside the reference (x_clip.py:779) and raise `Unsupported` here.
`sigmoid_loss=True` (an extension) trains with SigLIP's pairwise sigmoid loss (engine.SigmoidLossFn) in
place of InfoNCE: a new scalar parameter `logit_bias` (initial -10) and `temperature` initialised to
log 10.  It runs in the single pass, with augmented views, MLM / SimSiam / SimCLR and in the micro-batched
step; FILIP, DCL and the extra latent projection (and so the similarity regularisation) raise `Unsupported`.
"""
from __future__ import annotations

import copy
import math
from typing import Optional

import torch
import torch.distributed as dist
from torch import nn

from . import engine as E
from .filip import FilipLossFn

BF16 = torch.bfloat16


class Unsupported(NotImplementedError):
    pass


def _require(cond: bool, msg: str) -> None:
    if not cond:
        raise Unsupported("x_clip_b200: " + msg + " (no fallback path exists by design)")


# ----------------------------------------------------------------------------- containers
# The nesting below exists only to reproduce the reference's parameter names, e.g.
# `transformer.layers.3.0.fn.to_out.1.g` or `to_tokens.1.weight`.

class LayerNorm(nn.Module):
    """gain-only LayerNorm parameter (reference :112-121)."""

    def __init__(self, dim: int):
        super().__init__()
        self.g = nn.Parameter(torch.ones(dim))


class _Slot(nn.Module):
    """Parameter-free placeholder keeping nn.Sequential indices aligned with the reference."""


class PreNorm(nn.Module):
    def __init__(self, dim: int, fn: nn.Module):
        super().__init__()
        self.norm = LayerNorm(dim)
        self.fn = fn


class Attention(nn.Module):
    def __init__(self, dim: int, dim_head: int = 64, heads: int = 8, causal: bool = False,
                 dropout: float = 0.):
        super().__init__()
        _require(dim_head == 64, f"dim_head must be 64, got {dim_head}")
        self.heads = heads
        self.causal = causal
        self.scale = dim_head ** -0.5
        inner = dim_head * heads
        self.to_qkv = nn.Linear(dim, inner * 3, bias=False)
        self.to_out = nn.Sequential(nn.Linear(inner, dim, bias=False), LayerNorm(dim))
        # parameter-free, as in the reference (:211): holds p (range-checked by nn.Dropout) and follows
        # train() / eval(); the dropout itself runs in the attention kernels
        self.dropout = nn.Dropout(dropout)


class FeedForward(nn.Module):
    def __init__(self, dim: int, mult: int = 4, dropout: float = 0.):
        super().__init__()
        _require(mult == 4, "feed-forward multiplier must be 4")
        _require(dropout == 0., "feed-forward dropout > 0 is not implemented")
        inner = dim * mult
        self.net = nn.Sequential(
            nn.Linear(dim, inner * 2, bias=False),   # value | gate
            _Slot(),                                 # GEGLU
            LayerNorm(inner),
            _Slot(),                                 # Dropout(0)
            nn.Linear(inner, dim, bias=False),
        )


class Transformer(nn.Module):
    """norm_in -> depth x (attention, feed-forward) -> norm_out, executed by engine.TransformerFn.

    Attention dropout is active, as nn.Dropout is, iff the layer's `dropout` module is in training mode
    and its p > 0, under no_grad as well; engine.TransformerFn then gets one 64-bit seed per call, drawn
    from the CUDA generator of the input's device (so torch.manual_seed governs the masks).  `forced_dropout_seed` (an int) pins that seed for tests.  `ff_dropout` is accepted and not
    applied: the reference's Transformer never hands it to its FeedForward (x_clip.py:268)."""

    def __init__(self, dim: int, *, depth: int, dim_head: int = 64, heads: int = 8,
                 causal: bool = False, attn_dropout: float = 0., ff_dropout: float = 0.,
                 ff_mult: int = 4, checkpoint_during_training: bool = False):
        super().__init__()
        _require(dim % 128 == 0 and 128 <= dim <= 1024,
                 f"model dim must be a multiple of 128 from 128 to 1024, got {dim}")
        _require(depth >= 1, "depth must be >= 1")
        self.dim, self.depth, self.heads, self.causal = dim, depth, heads, causal
        # activation checkpointing only trades memory for recompute; accepted and ignored
        self.checkpoint_during_training = checkpoint_during_training
        self.layers = nn.ModuleList([
            nn.ModuleList([
                PreNorm(dim, Attention(dim, dim_head=dim_head, heads=heads, causal=causal,
                                       dropout=attn_dropout)),
                PreNorm(dim, FeedForward(dim, mult=ff_mult)),
            ]) for _ in range(depth)
        ])
        self.norm_in = LayerNorm(dim)
        self.norm_out = LayerNorm(dim)
        self.forced_dropout_seed: Optional[int] = None

    def flat_weights(self):
        w = [self.norm_in.g, self.norm_out.g]
        for attn, ff in self.layers:
            w += [attn.norm.g, attn.fn.to_qkv.weight, attn.fn.to_out[0].weight, attn.fn.to_out[1].g,
                  ff.norm.g, ff.fn.net[0].weight, ff.fn.net[2].g, ff.fn.net[4].weight]
        return w

    def forward(self, x, rotary_pos_emb=None, mask=None):
        """rotary_pos_emb: the reference's angle table [n, 32] (RotaryEmbedding.forward, :161-166);
        its two halves are equal, the kernel takes cos / sin of the first 16 columns."""
        _require(x.is_cuda, "inputs must live on a CUDA (sm_90) device")
        n = x.shape[1]
        _require(not self.causal or n <= 128, "the causal mask is implemented for sequences <= 128 tokens")
        cos = sin = None
        if rotary_pos_emb is not None:
            _require(tuple(rotary_pos_emb.shape) == (n, 32),
                     f"rotary table must be [n, 32] (dim_head 64 -> rot dim 32), got {tuple(rotary_pos_emb.shape)}")
            ang = rotary_pos_emb[:, :16].to(device=x.device, dtype=torch.float32)
            cos, sin = ang.cos().contiguous(), ang.sin().contiguous()
        ps = tuple(float(attn.fn.dropout.p) if attn.fn.dropout.training else 0.0 for attn, _ in self.layers)
        drop = (ps, self.dropout_seed(x.device)) if any(p > 0.0 for p in ps) else None
        return E.TransformerFn.apply(x, mask, self.heads, self.depth, self.causal, cos, sin,
                                     torch.is_grad_enabled(), drop, *self.flat_weights())

    def dropout_seed(self, device) -> torch.Tensor:
        """int64 [1] on `device`: the Philox key of this call's attention-dropout masks, drawn from the
        device's CUDA generator without a host sync, or `forced_dropout_seed`."""
        if self.forced_dropout_seed is not None:
            return torch.tensor([self.forced_dropout_seed], dtype=torch.int64, device=device)
        return torch.randint(-2 ** 63, 2 ** 63 - 1, (1,), dtype=torch.int64, device=device)


class PatchDropout(nn.Module):
    """Random patch keep (reference :134-151).  The indices are drawn with the same torch RNG
    recipe (randn -> topk); tests may pin them through `forced_keep`."""

    def __init__(self, prob: float):
        super().__init__()
        assert 0 <= prob < 1.
        self.prob = prob
        self.forced_keep: Optional[torch.Tensor] = None

    def indices(self, b: int, n: int, device, force_keep_all: bool = False) -> Optional[torch.Tensor]:
        """Kept patch indices int64 [b, keep] drawn exactly like the reference (:146-149), or None
        when every patch is kept (eval mode, prob 0, keep_all_patches)."""
        if not self.training or self.prob == 0. or force_keep_all:
            return None
        keep = max(1, int(n * (1 - self.prob)))
        if self.forced_keep is not None:
            return self.forced_keep.to(device)
        return torch.randn(b, n, device=device).topk(keep, dim=-1).indices

    def forward(self, x, force_keep_all: bool = False):
        b, n, d = x.shape
        idx = self.indices(b, n, x.device, force_keep_all)
        if idx is None:
            return x
        return torch.gather(x, 1, idx[:, :, None].expand(-1, -1, d))


class RotaryEmbedding(nn.Module):
    """Angle table of the rotary embedding (reference :155-166); `inv_freq` is a buffer so that
    reference checkpoints load unchanged."""

    def __init__(self, dim: int):
        super().__init__()
        self.register_buffer('inv_freq', 1. / (10000 ** (torch.arange(0, dim, 2).float() / dim)))

    def forward(self, seq_len: int, device):
        t = torch.arange(seq_len, device=device).type_as(self.inv_freq)
        freqs = torch.einsum('i , j -> i j', t, self.inv_freq.to(device))
        return torch.cat((freqs, freqs), dim=-1)


class TextTransformer(nn.Module):
    def __init__(self, dim: int, *, num_tokens: int, max_seq_len: int, dim_head: int,
                 rotary_pos_emb=None, causal: bool = False, **kwargs):
        super().__init__()
        _require(not (rotary_pos_emb and causal),
                 "text_rotary_pos_emb with text_causal_mask is broken in the reference itself "
                 "(n+1 rotary positions for n tokens, x_clip.py:328) and not offered here")
        _require(not causal or max_seq_len <= 128, "text_causal_mask needs text_seq_len <= 128")
        self.token_emb = nn.Embedding(num_tokens, dim)
        self.abs_pos_emb = nn.Embedding(max_seq_len, dim) if not rotary_pos_emb else None
        self.rotary_pos_emb = RotaryEmbedding(min(dim_head, 32)) if rotary_pos_emb else None
        self.cls_token = nn.Parameter(torch.randn(dim)) if not causal else None
        self.max_seq_len = max_seq_len
        self.transformer = Transformer(dim, dim_head=dim_head, causal=causal, **kwargs)

    def forward(self, x, mask=None):
        b, n = x.shape
        _require(x.is_cuda, "inputs must live on a CUDA (sm_90) device")
        _require(n <= self.max_seq_len, "text longer than text_seq_len")
        rotary = None
        if self.abs_pos_emb is not None and self.cls_token is not None:
            # default configuration: gather + position + CLS in one kernel
            h = E.TextEmbedFn.apply(x, self.token_emb.weight, self.abs_pos_emb.weight, self.cls_token)
        else:
            # rotary (no position table) or causal (no CLS token): plain embedding lookups
            h = self.token_emb(x)
            if self.abs_pos_emb is not None:
                h = h + self.abs_pos_emb(torch.arange(n, device=x.device))[None]
            if self.rotary_pos_emb is not None:
                rotary = self.rotary_pos_emb(n + 1, x.device)       # n + 1: the CLS position (:328)
            if self.cls_token is not None:
                h = torch.cat((self.cls_token.expand(b, 1, -1), h), dim=1)
            h = h.to(BF16)
        if mask is not None and self.cls_token is not None:
            mask = torch.cat((torch.ones(b, 1, dtype=torch.bool, device=mask.device), mask), dim=1)
        return self.transformer(h, rotary_pos_emb=rotary, mask=mask)


class VisionTransformer(nn.Module):
    def __init__(self, dim: int, *, image_size: int, patch_size: int, channels: int,
                 patch_dropout: float = 0.5, **kwargs):
        super().__init__()
        assert image_size % patch_size == 0, 'Image dimensions must be divisible by the patch size.'
        self.patch_size = patch_size
        num_patches = (image_size // patch_size) ** 2
        patch_dim = channels * patch_size ** 2
        self.to_tokens = nn.Sequential(_Slot(), nn.Linear(patch_dim, dim))
        self.pos_emb = nn.Embedding(num_patches, dim)
        self.patch_dropout = PatchDropout(patch_dropout)
        self.transformer = Transformer(dim, **kwargs)
        self.to_cls_tokens = nn.Sequential(_Slot(), nn.Linear(dim, dim, bias=False), _Slot())

    def forward(self, x, keep_all_patches: bool = False):
        """image f32 [b, c, H, W] -> [b, 1 + n_kept, dim] (CLS first).  Patchify, PatchDropout and the
        bf16 cast are ONE pass that reads only the kept patches (xclip_patchify_gather); the
        patch-embedding GEMM adds bias and the gathered position rows in its epilogue.  An image with
        requires_grad gets its gradient (xclip_patchify_scatter; 0 on dropped patches)."""
        b = x.shape[0]
        _require(x.is_cuda, "inputs must live on a CUDA (sm_90) device")
        p = self.patch_size
        _require(x.shape[2] % p == 0 and x.shape[3] % p == 0, "image size must be a multiple of the patch size")
        n = (x.shape[2] // p) * (x.shape[3] // p)
        _require(n == self.pos_emb.num_embeddings, "image size does not match the position table")
        lin = self.to_tokens[1]
        keep = self.patch_dropout.indices(b, n, x.device, keep_all_patches)
        if keep is None:
            index = torch.arange(n, device=x.device, dtype=torch.int32).repeat(b)
            k = n
        else:
            index = keep.reshape(-1).to(torch.int32)
            k = keep.shape[1]
        x = x.float()
        if x.requires_grad and torch.is_grad_enabled():
            # d loss / d image (adversarial training, guidance, saliency): the backward scatters the
            # patch gradients back to pixels; every other call keeps the launch sequence below
            tok = E.PatchifyFn.apply(x, p, keep, index, lin.weight, lin.bias, self.pos_emb.weight)
        else:
            patches = E.patch_rows(x, p, keep)
            tok = E.PatchEmbedFn.apply(patches, index, lin.weight, lin.bias, self.pos_emb.weight)
        out = self.transformer(tok.view(b, k, -1))
        pooled = out.float().mean(dim=1).to(BF16)
        cls = E.LinearFn.apply(pooled, self.to_cls_tokens[1].weight, None, None)
        return torch.cat((cls[:, None], out), dim=1)


# ----------------------------------------------------------------------------- CLIP

def _encode(fn, args, freeze: bool):
    if not freeze:
        return fn(*args)
    with torch.no_grad():
        return fn(*args).detach()


class CLIP(nn.Module):
    def __init__(
        self,
        *,
        image_encoder=None,
        text_encoder=None,
        dim_text=512,
        dim_image=512,
        dim_latent=512,
        num_text_tokens=10000,
        text_enc_depth=6,
        text_seq_len=256,
        text_heads=8,
        text_dim_head=64,
        text_has_cls_token=True,
        text_pad_id=0,
        text_rotary_pos_emb=False,
        text_causal_mask=False,
        text_eos_id=None,
        text_encode_without_mask=False,
        visual_enc_depth=6,
        visual_heads=8,
        visual_dim_head=64,
        visual_image_size=256,
        visual_patch_size=32,
        visual_patch_dropout=0.5,
        visual_has_cls_token=True,
        channels=3,
        use_all_token_embeds=False,
        downsample_image_embeds=False,
        decoupled_contrastive_learning=False,
        extra_latent_projection=False,
        use_mlm=False,
        text_ssl_loss_weight=0.05,
        use_visual_ssl=False,
        visual_ssl=None,
        visual_ssl_type='simsiam',
        visual_ssl_hidden_layer=-1,
        simclr_temperature=0.1,
        image_ssl_loss_weight=0.05,
        multiview_loss_weight=0.1,
        checkpoint_during_training=False,
        sim_reg_loss_weight=0.,
        microbatch=None,   # (extension) encoder micro-batch for the GradCache-style large-batch step
        microbatch_retain="auto",   # (extension) chunks whose activations stay in HBM: "auto" | int
        **kwargs,     # unknown keywords are swallowed, like the reference (:455)
    ):
        super().__init__()
        # (extension) sigmoid_loss=False: SigLIP's pairwise sigmoid loss in place of InfoNCE.  Taken from
        # **kwargs, so that the explicit signature stays the reference's plus the micro-batch options
        sigmoid_loss = bool(kwargs.pop("sigmoid_loss", False))
        assert use_all_token_embeds or (visual_has_cls_token or text_has_cls_token), \
            'CLS token must be included on both vision and text transformers if you are not using fine-grained contrastive learning loss'
        assert not (text_causal_mask and text_eos_id is None), \
            'text EOS token id must be given if using causal mask in text transformer'
        _require(not downsample_image_embeds, "downsample_image_embeds is not implemented")
        if sigmoid_loss:
            _require(not use_all_token_embeds, "sigmoid_loss with use_all_token_embeds (no FILIP variant of the sigmoid loss)")
            _require(not decoupled_contrastive_learning,
                     "sigmoid_loss with decoupled_contrastive_learning (DCL changes a softmax denominator the sigmoid loss does not have)")
            _require(not extra_latent_projection and sim_reg_loss_weight <= 0.,
                     "sigmoid_loss with extra_latent_projection or sim_reg_loss_weight > 0 (the sigmoid loss is "
                     "symmetric: it has no image-to-text direction for a second projection)")
        if sim_reg_loss_weight > 0.:
            # without the extra projection the reference's einsum at x_clip.py:779 gets the 2-D
            # un-rearranged text_latents_extra and fails; with FILIP its [1, B, B] mask cannot index
            # the [m, t, B, B] token similarities
            _require(extra_latent_projection,
                     "sim_reg_loss_weight > 0 needs extra_latent_projection=True (the reference fails at x_clip.py:779 without it)")
            _require(not use_all_token_embeds,
                     "sim_reg_loss_weight > 0 with use_all_token_embeds (the reference's mask at x_clip.py:779 does not fit the token similarities)")
        _require(dim_latent % 128 == 0 and 128 <= dim_latent <= 1024,
                 f"dim_latent must be a multiple of 128 from 128 to 1024, got {dim_latent}")
        _require(dim_text % 8 == 0 and dim_image % 8 == 0, "dim_text / dim_image must be multiples of 8")

        self.dim_text, self.dim_image, self.dim_latent = dim_text, dim_image, dim_latent
        self.image_channels = channels
        self.image_size = visual_image_size
        self.text_pad_id = text_pad_id
        self.text_has_cls_token = text_has_cls_token
        self.text_seq_len = text_seq_len
        self.text_encode_without_mask = text_encode_without_mask
        self.text_causal_mask = text_causal_mask
        self.text_eos_id = text_eos_id
        self.visual_has_cls_token = visual_has_cls_token

        if text_encoder is not None:
            self.text_transformer = text_encoder
        else:
            self.text_transformer = TextTransformer(
                dim=dim_text, num_tokens=num_text_tokens + (1 if use_mlm else 0), max_seq_len=text_seq_len,
                depth=text_enc_depth, heads=text_heads, causal=text_causal_mask,
                dim_head=text_dim_head, rotary_pos_emb=text_rotary_pos_emb,
                checkpoint_during_training=checkpoint_during_training)

        if image_encoder is not None:
            self.visual_transformer = image_encoder
        else:
            self.visual_transformer = VisionTransformer(
                dim=dim_image, image_size=visual_image_size, patch_size=visual_patch_size,
                channels=channels, depth=visual_enc_depth, heads=visual_heads,
                dim_head=visual_dim_head, patch_dropout=visual_patch_dropout,
                checkpoint_during_training=checkpoint_during_training)

        # auxiliary self-supervised losses through the fast encoders (reference :516-552; aux.py)
        self.use_mlm = use_mlm
        self.text_ssl_loss_weight = text_ssl_loss_weight if use_mlm else 0
        if use_mlm:
            from .aux import MLM
            mlm_kwargs = {k[len('mlm_'):]: kwargs.pop(k) for k in list(kwargs) if k.startswith('mlm_')}
            self.mlm = MLM(self.text_transformer, dim=dim_text, num_tokens=num_text_tokens, **mlm_kwargs)
        self.use_visual_ssl = use_visual_ssl or visual_ssl is not None
        self.image_ssl_loss_weight = image_ssl_loss_weight if use_visual_ssl else 0     # (sic, :536)
        if self.use_visual_ssl:
            if visual_ssl is not None:
                self.visual_ssl = visual_ssl
            else:
                from .aux import SimCLR, SimSiam
                if visual_ssl_type == 'simsiam':
                    self.visual_ssl = SimSiam(self.visual_transformer, image_size=visual_image_size,
                                              channels=channels, rep_dim=dim_image)
                elif visual_ssl_type == 'simclr':
                    self.visual_ssl = SimCLR(self.visual_transformer, image_size=visual_image_size,
                                             channels=channels, rep_dim=dim_image, temperature=simclr_temperature)
                else:
                    raise ValueError('unknown visual_ssl_type')

        self.to_text_latent = nn.Linear(dim_text, dim_latent, bias=False)
        self.to_visual_latent = nn.Linear(dim_image, dim_latent, bias=False)
        # SigLIP's initial logit scale 10 and bias -10 (Zhai et al. 2023; open_clip's SigLIP models)
        self.sigmoid_loss = sigmoid_loss
        self.temperature = nn.Parameter(torch.tensor(math.log(10.) if sigmoid_loss else 1.))
        if sigmoid_loss:
            self.logit_bias = nn.Parameter(torch.tensor(-10.))

        self.use_all_token_embeds = use_all_token_embeds
        self.decoupled_contrastive_learning = decoupled_contrastive_learning
        self.extra_latent_projection = extra_latent_projection
        # always present, initialised as copies, exactly like the reference (:585-586)
        self.to_text_latent_extra = copy.deepcopy(self.to_text_latent)
        self.to_visual_latent_extra = copy.deepcopy(self.to_visual_latent)

        self.multiview_loss_weight = multiview_loss_weight
        self.microbatch = microbatch
        assert microbatch_retain == "auto" or (isinstance(microbatch_retain, int) and microbatch_retain >= 0)
        self.microbatch_retain = microbatch_retain
        self.last_step_plan = None      # filled by engine.ChunkedClipLossFn: chunks / retained / bytes
        # latched at construction, like the reference (:591): the process group must exist first
        self.requires_all_gather = dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1
        # similarity regularisation (https://arxiv.org/abs/2309.08773), fused into ContrastiveLossFn
        self.sim_reg_loss_weight = sim_reg_loss_weight
        self.has_sim_reg_loss = sim_reg_loss_weight > 0.

    # -- helpers ---------------------------------------------------------------------
    def _eos_to_front(self, enc_text, text):
        """Causal text tower: the encoding at the first EOS token of every row moves to index 0,
        the others keep their order (reference :668-685; its undefined `b` is the batch size)."""
        eos = text == self.text_eos_id
        assert torch.all(torch.any(eos, dim=-1)), \
            f'some of the text rows does not have the eos id {self.text_eos_id}'
        b, n, d = enc_text.shape
        first = eos.float().argmax(dim=-1, keepdim=True)                       # [b, 1]
        pos = torch.arange(n, device=text.device)[None].expand(b, -1)
        rest = pos[pos != first].view(b, n - 1)
        order = torch.cat((first, rest), dim=1)
        return torch.gather(enc_text, 1, order[:, :, None].expand(-1, -1, d))

    def _encodings(self, text, image, text_mask, freeze_text=False, freeze_image=False):
        """(text encodings, image encodings) of both towers, a frozen tower without gradient."""
        text_args = (text,) if self.text_encode_without_mask else (text, text_mask)
        enc_text = _encode(self.text_transformer, text_args, freeze_text)
        if self.text_causal_mask:
            enc_text = self._eos_to_front(enc_text, text)
        return enc_text, _encode(self.visual_transformer, (image,), freeze_image)

    def _latents(self, enc_text, enc_image):
        """CLS select (FILIP: every token but the CLS) -> projections.
        Returns ([zt, zi(, zt_x, zi_x)], ops): latents [b, D], or [b, tokens, D] in FILIP mode."""
        if self.use_all_token_embeds:
            assert enc_text.ndim == 3, 'encoded text must have 3 dimensions (batch, seq, features)'
            assert enc_image.ndim == 3, 'encoded image must have 3 dimensions (batch, seq [height x width], features)'
            te = enc_text[:, 1:] if self.text_has_cls_token else enc_text
            ie = enc_image[:, 1:] if self.visual_has_cls_token else enc_image
        else:
            te = enc_text[:, 0] if enc_text.ndim == 3 else enc_text
            ie = enc_image[:, 0] if enc_image.ndim == 3 else enc_image
        zt, ops_t = self._project(te, self.to_text_latent)
        zi, ops_i = self._project(ie, self.to_visual_latent)
        zs, ops = [zt, zi], [ops_t, ops_i]
        if self.extra_latent_projection:
            zt_x, ops_tx = self._project(te, self.to_text_latent_extra)
            zi_x, ops_ix = self._project(ie, self.to_visual_latent_extra)
            zs += [zt_x, zi_x]
            ops += [ops_tx, ops_ix]
        return zs, ops

    def _encode_to_latents(self, text, image, text_mask):
        """encoders -> latents (_latents)."""
        return self._latents(*self._encodings(text, image, text_mask))

    def _chunkable_ssl(self) -> bool:
        """visual SSL the micro-batched step can split into encoder passes and a head"""
        from .aux import SimCLR, SimSiam
        return isinstance(self.visual_ssl, (SimSiam, SimCLR))

    def _aux_inputs(self, text, image) -> dict:
        """The random parts of the auxiliary losses for the whole batch, drawn once before any chunk
        and in the single pass's order: the MLM corruption, then both augmentations (the reference's
        augmentations draw one decision per call, so per-chunk augmentation would be another function)."""
        aux = dict(mlm=None, ssl=None, ssl_encoder=None, ssl_targets=False)
        if self.use_mlm:
            masked, labels = self.mlm.corrupt(text)
            sel = labels != self.mlm.pad_token_id
            aux["mlm"] = (masked, sel, labels[sel])
        if self.use_visual_ssl:
            ssl = self.visual_ssl
            assert image.shape[0] > 1, \
                'you must have greater than 1 sample when training, due to the batchnorm in the projection layer'
            aux["ssl"] = (ssl.augment1(image), ssl.augment2(image))
            from .aux import SimSiam
            aux["ssl_targets"] = isinstance(ssl, SimSiam)
            aux["ssl_encoder"] = ssl.online_encoder if aux["ssl_targets"] else ssl.net
        return aux

    def _project(self, embeds: torch.Tensor, linear: nn.Linear):
        """embeds [..., d] (any float dtype) -> (z fp32 [..., D], (zrow, zcol) bf16 [rows, 3D])."""
        lead = embeds.shape[:-1]
        e = embeds.reshape(-1, embeds.shape[-1])
        if e.dtype != BF16:
            e = e.to(BF16)
        z, zrow, zcol = E.ProjectL2NormFn.apply(e, linear.weight)
        return z.view(*lead, -1), (zrow, zcol)

    def _loss(self, zs, ops, text_mask, temperature, logit_bias=None, views=(1, 1), mlm=None, ssl=None,
              filip_stats=None):
        """The training loss of the single pass and of the micro-batched step (engine.ChunkedClipLossFn).

        zs / ops: _latents' outputs for m text views and n image views (views = (m, n)) of the same b pairs,
        stacked along the batch; text_mask [m b, n_text].  The FILIP, sigmoid or InfoNCE / DCL loss (with
        the similarity regularisation), weighted as the reference does (x_clip.py:851-873):
        cl_w * L[0, 0] + w_text * mlm + w_image * ssl + w_multiview * mean(the other view pairs), where
        cl_w = 1 - (w_text + w_image + w_multiview).  Without any auxiliary term the loss is returned
        unweighted.  `mlm` / `ssl`: the auxiliary losses, or None when off; `filip_stats` receives
        FilipLossFn's plan."""
        m, n = views
        multiview = m * n > 1
        has_aux = multiview or self.use_mlm or self.use_visual_ssl
        mv_w = self.multiview_loss_weight if multiview else 0
        cl_w = 1 - (self.text_ssl_loss_weight + self.image_ssl_loss_weight + mv_w)
        extra = self.extra_latent_projection
        dcl, gather = self.decoupled_contrastive_learning, self.requires_all_gather
        others = ()
        if self.use_all_token_embeds:
            # every (text view, image view) pair in one pair of segment-max passes, the view pairs
            # weighted inside the loss
            loss = FilipLossFn.apply(zs[0], zs[1], *(zs[2:] if extra else (None, None)), temperature,
                                     tuple(ops), text_mask.contiguous(), dcl, gather, filip_stats, views,
                                     (cl_w, mv_w))
            weighted = multiview
        else:
            b = zs[0].shape[0] // m

            def pick(k, t, i, j):
                """text view i (zs / ops 0 and 2) or image view j (1 and 3) of t: t itself for one view"""
                v, count = (i, m) if k % 2 == 0 else (j, n)
                return t if count == 1 else t[v * b:(v + 1) * b]

            def pair(i, j):
                """the loss of text view i against image view j"""
                z = [pick(k, t, i, j) for k, t in enumerate(zs)]
                o = tuple((pick(k, r, i, j), pick(k, c, i, j)) for k, (r, c) in enumerate(ops))
                if self.sigmoid_loss:
                    return E.SigmoidLossFn.apply(z[0], z[1], temperature, logit_bias, o, gather)
                # the similarity regularisation (single view: refused with views) weighs the
                # contrastive term itself: cl_w * contrastive + w * L_sim
                sim_reg = (self.sim_reg_loss_weight, cl_w if has_aux else 1.0) if self.has_sim_reg_loss else ()
                return E.ContrastiveLossFn.apply(z[0], z[1], *(z[2:] if extra else (None, None)), temperature,
                                                 o, dcl, gather, *sim_reg)

            loss, *others = [pair(i, j) for i in range(m) for j in range(n)]
            weighted = self.has_sim_reg_loss
        if has_aux and not weighted:
            loss = loss * cl_w
        if mlm is not None:
            loss = loss + mlm * self.text_ssl_loss_weight
        if ssl is not None:
            loss = loss + ssl * self.image_ssl_loss_weight
        if others:
            loss = loss + torch.stack(others).mean() * mv_w
        return loss

    def forward(
        self,
        text,
        image,
        return_loss=False,
        return_encodings=False,
        return_latents=False,
        freeze_image_encoder=False,
        freeze_text_encoder=False,
        text_to_image=True,
        aug_text=None,
        aug_image=None,
    ):
        # the reference's [1, B, B] off-diagonal mask (x_clip.py:779) cannot index the [m, B, B] view
        # similarities: it raises for every multiview step, so this one refuses before any encoder runs
        _require(not (self.has_sim_reg_loss and (aug_text is not None or aug_image is not None)),
                 "sim_reg_loss_weight > 0 with aug_text / aug_image (the reference fails at x_clip.py:779)")
        _require(text.is_cuda and image.is_cuda, "inputs must live on a CUDA (sm_90) device")

        text_mask = text != self.text_pad_id

        # large batches: the micro-batched step, auxiliary losses included (engine.ChunkedClipLossFn).
        # Multiview, frozen towers, a custom visual_ssl module, and visual SSL on an image that wants a
        # gradient run the single pass below.
        if (return_loss and self.microbatch and text.shape[0] > self.microbatch
                and aug_text is None and aug_image is None
                and not (freeze_image_encoder or freeze_text_encoder)
                and (not self.use_visual_ssl or (self._chunkable_ssl() and not image.requires_grad))):
            assert self.training, 'loss cannot be used if not training'
            aux = self._aux_inputs(text, image) if (self.use_mlm or self.use_visual_ssl) else None
            return E.ChunkedClipLossFn.apply(self, text, image, text_mask, int(self.microbatch),
                                             self.temperature, self.microbatch_retain, aux,
                                             *((self.logit_bias,) if self.sigmoid_loss else ()))

        # auxiliary losses on the un-augmented batch (reference :616-621)
        mlm = ssl = None
        if return_loss:
            mlm = self.mlm(text, mask=text_mask) if self.use_mlm else None
            ssl = self.visual_ssl(image) if self.use_visual_ssl else None

        # multiview: augmented texts / images are further "views" of the same pairs (:625-650)
        num_batch_texts = num_batch_images = 1
        if aug_text is not None:
            aug_text = aug_text if isinstance(aug_text, (tuple, list)) else (aug_text,)
            assert all(t.shape == text.shape for t in aug_text)
            num_batch_texts = len(aug_text) + 1
            text = torch.cat((text, *aug_text), dim=0)
            text_mask = text != self.text_pad_id
        if aug_image is not None:
            aug_image = aug_image if isinstance(aug_image, (tuple, list)) else (aug_image,)
            assert all(i.shape == image.shape for i in aug_image)
            num_batch_images = len(aug_image) + 1
            image = torch.cat((image, *aug_image), dim=0)
        is_multiview = num_batch_texts > 1 or num_batch_images > 1
        assert not (return_loss and not self.training), 'loss cannot be used if not training'
        assert not (not return_loss and is_multiview), 'do not pass in augmented texts or images if not training'
        assert not (self.multiview_loss_weight == 0 and is_multiview), \
            'multiview loss weight cannot be 0 if augmented text or images passed in'

        enc_text, enc_image = self._encodings(text, image, text_mask, freeze_text_encoder, freeze_image_encoder)
        if return_encodings:
            return enc_text.float(), enc_image.float()

        zs, ops = self._latents(enc_text, enc_image)
        if return_latents:
            return tuple(zs)

        if not return_loss:
            # exp(temperature) * similarity, as the reference returns; with sigmoid_loss the logit_bias
            # is not added (add clip.logit_bias for the logits the sigmoid loss sees)
            temp = self.temperature.exp()
            a, b = zs[2:] if (self.extra_latent_projection and not text_to_image) else zs[:2]
            if self.use_all_token_embeds:
                return torch.einsum('btd,bid->bti', a, b) * temp      # per-pair token sims (:740-742)
            return (a * b).sum(dim=-1) * temp                          # per-pair similarity (:744-746)

        return self._loss(zs, ops, text_mask, self.temperature, self.logit_bias if self.sigmoid_loss else None,
                          views=(num_batch_texts, num_batch_images), mlm=mlm, ssl=ssl)
