"""CPU oracle for the x-clip contrastive training hot path.  TEST INFRASTRUCTURE ONLY.

A functional, fp32, pure-torch restatement of what lucidrains/x-clip v0.14.4
computes on the path  encoders -> latent projection + l2norm -> (all-gather) ->
similarity -> InfoNCE / DCL / FILIP loss.  It works on a flat `state_dict`
(reference parameter names, SURVEY.md 8b) instead of nn.Modules, so that it shares
no code structure with either the reference modules or the product package.
Gradients come from torch autograd over these functions.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference
legs may import this file.  The product path (x_clip_b200/) never does.

Parity pinning: the reference ships NO tests or golden vectors (SURVEY.md 4, 8c), so
this oracle is pinned against outputs of the reference itself, generated in the build
container by tests/golden/make_golden.py and committed under tests/golden/*.json
(tests/test_oracle_golden.py checks them, incl. the SURVEY 4 known-answer anchors).

Every function cites the reference lines (x_clip/x_clip.py unless noted) it restates.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import torch

Tensor = torch.Tensor
Params = Dict[str, Tensor]


@dataclass
class ClipConfig:
    """Constructor arguments of the reference CLIP that matter on the hot path (:413-456)."""
    dim_text: int = 512
    dim_image: int = 512
    dim_latent: int = 512
    num_text_tokens: int = 10000
    text_enc_depth: int = 6
    text_seq_len: int = 256
    text_heads: int = 8
    text_dim_head: int = 64
    text_pad_id: int = 0
    visual_enc_depth: int = 6
    visual_heads: int = 8
    visual_dim_head: int = 64
    visual_image_size: int = 256
    visual_patch_size: int = 32
    channels: int = 3
    use_all_token_embeds: bool = False
    decoupled_contrastive_learning: bool = False
    extra_latent_projection: bool = False
    text_rotary_pos_emb: bool = False      # :428 - rotary instead of the absolute position table
    text_causal_mask: bool = False         # :429 - causal text tower, no CLS token, EOS pooling
    text_eos_id: Optional[int] = None      # :430

    def to_kwargs(self) -> dict:
        return dict(self.__dict__)


# --------------------------------------------------------------------------- blocks

# The reference's precision rules: LayerNorm eps 1e-3 for any non-fp32 input (:118) and the attention
# softmax in fp32 (:238).  tests/step_oracle.py pins them (PINNED_LN_EPS = 1e-5, SOFTMAX_FP32 = False)
# to run these same functions as an fp64 reference of the fp32 step.  The defaults change nothing.
PINNED_LN_EPS: Optional[float] = None
SOFTMAX_FP32 = True


def gain_layernorm(x: Tensor, g: Tensor) -> Tensor:
    """Gain-only LayerNorm, biased variance; eps 1e-5 for fp32 inputs (:112-121)."""
    if PINNED_LN_EPS is not None:
        eps = PINNED_LN_EPS
    else:
        eps = 1e-5 if x.dtype == torch.float32 else 1e-3
    mu = x.mean(dim=-1, keepdim=True)
    var = ((x - mu) ** 2).mean(dim=-1, keepdim=True)
    return (x - mu) * torch.rsqrt(var + eps) * g


def rotary_angles(n_pos: int, rot_dim: int, device=None) -> Tensor:
    """RotaryEmbedding(rot_dim)(n_pos) (:155-166): angle[pos, j] = pos / 10000^(2(j mod rot_dim/2)/rot_dim),
    the half-table repeated twice along the feature axis -> [n_pos, rot_dim] fp32 on `device`."""
    inv_freq = 1.0 / (10000 ** (torch.arange(0, rot_dim, 2, device=device).float() / rot_dim))
    ang = torch.arange(n_pos, device=device).float()[:, None] * inv_freq[None, :]
    return torch.cat([ang, ang], dim=-1)


def rotate_features(ang: Tensor, t: Tensor) -> Tensor:
    """apply_rotary_pos_emb (:168-176): the first rot_dim features of every head are rotated
    pairwise (feature j with j + rot_dim/2), the rest pass through."""
    r = ang.shape[-1]
    head, rest = t[..., :r], t[..., r:]
    a, b = head[..., : r // 2], head[..., r // 2:]
    turned = torch.cat([-b, a], dim=-1)
    return torch.cat([head * ang.cos() + turned * ang.sin(), rest], dim=-1)


def attention(x: Tensor, p: Params, prefix: str, heads: int, dim_head: int,
              key_mask: Optional[Tensor], causal: bool = False,
              rotary: Optional[Tensor] = None) -> Tensor:
    """Multi-head attention with a key-padding mask (and optionally a causal mask), followed by
    the output projection AND a LayerNorm (:201-245).  q is pre-scaled by dim_head**-0.5 (:219);
    rotary angles, when given, rotate q, k AND v (:221-223); masked keys are filled with
    -finfo.max, not -inf (:227-236); softmax in fp32 (:238)."""
    b, n, _ = x.shape
    qkv = x @ p[prefix + "to_qkv.weight"].t()                       # [b, n, 3*h*dh]
    qkv = qkv.view(b, n, 3, heads, dim_head).permute(2, 0, 3, 1, 4)  # [3, b, h, n, dh]
    q, k, v = qkv[0] * dim_head ** -0.5, qkv[1], qkv[2]
    if rotary is not None:
        q, k, v = rotate_features(rotary, q), rotate_features(rotary, k), rotate_features(rotary, v)
    scores = q @ k.transpose(-1, -2)                                 # [b, h, n, n]
    fill = -torch.finfo(scores.dtype).max
    if key_mask is not None:
        scores = torch.where(key_mask[:, None, None, :], scores, torch.full_like(scores, fill))
    if causal:
        future = torch.ones(n, n, dtype=torch.bool, device=x.device).triu(1)
        scores = scores.masked_fill(future, fill)
    probs = torch.softmax(scores.float() if SOFTMAX_FP32 else scores, dim=-1).to(scores.dtype)
    ctx = (probs @ v).permute(0, 2, 1, 3).reshape(b, n, heads * dim_head)
    out = ctx @ p[prefix + "to_out.0.weight"].t()
    return gain_layernorm(out, p[prefix + "to_out.1.g"])


def geglu_feedforward(x: Tensor, p: Params, prefix: str) -> Tensor:
    """Linear(d, 8d) -> value * gelu_erf(gate) -> LayerNorm(4d) -> Linear(4d, d), no biases
    (:180-199).  The FIRST half of the up-projection is the value, the second the gate."""
    u = x @ p[prefix + "net.0.weight"].t()
    half = u.shape[-1] // 2
    val, gate = u[..., :half], u[..., half:]
    hdn = val * (0.5 * gate * (1.0 + torch.erf(gate / math.sqrt(2.0))))
    hdn = gain_layernorm(hdn, p[prefix + "net.2.g"])
    return hdn @ p[prefix + "net.4.weight"].t()


def transformer_stack(x: Tensor, p: Params, prefix: str, depth: int, heads: int, dim_head: int,
                      key_mask: Optional[Tensor], causal: bool = False,
                      rotary: Optional[Tensor] = None) -> Tensor:
    """norm_in -> depth x (pre-norm attention + residual, pre-norm feed-forward + residual)
    -> norm_out (:247-291)."""
    x = gain_layernorm(x, p[prefix + "norm_in.g"])
    for layer in range(depth):
        a = f"{prefix}layers.{layer}.0."
        f = f"{prefix}layers.{layer}.1."
        x = attention(gain_layernorm(x, p[a + "norm.g"]), p, a + "fn.", heads, dim_head, key_mask,
                      causal, rotary) + x
        x = geglu_feedforward(gain_layernorm(x, p[f + "norm.g"]), p, f + "fn.") + x
    return gain_layernorm(x, p[prefix + "norm_out.g"])


# --------------------------------------------------------------------------- encoders

def encode_text(ids: Tensor, key_mask: Tensor, p: Params, cfg: ClipConfig) -> Tensor:
    """Token embedding + absolute position table (or rotary angles for n+1 positions, :326-328),
    CLS prepended and always attendable unless the tower is causal (:313, :330-335), transformer
    (:295-338).  Returns [b, 1+n, dim_text] (causal: [b, n, dim_text])."""
    b, n = ids.shape
    x = p["text_transformer.token_emb.weight"][ids]
    rotary = None
    if cfg.text_rotary_pos_emb:
        rotary = rotary_angles(n + 1, min(cfg.text_dim_head, 32), ids.device)
    else:
        x = x + p["text_transformer.abs_pos_emb.weight"][:n][None]
    mask = key_mask
    if not cfg.text_causal_mask:
        cls = p["text_transformer.cls_token"].expand(b, 1, -1)
        x = torch.cat([cls, x], dim=1)
        mask = torch.cat([torch.ones(b, 1, dtype=torch.bool, device=ids.device), key_mask], dim=1)
    return transformer_stack(x, p, "text_transformer.transformer.", cfg.text_enc_depth,
                             cfg.text_heads, cfg.text_dim_head, mask, cfg.text_causal_mask, rotary)


def eos_to_front(enc_text: Tensor, ids: Tensor, eos_id: int) -> Tensor:
    """Causal text tower: the encoding at the FIRST eos token of every row becomes token 0, the
    other tokens keep their order behind it (:668-685, with the undefined `b` read as the batch)."""
    is_eos = ids == eos_id
    assert bool(is_eos.any(dim=-1).all()), f"some of the text rows does not have the eos id {eos_id}"
    first = is_eos.float().argmax(dim=-1)                                # [b]
    b, n, d = enc_text.shape
    pos = torch.arange(n, device=ids.device)[None, :].expand(b, -1)
    rest = pos[pos != first[:, None]].view(b, n - 1)
    order = torch.cat([first[:, None], rest], dim=1)                      # [b, n]
    return torch.gather(enc_text, 1, order[:, :, None].expand(-1, -1, d))


def patchify(img: Tensor, patch: int) -> Tensor:
    """'b c (h p1) (w p2) -> b (h w) (p1 p2 c)' (:357)."""
    b, c, H, W = img.shape
    gh, gw = H // patch, W // patch
    x = img.view(b, c, gh, patch, gw, patch).permute(0, 2, 4, 3, 5, 1)
    return x.reshape(b, gh * gw, patch * patch * c)


def encode_image(img: Tensor, p: Params, cfg: ClipConfig,
                 keep: Optional[Tensor] = None) -> Tensor:
    """Patch embedding (Linear with bias) + position table, optional patch dropout given as
    explicit kept indices [b, n_keep] (the reference draws them with randn().topk, :149),
    transformer, then CLS = Linear(mean over tokens) prepended (:340-390)."""
    x = patchify(img, cfg.visual_patch_size)
    x = x @ p["visual_transformer.to_tokens.1.weight"].t() + p["visual_transformer.to_tokens.1.bias"]
    x = x + p["visual_transformer.pos_emb.weight"][: x.shape[1]][None]
    if keep is not None:
        x = torch.gather(x, 1, keep[:, :, None].expand(-1, -1, x.shape[-1]))
    out = transformer_stack(x, p, "visual_transformer.transformer.", cfg.visual_enc_depth,
                            cfg.visual_heads, cfg.visual_dim_head, None)
    cls = out.mean(dim=1) @ p["visual_transformer.to_cls_tokens.1.weight"].t()
    return torch.cat([cls[:, None], out], dim=1)


# --------------------------------------------------------------------------- latents + loss

def unit_rows(t: Tensor) -> Tensor:
    """F.normalize(dim=-1): x / max(||x||, 1e-12) (:54-55)."""
    return t / t.norm(dim=-1, keepdim=True).clamp_min(1e-12)


def project_latents(enc_text: Tensor, enc_image: Tensor, p: Params, cfg: ClipConfig):
    """Select CLS (or all non-CLS tokens for FILIP), project without bias, l2-normalise;
    the *_extra pair uses the second set of projections (:702-724)."""
    if cfg.use_all_token_embeds:
        te, ie = enc_text[:, 1:], enc_image[:, 1:]
    else:
        te, ie = enc_text[:, 0], enc_image[:, 0]
    zt = unit_rows(te @ p["to_text_latent.weight"].t())
    zi = unit_rows(ie @ p["to_visual_latent.weight"].t())
    if cfg.extra_latent_projection:
        zt_x = unit_rows(te @ p["to_text_latent_extra.weight"].t())
        zi_x = unit_rows(ie @ p["to_visual_latent_extra.weight"].t())
    else:
        zt_x, zi_x = zt, zi
    return zt, zi, zt_x, zi_x


def _nce_from_logits(t2i: Tensor, i2t: Tensor, dcl: bool) -> Tensor:
    """exp, positives = diagonal, denominators = row sums (diagonal zeroed for DCL),
    mean(-log pos + log denom) per direction, averaged (:821-847; log adds 1e-20, :51-52).
    No max-subtraction, as in the reference."""
    n = t2i.shape[0]
    eye = torch.eye(n, dtype=torch.bool, device=t2i.device)
    losses = []
    for s in (t2i, i2t):
        e = torch.exp(s)
        pos = e[eye]
        den = (e.masked_fill(eye, 0.0) if dcl else e).sum(dim=-1)
        losses.append((-torch.log(pos + 1e-20) + torch.log(den + 1e-20)).mean())
    return (losses[0] + losses[1]) / 2


def contrastive_loss(zt: Tensor, zi: Tensor, zt_x: Tensor, zi_x: Tensor, temperature: Tensor,
                     cfg: ClipConfig, text_mask: Optional[Tensor] = None) -> Tensor:
    """All-pairs similarity times exp(temperature) and the InfoNCE / DCL loss (:736, :797-847).
    CLS mode: t2i[t,i] = temp <zt_t, zi_i>; i2t is its transpose, or the extra-latent
    contraction when extra_latent_projection (:813-817).
    FILIP mode (zt [B,T,d], zi [B,I,d]): t2i[x,y] = masked-mean_t max_i sim, i2t[x,y] =
    mean_i max_t(sim with padded text tokens -> -max); NOTE the reference's i2t keeps the
    [text, image] orientation, so its 'rows' are still texts (:799-811, :822, :838)."""
    temp = temperature.exp()
    if not cfg.use_all_token_embeds:
        t2i = temp * (zt @ zi.t())
        i2t = temp * (zi_x @ zt_x.t()) if cfg.extra_latent_projection else t2i.t()
        return _nce_from_logits(t2i, i2t, cfg.decoupled_contrastive_learning)
    assert text_mask is not None
    sim = temp * torch.einsum("xtd,yid->xyti", zt, zi)
    sim_x = temp * torch.einsum("xtd,yid->xyti", zt_x, zi_x) if cfg.extra_latent_projection else sim
    m = text_mask[:, None, :]                                            # [x,1,t]
    t2i = sim.amax(dim=-1).masked_fill(~m, 0.0).sum(-1) / m.sum(-1).clamp_min(1e-6)
    fill = -torch.finfo(sim_x.dtype).max
    i2t = sim_x.masked_fill(~text_mask[:, None, :, None], fill).amax(dim=-2).mean(dim=-1)
    return _nce_from_logits(t2i, i2t, cfg.decoupled_contrastive_learning)


# --------------------------------------------------------------------------- whole step

def clip_forward(p: Params, text: Tensor, image: Tensor, cfg: ClipConfig,
                 keep: Optional[Tensor] = None, return_parts: bool = False):
    """CLIP.forward(text, image, return_loss=True) with SSL / multiview terms off
    (:597-875 with the defaults of :444-454): loss weight of the contrastive term is 1."""
    mask = text != cfg.text_pad_id                                       # :614
    enc_t = encode_text(text, mask, p, cfg)
    if cfg.text_causal_mask:
        enc_t = eos_to_front(enc_t, text, cfg.text_eos_id)
    enc_i = encode_image(image, p, cfg, keep)
    zt, zi, zt_x, zi_x = project_latents(enc_t, enc_i, p, cfg)
    loss = contrastive_loss(zt, zi, zt_x, zi_x, p["temperature"], cfg, mask)
    if return_parts:
        return loss, dict(enc_text=enc_t, enc_image=enc_i, text_latents=zt, image_latents=zi,
                          text_latents_extra=zt_x, image_latents_extra=zi_x)
    return loss


def clip_forward_multiview(p: Params, texts: Sequence[Tensor], images: Sequence[Tensor],
                           cfg: ClipConfig, multiview_loss_weight: float = 0.1) -> Tensor:
    """CLIP.forward(text, image, aug_text=..., aug_image=..., return_loss=True) (:623-650, :750-755,
    :851-868): texts[0] / images[0] are the originals, the others augmented views of the SAME pairs.
    Every (text view m, image view n) combination is an InfoNCE problem of its own; the loss is
    (1 - w) * loss[0,0] + w * mean(the other m*n - 1 losses)."""
    assert not cfg.use_all_token_embeds
    zs_t, zs_i = [], []
    for t in texts:
        m = t != cfg.text_pad_id
        et = encode_text(t, m, p, cfg)
        if cfg.text_causal_mask:
            et = eos_to_front(et, t, cfg.text_eos_id)
        te = et[:, 0]
        zt = unit_rows(te @ p["to_text_latent.weight"].t())
        ztx = unit_rows(te @ p["to_text_latent_extra.weight"].t()) if cfg.extra_latent_projection else zt
        zs_t.append((zt, ztx))
    for im in images:
        ie = encode_image(im, p, cfg)[:, 0]
        zi = unit_rows(ie @ p["to_visual_latent.weight"].t())
        zix = unit_rows(ie @ p["to_visual_latent_extra.weight"].t()) if cfg.extra_latent_projection else zi
        zs_i.append((zi, zix))
    losses = [contrastive_loss(zt, zi, ztx, zix, p["temperature"], cfg)
              for (zt, ztx) in zs_t for (zi, zix) in zs_i]
    if len(losses) == 1:
        return losses[0]
    w = multiview_loss_weight
    return losses[0] * (1 - w) + torch.stack(losses[1:]).mean() * w


def clip_forward_sharded(p: Params, texts: Sequence[Tensor], images: Sequence[Tensor],
                         cfg: ClipConfig, rank: int) -> Tensor:
    """What rank `rank` of a W-rank job computes (x_clip/distributed.py:41-56 +
    x_clip.py:759-769): every rank encodes ITS shard, latents are all-gathered, every rank
    evaluates the full-batch loss, and AllGather.backward returns only the local slice of the
    latent gradient.  Restated here by encoding every shard and detaching the non-local
    latents - the value equals the single-process loss on the concatenated batch and the
    parameter gradients equal d loss / d(local latents) chained through the local encoders."""
    assert not cfg.use_all_token_embeds, "the reference cannot gather FILIP latents (SURVEY 8c)"
    lat = []
    for r, (t, im) in enumerate(zip(texts, images)):
        ctx = torch.enable_grad() if r == rank else torch.no_grad()
        with ctx:
            m = t != cfg.text_pad_id
            et = encode_text(t, m, p, cfg)
            if cfg.text_causal_mask:
                et = eos_to_front(et, t, cfg.text_eos_id)
            z = project_latents(et, encode_image(im, p, cfg), p, cfg)
        lat.append(z)
    cat = [torch.cat([z[j] for z in lat], dim=0) for j in range(4)]
    return contrastive_loss(cat[0], cat[1], cat[2], cat[3], p["temperature"], cfg)


# --------------------------------------------------------------------------- fixtures protocol

def param_shapes(cfg: ClipConfig) -> Dict[str, Tuple[int, ...]]:
    """state_dict names and shapes of the reference CLIP for `cfg` (SURVEY.md 8b)."""
    s: Dict[str, Tuple[int, ...]] = {"temperature": ()}

    def tower(prefix: str, d: int, depth: int, heads: int, dh: int):
        inner = heads * dh
        for L in range(depth):
            a, f = f"{prefix}layers.{L}.0.", f"{prefix}layers.{L}.1."
            s[a + "norm.g"] = (d,)
            s[a + "fn.to_qkv.weight"] = (3 * inner, d)
            s[a + "fn.to_out.0.weight"] = (d, inner)
            s[a + "fn.to_out.1.g"] = (d,)
            s[f + "norm.g"] = (d,)
            s[f + "fn.net.0.weight"] = (8 * d, d)
            s[f + "fn.net.2.g"] = (4 * d,)
            s[f + "fn.net.4.weight"] = (d, 4 * d)
        s[prefix + "norm_in.g"] = (d,)
        s[prefix + "norm_out.g"] = (d,)

    if not cfg.text_causal_mask:                      # :313
        s["text_transformer.cls_token"] = (cfg.dim_text,)
    s["text_transformer.token_emb.weight"] = (cfg.num_text_tokens, cfg.dim_text)
    if not cfg.text_rotary_pos_emb:                   # :310
        s["text_transformer.abs_pos_emb.weight"] = (cfg.text_seq_len, cfg.dim_text)
    tower("text_transformer.transformer.", cfg.dim_text, cfg.text_enc_depth, cfg.text_heads,
          cfg.text_dim_head)
    n_patch = (cfg.visual_image_size // cfg.visual_patch_size) ** 2
    patch_dim = cfg.channels * cfg.visual_patch_size ** 2
    s["visual_transformer.to_tokens.1.weight"] = (cfg.dim_image, patch_dim)
    s["visual_transformer.to_tokens.1.bias"] = (cfg.dim_image,)
    s["visual_transformer.pos_emb.weight"] = (n_patch, cfg.dim_image)
    tower("visual_transformer.transformer.", cfg.dim_image, cfg.visual_enc_depth,
          cfg.visual_heads, cfg.visual_dim_head)
    s["visual_transformer.to_cls_tokens.1.weight"] = (cfg.dim_image, cfg.dim_image)
    s["to_text_latent.weight"] = (cfg.dim_latent, cfg.dim_text)
    s["to_visual_latent.weight"] = (cfg.dim_latent, cfg.dim_image)
    s["to_text_latent_extra.weight"] = (cfg.dim_latent, cfg.dim_text)
    s["to_visual_latent_extra.weight"] = (cfg.dim_latent, cfg.dim_image)
    return s


def protocol_state_dict(cfg: ClipConfig, seed: int) -> Params:
    """Deterministic weights shared by the golden generator, the oracle tests and the GPU
    parity tests: independent of any module construction order.  Names are visited in sorted
    order with one CPU generator; magnitudes mimic the reference's default init (kaiming-uniform
    bound 1/sqrt(fan_in) for Linear, N(0,1) embeddings) except that LayerNorm gains are
    1 + 0.1*N(0,1) and temperature 1.0 so that gains are exercised."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    out: Params = {}
    for name, shape in sorted(param_shapes(cfg).items()):
        if name == "temperature":
            out[name] = torch.tensor(1.0)
        elif name.endswith(".g"):
            out[name] = 1.0 + 0.1 * torch.randn(shape, generator=g)
        elif name.endswith("emb.weight") or name.endswith("cls_token"):
            out[name] = torch.randn(shape, generator=g)
        elif name.endswith(".bias"):
            out[name] = 0.02 * torch.randn(shape, generator=g)
        else:
            bound = 1.0 / math.sqrt(shape[-1])
            out[name] = (torch.rand(shape, generator=g) * 2 - 1) * bound
    return out


def protocol_inputs(cfg: ClipConfig, batch: int, seed: int, pad_fraction: float = 0.0):
    """text = randint(0, vocab) with an optional fraction of positions forced to the pad id
    (pads may sit mid-sequence, as with the benchmark's randint data); images = randn."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    text = torch.randint(0, cfg.num_text_tokens, (batch, cfg.text_seq_len), generator=g)
    if pad_fraction > 0:
        drop = torch.rand((batch, cfg.text_seq_len), generator=g) < pad_fraction
        text = text.masked_fill(drop, cfg.text_pad_id)
    if cfg.text_causal_mask:
        # every row needs an eos token (:670): one per row at a random position >= 1 (a second one
        # later in half of the rows - the reference takes the first), never anywhere else
        eos = cfg.text_eos_id
        other = 1 if eos != 1 else 2
        text = torch.where(text == eos, torch.full_like(text, other), text)
        where = torch.randint(1, cfg.text_seq_len, (batch,), generator=g)
        text[torch.arange(batch), where] = eos
        again = torch.randint(1, cfg.text_seq_len, (batch,), generator=g)
        for r in range(0, batch, 2):
            if again[r] > where[r]:
                text[r, again[r]] = eos
    image = torch.randn((batch, cfg.channels, cfg.visual_image_size, cfg.visual_image_size),
                        generator=g)
    return text, image
