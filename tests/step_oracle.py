"""Whole-step fp64 reference of x_clip_b200.CLIP (forward + backward).  TEST INFRASTRUCTURE ONLY.

Built on oracle/clip_oracle.py, run in fp64 on the model's device under `pinned()`: LayerNorm eps
1e-5 (engine.LN_EPS) and the attention softmax in the compute dtype, where the oracle otherwise
follows the reference's own precision rules (eps 1e-3 below fp32, an fp32 softmax).

Every tensor the GPU step casts to bf16 before use is bf16-exact here already (matmul weights, the
patch-embedding weight and bias, the embedding and position tables, the pixels); gains and the
temperature stay fp32.  The weight casts and the patch gather of the GPU step are then exact, and
what is left between the two is the kernels' own activation rounding.

The encoders and the loss terms are restated here (on the oracle's transformer stack) rather than
called through oracle.clip_forward because the step also covers terms clip_forward leaves out -
multiview, similarity regularisation, MLM with a pinned corruption, SimCLR with the identity
augmentation - and because test_step_gates.py measures each gate against glue defects (`DEFECTS`)
restated in the same functions.  test_step_gates.py also checks that without a defect the
restatement in fp32 is oracle.clip_forward.

Used by test_gpu_step_fp64.py (the cases below on an H100) and test_step_gates.py (CPU).
"""
from __future__ import annotations

import contextlib
from typing import Dict, Optional, Sequence

import torch
import torch.nn.functional as F

import simreg_oracle as SR
from oracle import clip_oracle as O

LN_EPS = 1e-5          # engine.LN_EPS

# Glue defects a whole-step gate must catch (test_step_gates.py):
#   pos_cls        the text position table is applied to the CLS slot too (CLS + pos[0])
#   pos_shift      the text position table is indexed by slot: CLS gets row 0, token i row i + 1
#   cls_sum        the vision CLS is projected from the sum of the tokens instead of their mean
#   eos_last       the causal tower pools the LAST eos token instead of the first
#   pos_kept_order under patch dropout the position rows follow the kept order, not the patch index
#   ln_eps         LayerNorm eps 1e-3 (the reference's rule for non-fp32 inputs)
#   filip_pad_mean the FILIP text-to-image mean includes the padded text tokens
#   mv_weight      the multiview main loss misses its (1 - multiview_loss_weight) weight
#   simreg_b2      the similarity regularisation divides by B^2 instead of B (B - 1)
#   mlm_all        the MLM cross entropy is averaged over all positions, not the chosen ones
DEFECTS = ("pos_cls", "pos_shift", "cls_sum", "eos_last", "pos_kept_order", "ln_eps", "filip_pad_mean",
           "mv_weight", "simreg_b2", "mlm_all")

TOK = "text_transformer.token_emb.weight"
POS = "text_transformer.abs_pos_emb.weight"
CLS = "text_transformer.cls_token"
VPOS = "visual_transformer.pos_emb.weight"


@contextlib.contextmanager
def pinned(eps: float = LN_EPS):
    """The oracle with LayerNorm eps `eps` at every dtype and the softmax in the compute dtype."""
    prev = O.PINNED_LN_EPS, O.SOFTMAX_FP32
    O.PINNED_LN_EPS, O.SOFTMAX_FP32 = eps, False
    try:
        yield
    finally:
        O.PINNED_LN_EPS, O.SOFTMAX_FP32 = prev


# --------------------------------------------------------------------------- encoders

def encode_text(p, ids, cfg: O.ClipConfig, key_mask: Optional[torch.Tensor], defects=()):
    """CLIP text tower (x_clip.py:295-338): token + position rows (or rotary angles over n + 1 slots),
    CLS in front unless causal, the transformer.  key_mask None: every token is attended."""
    b, n = ids.shape
    x = p[TOK][ids]
    rot = None
    pos = None
    if cfg.text_rotary_pos_emb:
        rot = O.rotary_angles(n + 1, min(cfg.text_dim_head, 32), ids.device)
    else:
        pos = p[POS][:n]
        if "pos_shift" not in defects:
            x = x + pos[None]
    if not cfg.text_causal_mask:
        cls = p[CLS].expand(b, 1, -1)
        if "pos_cls" in defects:
            cls = cls + pos[:1][None]
        x = torch.cat([cls, x], dim=1)
        if "pos_shift" in defects:
            x = x + torch.cat([pos, torch.zeros_like(pos[:1])])[None]
        if key_mask is not None:
            key_mask = torch.cat([torch.ones_like(key_mask[:, :1]), key_mask], dim=1)
    return O.transformer_stack(x, p, "text_transformer.transformer.", cfg.text_enc_depth, cfg.text_heads,
                               cfg.text_dim_head, key_mask, cfg.text_causal_mask, rot)


def eos_to_front(enc, ids, eos_id, last=False):
    """CLIP._eos_to_front: the encoding at the first (defect: last) eos token moves to index 0."""
    if not last:
        return O.eos_to_front(enc, ids, eos_id)
    b, n, d = enc.shape
    at = n - 1 - (ids == eos_id).flip(1).float().argmax(dim=-1)
    pos = torch.arange(n, device=ids.device)[None].expand(b, -1)
    order = torch.cat([at[:, None], pos[pos != at[:, None]].view(b, n - 1)], dim=1)
    return torch.gather(enc, 1, order[:, :, None].expand(-1, -1, d))


def encode_image(p, img, cfg: O.ClipConfig, keep=None, defects=()):
    """Vision tower (x_clip.py:340-390): patch embedding + position row of each patch, patch dropout by
    explicit kept indices [b, k], the transformer, CLS = to_cls_tokens(mean of the tokens) in front."""
    x = O.patchify(img, cfg.visual_patch_size)
    x = x @ p["visual_transformer.to_tokens.1.weight"].t() + p["visual_transformer.to_tokens.1.bias"]
    pos = p[VPOS][: x.shape[1]]
    if keep is None:
        x = x + pos[None]
    elif "pos_kept_order" in defects:
        x = torch.gather(x, 1, keep[:, :, None].expand(-1, -1, x.shape[-1])) + pos[: keep.shape[1]][None]
    else:
        x = torch.gather(x + pos[None], 1, keep[:, :, None].expand(-1, -1, x.shape[-1]))
    out = O.transformer_stack(x, p, "visual_transformer.transformer.", cfg.visual_enc_depth,
                              cfg.visual_heads, cfg.visual_dim_head, None)
    pooled = out.sum(dim=1) if "cls_sum" in defects else out.mean(dim=1)
    cls = pooled @ p["visual_transformer.to_cls_tokens.1.weight"].t()
    return torch.cat([cls[:, None], out], dim=1)


# --------------------------------------------------------------------------- loss terms

def filip_loss(zt, zi, zt_x, zi_x, temperature, cfg, text_mask, pad_mean=False):
    """oracle.contrastive_loss in FILIP mode; pad_mean: the t2i mean over every text token."""
    if not pad_mean:
        return O.contrastive_loss(zt, zi, zt_x, zi_x, temperature, cfg, text_mask)
    temp = temperature.exp()
    sim = temp * torch.einsum("xtd,yid->xyti", zt, zi)
    sim_x = temp * torch.einsum("xtd,yid->xyti", zt_x, zi_x) if cfg.extra_latent_projection else sim
    t2i = sim.amax(dim=-1).mean(-1)
    i2t = sim_x.masked_fill(~text_mask[:, None, :, None], -torch.finfo(sim_x.dtype).max).amax(dim=-2).mean(-1)
    return O._nce_from_logits(t2i, i2t, cfg.decoupled_contrastive_learning)


def mlm_loss(p, cfg, masked, labels, key_mask, pad_id, all_positions=False):
    """aux.MLM.loss_from (reference mlm.py:96-107): encode the corrupted text, project the chosen
    positions onto the vocabulary (Linear with bias), cross entropy against the original tokens."""
    enc = encode_text(p, masked, cfg, key_mask)[:, 1:]
    sel = labels != pad_id
    logits = enc[sel] @ p["mlm.to_logits.weight"].t() + p["mlm.to_logits.bias"]
    ce = F.cross_entropy(logits, labels[sel], reduction="sum")
    return ce / (sel.numel() if all_positions else sel.sum())


def simclr_loss(p, img, cfg, temperature):
    """aux.SimCLR with the identity augmentation: both views are the image, rep = vision CLS, projector
    Linear -> BatchNorm (batch statistics) -> ReLU -> Linear, NT-Xent without normalisation."""
    pre = "visual_ssl.net.projector."
    rep = encode_image(p, img, cfg)[:, 0]
    h = rep @ p[pre + "0.weight"].t() + p[pre + "0.bias"]
    mu, var = h.mean(0), h.var(0, unbiased=False)
    h = torch.relu((h - mu) * torch.rsqrt(var + 1e-5) * p[pre + "1.weight"] + p[pre + "1.bias"])
    z = h @ p[pre + "3.weight"].t() + p[pre + "3.bias"]
    b = z.shape[0]
    z = torch.cat([z, z])
    logits = (z @ z.t() / temperature).masked_fill(torch.eye(2 * b, dtype=torch.bool, device=z.device),
                                                   -torch.finfo(z.dtype).max)
    target = torch.cat([torch.arange(b, 2 * b), torch.arange(0, b)]).to(z.device)
    return F.cross_entropy(logits, target)


def step_loss(p, c, texts: Sequence[torch.Tensor], images: Sequence[torch.Tensor], keep=None, defects=()):
    """CLIP.forward(texts[0], images[0], return_loss=True, aug_text=texts[1:], aug_image=images[1:])
    (x_clip.py:597-875) for the case `c` (see make_case)."""
    cfg, kw = c["cfg"], c["kw"]
    pad = cfg.text_pad_id
    text_ssl_w = kw.get("text_ssl_loss_weight", 0.05) if kw.get("use_mlm") else 0.0
    image_ssl_w = kw.get("image_ssl_loss_weight", 0.05) if kw.get("use_visual_ssl") else 0.0
    multiview = len(texts) > 1 or len(images) > 1
    mv_w = kw.get("multiview_loss_weight", 0.1) if multiview else 0.0
    sim_w = kw.get("sim_reg_loss_weight", 0.0)

    lat_t, lat_i = [], []
    for t in texts:
        mask = t != pad
        et = encode_text(p, t, cfg, None if kw.get("text_encode_without_mask") else mask, defects)
        if cfg.text_causal_mask:
            et = eos_to_front(et, t, cfg.text_eos_id, "eos_last" in defects)
        lat_t.append(et[:, 1:] if cfg.use_all_token_embeds else et[:, 0])
    for v, im in enumerate(images):
        ei = encode_image(p, im, cfg, keep if v == 0 else None, defects)
        lat_i.append(ei[:, 1:] if cfg.use_all_token_embeds else ei[:, 0])

    def proj(e, name):
        return O.unit_rows(e @ p[name].t())

    extra = cfg.extra_latent_projection
    zs_t = [(proj(e, "to_text_latent.weight"), proj(e, "to_text_latent_extra.weight") if extra else None)
            for e in lat_t]
    zs_i = [(proj(e, "to_visual_latent.weight"), proj(e, "to_visual_latent_extra.weight") if extra else None)
            for e in lat_i]
    losses = []
    for (zt, ztx) in zs_t:
        for (zi, zix) in zs_i:
            ztx_, zix_ = (ztx, zix) if extra else (zt, zi)
            if cfg.use_all_token_embeds:
                losses.append(filip_loss(zt, zi, ztx_, zix_, p["temperature"], cfg, texts[0] != pad,
                                         "filip_pad_mean" in defects))
            else:
                losses.append(O.contrastive_loss(zt, zi, ztx_, zix_, p["temperature"], cfg))
    cl_w = 1.0 - (text_ssl_w + image_ssl_w + (0.0 if "mv_weight" in defects else mv_w))
    loss = cl_w * losses[0]
    if multiview:
        loss = loss + mv_w * torch.stack(losses[1:]).mean()
    if sim_w:
        (zt, ztx), (zi, zix) = zs_t[0], zs_i[0]
        ls = SR.sim_reg_loss(zt, zi, ztx, zix)
        if "simreg_b2" in defects:
            ls = ls * (zt.shape[0] - 1) / zt.shape[0]
        loss = loss + sim_w * ls
    if text_ssl_w:
        masked, labels = (t.to(texts[0].device) for t in c["mlm"])
        loss = loss + text_ssl_w * mlm_loss(p, cfg, masked, labels, texts[0] != pad, pad, "mlm_all" in defects)
    if image_ssl_w:
        loss = loss + image_ssl_w * simclr_loss(p, images[0], cfg, kw.get("simclr_temperature", 0.1))
    return loss


# --------------------------------------------------------------------------- cases

TINY = dict(dim_text=256, dim_image=256, dim_latent=256, num_text_tokens=128, text_enc_depth=2,
            text_seq_len=16, text_heads=4, visual_enc_depth=2, visual_heads=4, visual_image_size=64,
            visual_patch_size=16, visual_patch_dropout=0.0)
DCL_EXTRA = dict(decoupled_contrastive_learning=True, extra_latent_projection=True)
CFG3 = dict(dim_text=512, dim_image=768, dim_latent=512, num_text_tokens=1000, text_seq_len=77, text_heads=8,
            visual_heads=12, visual_image_size=224)
MICRO = dict(DCL_EXTRA, sim_reg_loss_weight=1.0, visual_patch_dropout=0.5, microbatch=3)

# name: CLIP keywords over TINY, and how the batch is made.
#   batch, pad (fraction of pad tokens), text_len (tokens fed, <= text_seq_len), keep ("pinned": a fixed
#   patch-dropout draw that drops patches 0 and 5 of every sample), eos (first / second eos position per
#   row of a causal case), aug (augmented text and image views), image_grad, frozen (requires_grad_(False)),
#   mlm (a pinned corruption), retain (micro-batched step), steps (steps without zero_grad)
CASES: Dict[str, dict] = {
    "default": dict(kw={}, text_len=13),
    "dcl_extra": dict(kw=DCL_EXTRA),
    "drop": dict(kw=dict(visual_patch_dropout=0.5), keep="pinned"),
    "filip_dcl_extra": dict(kw=dict(DCL_EXTRA, use_all_token_embeds=True), batch=5, pad=0.3),
    "rotary": dict(kw=dict(text_rotary_pos_emb=True)),
    "causal": dict(kw=dict(text_causal_mask=True, text_eos_id=5), eos=[(1, 9), (3, None), (7, 13), (10, None),
                                                                       (15, None), (12, 14)]),
    "nomask": dict(kw=dict(text_encode_without_mask=True)),
    "simreg": dict(kw=dict(DCL_EXTRA, decoupled_contrastive_learning=False, sim_reg_loss_weight=3.0)),
    "multiview": dict(kw=DCL_EXTRA, aug=1),
    "vits": dict(kw=dict(dim_text=384, dim_image=384, dim_latent=256, text_heads=6, visual_heads=6,
                         visual_image_size=96)),
    "w128": dict(kw=dict(dim_text=128, dim_image=128, dim_latent=256, text_heads=2, visual_heads=2)),
    "cfg3": dict(kw=CFG3, batch=4, pad=0.1),
    "long": dict(kw=dict(visual_image_size=336), batch=3),
    "imggrad": dict(kw=DCL_EXTRA, image_grad=True),
    "imggrad_drop": dict(kw=dict(DCL_EXTRA, visual_patch_dropout=0.5), keep="pinned", image_grad=True),
    "imggrad_frozen": dict(kw={}, image_grad=True, frozen=True),
    # simclr_temperature 10: at the default 0.1 the identical views make the NT-Xent term exactly 0 in fp64
    "aux": dict(kw=dict(num_text_tokens=120, use_mlm=True, mlm_mask_token_id=2, use_visual_ssl=True,
                        visual_ssl_type="simclr", simclr_temperature=10.0), mlm=True),
    "micro_r0": dict(kw=dict(MICRO, microbatch_retain=0), batch=7),
    "micro_r1": dict(kw=dict(MICRO, microbatch_retain=1), batch=7),
    "micro_auto": dict(kw=dict(MICRO, microbatch_retain="auto"), batch=7),
    "accum": dict(kw=DCL_EXTRA, batch=7, steps=2),
    "accum_micro": dict(kw=dict(DCL_EXTRA, microbatch=3, microbatch_retain=1), batch=7, steps=2),
}


def _bf16_exact(t: torch.Tensor) -> torch.Tensor:
    return t.bfloat16().float()


def _batch(cfg, spec, seed):
    text, image = O.protocol_inputs(cfg, spec.get("batch", 6), seed, spec.get("pad", 0.2))
    text = text[:, : spec.get("text_len", cfg.text_seq_len)]
    if spec.get("eos"):
        eos = cfg.text_eos_id
        text = torch.where(text == eos, torch.full_like(text, eos + 1), text)
        for r, (first, second) in enumerate(spec["eos"]):
            text[r, first] = eos
            if second is not None:
                text[r, second] = eos
    return text, _bf16_exact(image)


def make_case(name: str) -> dict:
    """The case's CLIP (on the CPU, weights made bf16-exact), its inputs and everything pinned."""
    import x_clip_b200
    spec = CASES[name]
    kw = dict(TINY, **spec["kw"])
    fields = set(O.ClipConfig().__dict__)
    cfg = O.ClipConfig(**{k: v for k, v in kw.items() if k in fields})
    if kw.get("use_mlm"):
        cfg.num_text_tokens += 1                      # the [MASK] row of the token table
    torch.manual_seed(17)                             # heads the oracle has no weights for (MLM, SimCLR)
    clip = x_clip_b200.CLIP(**kw)
    clip.load_state_dict(O.protocol_state_dict(cfg, 1234), strict=False)
    if kw.get("use_visual_ssl"):
        clip.visual_ssl.augment1 = clip.visual_ssl.augment2 = torch.nn.Identity()
    with torch.no_grad():
        for k, v in clip.named_parameters():
            if not (k.endswith(".g") or k == "temperature"):
                v.copy_(_bf16_exact(v))
    names = [k for k, _ in clip.named_parameters()]
    c = dict(name=name, spec=spec, kw=kw, cfg=cfg, model=clip, names=names,
             params={k: v.detach().clone() for k, v in clip.named_parameters()},
             image_grad=spec.get("image_grad", False), frozen=spec.get("frozen", False))
    c["batches"] = [_batch(cfg, spec, 4321 + 97 * s) for s in range(spec.get("steps", 1))]
    text, image = c["batches"][0]
    c["aug_text"] = [_batch(cfg, spec, 5000 + v)[0] for v in range(spec.get("aug", 0))]
    c["aug_image"] = [_batch(cfg, spec, 6000 + v)[1] for v in range(spec.get("aug", 0))]
    c["keep"] = None
    if spec.get("keep") == "pinned":
        n = (cfg.visual_image_size // cfg.visual_patch_size) ** 2
        g = torch.Generator().manual_seed(99)
        allowed = torch.tensor([i for i in range(n) if i not in (0, 5)])
        c["keep"] = torch.stack([allowed[torch.randperm(len(allowed), generator=g)[: n // 2]]
                                 for _ in range(text.shape[0])])
    c["mlm"] = None
    if spec.get("mlm"):
        text.clamp_(max=kw["num_text_tokens"] - 1)
        torch.manual_seed(3)
        c["mlm"] = clip.mlm.corrupt(text)
        assert (c["mlm"][1] != cfg.text_pad_id).any()
    return c


def reference(c, device, step: int = 0, keep=None, defects=(), eps: float = LN_EPS):
    """fp64 loss and gradients of one step of case `c` on `device`: dict(loss, grads {name: tensor or
    None}, image_grads [per view, or None])."""
    p = {k: v.to(device).double().requires_grad_(not c["frozen"]) for k, v in c["params"].items()}
    text, image = c["batches"][step]
    texts = [t.to(device) for t in [text] + c["aug_text"]]
    images = [im.to(device).double().requires_grad_(c["image_grad"]) for im in [image] + c["aug_image"]]
    if keep is None and c["keep"] is not None:
        keep = c["keep"]
    keep = None if keep is None else keep.to(device)
    with pinned(1e-3 if "ln_eps" in defects else eps):
        loss = step_loss(p, c, texts, images, keep, defects)
        loss.backward()
    return dict(loss=loss.item(), grads={k: v.grad for k, v in p.items()},
                image_grads=[im.grad for im in images] if c["image_grad"] else None)


# --------------------------------------------------------------------------- gates

def family(name: str) -> str:
    """Gate family of a parameter: the transformer kinds of block_oracle.BLOCK_GATES, the tables and the
    heads around the towers."""
    kinds = {"0.norm.g": "g1", "0.fn.to_qkv.weight": "wqkv", "0.fn.to_out.0.weight": "wo",
             "0.fn.to_out.1.g": "go", "1.norm.g": "g2", "1.fn.net.0.weight": "w1", "1.fn.net.2.g": "g4",
             "1.fn.net.4.weight": "w2"}
    if ".transformer." in name and ".layers." in name:
        return kinds[name.split(".layers.")[1].split(".", 1)[1]]
    if name.endswith("norm_in.g"):
        return "g_in"
    if name.endswith("norm_out.g"):
        return "g_out"
    table = {TOK: "token_emb", POS: "text_pos", CLS: "cls_token", VPOS: "image_pos",
             "visual_transformer.to_tokens.1.weight": "to_tokens_w", "visual_transformer.to_tokens.1.bias":
             "to_tokens_b", "visual_transformer.to_cls_tokens.1.weight": "to_cls_tokens"}
    if name in table:
        return table[name]
    if name.startswith("to_") and "_latent" in name:
        return "latent"
    if name.startswith("mlm."):
        return "mlm_head"
    if name.startswith("visual_ssl."):
        return "ssl_head"
    raise KeyError(name)


# Relative Frobenius gates of test_gpu_step_fp64.py per family, plus the loss (relative), d temperature
# (DTEMP_REL * |ref| + DTEMP_ABS) and d image (per sample): about twice the largest error measured on an
# H100 80GB HBM3 (700 W power limit) over the cases below, FILIP and aux aside.  Largest measured: loss 3.5e-4;
# transformer weights and gains 1.7e-2 .. 2.0e-2 (g1, g_in); token_emb 1.4e-2; text_pos 2.8e-2 and
# cls_token 2.6e-2 (nomask); to_tokens weight 1.3e-2, bias 3.5e-2 and image_pos 3.4e-2 (nomask:
# sums over the batch of per-sample gradients that partly cancel); to_cls_tokens and the latent
# projections 1.8e-2; the MLM head 5.9e-3; d image 1.3e-2; d temperature 0.48 of its gate.
STEP_GATES = {"loss": 7e-4, "g_in": 4e-2, "g_out": 3.5e-2, "g1": 4e-2, "wqkv": 4e-2, "wo": 3.5e-2,
              "go": 3.5e-2, "g2": 4e-2, "w1": 3.5e-2, "g4": 3.5e-2, "w2": 3.5e-2, "token_emb": 3e-2,
              "text_pos": 6e-2, "cls_token": 5e-2, "image_pos": 7e-2, "to_tokens_w": 2.5e-2,
              "to_tokens_b": 7e-2, "to_cls_tokens": 3.5e-2, "latent": 3.5e-2, "mlm_head": 1.2e-2,
              "ssl_head": 8e-2, "image": 2.5e-2}
# Two cases amplify the kernels' rounding, so their gradient gates (not the loss or d temperature
# gates) are scaled by GATE_SCALE.  Measured: rounding the encoder outputs once to bf16, in the reference,
# moves their gradients several times more than the default case's (same weights and batch).
# - FILIP: the segment maxima pick one token per row, and a rounding that reorders two near-equal
#   similarities moves that row's whole gradient to another token.  4-7x the default case's sensitivity;
#   on the H100 up to 2.5x the gates above (latent 8.9e-2, g2 9.0e-2).
# - aux: SimCLR's BatchNorm normalises each projector feature over the 6 samples of the batch.  About 2x
#   the default case's sensitivity in the vision tower and 10x in the projector; on the H100 the vision
#   tower reached 1.5x the gates above (to_tokens weight 3.7e-2) and the SimCLR projector 1.2e-1.
GATE_SCALE = {"filip_dcl_extra": 5.0, "aux": 3.0}
DTEMP_REL, DTEMP_ABS = 1e-2, 1e-3


def rel_fro(got, ref) -> float:
    return ((got.double() - ref.double()).norm() / ref.double().norm().clamp_min(1e-300)).item()


def is_zero(g) -> bool:
    return g is None or not bool(g.ne(0).any())


# Gradients that are zero in exact arithmetic but not in floating point: the bias of the Linear in front
# of SimCLR's training-mode BatchNorm (the normalisation removes any constant shift).  Both sides hold
# rounding noise there, so its error is measured against the gradient of that Linear's weight.
NORM_BY = {"visual_ssl.net.projector.0.bias": "visual_ssl.net.projector.0.weight"}


def ratios(got: dict, ref: dict, scale: float = 1.0) -> Dict[str, float]:
    """Fraction of its gate each gated quantity uses, max over the parameters of a family.  got / ref:
    dict(loss, grads {name: tensor or None}, optional image_grads).  A gradient the reference does not
    have (None or all zero) is not gated here: `structural_errors` checks that.  scale multiplies the
    gradient gates (GATE_SCALE)."""
    out = {"loss": abs(got["loss"] - ref["loss"]) / abs(ref["loss"]) / STEP_GATES["loss"]}
    for k, r in ref["grads"].items():
        if k == "temperature":
            if r is not None:
                g = got["grads"][k]
                out["dtemp"] = abs(g.item() - r.item()) / (DTEMP_REL * abs(r.item()) + DTEMP_ABS)
            continue
        if is_zero(r):
            continue
        g = got["grads"][k]
        f = family(k)
        gate = STEP_GATES[f] * scale
        if g is None:
            v = float("inf")
        elif k in NORM_BY:
            v = (g.double() - r).norm().item() / ref["grads"][NORM_BY[k]].norm().item() / gate
        else:
            v = rel_fro(g, r) / gate
        out[f] = max(out.get(f, 0.0), v)
    for gi, ri in zip(got.get("image_grads") or [], ref.get("image_grads") or []):
        for b in range(ri.shape[0]):
            out["image"] = max(out.get("image", 0.0), rel_fro(gi[b], ri[b]) / (STEP_GATES["image"] * scale))
    return out


def structural_errors(names, got: dict, ref: dict):
    """What must hold exactly, whatever the rounding: a parameter has a gradient (not None, not all 0)
    where and only where the reference has one; rows of the token and position tables that nothing in
    the batch reads (absent ids, positions past the text length, patches dropped in every sample), and
    pixels of dropped patches, get exactly 0."""
    bad = []
    for k in names:
        r, g = ref["grads"][k], got["grads"][k]
        if is_zero(r) and not is_zero(g):
            bad.append(f"{k}: a gradient where the reference has none")
        if not is_zero(r) and is_zero(g) and k not in NORM_BY:
            bad.append(f"{k}: no gradient")
    for k in (TOK, POS, VPOS):
        r, g = ref["grads"].get(k), got["grads"].get(k)
        if r is not None and g is not None and g[~r.ne(0).any(dim=1)].ne(0).any():
            bad.append(f"{k}: non-zero rows where the reference's are 0")
    for gi, ri in zip(got.get("image_grads") or [], ref.get("image_grads") or []):
        if gi[ri == 0].ne(0).any():
            bad.append("image: non-zero gradient on pixels of dropped patches")
    return bad
