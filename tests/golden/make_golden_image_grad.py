"""Generate tests/golden/imggrad_*.json: the gradient of the loss with respect to the INPUT IMAGE, from the
reference (lucidrains/x-clip, imported read-only) run with image.requires_grad_(True).

    python tests/golden/make_golden_image_grad.py

Built on make_golden.py (protocol weights and inputs, import_reference, build_reference).  Every case is
cross-checked against oracle/clip_oracle.py, which differentiates to the image through its torch
patchify, before anything is written.  The fixtures record the loss, the parameter-gradient norms, a
summary of d loss / d image, its norm per sample and per (sample, patch), 256 sampled entries and the
PatchDropout `keep`.  Cases: TINY without and with patch dropout, the cfg3-shaped ViT-B/16 tower with
dropout 0.5 (98 of 196 patches), FILIP + DCL + extra projections, multiview with two aug_image views
(one gradient per view), and a guidance objective (eval mode, return_latents=True, (zi * target).sum()).
"""
from __future__ import annotations

import json
import os
import sys
from pathlib import Path

import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent.parent))

import make_golden as MG  # noqa: E402
from oracle import clip_oracle as O  # noqa: E402

IMG_SAMPLES = 256
TARGET_SEED = 555

CASES = {
    # name: (cfg overrides, batch, pad fraction, patch dropout, kind)
    "imggrad_tiny": (dict(MG.TINY), 4, 0.2, 0.0, "loss"),
    "imggrad_tiny_drop": (dict(MG.TINY), 4, 0.2, 0.5, "loss"),
    "imggrad_vitb16_drop": (dict(MG.VITB16_2L), 3, 0.1, 0.5, "loss"),
    "imggrad_tiny_filip_dcl_extra": (dict(MG.TINY, use_all_token_embeds=True, decoupled_contrastive_learning=True,
                                          extra_latent_projection=True), 4, 0.25, 0.0, "loss"),
    "imggrad_tiny_multiview": (dict(MG.TINY), 4, 0.2, 0.0, "multiview"),
    "imggrad_tiny_guidance": (dict(MG.TINY), 4, 0.2, 0.5, "guidance"),
}
AUG_SEED_STRIDE = 17


def patch_norms(g: torch.Tensor, patch: int) -> torch.Tensor:
    """per-(sample, patch) norms [B, n] of an image-shaped tensor, patches in row-major order"""
    return O.patchify(g.detach().double(), patch).norm(dim=-1)


def image_record(g: torch.Tensor, patch: int) -> dict:
    return dict(summ=MG.summ(g), sample_norms=g.detach().double().flatten(1).norm(dim=1).tolist(),
                patch_norms=patch_norms(g, patch).tolist(), samples=MG.sample(g, IMG_SAMPLES, 3))


def guidance_target(cfg: O.ClipConfig, batch: int) -> torch.Tensor:
    g = torch.Generator(device="cpu").manual_seed(TARGET_SEED)
    return torch.randn(batch, cfg.dim_latent, generator=g)


def aug_images(cfg: O.ClipConfig, batch: int, n_aug: int):
    return [O.protocol_inputs(cfg, batch, MG.INPUT_SEED + AUG_SEED_STRIDE * (v + 1), 0.2)[1] for v in range(n_aug)]


def oracle_image_grads(name, cfg, kind, state, text, images, keep, clip_mv_weight=0.1):
    """d objective / d image(s) by the oracle, fp32 CPU; returns (objective, [grad per image])"""
    p = {k: v.clone().requires_grad_(True) for k, v in state.items()}
    ims = [im.clone().requires_grad_(True) for im in images]
    if kind == "loss":
        obj = O.clip_forward(p, text, ims[0], cfg, keep=keep)
    elif kind == "multiview":
        obj = O.clip_forward_multiview(p, [text], ims, cfg, clip_mv_weight)
    else:   # guidance: eval mode (no patch dropout), image latents against a fixed target
        mask = text != cfg.text_pad_id
        zt, zi, _, _ = O.project_latents(O.encode_text(text, mask, p, cfg), O.encode_image(ims[0], p, cfg), p, cfg)
        obj = (zi * guidance_target(cfg, text.shape[0])).sum()
    obj.backward()
    return obj, [im.grad for im in ims], p


def run(x_clip, name, cfg_kwargs, batch, pad, drop, kind):
    cfg = O.ClipConfig(**cfg_kwargs)
    state = O.protocol_state_dict(cfg, MG.WEIGHT_SEED)
    text, image = O.protocol_inputs(cfg, batch, MG.INPUT_SEED, pad)
    clip = MG.build_reference(x_clip, cfg_kwargs, drop, state)
    import x_clip.x_clip as _xc
    _xc.b = batch

    keep = None
    if drop > 0 and kind != "guidance":
        n = (cfg.visual_image_size // cfg.visual_patch_size) ** 2
        torch.manual_seed(MG.DROP_SEED)
        keep = torch.randn(batch, n).topk(max(1, int(n * (1 - drop))), dim=-1).indices
    images = [image] + (aug_images(cfg, batch, 2) if kind == "multiview" else [])
    leaves = [im.clone().requires_grad_(True) for im in images]
    torch.manual_seed(MG.DROP_SEED)
    if kind == "loss":
        obj = clip(text, leaves[0], return_loss=True)
    elif kind == "multiview":
        obj = clip(text, leaves[0], return_loss=True, aug_image=tuple(leaves[1:]))
    else:
        clip.eval()
        lat = clip(text, leaves[0], return_latents=True)
        obj = (lat[1] * guidance_target(cfg, batch)).sum()
    obj.backward()
    grads = {k: q.grad for k, q in clip.named_parameters() if q.grad is not None}
    igrads = [im.grad for im in leaves]

    # --- oracle cross-check against the live reference, before anything is written
    o_obj, o_igrads, p = oracle_image_grads(name, cfg, kind, state, text, images, keep, clip.multiview_loss_weight)
    assert abs(o_obj.item() - obj.item()) <= 3e-6 * max(1.0, abs(obj.item())), (name, o_obj.item(), obj.item())
    for v, (g, og) in enumerate(zip(igrads, o_igrads)):
        assert g is not None and og is not None, (name, v)
        rel = (og - g).norm().item() / (g.norm().item() + 1e-30)
        assert rel < 2e-4, (name, v, rel)
        if keep is not None:        # dropped patches: exactly zero in both
            pn, on = patch_norms(g, cfg.visual_patch_size), patch_norms(og, cfg.visual_patch_size)
            dropped = torch.ones_like(pn, dtype=torch.bool).scatter_(1, keep, False)
            assert (pn[dropped] == 0).all() and (on[dropped] == 0).all(), name
            assert (pn[~dropped] > 0).all(), name
    for k, g in grads.items():
        og = p[k].grad
        assert og is not None and (og - g).norm().item() / (g.norm().item() + 1e-12) < 2e-4, (name, k)

    out = dict(case=name, kind=kind, cfg=cfg_kwargs, batch=batch, pad_fraction=pad, patch_dropout=drop,
               weight_seed=MG.WEIGHT_SEED, input_seed=MG.INPUT_SEED, drop_seed=MG.DROP_SEED,
               loss=obj.item(), grad_norms={k: g.double().norm().item() for k, g in grads.items()},
               images=[image_record(g, cfg.visual_patch_size) for g in igrads],
               keep=None if keep is None else keep.tolist(), torch_version=torch.__version__)
    if kind == "multiview":
        out.update(aug_seed_stride=AUG_SEED_STRIDE, multiview_loss_weight=clip.multiview_loss_weight)
    if kind == "guidance":
        out["target_seed"] = TARGET_SEED
    return out


def freeze_check(x_clip) -> dict:
    """freeze_image_encoder=True: the reference encodes the image under no_grad and detaches
    (x_clip.py:692-698), so image.grad stays None."""
    cfg = O.ClipConfig(**MG.TINY)
    state = O.protocol_state_dict(cfg, MG.WEIGHT_SEED)
    text, image = O.protocol_inputs(cfg, 4, MG.INPUT_SEED, 0.2)
    clip = MG.build_reference(x_clip, dict(MG.TINY), 0.0, state)
    img = image.clone().requires_grad_(True)
    clip(text, img, return_loss=True, freeze_image_encoder=True).backward()
    return dict(case="imggrad_freeze", image_grad_is_none=img.grad is None)


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    x_clip = MG.import_reference()
    for name, (cfgk, batch, pad, drop, kind) in CASES.items():
        out = run(x_clip, name, cfgk, batch, pad, drop, kind)
        (HERE / f"{name}.json").write_text(json.dumps(out))
        print(f"{name}: objective={out['loss']:.7f} |d image|={[im['summ']['sq_sum'] ** 0.5 for im in out['images']]}")
    fr = freeze_check(x_clip)
    assert fr["image_grad_is_none"]
    (HERE / "imggrad_freeze.json").write_text(json.dumps(fr))
    print(fr)


if __name__ == "__main__":
    main()
