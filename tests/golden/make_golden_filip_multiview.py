"""Generate the FILIP multiview fixtures: CLIP(use_all_token_embeds=True) with aug_text / aug_image, run
by the REFERENCE on the CPU with the protocol weights and inputs of make_golden.py, cross-checked against
tests/filip_multiview_oracle.py (the oracle's encoders and FILIP loss with per-view text masks) before
anything is written.

Run in the build container only (the GPU box has no /root/reference):

    python tests/golden/make_golden_filip_multiview.py

View v's inputs are protocol_inputs(seed INPUT_SEED + 17 v), so an augmented caption has a pad pattern of
its own; `empty` lists (text view, row) pairs set entirely to padding.  Every case records the loss,
d temperature and the gradient norm of every parameter; the image-gradient case also records the norm
of d loss / d image per sample of every image view.
"""
from __future__ import annotations

import json
import os
import sys
from pathlib import Path

import torch

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE))
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE.parent.parent))

import make_golden as M  # noqa: E402
import filip_multiview_oracle as FMV  # noqa: E402
from oracle import clip_oracle as O  # noqa: E402

VIEW_SEED_STRIDE = 17
TINY_FILIP = dict(M.TINY, use_all_token_embeds=True)
DCL_EXTRA = dict(decoupled_contrastive_learning=True, extra_latent_projection=True)
# 48 text tokens x 144 image tokens: neither a divisor of the segment-max GEMM's 256-column tile
T48_I144 = dict(TINY_FILIP, text_seq_len=48, visual_image_size=192)

CASES = {
    # name: (cfg overrides, batch, pad fraction, text views, image views, empty (view, row), image grad)
    "filip_mv_t1i2": (dict(TINY_FILIP), 4, 0.25, 1, 2, (), False),
    "filip_mv_t2i1": (dict(TINY_FILIP), 4, 0.25, 2, 1, (), False),
    "filip_mv_t2i2": (dict(TINY_FILIP), 4, 0.25, 2, 2, (), False),
    "filip_mv_t2i2_dcl_extra": (dict(TINY_FILIP, **DCL_EXTRA), 4, 0.25, 2, 2, ((1, 2),), False),
    "filip_mv_t3i2_empty": (dict(TINY_FILIP), 5, 0.3, 3, 2, ((1, 0), (2, 3)), False),
    "filip_mv_t48_i144_dcl_extra": (dict(T48_I144, **DCL_EXTRA), 3, 0.3, 2, 2, ((1, 1),), False),
    "filip_mv_imggrad_dcl_extra": (dict(TINY_FILIP, **DCL_EXTRA), 4, 0.25, 2, 2, ((1, 3),), True),
}


def view_inputs(cfg: O.ClipConfig, batch: int, pad: float, m: int, n: int, empty):
    """(texts [m], images [n]) of a case: view v from protocol_inputs at seed INPUT_SEED + 17 v."""
    views = [O.protocol_inputs(cfg, batch, M.INPUT_SEED + VIEW_SEED_STRIDE * v, pad) for v in range(max(m, n))]
    texts = [views[v][0].clone() for v in range(m)]
    images = [views[v][1] for v in range(n)]
    for v, row in empty:
        texts[v][row] = cfg.text_pad_id
    return texts, images


def run(x_clip, name, cfgk, batch, pad, m, n, empty, image_grad):
    cfg = O.ClipConfig(**cfgk)
    state = O.protocol_state_dict(cfg, M.WEIGHT_SEED)
    texts, images = view_inputs(cfg, batch, pad, m, n, empty)
    clip = M.build_reference(x_clip, cfgk, 0.0, state)
    import x_clip.x_clip as _xc
    _xc.b = batch
    leaves = [im.clone().requires_grad_(image_grad) for im in images]
    loss = clip(texts[0], leaves[0], return_loss=True,
                aug_text=tuple(texts[1:]) if m > 1 else None,
                aug_image=tuple(leaves[1:]) if n > 1 else None)
    loss.backward()
    grads = {k: q.grad for k, q in clip.named_parameters() if q.grad is not None}

    # --- oracle cross-check against the live reference, before anything is written
    p = {k: v.clone().requires_grad_(True) for k, v in state.items()}
    o_leaves = [im.clone().requires_grad_(image_grad) for im in images]
    o_loss = FMV.clip_forward_filip_multiview(p, texts, o_leaves, cfg, clip.multiview_loss_weight)
    o_loss.backward()
    assert torch.isfinite(loss), name
    assert abs(o_loss.item() - loss.item()) <= 3e-6 * max(1.0, abs(loss.item())), (name, o_loss.item(), loss.item())
    for k, g in grads.items():
        assert p[k].grad is not None, (name, k)
        rel = (p[k].grad - g).norm().item() / (g.norm().item() + 1e-12)
        assert rel < 2e-4, (name, k, rel)
    if image_grad:
        for v, (g, og) in enumerate(zip(leaves, o_leaves)):
            rel = (og.grad - g.grad).norm().item() / (g.grad.norm().item() + 1e-30)
            assert rel < 2e-4, (name, v, rel)

    total = torch.sqrt(sum((g.double() ** 2).sum() for g in grads.values())).item()
    out = dict(case=name, cfg=cfgk, batch=batch, pad_fraction=pad, n_text_views=m, n_image_views=n,
               empty=[list(e) for e in empty], view_seed_stride=VIEW_SEED_STRIDE,
               weight_seed=M.WEIGHT_SEED, input_seed=M.INPUT_SEED,
               multiview_loss_weight=clip.multiview_loss_weight, loss=loss.item(),
               dtemperature=grads["temperature"].item(), grad_norm=total,
               grad_norms={k: g.double().norm().item() for k, g in grads.items()},
               torch_version=torch.__version__)
    if image_grad:
        out["images"] = [dict(sample_norms=im.grad.double().flatten(1).norm(dim=1).tolist()) for im in leaves]
    return out


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    x_clip = M.import_reference()
    for name, args in CASES.items():
        out = run(x_clip, name, *args)
        (HERE / f"{name}.json").write_text(json.dumps(out))
        print(f"{name}: loss={out['loss']:.7f} grad_norm={out['grad_norm']:.6f} dtemp={out['dtemperature']:.7f}")


if __name__ == "__main__":
    main()
