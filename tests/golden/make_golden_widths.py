"""Generate the model-width fixtures (widths that are odd multiples of 128, and attention widths
heads * 64 that differ from the model width) with the machinery of make_golden.py: the REFERENCE on
deterministic protocol weights and inputs, cross-checked against the oracle before anything is written.
The similarity-regularisation case follows make_golden_simreg.py.

Run in the build container only (the GPU box has no /root/reference):

    python tests/golden/make_golden_widths.py

Writes only the cases below; the other generators keep writing every other fixture.
"""
from __future__ import annotations

import json
import os
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import make_golden as M  # noqa: E402
import make_golden_simreg as MS  # noqa: E402

# 128 wide with 2 heads: the smallest width (no full 256-column vector in the row-wise kernels)
TINY128 = dict(M.TINY, dim_text=128, dim_image=128, dim_latent=128, text_heads=2, visual_heads=2)
# ViT-S/16-shaped towers at depth 2: width 384, 6 heads, 224 px / patch 16 (196 patches, 98 under patch
# dropout), 77 text tokens + CLS, latent 384
VITS16_2L = dict(dim_text=384, dim_image=384, dim_latent=384, num_text_tokens=1000, text_enc_depth=2,
                 text_seq_len=77, text_heads=6, visual_enc_depth=2, visual_heads=6,
                 visual_image_size=224, visual_patch_size=16)
# 384 wide with the default 8 heads: attention width 512 != model width
W384_H8 = dict(M.TINY, dim_text=384, dim_image=384, dim_latent=384, text_heads=8, visual_heads=8)
# ViT-B/16-plus-shaped at depth 1: text 640 / 10 heads, image 896 / 14 heads at 240 px / 16 (225 patches),
# latent 640
B16PLUS_1L = dict(dim_text=640, dim_image=896, dim_latent=640, num_text_tokens=1000, text_enc_depth=1,
                  text_seq_len=77, text_heads=10, visual_enc_depth=1, visual_heads=14,
                  visual_image_size=240, visual_patch_size=16)

CASES = {
    # name: (cfg overrides, batch, pad_fraction, patch_dropout)
    "tiny128_h2": (dict(TINY128), 6, 0.2, 0.0),
    "vits16_shaped": (dict(VITS16_2L), 4, 0.1, 0.0),            # image attention n = 196, text n = 78
    "vits16_shaped_drop": (dict(VITS16_2L), 4, 0.1, 0.5),       # image attention n = 98
    "w384_h8": (dict(W384_H8), 6, 0.2, 0.0),
    "b16plus_shaped_dcl_extra": (dict(B16PLUS_1L, decoupled_contrastive_learning=True,
                                      extra_latent_projection=True), 4, 0.1, 0.0),
    "vits16_filip": (dict(VITS16_2L, text_enc_depth=1, visual_enc_depth=1, use_all_token_embeds=True),
                     4, 0.25, 0.5),
    "vits16_text_causal": (dict(VITS16_2L, text_causal_mask=True, text_eos_id=999, visual_enc_depth=1),
                           4, 0.1, 0.5),
}
SIMREG_CASES = {
    "vits16_simreg_extra": (dict(VITS16_2L, text_enc_depth=1, visual_enc_depth=1, extra_latent_projection=True),
                            4, 0.1, 0.0),
}


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    x_clip = M.import_reference()
    for name, (cfgk, batch, padf, drop) in CASES.items():
        out = M.run_case(x_clip, name, cfgk, batch, padf, drop)
        # latents are kept as summaries (shape, sums, first values), as for the FILIP fixtures: the
        # full [B, D] lists would make up nearly all of each file
        out.pop("text_latents", None)
        out.pop("image_latents", None)
        (M.HERE / f"{name}.json").write_text(json.dumps(out))
        print(f"{name}: loss={out['loss']:.7f} grad_norm={out['grad_norm']:.6f} dtemp={out['dtemperature']:.7f}")
    for name, (cfgk, batch, padf, drop) in SIMREG_CASES.items():
        w = MS.pick_weight(cfgk, batch, padf)
        out = MS.run_case(x_clip, name, cfgk, batch, padf, drop, w)
        (M.HERE / f"{name}.json").write_text(json.dumps(out))
        print(f"{name}: w={w} loss={out['loss']:.7f} (w=0: {out['loss_without_sim_reg']:.7f}) "
              f"grad_norm={out['grad_norm']:.6f} dtemp={out['dtemperature']:.7f}")


if __name__ == "__main__":
    main()
