"""Generate the long-sequence fixtures (attention n > 320, the streaming kernels) with the machinery
of make_golden.py: the REFERENCE on deterministic protocol weights and inputs, cross-checked against
the oracle before anything is written.

Run in the build container only (the GPU box has no /root/reference):

    python tests/golden/make_golden_long.py

Writes only the cases below; make_golden.py keeps writing every other fixture.
"""
from __future__ import annotations

import json
import os
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import make_golden as M  # noqa: E402

# 400 text tokens + CLS (n = 401), 400 px / patch 16 -> 625 image tokens
LONG = dict(dim_text=256, dim_image=256, dim_latent=256, num_text_tokens=512, text_enc_depth=1,
            text_seq_len=400, text_heads=4, visual_enc_depth=1, visual_heads=4,
            visual_image_size=400, visual_patch_size=16)

CASES = {
    # name: (cfg overrides, batch, pad_fraction, patch_dropout); patch dropout 0: every token reaches attention
    "long_t401_i625": (dict(LONG), 4, 0.2, 0.0),                  # text 401, image 625 (ragged last blocks)
    "long_rotary_t401": (dict(LONG, text_rotary_pos_emb=True), 4, 0.2, 0.0),   # rotary beyond position 320
    # ViT-B/16 at 384 px: image 576, text 78
    "vitb16_384_shaped": (dict(M.VITB16_2L, visual_image_size=384, text_enc_depth=1, visual_enc_depth=1),
                          4, 0.2, 0.0),
}


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    x_clip = M.import_reference()
    for name, (cfgk, batch, padf, drop) in CASES.items():
        out = M.run_case(x_clip, name, cfgk, batch, padf, drop)
        (M.HERE / f"{name}.json").write_text(json.dumps(out))
        print(f"{name}: loss={out['loss']:.7f} grad_norm={out['grad_norm']:.6f} dtemp={out['dtemperature']:.7f}")


if __name__ == "__main__":
    main()
