"""Generate the FILIP fixtures at token counts other than 16, 32, 64 and 256 with the machinery of
make_golden.py: the REFERENCE on deterministic protocol weights and inputs, cross-checked against
the oracle before anything is written.

Run in the build container only (the GPU box has no /root/reference):

    python tests/golden/make_golden_filip.py

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

# 48 text tokens, 192 px / patch 16 -> 144 image tokens: the segment-max GEMMs run with seg_len 144
# over the image tokens and seg_len 48 over the text tokens, neither a divisor of the 256-column tile
FILIP_T48_I144 = dict(M.TINY, text_seq_len=48, visual_image_size=192, use_all_token_embeds=True)

CASES = {
    # name: (cfg overrides, batch, pad_fraction, patch_dropout)
    "filip_t48_i144": (dict(FILIP_T48_I144), 5, 0.3, 0.0),
    "filip_t48_i144_dcl_extra": (dict(FILIP_T48_I144, decoupled_contrastive_learning=True,
                                      extra_latent_projection=True), 5, 0.3, 0.0),
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
