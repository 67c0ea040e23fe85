"""Generate the FILIP fixtures at token counts that are not multiples of 16 or exceed 256, with the
machinery of make_golden.py: the REFERENCE on deterministic protocol weights and inputs,
cross-checked against the oracle before anything is written.

Run in the build container only (the GPU box has no /root/reference):

    python tests/golden/make_golden_filip_any.py

Writes only the cases below; make_golden.py and make_golden_filip.py keep writing every other
fixture.
"""
from __future__ import annotations

import json
import os
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import make_golden as M  # noqa: E402

# cfg3's towers at depth 2: 77 text tokens against 196 image tokens (98 with patch dropout 0.5)
VITB16_FILIP = dict(M.VITB16_2L, use_all_token_embeds=True)
# 300 text tokens against 384 px / patch 16 = 576 image tokens: both sides longer than a 256-column
# tile, so segments cross one or two tile edges
FILIP_T300_I576 = dict(M.TINY, text_seq_len=300, visual_image_size=384, use_all_token_embeds=True)
# 7 text tokens against 48 px / patch 16 = 9 image tokens: several segments per 16-column chunk
FILIP_T7_I9 = dict(M.TINY, text_seq_len=7, visual_image_size=48, use_all_token_embeds=True)

CASES = {
    # name: (cfg overrides, batch, pad_fraction, patch_dropout)
    "vitb16_shaped_filip": (dict(VITB16_FILIP), 4, 0.1, 0.0),
    "vitb16_shaped_filip_drop": (dict(VITB16_FILIP), 4, 0.1, 0.5),
    "vitb16_shaped_filip_dcl_extra": (dict(VITB16_FILIP, decoupled_contrastive_learning=True,
                                           extra_latent_projection=True), 4, 0.1, 0.0),
    "filip_t300_i576": (dict(FILIP_T300_I576), 4, 0.3, 0.0),
    "filip_t7_i9": (dict(FILIP_T7_I9), 33, 0.3, 0.0),
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
