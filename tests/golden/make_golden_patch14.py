"""Generate the patch-size goldens: CLIP image towers whose patches hold a number of values that is not
a multiple of 8 (ViT-L/14's 14 x 14 x 3 = 588, one-channel 14 x 14 = 196, 7 x 7 x 3 = 147), from the
reference (lucidrains/x-clip, imported read-only) on the protocol weights and inputs.

    python tests/golden/make_golden_patch14.py

Built on make_golden.py (run_case: loss, gradients, encodings, latents) and make_golden_image_grad.py
(d loss / d image); both cross-check the oracle against the live reference before anything is
written.  Writes only its own cases:

  tiny_p14, tiny_p14_drop  the TINY towers at 56 px / patch 14 (16 patches), patch dropout 0 and 0.5
  tiny_p14_c1              one channel: 196 values per patch
  tiny_p7                  28 px / patch 7: an odd 147 values per patch
  vitl14_shaped            ViT-L/14-shaped image tower (1024 wide, 16 heads, 224 px / 14 = 256 patches,
                           128 kept) with a causal 77-token text tower (768 wide, 12 heads, EOS
                           pooling), latent 768, depth 2 / 1
  vitl14_336_filip         336 px / 14 (576 patches, 288 kept) with use_all_token_embeds=True
  imggrad_p14              d loss / d image at patch 14 with patch dropout 0.5
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
import make_golden_image_grad as MGI  # noqa: E402

TINY_P14 = dict(MG.TINY, visual_image_size=56, visual_patch_size=14)
VITL14_2L = dict(dim_text=768, dim_image=1024, dim_latent=768, num_text_tokens=1000, text_enc_depth=1,
                 text_seq_len=77, text_heads=12, visual_enc_depth=2, visual_heads=16,
                 visual_image_size=224, visual_patch_size=14)

CASES = {
    # name: (cfg overrides, batch, pad fraction, patch dropout)
    "tiny_p14": (dict(TINY_P14), 4, 0.2, 0.0),
    "tiny_p14_drop": (dict(TINY_P14), 4, 0.2, 0.5),
    "tiny_p14_c1": (dict(TINY_P14, channels=1), 4, 0.2, 0.0),
    "tiny_p7": (dict(MG.TINY, visual_image_size=28, visual_patch_size=7), 4, 0.2, 0.5),
    "vitl14_shaped": (dict(VITL14_2L, text_causal_mask=True, text_eos_id=999), 3, 0.1, 0.5),
    # (FILIP needs the CLS text tower: the reference's causal tower does not run with it, make_golden.py)
    "vitl14_336_filip": (dict(VITL14_2L, visual_image_size=336, visual_enc_depth=1, use_all_token_embeds=True),
                         2, 0.3, 0.5),
}
IMGGRAD_CASES = {
    "imggrad_p14": (dict(TINY_P14), 4, 0.2, 0.5, "loss"),
}


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    x_clip = MG.import_reference()
    for name, (cfgk, batch, pad, drop) in CASES.items():
        out = MG.run_case(x_clip, name, cfgk, batch, pad, drop)
        (HERE / f"{name}.json").write_text(json.dumps(out))
        print(f"{name}: loss={out['loss']:.7f} dT={out['dtemperature']:.6f} |g|={out['grad_norm']:.6f}")
    for name, (cfgk, batch, pad, drop, kind) in IMGGRAD_CASES.items():
        out = MGI.run(x_clip, name, cfgk, batch, pad, drop, kind)
        (HERE / f"{name}.json").write_text(json.dumps(out))
        print(f"{name}: loss={out['loss']:.7f} |d image|={out['images'][0]['summ']['sq_sum'] ** 0.5:.6e}")


if __name__ == "__main__":
    main()
