"""Generate the odd-batch fixtures with the machinery of make_golden.py: the REFERENCE on deterministic
protocol weights and inputs, cross-checked against the oracle before anything is written.

Odd global batches put the image-direction log-denominators of ContrastiveLossFn at an odd float
offset inside the gathered [4, B] statistics, and B >= 33 gives every 32-column chunk of the InfoNCE
backward its vectorised interior path.  B = 65 also splits into micro-batches of 32, 32 and 1.

Run in the build container only (the GPU box has no /root/reference):

    python tests/golden/make_golden_odd.py

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

CASES = {
    # name: (cfg overrides, batch, pad_fraction, patch_dropout)
    "tiny_b65": (dict(M.TINY), 65, 0.2, 0.0),
    "tiny_b33_dcl_extra": (dict(M.TINY, decoupled_contrastive_learning=True, extra_latent_projection=True),
                           33, 0.2, 0.0),
}


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    x_clip = M.import_reference()
    for name, (cfgk, batch, padf, drop) in CASES.items():
        out = M.run_case(x_clip, name, cfgk, batch, padf, drop)
        # keep the latents' summaries (shape, sums, first values) only: every sample's full latent
        # would make these fixtures ~0.5 MB each; the parity tests check the summaries when the lists
        # are absent, and the gradients of every parameter either way
        for k in ("text_latents", "image_latents"):
            out.pop(k)
        (M.HERE / f"{name}.json").write_text(json.dumps(out))
        print(f"{name}: loss={out['loss']:.7f} grad_norm={out['grad_norm']:.6f} dtemp={out['dtemperature']:.7f}")


if __name__ == "__main__":
    main()
