"""Cross-check of the CPU oracle against the REFERENCE on randomly drawn small configurations.

What the reference (lucidrains/x-clip v0.14.4) computed on each configuration is stored by
tests/golden/make_golden.py (random_cases): loss, temperature gradient, per-parameter gradient norms,
encoding and latent summaries in random_configs.json, and fixed samples of every gradient and of both
encodings in random_configs_samples.npy.  The configurations sweep what the named fixtures
(tests/golden/*.json, test_oracle_golden.py) cannot enumerate: widths, head counts, depths, sequence
lengths, batch sizes, pad fractions, patch dropout and every combination of the loss flags."""
import importlib.util
import json
from pathlib import Path

import numpy as np
import pytest
import torch

from oracle import clip_oracle as O

GOLDEN = Path(__file__).parent / "golden"


def _mg():
    spec = importlib.util.spec_from_file_location("make_golden", GOLDEN / "make_golden.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


MG = _mg()
CASES = json.loads((GOLDEN / "random_configs.json").read_text())
SAMPLES = np.load(GOLDEN / "random_configs_samples.npy")


def _summ_close(t, ref, tol=2e-4):
    d = t.detach().double().flatten()
    assert list(t.shape) == ref["shape"]
    assert abs(d.sum().item() - ref["sum"]) <= tol * max(1.0, ref["abs_sum"])
    assert abs(d.abs().sum().item() - ref["abs_sum"]) <= tol * max(1.0, ref["abs_sum"])
    assert abs((d * d).sum().item() - ref["sq_sum"]) <= tol * max(1.0, ref["sq_sum"])
    assert torch.allclose(d[:8], torch.tensor(ref["head"], dtype=torch.float64), atol=5e-4, rtol=1e-3)


@pytest.mark.parametrize("seed", MG.RANDOM_SEEDS)
def test_oracle_equals_live_reference_on_random_configuration(seed):
    out = CASES[seed]
    cfg_kwargs, batch, pad, drop = MG.draw_random_case(seed)
    assert (out["seed"], cfg_kwargs, batch, pad, drop) == (seed, out["cfg"], out["batch"], out["pad_fraction"],
                                                           out["patch_dropout"])
    torch.set_num_threads(4)
    cfg = O.ClipConfig(**cfg_kwargs)
    state = O.protocol_state_dict(cfg, out["weight_seed"])
    text, image = O.protocol_inputs(cfg, batch, out["input_seed"], pad)
    keep = None if out["keep"] is None else torch.tensor(out["keep"])
    p = {k: v.clone().requires_grad_(True) for k, v in state.items()}
    loss, parts = O.clip_forward(p, text, image, cfg, keep=keep, return_parts=True)
    loss.backward()
    assert abs(loss.item() - out["loss"]) <= 5e-6 * max(1.0, abs(out["loss"])), (cfg_kwargs, loss.item(), out["loss"])
    assert abs(p["temperature"].grad.item() - out["dtemperature"]) <= 5e-6

    # element by element at the stored positions: catches permuted / transposed gradients that a norm cannot
    off = out["sample_offset"]

    def take(t, n, sample_seed):
        nonlocal off
        d = t.detach().flatten()
        pos = MG.sample_positions(d.numel(), n, sample_seed)
        ref = torch.from_numpy(SAMPLES[off:off + len(pos)].astype(np.float64))
        off += len(pos)
        return d[pos].double(), ref

    for k, n in out["grad_norms"].items():
        g = p[k].grad
        assert g is not None, (cfg_kwargs, k)
        assert abs(g.double().norm().item() - n) <= 5e-4 * max(n, 1e-5) + 1e-8, (cfg_kwargs, k)
        ours, ref = take(g, MG.RANDOM_SAMPLES, 0)
        scale = n / g.numel() ** 0.5                       # rms of the reference gradient
        assert torch.allclose(ours, ref, rtol=2e-4, atol=2e-4 * scale + 1e-9), (cfg_kwargs, k, ours, ref)
    for name, sample_seed in (("enc_text", 1), ("enc_image", 2)):
        ours, ref = take(parts[name], 2 * MG.RANDOM_SAMPLES, sample_seed)
        assert torch.allclose(ours, ref, atol=2e-4, rtol=1e-4), (cfg_kwargs, name)
        _summ_close(parts[name], out[name])
    _summ_close(parts["text_latents"], out["latents"][0])
    _summ_close(parts["image_latents"], out["latents"][1])
    assert off == (CASES[seed + 1]["sample_offset"] if seed + 1 < len(CASES) else SAMPLES.size)
