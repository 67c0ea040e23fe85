"""ContrastiveLossFn (engine.py: InfoNCE / DCL, with and without extra latents) against
oracle.clip_oracle.contrastive_loss in fp64, at global batches from 1 to 4096, odd ones included.

The latents come out of ProjectL2NormFn (a bf16 GEMM and xclip_l2norm_fwd), so the loss runs on the
same split-bf16 operands as in the model; the oracle gets those fp32 latents in fp64.  No encoder runs,
so the comparison sees only the similarity and loss kernels.  With an odd batch the image-direction
log-denominators sit at an odd float offset inside the gathered [4, B] statistics, and from B = 33 on
every row has 32-column chunks on the backward's vectorised interior path."""
import math

import pytest
import torch

from test_gpu_filip import _report_peak, _start_peak

pytestmark = pytest.mark.gpu

BF16, F32 = torch.bfloat16, torch.float32
D_IN, D_LAT = 256, 512
BATCHES = [1, 33, 63, 65, 127, 129, 257, 1000, 4095, 4096]
MODES = {"plain": (False, False), "dcl": (True, False), "extra": (False, True), "dcl_extra": (True, True)}

# Measured on an H100 80GB HBM3 (400 W power limit) over every case below: loss rel at most 2.7e-6,
# d temperature rel at most 4.5e-5, latent gradient rel at most 2.75e-3 (two bf16 roundings of ~2^-9
# each, uncorrelated: ~2^-8.5).  The gates keep ~2x headroom (4x for d temperature).
LOSS_REL = 5e-6
DTEMP_REL, DTEMP_ABS = 2e-4, 1e-6
GRAD_REL = 5e-3


def _latents(B, n_sets, dev, seed):
    """n_sets of (fp32 unit latents z carrying the graph, zrow, zcol) through ProjectL2NormFn."""
    from x_clip_b200 import engine as E
    gen = torch.Generator(device=dev).manual_seed(seed)
    out = []
    for _ in range(n_sets):
        e = torch.randn((B, D_IN), generator=gen, device=dev).to(BF16)
        w = (torch.randn((D_LAT, D_IN), generator=gen, device=dev) * D_IN ** -0.5).requires_grad_(True)
        z, zrow, zcol = E.ProjectL2NormFn.apply(e, w)
        z.retain_grad()
        out.append((z, zrow, zcol))
    return out


def _run_loss(B, dcl, extra, temperature, seed):
    """ContrastiveLossFn -> (loss, d temperature, d latents, the fp32 latents)."""
    from x_clip_b200 import engine as E
    dev = torch.device("cuda:0")
    sets = _latents(B, 4 if extra else 2, dev, seed)
    z = [s[0] for s in sets]
    ops = tuple((s[1], s[2]) for s in sets)
    temp = torch.tensor(temperature, device=dev, dtype=F32, requires_grad=True)
    loss = E.ContrastiveLossFn.apply(z[0], z[1], z[2] if extra else None, z[3] if extra else None, temp, ops,
                                     dcl, False)
    loss.backward()
    return loss.item(), temp.grad.item(), [t.grad for t in z], [t.detach() for t in z]


def _oracle(lat, dcl, extra, temperature):
    """oracle.contrastive_loss in fp64 autograd on the GPU -> (loss, d temperature, d latents)."""
    from oracle import clip_oracle as O
    z = [t.double().requires_grad_(True) for t in lat]
    t64 = torch.tensor(temperature, dtype=F32).double().to(lat[0].device).requires_grad_(True)
    zt_x, zi_x = (z[2], z[3]) if extra else (z[0], z[1])
    cfg = O.ClipConfig(decoupled_contrastive_learning=dcl, extra_latent_projection=extra)
    loss = O.contrastive_loss(z[0], z[1], zt_x, zi_x, t64, cfg)
    loss.backward()
    return loss.item(), t64.grad.item(), [t.grad for t in z]


CASES = [(B, mode, temperature) for B in BATCHES for mode in MODES for temperature in (1.0, math.log(100.0))
         if B > 1 or MODES[mode][0]]


@pytest.mark.parametrize("B,mode,temperature", CASES,
                         ids=[f"B{B}-{m}-{'e' if t == 1.0 else '100'}" for B, m, t in CASES])
def test_contrastive_loss_fn_matches_fp64_oracle(cuda_device, B, mode, temperature):
    """Loss rel <= LOSS_REL, d temperature within DTEMP_REL rel + DTEMP_ABS, each latent gradient's
    relative error norm <= GRAD_REL (dZ = bf16(temp g) @ the bf16 hi columns: two bf16 roundings).
    B = 1 runs only under DCL: its denominator is empty, and the loss must be the oracle's finite
    ln(1e-20) - s (measured: rel 4e-8).  At B = 4096 the case with its fp64 reference takes < 0.1 s
    and at most 1.1 GiB on an H100."""
    dcl, extra = MODES[mode]
    t0 = _start_peak()
    loss, dt, grads, lat = _run_loss(B, dcl, extra, temperature, seed=B * 10 + len(mode))
    r_loss, r_dt, r_grads = _oracle(lat, dcl, extra, temperature)
    label = f"B={B} {mode} exp(temperature)={math.exp(temperature):.4g}"
    assert math.isfinite(loss) and math.isfinite(r_loss), (label, loss, r_loss)
    e_loss = abs(loss - r_loss) / abs(r_loss)
    e_dt = abs(dt - r_dt) / (DTEMP_REL * abs(r_dt) + DTEMP_ABS)
    rels = []
    for j, (g, r) in enumerate(zip(grads, r_grads)):
        assert g is not None and bool(torch.isfinite(g).all()), (label, j)
        rels.append((g.double() - r).norm().item() / r.norm().item())
    print(f"nce loss {label}: loss rel {e_loss:.2e} dtemp {dt:.6e} vs {r_dt:.6e} (error/gate {e_dt:.3f}) "
          f"grad rel {max(rels):.2e}")
    assert e_loss <= LOSS_REL, (label, loss, r_loss)
    assert e_dt <= 1.0, (label, dt, r_dt)
    assert max(rels) <= GRAD_REL, (label, rels)
    if B == 4096:
        _report_peak(f"ContrastiveLossFn {label} with its fp64 reference", t0)
