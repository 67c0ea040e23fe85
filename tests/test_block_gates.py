"""CPU checks of the transformer-block tests' references and gates (no GPU).

- The fp64 encoder restatement (block_oracle.transformer_stack) agrees with oracle.transformer_stack
  in fp32, where both use eps = 1e-5.
- Each gate of the GPU tests is at most a quarter of the effect of the defect it exists to catch, on
  the inputs those tests build from the same seeds: the largest per-element effect spans at least 4
  gates (`bite` >= 4), so the defect still fails the test after the kernel's own rounding error (at
  most 1 gate) is subtracted.  Loosening a gate later fails here, not silently on the GPU.
"""
import pytest
import torch

import block_oracle as BO
from oracle import clip_oracle as O

BITE = 4.0


@pytest.mark.parametrize("name", ["d512_mask_causal", "d256_rotary"])
def test_restatement_matches_oracle_fp32(name):
    case = BO.block_case(name)
    B, n, d, heads, masked, causal, rotary = BO.BLOCK_CASES[name]
    x = case["x"].float()
    mine = BO.transformer_stack(x, case["weights"], BO.BLOCK_DEPTH, heads, case["mask"], causal, case["rot"])
    p = BO.oracle_params(case["weights"], BO.BLOCK_DEPTH)
    ang = O.rotary_angles(n, 32) if rotary else None
    ref = O.transformer_stack(x, p, "t.", BO.BLOCK_DEPTH, heads, 64, case["mask"], causal, ang)
    err = (mine - ref).abs().max().item()
    assert err <= 1e-4 * ref.abs().max().item(), err


def test_rotary_tables_match_oracle():
    from x_clip_b200.clip import RotaryEmbedding
    for n in (1, 33, 78, 401):
        assert torch.equal(RotaryEmbedding(32)(n, torch.device("cpu")), O.rotary_angles(n, 32))


@pytest.mark.parametrize("rows,d", [(7, 256), (1003, 512), (1003, 1024)])
def test_layernorm_gates_bite(rows, d):
    """Dropping s1 = mean(g dy) or s2 = mean(g dy xhat) from the LayerNorm backward."""
    t = BO.ln_case(rows, d)
    mean, rstd = BO.ln_stats64(t["x"])
    dx, _, s1, s2 = BO.ln_bwd64(t["dy"], t["x"], mean, rstd, t["g"])
    gate = BO.elem_gate(dx + t["add"].double())
    xh = (t["x"].double() - mean[:, None]) * rstd[:, None]
    assert BO.bite(rstd[:, None] * s1.expand_as(dx), gate) >= BITE
    assert BO.bite(rstd[:, None] * xh * s2, gate) >= BITE


def _ff_ref(M, d):
    t = BO.ff_case(M, d)
    w2g = (t["w2"] * t["g4"]).bfloat16()
    colvec = w2g.double().sum(1)
    u, hp64, _ = BO.ff_forward64(t["x"], t["w1"].bfloat16(), t["w2"], t["g4"])
    u, hp = u.bfloat16(), hp64.bfloat16()
    mean, rstd = BO.ln_stats64(hp)
    x2, acc, _ = BO.ff_down64(hp, w2g, colvec, mean, rstd, t["res"])
    a, b = BO.ff_ab64(t["dx"], acc.bfloat16(), colvec, mean, rstd, 4 * d)
    return t, w2g, colvec, u, hp, mean, rstd, x2, a, b


@pytest.mark.parametrize("M,d", [(129, 256), (128, 1024), (1413, 768)])
def test_ff_gates_bite(M, d):
    """Dropping a or b from ff_bwd, mean * colvec from ff_down, vsum from dg4."""
    t, w2g, colvec, u, hp, mean, rstd, x2, a, b = _ff_ref(M, d)
    D4 = 4 * d
    du = BO.ff_bwd64(t["dx"], w2g, u, mean, rstd, a, b).view(M, 2, D4)
    gate = BO.elem_gate(du)
    no_a = BO.ff_bwd64(t["dx"], w2g, u, mean, rstd, torch.zeros_like(a), b).view(M, 2, D4)
    no_b = BO.ff_bwd64(t["dx"], w2g, u, mean, rstd, a, torch.zeros_like(b)).view(M, 2, D4)
    assert BO.bite(no_a - du, gate) >= BITE
    assert BO.bite(no_b - du, gate) >= BITE
    assert BO.bite(rstd[:, None] * mean[:, None] * colvec[None, :], BO.elem_gate(x2)) >= BITE
    # vsum: dW2 is checked bit for bit against g4 (raw - vsum), so any vsum defect fails it; dg4
    dxs = (t["dx"].float() * rstd.float()[:, None]).bfloat16().double()
    vsum = (dxs * mean[:, None]).sum(0)
    raw = dxs.t() @ hp.double()
    tt = (raw - vsum[:, None]) * t["w2"].double()
    dg_gate = BO.RED_REL * (tt.abs().sum(0) + t["dg0"].double().abs())
    assert BO.bite((vsum[:, None] * t["w2"].double()).sum(0), dg_gate) >= BITE
    assert vsum.abs().max() > 0


@pytest.mark.parametrize("name", ["d256_rotary"])
def test_block_gates_bite(name):
    """A reference that skips the rotary inverse in the backward, and one that swaps value and gate,
    move some flat-weight gradient by at least 4 of that weight's gates."""
    case = BO.block_case(name)
    out, grads = BO.block_reference64(case)
    names = BO.flat_names(BO.BLOCK_DEPTH)

    def worst(defect):
        o2, g2 = BO.block_reference64(case, **{defect: True})
        bites = [BO.rel_fro(o2, out) / BO.BLOCK_GATES["out"]]
        bites += [BO.rel_fro(b, a) / BO.BLOCK_GATES[nm.split(".")[0]] for nm, a, b in zip(names, grads, g2)]
        return max(bites)

    assert worst("rotary_bwd_identity") >= BITE
    assert worst("swap_value_gate") >= BITE
