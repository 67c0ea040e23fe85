"""fp64 references and gates of the logits + InfoNCE / DCL kernels (xclip_nce_fwd / xclip_nce_bwd).
TEST INFRASTRUCTURE ONLY.

Shared by test_gpu_nce.py and by the per-call checks of bench_call_oracle.py.  The error budget is
test_gpu_nce.py's: logits within temp 2^-16 (what the split-bf16 product keeps of fp32 latents), lse /
pos inherit it plus the fp32 log-sum-exp, g = bf16(temp gscale (...)) per element, d temperature
against the magnitudes of its terms and the count of its fp32 additions.
"""
from __future__ import annotations

import math

import torch

F32 = torch.float32
BF16 = torch.bfloat16
LN_1E20 = math.log(1e-20)
LOGIT_GATE = 2.0 ** -16
BF16_REL = 2.0 ** -7                    # bf16 keeps 8 significant bits: one rounding <= 2^-8 relative


def ref_rows(s, first_pos, dcl):
    """fp64 (lse, pos) of logit rows s [r, C] whose row i has its positive at column first_pos + i.
    An empty DCL denominator (C == 1) gives the reference's ln(1e-20)."""
    r = s.shape[0]
    rows = torch.arange(r, device=s.device)
    pos = s[rows, rows + first_pos]
    if dcl:
        s = s.clone()
        s[rows, rows + first_pos] = -math.inf
    lse = torch.logsumexp(s, dim=1)
    return torch.where(torch.isinf(lse), LN_1E20, lse), pos


def lse_gate(temp, ref_lse):
    """logit error, plus fp32 rounding and exp2 / log2 approximations of the log-sum-exp"""
    return temp * LOGIT_GATE + 2.0 ** -20 * (1.0 + ref_lse.abs())


def exp_rel(temp):
    """Relative error of one exp term of g: the logit error temp * 2^-16 as a relative error of
    exp, with 2x headroom, plus the exp2 argument's fp32 rounding and ex2.approx (2^-18)."""
    return temp * 2.0 * LOGIT_GATE + 2.0 ** -18


def check_bwd_rows(g, s, first_pos, dcl, lse_row, lse_col, w, gs, temp):
    """g [r, >= C] (bf16 temp * g from xclip_nce_bwd) against fp64 for logit rows s [r, C] (temp
    included) with the kernel's own lse_row [r] / lse_col [C].  Returns (max error / gate, sum g s,
    sum |g| |s|, sum |g|) of this block, |g| the magnitude of an element's terms.  The pad columns must
    be exactly zero; under DCL each positive must be exactly bf16(fp32(-w_diag * gs) * temp)."""
    w_row, w_col, w_diag = w
    r, C = s.shape
    rows = torch.arange(r, device=s.device)
    ex = torch.zeros_like(s)
    if w_row:
        ex += w_row * torch.exp(s - lse_row.double()[:, None])
    if w_col:
        ex += w_col * torch.exp(s - lse_col.double()[None, :])
    if dcl:
        ex[rows, rows + first_pos] = 0.0
    g64 = gs * ex
    g64[rows, rows + first_pos] -= gs * w_diag
    ref = temp * g64
    gate = BF16_REL * ref.abs() + temp * gs * ex * exp_rel(temp) + temp * gs * 2.0 ** -120
    got = g[:, :C].double()
    err = ((got - ref).abs() / gate).max().item()
    assert bool((g[:, C:] == 0).all()), "pad columns of g are not zero"
    if dcl:
        want = ((torch.tensor([-w_diag], dtype=F32) * torch.tensor([gs], dtype=F32))
                * torch.tensor([temp], dtype=F32)).to(BF16).to(s.device)
        assert bool((g[rows, rows + first_pos] == want).all()), "DCL positives are not exactly -w_diag"
    # magnitude of each element's terms (its exp terms and the positive's -w_diag cancel at the diagonal)
    mag = gs * ex.abs()
    mag[rows, rows + first_pos] += gs * abs(w_diag)
    return err, (g64 * s).sum().item(), (mag * s.abs()).sum().item(), mag.sum().item()


def dtemp_gate(temp, abs_gs, abs_g, R, C):
    """d temperature = sum g s, gated against the magnitudes of its terms (sum |g| |s| and sum |g| with
    |g| the sum of an element's term magnitudes): the logit error through sum |g|, the exp error through
    sum |g| |s|, and the fp32 summation - 256 sequential terms per thread, a 32-lane tree, one atomic per
    warp and column block."""
    nblk = (C + 255) // 256 if C >= 256 else (C + 127) // 128
    n_add = 256 + 5 + -(-R // 32) * nblk
    return abs_g * temp * LOGIT_GATE + abs_gs * (exp_rel(temp) + n_add * 2.0 ** -24)
