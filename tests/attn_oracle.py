"""fp64 reference, gates and input recipes for the fused attention kernels.  TEST INFRASTRUCTURE ONLY.

Shared by the GPU tests (test_gpu_attention.py, test_gpu_attention_long.py) and by the CPU test
test_attn_gates.py, which builds the same inputs from the same seeds and checks that every gate is
small against the defect it guards.  The gate helpers (check, bite, ...) are block_oracle's.

Semantics (x_clip.py:217-244).  s = scale q k^T.  A key is hidden from row i when key_mask[b, j] is
False or, under the causal mask, j > i; hidden scores are set to -max, keys j >= n do not exist.
- A row with a visible key gets the softmax over its visible keys: every hidden p is exactly 0.
- A row with no visible key gets a softmax over n equal scores, p = 1/n for every key.  The kernel
  stores lse = -FLT_MAX for it (m = -FLT_MAX, and -FLT_MAX + log2(n) rounds to -FLT_MAX).
- Backward: masked_fill passes no gradient to a hidden score, so dS = 0 there (and on the whole of
  a row with no visible key); dV still gets P^T dO, with p = 1/n on such rows.
The backward's delta = rowsum(dO * o) uses the kernel's own bf16 o, the operand the kernel reads.

Gates (per element, upper bounds on the kernel's error; u = 2^-8 is one bf16 rounding).
Let T_ij = scale log2(e) sum_d |q_id k_jd| bound the base-2 score t_ij, Tm_i = max over row i's
visible keys.  A 64-long fp32 dot product on the tensor cores (4 chained m16n8k16 MMAs, exact bf16
products) is off by at most 8 roundings of its sum of |terms|: DOT = 2^-21 relative to that sum.
- lse = m + log2(l).  The scores are off by <= DOT Tm; l = sum exp2(t - m) has n fp32 additions
  (n 2^-24 relative), exp2 / log2 approximations add ~2^-22 each, the final add 2^-24 |lse|:
      g_lse = 2^-21 (Tm + |lse|) + (n + 8) 2^-24 log2(e)          (0 on rows with no visible key:
  the kernel must store -FLT_MAX exactly).
- Every recomputed p = exp2(t - lse) then carries a relative error
      eps_i = ln2 (2^-21 Tm_i + g_lse_i) + 2^-22,
  and every p that feeds an MMA is rounded to bf16 (u).  SLACK = 2^-15 covers the second-order
  terms (u^2 = 2^-16), fp32 accumulation of the products (2^-21) and the rescale / 1/l products.
- o = sum_j bf16(p_j) v_j / l, rounded to bf16:
      g_o = u |o| + (u + SLACK + eps_i) (P|V|)_i                (P|V| is also the fp32 floor)
- dv_j = sum_i bf16(p_ij) dO_i, rounded:   g_dv = u |dv| + ((u + SLACK + eps) P)^T |dO|
- dS = p (dp - delta) with dp = dO V^T and delta in fp32: p's error gives eps |dS|, the rounding of
  ds to bf16 u |dS|, and the fp32 errors of dp (DOT D_ij, D = |dO| |V|^T) and of delta (<= 11
  roundings: 2^-20 R_i, R = rowsum |dO| |o|) survive the cancellation dp - delta, scaled by p:
      A = (u + SLACK + eps) |dS| + (1 + 2^-7) P (2^-21 D + 2^-20 R)     on visible entries, 0 else
      g_dq = u |dq| + scale A |K|,    g_dk = u |dk| + scale A^T |Q|
  The cancellation term is what gates n = 1, where dS is exactly 0 and the kernel gives fp32 noise.
"""
from __future__ import annotations

import math
from typing import Optional

import torch

from block_oracle import BF16_REL as U

FLT_MAX = torch.finfo(torch.float32).max
LOG2E = 1.0 / math.log(2.0)
LN2 = math.log(2.0)
DOT = 2.0 ** -21          # fp32 tensor-core dot product over 64 features, relative to sum |terms|
DELTA_ERR = 2.0 ** -20    # fp32 rowsum(dO * o) of the delta kernel, relative to sum |terms|
SLACK = 2.0 ** -15        # second-order and fp32 terms of the bf16-operand gates
CHUNK_ELEMS = 2 ** 25     # (b, h, i, j) elements per reference chunk (256 MB per fp64 n x n tensor)


# --------------------------------------------------------------------------- layout

def split_heads(t: torch.Tensor, B: int, n: int, H: int, parts: int):
    """[B n, parts H 64] -> `parts` fp64 tensors [B, H, n, 64]."""
    x = t.double().reshape(B, n, parts, H, 64).permute(2, 0, 3, 1, 4)
    return tuple(x[i] for i in range(parts))


def merge_heads(*ts: torch.Tensor) -> torch.Tensor:
    """fp64 [B, H, n, 64] tensors -> [B n, len(ts) H 64]."""
    B, H, n, _ = ts[0].shape
    return torch.stack(ts, 0).permute(1, 3, 0, 2, 4).reshape(B * n, len(ts) * H * 64)


def visible(mask: Optional[torch.Tensor], B: int, n: int, causal: bool, device, mask_shift: int = 0,
            causal_diag: bool = True) -> torch.Tensor:
    """[B, 1, n (query), n (key)] bool: key j is visible to row i.  The two keywords build the
    defective variants of the gate tests (a key mask shifted by one key, a causal mask that hides
    the diagonal)."""
    vis = torch.ones(B, 1, n, n, dtype=torch.bool, device=device)
    if mask is not None:
        m = mask if mask_shift == 0 else torch.roll(mask, mask_shift, dims=1)
        vis = vis & m[:, None, None, :]
    if causal:
        vis = vis & torch.ones(n, n, dtype=torch.bool, device=device).tril(0 if causal_diag else -1)
    return vis


# --------------------------------------------------------------------------- reference

def _chunk(qkv, mask, Bc, n, H, scale, causal, o_k, d_o, defect):
    q, k, v = split_heads(qkv, Bc, n, H, 3)
    vis = visible(mask, Bc, n, causal, qkv.device, mask_shift=1 if defect == "mask_shift" else 0,
                  causal_diag=defect != "causal_no_diag")
    empty = ~vis.any(-1, keepdim=True)                                   # [Bc, 1, n, 1]
    z = (scale * (q @ k.transpose(-1, -2))).masked_fill(~vis, -math.inf).masked_fill(empty, 0.0)
    m = z.amax(-1, keepdim=True)
    P = torch.exp(z - m)
    del z
    lsum = P.sum(-1, keepdim=True)
    P /= lsum
    lse = ((m + torch.log(lsum)) * LOG2E).squeeze(-1)
    lse = lse.masked_fill(empty.squeeze(-1), -FLT_MAX)
    o = P @ v
    Tm = (scale * LOG2E * (q.abs() @ k.abs().transpose(-1, -2))).masked_fill(~vis, 0.0).amax(-1)
    g_lse = (2.0 ** -21 * (Tm + lse.abs()) + (n + 8) * 2.0 ** -24 * LOG2E).masked_fill(empty.squeeze(-1), 0.0)
    eps = (LN2 * (2.0 ** -21 * Tm + g_lse) + 2.0 ** -22)[..., None]       # [Bc, H, n, 1]
    out = dict(o=merge_heads(o), lse=lse, P=P,
               g_o=merge_heads(U * o.abs() + (U + SLACK + eps) * (P @ v.abs())), g_lse=g_lse)
    if d_o is None:
        return out
    (do,) = split_heads(d_o, Bc, n, H, 1)
    (ok,) = split_heads(o_k, Bc, n, H, 1)
    delta = 0.0 if defect == "no_delta" else (do * ok).sum(-1, keepdim=True)
    dP = do @ v.transpose(-1, -2)
    if defect == "masked_grad":
        # the backward before rows without a visible key were handled: p = exp2(t - lse) = 1 on every
        # key of such a row, and ds = p (dp - delta) on hidden entries too
        Pb = torch.where(empty, torch.ones_like(P), P)
        dS = Pb * (dP - delta)
    else:
        Pb = P
        dS = (P * (dP - delta)).masked_fill(~vis, 0.0)
    dv = Pb.transpose(-1, -2) @ do
    dq = scale * (dS @ k)
    dk = scale * (dS.transpose(-1, -2) @ q)
    Pe = (U + SLACK + eps) * P
    g_dv = U * dv.abs() + Pe.transpose(-1, -2) @ do.abs()
    D = do.abs() @ v.abs().transpose(-1, -2)
    R = (do.abs() * ok.abs()).sum(-1, keepdim=True)
    A = ((U + SLACK + eps) * dS.abs() + (1 + 2.0 ** -7) * P * (DOT * D + DELTA_ERR * R)).masked_fill(~vis, 0.0)
    g_dq = U * dq.abs() + scale * (A @ k.abs())
    g_dk = U * dk.abs() + scale * (A.transpose(-1, -2) @ q.abs())
    out.update(dqkv=merge_heads(dq, dk, dv), g_dqkv=merge_heads(g_dq, g_dk, g_dv))
    return out


def attn_ref64(qkv, mask, B, n, H, scale, causal=False, o=None, d_o=None, defect=None, keep_p=False):
    """fp64 attention of the bf16 qkv [B n, 3 H 64] the kernel read, and the gates of every output.
    -> dict(o [B n, H 64], lse [B, H, n] (base 2), g_o, g_lse; with d_o also dqkv, g_dqkv).
    o is the kernel's bf16 o (delta's operand); None uses bf16(the reference o).  Runs in chunks of
    batch items so that no fp64 n x n tensor outgrows CHUNK_ELEMS.  defect: None or one of
    "no_delta", "masked_grad", "mask_shift", "causal_no_diag" (CPU gate test only)."""
    per = max(1, CHUNK_ELEMS // (H * n * n))
    parts = []
    for b0 in range(0, B, per):
        b1 = min(B, b0 + per)
        rows = slice(b0 * n, b1 * n)
        mk = None if mask is None else mask[b0:b1]
        ok = None
        if d_o is not None:
            ok = o[rows] if o is not None else None
            if ok is None:
                ok = _chunk(qkv[rows], mk, b1 - b0, n, H, scale, causal, None, None, defect)["o"].bfloat16()
        r = _chunk(qkv[rows], mk, b1 - b0, n, H, scale, causal, ok, None if d_o is None else d_o[rows], defect)
        if not keep_p:
            del r["P"]
        parts.append(r)
    if len(parts) == 1:
        return parts[0]
    return {key: torch.cat([p[key] for p in parts]) for key in parts[0]}


def attn_fwd_blocks64(qkv, mask, B, n, H, scale, causal=False, rescale_l=True, rescale_o=True,
                      lse_skip_block0=False):
    """The kernels' online softmax, one 64-key block at a time, in fp64 on base-2 scores (hidden
    scores -FLT_MAX, as the kernel sets them).  -> (o [B n, H 64], lse [B, H, n]).  Without its
    keywords it is the reference; they build the defects of the gate test: an update that does not
    rescale l (or oacc) when the row maximum grows, and an lse that leaves out block 0's share of l."""
    q, k, v = split_heads(qkv, B, n, H, 3)
    vis = visible(mask, B, n, causal, qkv.device)
    t = (scale * LOG2E * (q @ k.transpose(-1, -2))).masked_fill(~vis, -FLT_MAX)
    m = torch.full((B, H, n, 1), -math.inf, dtype=torch.float64, device=qkv.device)
    lsum = torch.zeros_like(m)
    l0 = torch.zeros_like(m)
    acc = torch.zeros(B, H, n, 64, dtype=torch.float64, device=qkv.device)
    for kb in range(0, n, 64):
        tb = t[..., kb:kb + 64]
        mn = torch.maximum(m, tb.amax(-1, keepdim=True))
        corr = torch.exp2(m - mn)
        p = torch.exp2(tb - mn)
        lsum = (lsum * corr if rescale_l else lsum) + p.sum(-1, keepdim=True)
        l0 = l0 * corr + (p.sum(-1, keepdim=True) if kb == 0 else 0.0)
        acc = (acc * corr if rescale_o else acc) + p @ v[..., kb:kb + 64, :]
        m = mn
    lse = m + torch.log2(lsum - l0 if lse_skip_block0 else lsum)
    return merge_heads(acc / lsum), lse.squeeze(-1)


# --------------------------------------------------------------------------- input recipes

RECIPES = ("flat", "peaked", "late_max", "block_masked", "no_visible")
PEAK = 2.5        # q, k x 2.5: natural-unit scores at scale 1/8 have std ~6 (flat: ~1)
DO_ALONG_O = 3.0  # dO = noise + 3 o / rms(o): delta = rowsum(dO o) is large


def _mask(recipe, B, n, masked, gen):
    if recipe == "block_masked":
        # even items: block 0 masked apart from key 0; odd items: block 0 wholly masked (its rows
        # start from m = -FLT_MAX and must drop what they summed when a visible key arrives).  Both:
        # a middle block and the tail block masked.
        mask = torch.ones(B, n, dtype=torch.bool)
        nb = (n + 63) // 64
        for b in range(B):
            mask[b, :64] = False
            if b % 2 == 0 or nb == 1:
                mask[b, 0] = True
            if nb >= 3:
                mask[b, 64 * (nb // 2):64 * (nb // 2 + 1)] = False
            if nb >= 2:
                mask[b, 64 * (nb - 1):] = False
        return mask
    if recipe == "no_visible":
        # item 3c: the first max(1, n // 3) keys masked (causal rows before them see no key);
        # item 3c + 1: every key masked; item 3c + 2: a random mask that keeps key 0
        mask = torch.rand(B, n, generator=gen) > 0.3
        for b in range(B):
            if b % 3 == 0:
                mask[b, :max(1, n // 3)] = False
            elif b % 3 == 1:
                mask[b] = False
            else:
                mask[b, 0] = True
        return mask
    if not masked:
        return None
    mask = torch.rand(B, n, generator=gen) > 0.3
    mask[:, 0] = True     # the CLS key is always attendable (x_clip.py:335)
    return mask


def attn_case(recipe, B, n, H, causal=False, masked=True, scale=64 ** -0.5, seed=0, device="cpu", mask=None):
    """Seeded inputs of one attention case -> dict(qkv bf16 [B n, 3 H 64], mask bool [B, n] or None,
    d_o bf16 [B n, H 64]).  A given mask replaces the recipe's.
    - flat: randn q, k, v (scores ~ N(0, 1) at scale 1/8).
    - peaked: q and k x PEAK.
    - late_max: q shares a direction c; the first key of every 64-key block after block 0 and the
      last key (the one-key tail block at n = 64k + 1) are planted along c with growing weight, so
      the row maximum of every row beyond block 0 arrives in a late block, by a wide margin.
    - block_masked / no_visible: the masks of _mask; no_visible has rows with no visible key.
    d_o has a component along the reference o (DO_ALONG_O), so the - delta term of dS is large."""
    gen = torch.Generator().manual_seed(1000003 * seed + 7919 * n + 131 * H + 17 * B + RECIPES.index(recipe))

    def r(*s):
        return torch.randn(*s, generator=gen)

    q, k, v = r(B, n, H, 64), r(B, n, H, 64), r(B, n, H, 64)
    if recipe == "peaked":
        q, k = q * PEAK, k * PEAK
    if recipe == "late_max":
        c = torch.ones(64) / 8.0
        q = q + 4.0 * c
        planted = sorted(set(range(64, n, 64)) | {n - 1})
        for j in planted:
            k[:, j] = 16.0 * (1.0 + j / n) * c
    recipe_mask = _mask(recipe, B, n, masked, gen)
    mask = recipe_mask if mask is None else mask
    qkv = torch.stack([q, k, v], 2).reshape(B * n, 3 * H * 64).bfloat16().to(device)
    mask = None if mask is None else mask.to(device)
    noise = r(B * n, H, 64).to(device)
    o = attn_ref64(qkv, mask, B, n, H, scale, causal)["o"].view(B * n, H, 64)
    rms = o.pow(2).mean(-1, keepdim=True).sqrt().clamp_min(1e-30)
    d_o = (noise.double() + DO_ALONG_O * o / rms).reshape(B * n, H * 64).bfloat16()
    return dict(qkv=qkv, mask=mask, d_o=d_o)
