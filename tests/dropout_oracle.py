"""numpy restatement of the attention-dropout mask (csrc/philox.cuh, xclip_attn_dropout_fwd).  TEST
INFRASTRUCTURE ONLY.

Philox4x32-10 (Salmon et al., SC 2011) with the Random123 round constants.  Element (b, h, i, j) of
layer L is kept iff word j & 3 of philox((j >> 2, i, b H + h, L), seed) is below
round((1 - p) 2^32), p taken as fp32 (the C-ABI's type); a kept probability is scaled by 1 / (1 - p).
"""
from __future__ import annotations

import numpy as np
import torch

import attn_oracle as AO
import block_oracle as BO

M0, M1 = 0xD2511F53, 0xCD9E8D57
W0, W1 = 0x9E3779B9, 0xBB67AE85
_LO = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr uint32 [..., 4], key (k0, k1) -> uint32 [..., 4]."""
    ctr = np.asarray(ctr, dtype=np.uint64)
    c0, c1, c2, c3 = (ctr[..., i] for i in range(4))
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    for r in range(10):
        if r:
            k0, k1 = (k0 + np.uint64(W0)) & _LO, (k1 + np.uint64(W1)) & _LO
        p0, p1 = c0 * np.uint64(M0), c2 * np.uint64(M1)
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _LO, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _LO
    return np.stack([c0, c1, c2, c3], -1).astype(np.uint32)


def seed_key(seed: int):
    """int64 seed (as the device tensor holds it) -> Philox key (low word, high word)."""
    s = int(seed) & 0xFFFFFFFFFFFFFFFF
    return s & 0xFFFFFFFF, s >> 32


def keep_threshold(p: float) -> int:
    """keep iff word < this; p rounded to fp32 first"""
    return int(np.rint((1.0 - float(np.float32(p))) * 2.0 ** 32))


def attn_keep(seed: int, B: int, H: int, n: int, layer: int, p: float, rows=None) -> np.ndarray:
    """bool [B, H, len(rows), n]: the kept elements of one layer's attention (rows default: all n)."""
    rows = np.arange(n) if rows is None else np.asarray(rows)
    ng = (n + 3) // 4
    b, h, i, g = np.meshgrid(np.arange(B), np.arange(H), rows, np.arange(ng), indexing="ij")
    ctr = np.stack([g, i, b * H + h, np.full_like(g, layer)], -1).astype(np.uint32)
    words = philox4x32_10(ctr, seed_key(seed)).reshape(B, H, len(rows), 4 * ng)[..., :n]
    return words.astype(np.uint64) < np.uint64(keep_threshold(p))


# --------------------------------------------------------------------------- the same mask in torch
# philox4x32_10 / attn_keep restated on int64 tensors, so the mask of a whole training-shape layer can be
# drawn on the device.  Every 32 x 32-bit product is formed from 16-bit halves, so no intermediate
# leaves the int64 range.

_M32 = 0xFFFFFFFF


def _mulhilo(a: torch.Tensor, m: int):
    """(hi, lo) 32-bit words of the 64-bit product of a (int64 holding uint32) and the constant m."""
    al, ah = a & 0xFFFF, a >> 16
    ml, mh = m & 0xFFFF, m >> 16
    t0 = al * ml
    t1 = al * mh + ah * ml + (t0 >> 16)
    return ah * mh + (t1 >> 16), (t0 & 0xFFFF) | ((t1 & 0xFFFF) << 16)


def philox4x32_10_torch(c0, c1, c2, c3, key):
    """Philox4x32-10 of the counter words (int64 tensors holding uint32) -> 4 int64 tensors of uint32."""
    k0, k1 = key
    for r in range(10):
        if r:
            k0, k1 = (k0 + W0) & _M32, (k1 + W1) & _M32
        h0, l0 = _mulhilo(c0, M0)
        h1, l1 = _mulhilo(c2, M1)
        c0, c1, c2, c3 = h1 ^ c1 ^ k0, l1, h0 ^ c3 ^ k1, l0
    return c0, c1, c2, c3


def attn_keep_torch(seed: int, b0: int, b1: int, H: int, n: int, layer: int, p: float, device="cpu") -> torch.Tensor:
    """attn_keep for the batch items [b0, b1) of a layer: bool [b1 - b0, H, n, n], on `device`."""
    ng = (n + 3) // 4
    dev = torch.device(device)
    bh = torch.arange(b0 * H, b1 * H, device=dev, dtype=torch.int64).view(-1, 1, 1)
    i = torch.arange(n, device=dev, dtype=torch.int64).view(1, -1, 1)
    g = torch.arange(ng, device=dev, dtype=torch.int64).view(1, 1, -1)
    shape = (bh.shape[0], n, ng)
    ctr = [g.expand(shape), i.expand(shape), bh.expand(shape), torch.full(shape, int(layer), device=dev)]
    words = torch.stack(philox4x32_10_torch(*ctr, seed_key(seed)), -1)
    words = words.reshape(b1 - b0, H, n, 4 * ng)[..., :n]
    return words < keep_threshold(p)


def attn_drop_mul_torch(seed: int, b0: int, b1: int, H: int, n: int, layer: int, p: float, device="cpu"):
    """attn_drop_mul for the batch items [b0, b1), drawn with attn_keep_torch."""
    pf = float(np.float32(p))
    keep = attn_keep_torch(seed, b0, b1, H, n, layer, p, device)
    return keep.double() * (0.0 if pf == 1.0 else 1.0 / (1.0 - pf))


def attn_drop_mul(seed: int, B: int, H: int, n: int, layer: int, p: float, device="cpu") -> torch.Tensor:
    """fp64 [B, H, n, n] multiplier M / (1 - p) of the probabilities (0 everywhere at p = 1)."""
    keep = torch.from_numpy(attn_keep(seed, B, H, n, layer, p)).to(device)
    pf = float(np.float32(p))
    return keep.double() * (0.0 if pf == 1.0 else 1.0 / (1.0 - pf))


# --------------------------------------------------------------------------- fp64 references with dropout
# attn_oracle.attn_ref64 and block_oracle.transformer_stack restated with the dropout multiplier
# `drop` (attn_drop_mul) applied to the probabilities after the softmax (x_clip.py:241-243).  Their
# helpers and gate constants are reused; the gates carry the multiplier wherever P meets V or dP.

def _attn_chunk64(qkv, mask, Bc, n, H, scale, causal, o_k, d_o, drop):
    q, k, v = AO.split_heads(qkv, Bc, n, H, 3)
    vis = AO.visible(mask, Bc, n, causal, qkv.device)
    empty = ~vis.any(-1, keepdim=True)
    z = (scale * (q @ k.transpose(-1, -2))).masked_fill(~vis, -float("inf")).masked_fill(empty, 0.0)
    m = z.amax(-1, keepdim=True)
    P = torch.exp(z - m)
    del z
    lsum = P.sum(-1, keepdim=True)
    P /= lsum
    lse = ((m + torch.log(lsum)) * AO.LOG2E).squeeze(-1).masked_fill(empty.squeeze(-1), -AO.FLT_MAX)
    Pd = P * drop
    o = Pd @ v
    Tm = (scale * AO.LOG2E * (q.abs() @ k.abs().transpose(-1, -2))).masked_fill(~vis, 0.0).amax(-1)
    g_lse = (2.0 ** -21 * (Tm + lse.abs()) + (n + 8) * 2.0 ** -24 * AO.LOG2E).masked_fill(empty.squeeze(-1), 0.0)
    eps = (AO.LN2 * (2.0 ** -21 * Tm + g_lse) + 2.0 ** -22)[..., None]
    rel = AO.U + AO.SLACK + eps
    out = dict(o=AO.merge_heads(o), lse=lse, g_o=AO.merge_heads(AO.U * o.abs() + rel * (Pd @ v.abs())), g_lse=g_lse)
    if d_o is None:
        return out
    (do,) = AO.split_heads(d_o, Bc, n, H, 1)
    (ok,) = AO.split_heads(o_k, Bc, n, H, 1)
    delta = (do * ok).sum(-1, keepdim=True)
    dP = (do @ v.transpose(-1, -2)) * drop
    dS = (P * (dP - delta)).masked_fill(~vis, 0.0)
    dv = Pd.transpose(-1, -2) @ do
    dq = scale * (dS @ k)
    dk = scale * (dS.transpose(-1, -2) @ q)
    g_dv = AO.U * dv.abs() + (rel * Pd).transpose(-1, -2) @ do.abs()
    D = (do.abs() @ v.abs().transpose(-1, -2)) * drop
    R = (do.abs() * ok.abs()).sum(-1, keepdim=True)
    A = (rel * dS.abs() + (1 + 2.0 ** -7) * P * (AO.DOT * D + AO.DELTA_ERR * R)).masked_fill(~vis, 0.0)
    g_dq = AO.U * dq.abs() + scale * (A @ k.abs())
    g_dk = AO.U * dk.abs() + scale * (A.transpose(-1, -2) @ q.abs())
    out.update(dqkv=AO.merge_heads(dq, dk, dv), g_dqkv=AO.merge_heads(g_dq, g_dk, g_dv))
    return out


def attn_dropout_ref64(qkv, mask, B, n, H, scale, causal, drop, o, d_o):
    """fp64 attention with dropout of the bf16 qkv the kernel read, and attn_oracle's gates of every
    output: dict(o, lse, g_o, g_lse, dqkv, g_dqkv).  o is the kernel's bf16 o (delta's operand);
    drop fp64 [B, H, n, n].  Runs in chunks of batch items, as attn_oracle.attn_ref64 does."""
    per = max(1, AO.CHUNK_ELEMS // (H * n * n))
    parts = []
    for b0 in range(0, B, per):
        b1 = min(B, b0 + per)
        rows = slice(b0 * n, b1 * n)
        parts.append(_attn_chunk64(qkv[rows], None if mask is None else mask[b0:b1], b1 - b0, n, H, scale, causal,
                                   o[rows], d_o[rows], drop[b0:b1]))
    if len(parts) == 1:
        return parts[0]
    return {key: torch.cat([p[key] for p in parts]) for key in parts[0]}


def transformer_stack_dropout(x, weights, depth, heads, key_mask, causal, rot, attn_drop):
    """block_oracle.transformer_stack (eps pinned, in the dtype of x) with attention dropout: attn_drop
    holds per layer the [B, heads, n, n] multiplier of the probabilities."""
    B, n, d = x.shape
    dt = x.dtype
    eps = BO.LN_EPS
    w = [t.to(dt) for t in weights]
    h = BO._ln(x, w[0], eps)
    for L in range(depth):
        g1, wqkv, wo, go, g2, w1, g4, w2 = w[2 + 8 * L: 10 + 8 * L]
        qkv = (BO._ln(h, g1, eps) @ wqkv.t()).view(B, n, 3, heads, 64).permute(2, 0, 3, 1, 4)
        q, k, v = qkv[0] * 64 ** -0.5, qkv[1], qkv[2]
        if rot is not None:
            c, s = (t.to(dt)[None, None] for t in rot)
            q, k, v = BO._rotate(q, c, s), BO._rotate(k, c, s), BO._rotate(v, c, s)
        sc = q @ k.transpose(-1, -2)
        fill = -torch.finfo(dt).max
        if key_mask is not None:
            sc = sc.masked_fill(~key_mask[:, None, None, :], fill)
        if causal:
            sc = sc.masked_fill(torch.ones(n, n, dtype=torch.bool, device=x.device).triu(1), fill)
        pr = torch.softmax(sc, -1) * attn_drop[L].to(dt)
        o = (pr @ v).permute(0, 2, 1, 3).reshape(B, n, heads * 64)
        h = BO._ln(o @ wo.t(), go, eps) + h
        uu = BO._ln(h, g2, eps) @ w1.t()
        val, gate = uu[..., :4 * d], uu[..., 4 * d:]
        hp = val * (0.5 * gate * (1.0 + torch.erf(gate / 2.0 ** 0.5)))
        h = BO._ln(hp, g4, eps) @ w2.t() + h
    return BO._ln(h, w[1], eps)
