"""fp64 references, gates and input recipes for the generic wgmma GEMM (xclip_gemm_bf16, EPI_STORE).
TEST INFRASTRUCTURE ONLY.

Shared by test_gpu_gemm_fp64.py and by the CPU test test_gemm_edges_gates.py, which builds the same
inputs from the same seeds and checks that every gate is small against the defect it guards.

Gates.  Per element (i, j) of C = alpha A B^T (+ bias) (+ residual) (+ prefill):
- GAMMA * |alpha| * S_ij with S = |A| |B|^T, the sum of |a_ik b_jk| over k: the fp32 accumulation of the
  tensor cores.  A gate relative to S_ij, not to the largest |C|, makes a missing or doubled k-block
  visible in every element, whatever the size of the rest of the output;
- ADD_ULP * (splits + 2) * (|alpha| S_ij + |bias_j| + |res_ij| + |prefill_ij|): the fp32 additions of the
  epilogue and of the split-K reductions (red.add) into the output;
- BF16_REL * |C_ij| for a bf16 output (one rounding of the fp32 result).
Measured on an H100 80GB HBM3 (700 W power limit) over test_gpu_gemm_fp64.py: plain f32 products use at
most 0.034 of their gate (the accumulation error stays below GAMMA / 29), epilogue and split-K cases
at most 0.42 (the fp32 additions), and bf16 outputs 0.996, which is the bf16 rounding bound itself
(a value just above a power of two).  GAMMA keeps that headroom; every bite of
test_gemm_edges_gates.py holds with it.

GAMMA does not hold for long k-block chains: the tensor cores do not round the fp32 accumulation to
nearest, so its error grows with the MMAs of a chain.  At the training step's shapes a latent gradient
(128 k-blocks, one large term early in many rows) erred by 4.1 x GAMMA S, a weight gradient of 1568
k-blocks by 1.8 x.  gemm_gate therefore takes, where given, the larger of GAMMA S and chain_bound: four
ulp per MMA of the running partial sum of the element's own chain (chain_sums64).  Four, not two: one
wgmma (k = 16) aligns its 16 products to the largest exponent among them and the accumulator and
truncates each to two bits below that ulp, so it loses up to 16 / 4 = 4 ulp, all in one direction when
the products share a sign.  Measured on an H100 80GB HBM3 with one MMA of 16 positive products 2^-12 to
2^-32 of a running sum of 1.0: at most 3.995 ulp, 2.2 on average; with mixed signs 3.3.  A bound of
2^-22 |x| (two ulp at the top of a binade) is exceeded there, and was, by 1.05 x, on the MLM head's
weight gradient (168 k-blocks of small same-sign softmax terms).  The bound follows the data: with
products of both signs the running sum grows like the square root of the chain, and a missing or
doubled k-block still spans many gates (test_gemm_edges_gates.py).

Operands have rows of A and rows of B (the output's columns) scaled over three orders of magnitude,
so output tiles of small values exist and their gates are small with them.
"""
from __future__ import annotations

import math
from typing import Optional

import torch

GAMMA = 2.0 ** -16        # fp32 accumulation, as a fraction of S = |A| |B|^T (measured: <= 2^-20.9)
ADD_ULP = 2.0 ** -23      # one fp32 addition, as a fraction of the sum of |terms|
BF16_REL = 2.0 ** -8      # |bf16(v) - v| <= 2^-8 |v|
BLOCK_M, BLOCK_K = 128, 64


def block_n(N: int, K: int) -> int:
    """Tile width xclip_gemm_bf16 picks (csrc/gemm.cu:69-70): 128 where 256 would waste columns (N not a
    multiple of 256 and N <= 1024) and for narrow outputs with short K (N, K <= 768), else 256."""
    narrow_short_k = N <= 768 and K <= 768
    return 128 if ((N % 256 != 0 and N <= 1024) or narrow_short_k) else 256


def split_plan(M: int, N: int, K: int, accumulate: bool, sms: int) -> dict:
    """Split-K count xclip_gemm_bf16 chooses (csrc/gemm.cu:86-113), with the intermediate lo / hi."""
    bn = block_n(N, K)
    num_m, num_n, num_kb = -(-M // BLOCK_M), -(-N // bn), -(-K // BLOCK_K)
    tiles = num_m * num_n
    plan = dict(block_n=bn, tiles=tiles, num_kb=num_kb, splits=1, kb_per=num_kb, lo=None, hi=None)
    if not accumulate or tiles >= sms:
        return plan
    lo = -(-2 * sms // tiles)
    hi = (8 * sms) // tiles
    max_by_k = max(num_kb // 8, 1)
    hi = min(hi, max_by_k)
    best = max(min(lo, max_by_k), 1)
    best_fill = 0.0
    for sp in range(best, hi + 1):
        t = tiles * sp
        fill = t / (-(-t // sms) * sms)
        if fill > best_fill + 0.02:
            best_fill, best = fill, sp
    kb_per = -(-num_kb // best)
    plan.update(splits=-(-num_kb // kb_per), kb_per=kb_per, lo=lo, hi=hi)
    return plan


def split_ranges(plan: dict):
    """[(kb0, kb1)) k-block range of every split."""
    return [(s * plan["kb_per"], min((s + 1) * plan["kb_per"], plan["num_kb"])) for s in range(plan["splits"])]


# --------------------------------------------------------------------------- inputs

def _gen(seed: int) -> torch.Generator:
    return torch.Generator().manual_seed(seed)


def _scales(n: int, gen) -> torch.Tensor:
    """Per-row scales 10^U(-3, 0): tiles of small values next to tiles of large ones."""
    return 10.0 ** (-3.0 * torch.rand(n, 1, generator=gen))


def operands(M: int, N: int, K: int, a_major: int, b_major: int, seed: int):
    """bf16 A (logical [M, K]) and B (logical [N, K]) stored in the given majors ([K, M] / [K, N] for
    MN-major), rows scaled over three orders of magnitude.  CPU tensors."""
    gen = _gen(seed)
    A = (torch.randn(M, K, generator=gen) * _scales(M, gen)).bfloat16()
    B = (torch.randn(N, K, generator=gen) * _scales(N, gen)).bfloat16()
    a = A if a_major == 0 else A.t().contiguous()
    b = B if b_major == 0 else B.t().contiguous()
    return a, b


def epilogue_inputs(M: int, N: int, K: int, res_mode: Optional[str], seed: int):
    """bias fp32 [N], residual bf16 [R, N] and the residual row of every output row (int64 [M]) for
    res_mode None / "row" / "mod" (period 97) / "idx" (rows drawn with repeats from 50).  Their size
    is that of a typical |A B^T| entry of the same column, so every term shows in the output."""
    gen = _gen(seed + 1)
    col = _scales(N, gen).squeeze(1) * K ** 0.5 * 0.3
    bias = torch.randn(N, generator=gen) * col
    if res_mode is None:
        return bias, None, None
    R = {"row": M, "mod": 97, "idx": 50}[res_mode]
    res = (torch.randn(R, N, generator=gen) * col * _scales(R, gen)).bfloat16()
    if res_mode == "row":
        rows = torch.arange(M)
    elif res_mode == "mod":
        rows = torch.arange(M) % R
    else:
        rows = torch.randint(0, R, (M,), generator=gen)
        rows[: min(M, 4)] = rows[0]                  # repeated indices for certain
    return bias, res, rows


def prefill(M: int, N: int, seed: int) -> torch.Tensor:
    """Random non-zero fp32 content of an accumulated output, about as large as the product."""
    gen = _gen(seed + 2)
    return torch.randn(M, N, generator=gen) * _scales(M, gen) * _scales(N, gen).t()


# --------------------------------------------------------------------------- reference and gate

def logical(t: torch.Tensor, major: int) -> torch.Tensor:
    """fp64 [rows, K] view of an operand stored K-major ([rows, K]) or MN-major ([K, rows])."""
    return t.double() if major == 0 else t.double().t()


def gemm64(a, b, a_major=0, b_major=0, alpha=1.0, bias=None, residual=None, res_rows=None, prefill=None,
           k_blocks=None):
    """fp64 alpha A B^T (+ bias) (+ residual[res_rows]) (+ prefill) of the stored operands.  k_blocks
    (a list of (kb0, kb1) ranges of 64-wide k-blocks, repeats allowed) restricts / repeats the sum:
    the gate tests build defective products with it."""
    A, B = logical(a, a_major), logical(b, b_major)
    if k_blocks is None:
        acc = A @ B.t()
    else:
        acc = torch.zeros(A.shape[0], B.shape[0], dtype=torch.float64, device=A.device)
        for kb0, kb1 in k_blocks:
            k0, k1 = kb0 * BLOCK_K, min(kb1 * BLOCK_K, A.shape[1])
            acc += A[:, k0:k1] @ B[:, k0:k1].t()
    out = alpha * acc
    if bias is not None:
        out = out + bias.double()
    if residual is not None:
        out = out + residual.double()[res_rows]
    if prefill is not None:
        out = out + prefill.double()
    return out


def abs_sum64(a, b, a_major=0, b_major=0):
    """S = |A| |B|^T in fp64."""
    return logical(a, a_major).abs() @ logical(b, b_major).abs().t()


# One wgmma (k = 16 for bf16) aligns its 16 products to the largest exponent among them and the fp32
# accumulator and truncates each two bits below that ulp: at most 4 ulp of the largest magnitude it
# adds (measured 3.995).  An ulp of x is 2^-23 floor2(x), floor2(x) = 2^floor(log2 x).
MMA_ULPS = 4.0
ULP = 2.0 ** -23
DRIFT = 1.0 + 2.0 ** -8        # the accumulator the MMA sees may exceed the exact running sum by its error


def _kslice(t, major: int, k0: int, k1: int):
    return t[:, k0:k1] if major == 0 else t[k0:k1]


def floor2(x: torch.Tensor) -> torch.Tensor:
    """2^floor(log2 x) for x > 0, 0 for x = 0."""
    m, e = torch.frexp(x)
    return torch.where(x > 0, torch.ldexp(torch.full_like(x, 0.5), e), torch.zeros_like(x))


def chain_sums64(a, b, a_major=0, b_major=0, ranges=None, k_chunk=8192):
    """fp64 (A B^T, S = |A| |B|^T, P) of the stored operands, P the sum over every 64-wide k-block b of
    floor2(DRIFT (|P_b| + s_b)), P_b the running partial sum of its split's chain after block b and s_b
    the block's share of S: each of the block's four MMAs adds terms no larger than |P_b| + s_b (ranges:
    the k-block ranges of the splits, split_ranges; None: one chain).  Converted to fp64 k_chunk columns
    of K at a time."""
    K = a.shape[1] if a_major == 0 else a.shape[0]
    starts = {0} if ranges is None else {r[0] for r in ranges}
    acc = S = P = run = None
    for k0 in range(0, K, k_chunk):
        k1 = min(K, k0 + k_chunk)
        A, B = logical(_kslice(a, a_major, k0, k1), a_major), logical(_kslice(b, b_major, k0, k1), b_major)
        Aa, Ba = A.abs(), B.abs()
        for j0 in range(0, k1 - k0, BLOCK_K):
            j1 = min(k1 - k0, j0 + BLOCK_K)
            p = A[:, j0:j1] @ B[:, j0:j1].t()
            s = Aa[:, j0:j1] @ Ba[:, j0:j1].t()
            if acc is None:
                acc, S, P = p.clone(), s.clone(), torch.zeros_like(p)
            else:
                acc += p
                S += s
            run = p if (k0 + j0) // BLOCK_K in starts else run + p
            P += floor2(DRIFT * (run.abs() + s))
    return acc, S, P


def chain_bound(S, P):
    """Per-element bound on the accumulation error of the k-block chains: MMA_ULPS ulp for each of the
    four MMAs of every k-block, 16 ULP P, plus ULP S for the final conversion.  The running sum, not
    S, carries the bound: with products of both signs it grows like the square root of the chain and
    one k-block stays visible."""
    return 4.0 * MMA_ULPS * ULP * P + ULP * S


def gemm_gate(a, b, a_major=0, b_major=0, alpha=1.0, bias=None, residual=None, res_rows=None, prefill=None,
              bf16_out=False, splits=1, ref=None, S=None, P=None):
    """Per-element gate of the GEMM output (see the module docstring).  With P (chain_sums64) the
    accumulation term is the larger of GAMMA S and chain_bound(S, P)."""
    if S is None:
        S = abs_sum64(a, b, a_major, b_major)
    terms = abs(alpha) * S
    if bias is not None:
        terms = terms + bias.double().abs()
    if residual is not None:
        terms = terms + residual.double().abs()[res_rows]
    if prefill is not None:
        terms = terms + prefill.double().abs()
    acc = GAMMA * S if P is None else torch.maximum(GAMMA * S, chain_bound(S, P))
    gate = abs(alpha) * acc + ADD_ULP * (splits + 2) * terms
    if bf16_out:
        if ref is None:
            ref = gemm64(a, b, a_major, b_major, alpha, bias, residual, res_rows, prefill)
        gate = gate + BF16_REL * ref.abs()
    return gate


# --------------------------------------------------------------------------- call classes

def res_mode_of(residual, res_row_mod, res_row_idx) -> str:
    if residual is None:
        return "none"
    if res_row_idx is not None:
        return "idx"
    return "mod" if res_row_mod > 0 else "row"


def call_class(M, N, K, a_major, b_major, out_kind, bias, res_mode, alpha) -> tuple:
    """What decides the code path of one EPI_STORE GEMM call: (block_n, a_major, b_major, output kind
    "bf16" / "f32" / "f32acc", bias, residual mode, alpha != 1, partial last N tile, K tail)."""
    bn = block_n(N, K)
    return (bn, a_major, b_major, out_kind, bool(bias), res_mode, alpha != 1.0, N % bn != 0, K % BLOCK_K != 0)


CLASS_FIELDS = ("block_n", "a_major", "b_major", "out", "bias", "residual", "alpha!=1", "partial_n", "k_tail")


# --------------------------------------------------------------------------- embedding backward

RED_REL = 2.0 ** -16      # fp32 sums (red.add / atomicAdd / column sums), as a fraction of the sum of |terms|


def text_embed_bsplit(B: int, n: int, d: int, sms: int) -> int:
    """Batch slices of the text-embedding column sums (csrc/embed.cu:136-138)."""
    return max(1, min(B, (sms * 4) // ((n + 1) * -(-d // 512))))


def text_embed_case(B: int, n: int, d: int, vocab: int, seed: int = 0):
    """ids int64 [B, n] over the whole vocabulary and a bf16 cotangent dx [B, n + 1, d]."""
    gen = _gen(1009 * B + 31 * n + d + vocab + seed)
    ids = torch.randint(0, vocab, (B, n), generator=gen)
    dx = torch.randn(B, n + 1, d, generator=gen).bfloat16()
    return ids, dx


def text_embed_bwd64(ids, dx, vocab: int, pos_rows: int):
    """fp64 (dtok, dpos, dcls) and the per-element sums of |terms| of each."""
    B, n = ids.shape
    d = dx.shape[-1]
    x = dx.double()
    tok = x[:, 1:].reshape(B * n, d)
    idx = ids.reshape(-1).to(x.device)
    dtok = torch.zeros(vocab, d, dtype=torch.float64, device=x.device).index_add_(0, idx, tok)
    atok = torch.zeros(vocab, d, dtype=torch.float64, device=x.device).index_add_(0, idx, tok.abs())
    dpos = torch.zeros(pos_rows, d, dtype=torch.float64, device=x.device)
    apos = torch.zeros_like(dpos)
    dpos[:n] = x[:, 1:].sum(0)
    apos[:n] = x[:, 1:].abs().sum(0)
    return (dtok, atok), (dpos, apos), (x[:, 0].sum(0), x[:, 0].abs().sum(0))


def red_gate(abs_terms: torch.Tensor) -> torch.Tensor:
    return RED_REL * abs_terms


def patch_embed_case(B: int, n: int, k: int, patch_dim: int, d: int, seed: int = 0):
    """Patch-embedding operands: bf16 patches [B k, patch_dim] (rows scaled over three orders of
    magnitude), keep indices [B, k] drawn per sample (so patches repeat across samples), weight fp32
    [d, patch_dim] (bf16-exact), bias [d], position table [n, d] and a bf16 cotangent [B k, d]."""
    gen = _gen(7 * B + 131 * k + d + patch_dim + seed)
    keep = torch.stack([torch.randperm(n, generator=gen)[:k] for _ in range(B)])
    patches = (torch.randn(B * k, patch_dim, generator=gen) * _scales(B * k, gen)).bfloat16()
    w = ((torch.rand(d, patch_dim, generator=gen) * 2 - 1) / patch_dim ** 0.5).bfloat16().float()
    bias = 0.1 * torch.randn(d, generator=gen)
    table = torch.randn(n, d, generator=gen)
    dy = (torch.randn(B * k, d, generator=gen) * _scales(B * k, gen)).bfloat16()
    return dict(keep=keep, patches=patches, w=w, bias=bias, table=table, dy=dy)


def patchify64(img, p):
    """[B, C, H, W] -> [B, (H/p)(W/p), p p C] patch rows in the reference's (p1 p2 c) order, in the
    dtype of img (exact: a permutation)."""
    b, c, H, W = img.shape
    x = img.view(b, c, H // p, p, W // p, p).permute(0, 2, 4, 3, 5, 1)
    return x.reshape(b, (H // p) * (W // p), p * p * c)


# --------------------------------------------------------------------------- AdamW

ADAM_ULP = 2.0 ** -21     # eight fp32 ulp: the roundings of each term of the update (v takes five)


def adamw64(p, g, m, v, lr, b1, b2, eps, wd, step, grad_scale=1.0, defect=None):
    """One AdamW step (csrc/rowwise.cu:826-830, torch.optim.AdamW) in fp64 from the fp32 state, with
    every hyper-parameter rounded to the fp32 the kernel receives -> (p, m, v, gates of p, m, v).

    The gates are ADAM_ULP times the sum of |terms| of each update; that of p takes step_size times
    the sum of |terms| of m over denom as the size of the Adam term.  `defect` builds the wrong
    updates the gate test guards against."""
    f = lambda x: float(torch.tensor(x, dtype=torch.float32))          # noqa: E731
    lr, b1, b2, eps, wd, gs = f(lr), f(b1), f(b2), f(eps), f(wd), f(grad_scale)
    p, g, m, v = (t.double() for t in (p, g, m, v))
    gr = g * gs
    gm = g if defect == "scale_v_only" else gr          # the gradient m sees
    gv = g if defect == "scale_m_only" else gr          # the gradient v sees
    m1 = b1 * m + (1 - b1) * gm
    v1 = b2 * v + (1 - b2) * gv * gv
    t1 = step - 1 if defect == "bc1_step_minus_1" else step
    bc1 = 1.0 if defect == "no_bc1" else 1 - b1 ** t1
    bc2 = 1 - b2 ** step
    step_size = lr / bc1
    if defect == "eps_in_sqrt":
        denom = torch.sqrt(v1 / bc2 + eps)
    else:
        denom = torch.sqrt(v1) / math.sqrt(bc2) + eps
    decay = f(1 - lr * wd)
    if defect == "decay_after":
        p1 = (p - step_size * m1 / denom) * decay
    else:
        p1 = p * decay - step_size * m1 / denom
    am = b1 * m.abs() + (1 - b1) * gm.abs()
    av = b2 * v.abs() + (1 - b2) * gv * gv
    ap = (p * decay).abs() + step_size * am / denom
    return p1, m1, v1, ADAM_ULP * ap, ADAM_ULP * am, ADAM_ULP * av


def adamw_state(n: int, seed: int, step: int, near_eps: bool = False):
    """fp32 p, g, m, v of n elements in a plausible mid-training state; every 7th p is 0 (a zero-initialised
    bias: there the Adam term is all of the update), g has exact zeros and, with near_eps, magnitudes
    around 1e-8 so that eps matters in the denominator."""
    gen = _gen(n % 100003 + 17 * step + seed)
    p = torch.randn(n, generator=gen)
    p[1::7] = 0.0
    g = torch.randn(n, generator=gen) * 10.0 ** (-4 * torch.rand(n, generator=gen))
    g[torch.rand(n, generator=gen) < 0.05] = 0.0
    if near_eps:
        g[::3] = 1e-8 * torch.randn(g[::3].shape, generator=gen)
    if step == 1:
        m = torch.zeros(n)
        v = torch.zeros(n)
    else:
        m = 0.1 * g + 1e-3 * torch.randn(n, generator=gen)
        v = (g * g) * 0.5 + 1e-8 * torch.rand(n, generator=gen)
        if near_eps:
            v[::3] = 1e-17 * torch.rand(v[::3].shape, generator=gen)
    return p, g, m, v
