"""fp64 references and input recipes for the transformer-block kernels.  TEST INFRASTRUCTURE ONLY.

Shared by the GPU kernel tests (test_gpu_rowwise.py, test_gpu_ff.py, test_gpu_rotary.py,
test_gpu_transformer_fp64.py) and by the CPU test test_block_gates.py, which builds the same inputs
from the same seeds and checks that every gate is small against the defect it guards.

Gates.  A kernel that computes in fp32 and rounds its output once to bf16 is off from the exact
result by at most 2^-8 |ref| (round to nearest, 8 significant bits) plus its fp32 error.  The gates
are per element: `BF16_REL * |ref|` plus an absolute floor of `FLOOR * max |ref|` over the row, which
covers the fp32 accumulation error and the absolute (not relative) accuracy of the GELU's negative
tail (A&S 7.1.26, and Phi = 0.5 - q in gelu_parts2), both around 1e-7 of the row's scale.

The encoder restatement (`transformer_stack`) pins the LayerNorm eps to 1e-5 (engine.LN_EPS):
oracle.gain_layernorm picks eps by dtype, 1e-5 for fp32 and 1e-3 otherwise, so the oracle run in
fp64 would be a different function.
"""
from __future__ import annotations

import math
from typing import Optional, Sequence

import torch

BF16_REL = 2.0 ** -8      # |bf16(v) - v| <= 2^-8 |v|
FLOOR = 2.0 ** -16        # absolute floor, as a fraction of the row's largest |ref|
LN_EPS = 1e-5             # engine.LN_EPS
STAT_REL = 1e-5           # LayerNorm statistics (fp32 reductions)
RED_REL = 2.0 ** -16      # fp32 column / row sums, as a fraction of the sum of |terms|


# --------------------------------------------------------------------------- gates

def elem_gate(ref: torch.Tensor, rel: float = BF16_REL, floor: float = FLOOR) -> torch.Tensor:
    """Per element: rel * |ref| + floor * max |ref| over the last dim."""
    a = ref.abs()
    return rel * a + floor * a.amax(-1, keepdim=True)


def gate_ratio(got: torch.Tensor, ref: torch.Tensor, gate: torch.Tensor) -> float:
    """max over elements of |got - ref| / gate (0 where both are 0)."""
    err = (got.double() - ref.double()).abs()
    return (err / gate.double().clamp_min(1e-300)).max().item() if err.numel() else 0.0


def bite(effect: torch.Tensor, gate: torch.Tensor) -> float:
    """How many gates the largest effect of a defect spans (max over elements of |effect| / gate)."""
    return (effect.double().abs() / gate.double().clamp_min(1e-300)).max().item()


def check(name: str, got: torch.Tensor, ref: torch.Tensor, gate: torch.Tensor) -> float:
    """Assert |got - ref| <= gate everywhere; print the largest fraction of the gate used."""
    r = gate_ratio(got, ref, gate)
    print(f"GATE {name} {r:.4f}")
    assert r <= 1.0, f"{name}: error is {r:.3f} x its gate"
    return r


def gelu64(x):
    return 0.5 * x * (1.0 + torch.erf(x / math.sqrt(2.0)))


def gelu_grad64(x):
    return 0.5 * (1.0 + torch.erf(x / math.sqrt(2.0))) + x * torch.exp(-0.5 * x * x) / math.sqrt(2.0 * math.pi)


# --------------------------------------------------------------------------- LayerNorm

def ln_stats64(x, eps=LN_EPS):
    x = x.double()
    mean = x.mean(-1)
    var = ((x - mean[:, None]) ** 2).mean(-1)
    return mean, 1.0 / torch.sqrt(var + eps)


def ln_bwd64(dy, x, mean, rstd, g):
    """-> (dx, dg, s1, s2) of the gain-only LayerNorm at the given statistics (all fp64)."""
    xh = (x.double() - mean.double()[:, None]) * rstd.double()[:, None]
    gd = dy.double() * g.double()
    s1 = gd.mean(-1, keepdim=True)
    s2 = (gd * xh).mean(-1, keepdim=True)
    dx = rstd.double()[:, None] * (gd - s1 - xh * s2)
    return dx, (dy.double() * xh).sum(0), s1, s2


def ln_case(rows: int, d: int, device="cpu"):
    """LayerNorm inputs whose row terms are large: x rows with a sizeable mean, dy with a component
    along g (so mean(g dy) is O(1), not ~1/sqrt(d)) and one along xhat (so is mean(g dy xhat))."""
    gen = torch.Generator().manual_seed(7919 * rows + d)

    def r(*s):
        return torch.randn(*s, generator=gen)

    x = (r(rows, d) * (0.5 + r(rows, 1).abs()) + 3 * r(rows, 1)).bfloat16()
    g = 1 + 0.1 * r(d)
    g2 = 1 + 0.1 * r(d)
    res = r(rows, d).bfloat16()
    add = r(rows, d).bfloat16()
    mean, rstd = ln_stats64(x)
    xh = ((x.double() - mean[:, None]) * rstd[:, None]).float()
    dy = (r(rows, d) + (1 + 0.5 * r(rows, 1)) * g + (1 + 0.5 * r(rows, 1)) * xh).bfloat16()
    dg0 = 10 * r(d)                                   # non-zero prefill of the gain gradient
    t = dict(x=x, g=g, g2=g2, res=res, add=add, dy=dy, dg0=dg0)
    return {k: v.to(device) for k, v in t.items()}


# --------------------------------------------------------------------------- fused feed-forward

GATE_CORR = 1.5     # gate rows = 1.5 x their value rows + noise: hp rows get |mean| ~ std


def ff_permute(w1: torch.Tensor) -> torch.Tensor:
    """Row order of xclip_ff_permute_cast: tile t holds value rows [64t, 64t+64) then the matching gate rows."""
    d = w1.shape[1]
    v, g = w1[:4 * d].view(-1, 64, d), w1[4 * d:].view(-1, 64, d)
    return torch.cat([v, g], dim=1).reshape(8 * d, d)


def ff_unpermute(w1p: torch.Tensor) -> torch.Tensor:
    """Inverse of ff_permute: [value rows | gate rows] from the tile order of xclip_ff_permute_cast."""
    d = w1p.shape[1]
    t = w1p.view(-1, 128, d)
    return torch.cat([t[:, :64].reshape(4 * d, d), t[:, 64:].reshape(4 * d, d)])


def ff_forward64(x, w1b, w2, g4, eps=LN_EPS):
    """fp64 restatement of x_clip.py:180-199 (value first, gate second): -> (u, hp, y = LN(hp) g4 W2^T)."""
    u = x.double() @ w1b.double().t()
    h = u.shape[1] // 2
    hp = u[:, :h] * gelu64(u[:, h:])
    mean, rstd = ln_stats64(hp, eps)
    y = ((hp - mean[:, None]) * rstd[:, None] * g4.double()) @ w2.double().t()
    return u, hp, y


def ff_case(M: int, d: int, device="cpu"):
    """Fused feed-forward inputs whose LayerNorm-fold terms are large.
    - W1's gate rows are correlated with their value rows, so hp rows have |mean| comparable to std
      (with independent rows |mean|/std ~ 0.02 and every fold term hides under bf16 noise).
    - dx has a component along colvec, so a = mean_k gdh is large, and the odd rows one along the
      block's output y_r, so b = mean_k gdh hn is large there."""
    gen = torch.Generator().manual_seed(7919 * M + d + 1)

    def r(*s):
        return torch.randn(*s, generator=gen)

    def u(*s):
        return torch.rand(*s, generator=gen) * 2 - 1

    x = r(M, d).bfloat16()
    wv = u(4 * d, d) / d ** 0.5
    wg = GATE_CORR * wv + 0.5 * u(4 * d, d) / d ** 0.5
    w1 = torch.cat([wv, wg])
    w2 = u(d, 4 * d) / (4 * d) ** 0.5
    g4 = 1 + 0.1 * r(4 * d)
    res = r(M, d).bfloat16()
    noise = r(M, d)
    dg0 = r(4 * d)                                    # non-zero prefill of the gain gradient
    t = {k: v.to(device) for k, v in dict(x=x, w1=w1, w2=w2, g4=g4, res=res, noise=noise, dg0=dg0).items()}
    colvec = (t["w2"] * t["g4"]).bfloat16().double().sum(1)
    _, _, y = ff_forward64(t["x"], t["w1"].bfloat16(), t["w2"], t["g4"])
    sd = 3 * d ** 0.5
    dx = t["noise"].double() + sd * colvec / colvec.norm()
    odd = torch.arange(M, device=dx.device) % 2 == 1
    dx[odd] += sd * y[odd] / y[odd].norm(dim=1, keepdim=True).clamp_min(1e-30)
    t["dx"] = dx.bfloat16()
    del t["noise"]
    return t


def ff_rowsum64(hp):
    """Per row and 64-column box: (sum, sum of squares) of hp, [M, 4d/64, 2]."""
    h = hp.double().view(hp.shape[0], -1, 64)
    return torch.stack([h.sum(-1), (h * h).sum(-1)], dim=-1)


def ff_down64(hp, w2g, colvec, mean, rstd, res):
    """x2 = rstd (hp w2g^T - mean colvec) + res and acc = hp w2g^T at the given statistics."""
    acc = hp.double() @ w2g.double().t()
    y = rstd.double()[:, None] * (acc - mean.double()[:, None] * colvec.double()[None, :])
    return y + res.double(), acc, y


def ff_ab64(dx, acc, colvec, mean, rstd, D4):
    a = (dx.double() @ colvec.double()) / D4
    t = (dx.double() * acc.double()).sum(1)
    b = rstd.double() * (t - mean.double() * a * D4) / D4
    return a, b


def ff_bwd64(dx, w2g, u, mean, rstd, a, b):
    """du = [d value | d gate] of LN(4d) + GEGLU at the given row statistics and row means."""
    h = u.shape[1] // 2
    gdh = dx.double() @ w2g.double()
    val, gate = u[:, :h].double(), u[:, h:].double()
    ge = gelu64(gate)
    hn = (val * ge - mean.double()[:, None]) * rstd.double()[:, None]
    dhp = rstd.double()[:, None] * (gdh - a.double()[:, None] - hn * b.double()[:, None])
    return torch.cat([dhp * ge, dhp * val * gelu_grad64(gate)], dim=1)


# --------------------------------------------------------------------------- rotary

def rotary_tables(n: int, device="cpu"):
    """fp32 cos / sin [n, 16] exactly as clip.TextTransformer hands them to the kernel."""
    from x_clip_b200.clip import RotaryEmbedding
    ang = RotaryEmbedding(32)(n, torch.device("cpu"))[:, :16].float()
    return ang.cos().contiguous().to(device), ang.sin().contiguous().to(device)


class TableAngles:
    """Stands in for the angle table of oracle.rotate_features, whose cos() / sin() return the fp32
    tables the kernel reads (in fp64), so the reference rotates by exactly the kernel's numbers."""

    def __init__(self, cos, sin):
        self.c = torch.cat([cos, cos], -1).double()
        self.s = torch.cat([sin, sin], -1).double()
        self.shape = self.c.shape

    def cos(self):
        return self.c

    def sin(self):
        return self.s


def rotate64(t, cos, sin, inverse=False):
    """Rotary of the first 32 features of each 64-wide slice of t [rows = B n, nslices * 64], in fp64."""
    from oracle import clip_oracle as O
    n = cos.shape[0]
    rows, w = t.shape
    x = t.double().view(rows // n, n, w // 64, 64).transpose(1, 2)        # [B, slices, n, 64]
    out = O.rotate_features(TableAngles(cos, -sin if inverse else sin), x)
    return out.transpose(1, 2).reshape(rows, w)


# --------------------------------------------------------------------------- the encoder

PARAM_KINDS = ("g1", "wqkv", "wo", "go", "g2", "w1", "g4", "w2")


def flat_names(depth: int):
    """Names of TransformerFn's flat weights: [norm_in.g, norm_out.g] + depth * PARAM_KINDS."""
    return ["g_in", "g_out"] + [f"{k}.{L}" for L in range(depth) for k in PARAM_KINDS]


def oracle_params(weights: Sequence[torch.Tensor], depth: int, prefix: str = "t.") -> dict:
    """The flat weights under the parameter names of oracle.transformer_stack."""
    p = {prefix + "norm_in.g": weights[0], prefix + "norm_out.g": weights[1]}
    names = ("0.norm.g", "0.fn.to_qkv.weight", "0.fn.to_out.0.weight", "0.fn.to_out.1.g",
             "1.norm.g", "1.fn.net.0.weight", "1.fn.net.2.g", "1.fn.net.4.weight")
    for L in range(depth):
        for i, nm in enumerate(names):
            p[f"{prefix}layers.{L}.{nm}"] = weights[2 + 8 * L + i]
    return p


def _ln(x, g, eps):
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) * torch.rsqrt(var + eps) * g


class _RotateNoInverse(torch.autograd.Function):
    """A rotation whose backward passes the gradient through unrotated (a defect to guard against)."""

    @staticmethod
    def forward(ctx, t, c, s):
        return _rotate(t, c, s)

    @staticmethod
    def backward(ctx, g):
        return g, None, None


def _rotate(t, c, s):
    a, b, rest = t[..., :16], t[..., 16:32], t[..., 32:]
    return torch.cat([a * c - b * s, b * c + a * s, rest], dim=-1)


def transformer_stack(x, weights, depth, heads, key_mask=None, causal=False, rot=None, eps=LN_EPS,
                      swap_value_gate=False, rotary_bwd_identity=False):
    """norm_in -> depth x (pre-norm attention + residual, pre-norm GEGLU feed-forward + residual)
    -> norm_out, as oracle.transformer_stack (x_clip.py:201-291) but with eps pinned, in the dtype of
    x.  rot = (cos, sin) [n, 16] tables.  The two flags build defective variants for the gate tests."""
    B, n, d = x.shape
    dt = x.dtype
    w = [t.to(dt) for t in weights]
    h = _ln(x, w[0], eps)
    for L in range(depth):
        g1, wqkv, wo, go, g2, w1, g4, w2 = w[2 + 8 * L: 10 + 8 * L]
        qkv = (_ln(h, g1, eps) @ wqkv.t()).view(B, n, 3, heads, 64).permute(2, 0, 3, 1, 4)
        q, k, v = qkv[0] * 64 ** -0.5, qkv[1], qkv[2]
        if rot is not None:
            c, s = (t.to(dt)[None, None] for t in rot)
            rf = _RotateNoInverse.apply if rotary_bwd_identity else _rotate
            q, k, v = rf(q, c, s), rf(k, c, s), rf(v, c, s)
        sc = q @ k.transpose(-1, -2)
        fill = -torch.finfo(dt).max
        if key_mask is not None:
            sc = sc.masked_fill(~key_mask[:, None, None, :], fill)
        if causal:
            sc = sc.masked_fill(torch.ones(n, n, dtype=torch.bool, device=x.device).triu(1), fill)
        o = (torch.softmax(sc, -1) @ v).permute(0, 2, 1, 3).reshape(B, n, heads * 64)
        h = _ln(o @ wo.t(), go, eps) + h
        uu = _ln(h, g2, eps) @ w1.t()
        val, gate = uu[..., :4 * d], uu[..., 4 * d:]
        if swap_value_gate:
            val, gate = gate, val
        hp = val * (0.5 * gate * (1.0 + torch.erf(gate / math.sqrt(2.0))))
        h = _ln(hp, g4, eps) @ w2.t() + h
    return _ln(h, w[1], eps)


BLOCK_CASES = {
    # name: (B, n, d, heads, masked, causal, rotary)
    "d512_mask": (6, 78, 512, 8, True, False, False),
    "d512_mask_causal": (6, 78, 512, 8, True, True, False),
    "d768_n197": (4, 197, 768, 12, False, False, False),
    "d256_rotary": (6, 33, 256, 4, True, False, True),
}
BLOCK_DEPTH = 2


def block_case(name: str, seed: int = 0, device="cpu"):
    """Inputs of one encoder case: bf16-rounded x and matmul weights, fp32 gains, key mask (every
    row keeps its first key), rotary tables, and a fixed bf16 cotangent of the output."""
    B, n, d, heads, masked, causal, rotary = BLOCK_CASES[name]
    gen = torch.Generator().manual_seed(seed)

    def r(*s):
        return torch.randn(*s, generator=gen)

    def lin(o, i):
        return ((torch.rand(o, i, generator=gen) * 2 - 1) / i ** 0.5).bfloat16().float()

    x = r(B, n, d).bfloat16()
    weights = [1 + 0.1 * r(d), 1 + 0.1 * r(d)]
    for _ in range(BLOCK_DEPTH):
        weights += [1 + 0.1 * r(d), lin(3 * heads * 64, d), lin(d, heads * 64), 1 + 0.1 * r(d),
                    1 + 0.1 * r(d), lin(8 * d, d), 1 + 0.1 * r(4 * d), lin(d, 4 * d)]
    mask = None
    if masked:
        mask = torch.rand(B, n, generator=gen) < 0.8
        mask[:, 0] = True
    dout = r(B, n, d).bfloat16()
    rot = rotary_tables(n) if rotary else None
    mv = (lambda t: None if t is None else t.to(device))
    return dict(x=x.to(device), weights=[w.to(device) for w in weights], mask=mv(mask), dout=dout.to(device),
                rot=None if rot is None else tuple(t.to(device) for t in rot), heads=heads, causal=causal)


def block_reference64(case, **defects):
    """fp64 forward and flat-weight gradients of the encoder for a block_case -> (out, [grads])."""
    ws = [w.double().requires_grad_(True) for w in case["weights"]]
    out = transformer_stack(case["x"].double(), ws, BLOCK_DEPTH, case["heads"], case["mask"], case["causal"],
                            case["rot"], **defects)
    out.backward(case["dout"].double())
    return out.detach(), [w.grad for w in ws]


def rel_fro(got, ref) -> float:
    return ((got.double() - ref.double()).norm() / ref.double().norm().clamp_min(1e-300)).item()


# Relative Frobenius gates of test_gpu_transformer_fp64.py, per output / flat-weight kind.  Largest
# error measured on an H100 80GB HBM3 (400 W power limit), over the four BLOCK_CASES and both layers:
# out 5.5e-3, dx 6.6e-3, gains and matmul weights 5.5e-3 .. 9.0e-3 (g2 of layer 1, d512_mask).
BLOCK_GATES = {"out": 1e-2, "dx": 1.5e-2, "g_in": 1.5e-2, "g_out": 1.5e-2, "g1": 1.5e-2, "wqkv": 1.5e-2,
               "wo": 1.5e-2, "go": 1.5e-2, "g2": 1.5e-2, "w1": 1.5e-2, "g4": 1.5e-2, "w2": 1.5e-2}
