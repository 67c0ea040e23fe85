"""Rotary embedding kernel (xclip_rotary_inplace, csrc/embed.cu) against fp64 oracle.rotate_features,
applied with the same fp32 cos / sin tables the kernel reads.

The kernel rotates features j and j + 16 (j < 16) of every 64-wide slice of a row by the angle of
position row % n, in place; inverse = 1 applies the transpose (the backward on dq | dk | dv).
Gates per element: 2^-8 |ref| (one bf16 rounding) + 2^-20 (|t_j c| + |t_j+16 s|) for the fp32
products.  Largest error measured on an H100 80GB HBM3 at a 400 W power limit, as a fraction of
its gate: forward 0.996, inverse 0.996 (the bf16 rounding bound is tight by construction), inverse
of the forward 0.984.
"""
import pytest
import torch

import block_oracle as BO

pytestmark = pytest.mark.gpu

# (B, n, heads, extra columns past the 3 * heads slices)
ROT_CASES = [(1, 1, 1, 0), (2, 33, 4, 0), (3, 77, 8, 0), (4, 50, 4, 64),
             (300, 78, 8, 0)]     # 23400 rows x 24 slices > 132 x 16 x 256 grid-stride items


def _gate(t, cos, sin, ref):
    """2^-8 |ref| + 2^-20 (|a c| + |b s|) on the rotated half; 0 on the untouched half."""
    rows, w = t.shape
    n = cos.shape[0]
    c = torch.cat([cos, cos], -1).double().abs()
    s = torch.cat([sin, sin], -1).double().abs()
    x = t.double().abs().view(rows // n, n, w // 64, 64)
    a = x[..., :32]
    b = torch.cat([x[..., 16:32], x[..., :16]], -1)
    term = a * c[None, :, None] + b * s[None, :, None]
    g = torch.zeros_like(x)
    g[..., :32] = term * 2.0 ** -20
    return BO.BF16_REL * ref.abs() + g.view(rows, w)


@pytest.mark.parametrize("B,n,heads,extra", ROT_CASES)
def test_rotary_fp64(cuda_device, B, n, heads, extra):
    from x_clip_b200 import kernels as K
    tag = f"{B}x{n}x{heads}+{extra}"
    ns = 3 * heads
    gen = torch.Generator().manual_seed(B * 1000 + n)
    buf = torch.randn(B * n, ns * 64 + extra, generator=gen).bfloat16().to(cuda_device)
    cos, sin = BO.rotary_tables(n, cuda_device)
    x = buf.clone()
    K.rotary_(x, n, ns, cos, sin)
    torch.cuda.synchronize()
    view = buf[:, :ns * 64]
    ref = BO.rotate64(view, cos, sin)
    BO.check(f"rot_fwd[{tag}]", x[:, :ns * 64], ref, _gate(view, cos, sin, ref))
    # features 32..63 of every slice and the columns past the slices are untouched, bit for bit
    keep = torch.ones_like(buf, dtype=torch.bool)
    keep[:, :ns * 64].view(B * n, ns, 64)[..., :32] = False
    assert torch.equal(x[keep], buf[keep])

    # inverse against the fp64 transpose
    y = buf.clone()
    K.rotary_(y, n, ns, cos, sin, inverse=True)
    torch.cuda.synchronize()
    ref_i = BO.rotate64(view, cos, sin, inverse=True)
    BO.check(f"rot_inv[{tag}]", y[:, :ns * 64], ref_i, _gate(view, cos, sin, ref_i))
    assert torch.equal(y[keep], buf[keep])

    # inverse(forward(x)) = x to within the two bf16 roundings
    z = x.clone()
    K.rotary_(z, n, ns, cos, sin, inverse=True)
    torch.cuda.synchronize()
    f = x[:, :ns * 64]
    # |R^T e1 + e2| <= 2^-8 (|c| |f_j| + |s| |f_pair|) + 2^-8 |x| (1 + 2^-7), f = bf16 forward output
    turned = _gate(f, cos, sin, torch.zeros_like(f, dtype=torch.float64)) * 2.0 ** 20
    g2 = 1.01 * BO.BF16_REL * (view.double().abs() + turned)
    BO.check(f"rot_roundtrip[{tag}]", z[:, :ns * 64], view, g2)
