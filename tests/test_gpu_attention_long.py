"""Attention beyond 320 tokens (the streaming kernels) against the fp32 torch restatement of the
reference core, and bit-identity of the streaming and resident kernels where both run (n <= 320)."""
import pytest
import torch

from test_gpu_attention import _mk, _ref_attention

pytestmark = pytest.mark.gpu

ATTN_STREAM = 5     # XCLIP_TUNE_ATTN_STREAM (include/xclip_b200.h)

LONG_CASES = [(2, 321, 4, True), (2, 401, 8, True), (3, 576, 12, False), (2, 625, 4, True),
              (1, 1025, 4, True), (1, 2048, 2, False),
              (24, 577, 12, True)]      # many CTAs per SM; a last 64-row block with one row
LONG_CAUSAL_CASES = [(2, 385, 4, True), (1, 640, 2, False)]


def _check_fwd(o, lse, ref, s):
    err = (o.float() - ref).abs().max().item()
    assert err <= 2e-2 * ref.abs().max().item(), f"o err {err}"
    ref_lse = torch.logsumexp(s, dim=-1) / 0.6931471805599453
    assert torch.allclose(lse, ref_lse, atol=2e-2, rtol=1e-3)


@pytest.mark.parametrize("B,n,H,masked", LONG_CASES)
def test_attn_fwd_long(cuda_device, B, n, H, masked):
    from x_clip_b200 import kernels as K
    qkv, mask = _mk(B, n, H, masked, cuda_device)
    scale = 64 ** -0.5
    o, lse = K.attn_fwd(qkv, mask, B, n, H, scale)
    torch.cuda.synchronize()
    ref, s = _ref_attention(qkv, mask, B, n, H, scale)
    _check_fwd(o, lse, ref, s)


@pytest.mark.parametrize("B,n,H,masked", LONG_CASES)
def test_attn_bwd_long(cuda_device, B, n, H, masked):
    from x_clip_b200 import kernels as K
    qkv, mask = _mk(B, n, H, masked, cuda_device, seed=1)
    scale = 64 ** -0.5
    o, lse = K.attn_fwd(qkv, mask, B, n, H, scale)
    d_o = torch.randn(B * n, H * 64, device=cuda_device).bfloat16()
    dqkv = K.attn_bwd(qkv, mask, o, d_o, lse, B, n, H, scale)
    torch.cuda.synchronize()
    qf = qkv.float().requires_grad_(True)
    ref, _ = _ref_attention(qf, mask, B, n, H, scale)
    ref.backward(d_o.float())
    g = qf.grad
    inner = H * 64
    for name, sl in (("dq", slice(0, inner)), ("dk", slice(inner, 2 * inner)), ("dv", slice(2 * inner, 3 * inner))):
        err = (dqkv[:, sl].float() - g[:, sl]).abs().max().item()
        sc = g[:, sl].abs().max().item()
        assert err <= 3e-2 * sc + 1e-5, f"{name}: err {err} vs scale {sc}"
        rel = (dqkv[:, sl].float() - g[:, sl]).norm().item() / (g[:, sl].norm().item() + 1e-3)
        assert rel < 1e-2, f"{name}: rel fro err {rel}"


@pytest.mark.parametrize("B,n,H,masked", LONG_CAUSAL_CASES)
def test_attn_causal_long(cuda_device, B, n, H, masked):
    """The causal mask at kernel level (the text tower itself keeps causal sequences <= 128 tokens)."""
    from x_clip_b200 import kernels as K
    qkv, mask = _mk(B, n, H, masked, cuda_device, seed=2)
    scale = 64 ** -0.5
    o, lse = K.attn_fwd(qkv, mask, B, n, H, scale, causal=True)
    d_o = torch.randn(B * n, H * 64, device=cuda_device).bfloat16()
    dqkv = K.attn_bwd(qkv, mask, o, d_o, lse, B, n, H, scale, causal=True)
    torch.cuda.synchronize()
    qf = qkv.float().requires_grad_(True)
    ref, s = _ref_attention(qf, mask, B, n, H, scale, causal=True)
    _check_fwd(o, lse, ref.detach(), s.detach())
    ref.backward(d_o.float())
    rel = (dqkv.float() - qf.grad).norm().item() / qf.grad.norm().item()
    assert rel < 1e-2, f"rel fro err {rel}"


def _fwd_bwd(qkv, mask, d_o, B, n, H, causal):
    from x_clip_b200 import kernels as K
    o, lse = K.attn_fwd(qkv, mask, B, n, H, 0.125, causal=causal)
    dqkv = K.attn_bwd(qkv, mask, o, d_o, lse, B, n, H, 0.125, causal=causal)
    torch.cuda.synchronize()
    return o, lse, dqkv


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("n", [1, 16, 17, 64, 78, 98, 129, 197, 257, 320])
def test_streaming_equals_resident_bitwise(cuda_device, n, masked, causal):
    """Both schedules run the same per-block arithmetic in the same block order: o, lse and dqkv agree
    bit for bit."""
    from x_clip_b200 import _lib
    B, H = 3, 4
    qkv, mask = _mk(B, n, H, masked, cuda_device, seed=3)
    d_o = torch.randn(B * n, H * 64, generator=torch.Generator().manual_seed(4)).to(cuda_device).bfloat16()
    lib = _lib.load()
    resident = _fwd_bwd(qkv, mask, d_o, B, n, H, causal)
    prev = lib.xclip_tune_set(ATTN_STREAM, 1)
    assert prev == 0
    try:
        streaming = _fwd_bwd(qkv, mask, d_o, B, n, H, causal)
    finally:
        lib.xclip_tune_set(ATTN_STREAM, prev)
    for name, a, b in zip(("o", "lse", "dqkv"), resident, streaming):
        assert torch.equal(a, b), name
