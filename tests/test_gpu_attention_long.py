"""Attention beyond 320 tokens (the streaming kernels) against the fp64 reference of attn_oracle.py, and
bit-identity of the streaming and resident kernels where both run (n <= 320)."""
import pytest
import torch

import attn_oracle as AO
from test_gpu_attention import ATTN_STREAM, _mk, check_attn, fwd_bwd

pytestmark = pytest.mark.gpu

LONG_CASES = [(2, 321, 4, True), (2, 401, 8, True), (3, 576, 12, False), (2, 625, 4, True),
              (1, 1025, 4, True), (1, 2048, 2, False),
              (24, 577, 12, True)]      # many CTAs per SM; a last 64-row block with one row
LONG_CAUSAL_CASES = [(2, 385, 4, True), (1, 640, 2, False)]


@pytest.mark.parametrize("B,n,H,masked", LONG_CASES)
def test_attn_fwd_long(cuda_device, B, n, H, masked):
    case = AO.attn_case("peaked", B, n, H, masked=masked, device=cuda_device)
    o, lse, _ = fwd_bwd(case, B, n, H, bwd=False)
    check_attn(f"peaked B{B} n{n} H{H}", case, B, n, H, o, lse)


@pytest.mark.parametrize("B,n,H,masked", LONG_CASES)
def test_attn_bwd_long(cuda_device, B, n, H, masked):
    case = AO.attn_case("flat", B, n, H, masked=masked, seed=1, device=cuda_device)
    check_attn(f"flat B{B} n{n} H{H}", case, B, n, H, *fwd_bwd(case, B, n, H))


@pytest.mark.parametrize("B,n,H,masked", LONG_CAUSAL_CASES)
def test_attn_causal_long(cuda_device, B, n, H, masked):
    """The causal mask at kernel level (the text tower itself keeps causal sequences <= 128 tokens)."""
    case = AO.attn_case("flat", B, n, H, causal=True, masked=masked, seed=2, device=cuda_device)
    check_attn(f"causal B{B} n{n} H{H}", case, B, n, H, *fwd_bwd(case, B, n, H, causal=True), causal=True)


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


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("n", [1, 5, 17, 64, 129, 257, 320])
def test_streaming_equals_resident_bitwise_no_visible_key(cuda_device, n, causal):
    """The same on the no_visible recipe: rows with no visible key, and items whose mask is all False."""
    from x_clip_b200 import _lib
    B, H = 3, 4
    case = AO.attn_case("no_visible", B, n, H, causal=causal, seed=8, device=cuda_device)
    lib = _lib.load()
    resident = _fwd_bwd(case["qkv"], case["mask"], case["d_o"], B, n, H, causal)
    prev = lib.xclip_tune_set(ATTN_STREAM, 1)
    assert prev == 0
    try:
        streaming = _fwd_bwd(case["qkv"], case["mask"], case["d_o"], B, n, H, causal)
    finally:
        lib.xclip_tune_set(ATTN_STREAM, prev)
    for name, a, b in zip(("o", "lse", "dqkv"), resident, streaming):
        assert torch.equal(a, b), name
