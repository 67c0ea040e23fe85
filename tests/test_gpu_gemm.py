"""wgmma GEMM vs a plain fp32 torch matmul of the same bf16-rounded operands."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(a, b, a_major, b_major):
    A = a.float() if a_major == 0 else a.float().t()
    B = b.float() if b_major == 0 else b.float().t()
    return A @ B.t()


def _mk(M, N, K, a_major, b_major, dev, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    a = torch.randn((M, K) if a_major == 0 else (K, M), generator=g).to(dev).bfloat16()
    b = torch.randn((N, K) if b_major == 0 else (K, N), generator=g).to(dev).bfloat16()
    return a, b


SHAPES = [(128, 128, 64), (256, 256, 128), (384, 512, 512), (200, 136, 72), (1000, 1536, 512),
          (4096, 4096, 2048)]


def _check_layout(dev, a_major, b_major, M, N, K):
    from x_clip_b200 import kernels
    a, b = _mk(M, N, K, a_major, b_major, dev)
    out = kernels.gemm(a, b, a_major=a_major, b_major=b_major, out_dtype=torch.float32)
    torch.cuda.synchronize()
    ref = _ref(a, b, a_major, b_major)
    err = (out - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert err <= 2e-3 * scale + 1e-3, f"max err {err} (scale {scale})"


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_gemm_kmajor_kmajor(cuda_device, M, N, K):      # forward: X @ W^T
    _check_layout(cuda_device, 0, 0, M, N, K)


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_gemm_kmajor_mnmajor(cuda_device, M, N, K):     # dgrad: dY @ W
    _check_layout(cuda_device, 0, 1, M, N, K)


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_gemm_mnmajor_kmajor(cuda_device, M, N, K):
    _check_layout(cuda_device, 1, 0, M, N, K)


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_gemm_mnmajor_mnmajor(cuda_device, M, N, K):    # wgrad: dY^T @ X
    _check_layout(cuda_device, 1, 1, M, N, K)


def test_gemm_bf16_out_bias_residual(cuda_device):
    from x_clip_b200 import kernels
    M, N, K = 640, 512, 768
    a, b = _mk(M, N, K, 0, 0, cuda_device, seed=1)
    bias = torch.randn(N, device=cuda_device)
    res = torch.randn(64, N, device=cuda_device).bfloat16()
    out = kernels.gemm(a, b, alpha=0.5, bias=bias, residual=res, res_row_mod=64)
    torch.cuda.synchronize()
    ref = 0.5 * _ref(a, b, 0, 0) + bias + res.float().repeat(M // 64, 1)
    assert out.dtype == torch.bfloat16
    err = (out.float() - ref).abs().max().item()
    assert err <= 1e-2 * ref.abs().max().item()


def test_gemm_strided_output_and_operand(cuda_device):
    from x_clip_b200 import kernels
    M, N, K = 256, 128, 64
    big = torch.randn(M, 3 * K, device=cuda_device).bfloat16()
    a = big[:, K:2 * K]           # lda = 3K, offset K
    _, b = _mk(M, N, K, 0, 0, cuda_device, seed=2)
    outbig = torch.zeros(M, 2 * N, device=cuda_device, dtype=torch.bfloat16)
    kernels.gemm(a, b, out=outbig[:, N:])
    torch.cuda.synchronize()
    ref = a.float() @ b.float().t()
    assert (outbig[:, :N] == 0).all()
    assert (outbig[:, N:].float() - ref).abs().max().item() <= 1e-2 * ref.abs().max().item()


@pytest.mark.parametrize("M,N,K", [(512, 512, 33792), (1536, 512, 8192), (136, 264, 1000)])
def test_gemm_wgrad_splitk_accumulate(cuda_device, M, N, K):
    """dW[N_out, d] += dY^T X : both operands MN-major, fp32 atomic accumulate, split-K."""
    from x_clip_b200 import kernels
    a, b = _mk(M, N, K, 1, 1, cuda_device, seed=3)
    out = torch.ones(M, N, device=cuda_device)
    kernels.gemm(a, b, a_major=1, b_major=1, out=out, accumulate=True)
    torch.cuda.synchronize()
    ref = _ref(a, b, 1, 1) + 1.0
    err = (out - ref).abs().max().item()
    assert err <= 2e-3 * ref.abs().max().item() + 1e-2


def test_gemm_rejects_bad_args(cuda_device):
    from x_clip_b200 import kernels, _lib
    a = torch.randn(128, 64, device=cuda_device).bfloat16()
    b = torch.randn(100, 64, device=cuda_device).bfloat16()   # N % 8 != 0
    with pytest.raises(_lib.XClipB200Error):
        kernels.gemm(a, b)
    with pytest.raises(_lib.XClipB200Error):
        kernels.gemm(a.float(), b)
