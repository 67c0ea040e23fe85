"""The ping-pong schedule of the wgmma GEMM (128-wide tiles, one tile per consumer warpgroup) vs fp32
torch, at tile counts that leave warpgroup 1 idle, give a CTA an odd number of tiles or leave a
partial last wave, and bit-reproducibility of the fused epilogues that run on it."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _mk(M, N, K, a_major, b_major, dev, seed=0):
    g = torch.Generator(device="cpu").manual_seed(seed)
    a = torch.randn((M, K) if a_major == 0 else (K, M), generator=g).to(dev).bfloat16()
    b = torch.randn((N, K) if b_major == 0 else (K, N), generator=g).to(dev).bfloat16()
    return a, b


def _ref(a, b, a_major, b_major):
    A = a.float() if a_major == 0 else a.float().t()
    B = b.float() if b_major == 0 else b.float().t()
    return A @ B.t()


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# N = 128 and 384 are not multiples of 256 and stay below 1024: the 128-wide (ping-pong) tiles
@pytest.mark.parametrize("tiles", [1, 2, "sms-1", "sms", "sms+1", "2sms-1", "2sms", "2sms+1"])
@pytest.mark.parametrize("N", [128, 384])
def test_pingpong_tile_counts(cuda_device, tiles, N):
    from x_clip_b200 import kernels
    s = _sms()
    t = {"sms-1": s - 1, "sms": s, "sms+1": s + 1, "2sms-1": 2 * s - 1, "2sms": 2 * s,
         "2sms+1": 2 * s + 1}.get(tiles, tiles)
    M = -(-t // (N // 128)) * 128 - 40            # ragged last row block
    a, b = _mk(M, N, 200, 0, 0, cuda_device)
    out = kernels.gemm(a, b, out_dtype=torch.float32)
    torch.cuda.synchronize()
    ref = _ref(a, b, 0, 0)
    assert (out - ref).abs().max().item() <= 2e-3 * ref.abs().max().item() + 1e-3


@pytest.mark.parametrize("K", [64, 72, 192, 200])
@pytest.mark.parametrize("a_major,b_major", [(0, 0), (0, 1), (1, 0), (1, 1)])
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16])
def test_pingpong_k_majors_dtypes(cuda_device, K, a_major, b_major, out_dtype):
    from x_clip_b200 import kernels
    M, N = 3 * _sms() * 128 // 2 + 72, 128       # 1.5 tiles per CTA, ragged M
    a, b = _mk(M, N, K, a_major, b_major, cuda_device, seed=K)
    out = kernels.gemm(a, b, a_major=a_major, b_major=b_major, out_dtype=out_dtype)
    torch.cuda.synchronize()
    ref = _ref(a, b, a_major, b_major)
    tol = (2e-3 if out_dtype == torch.float32 else 1e-2) * ref.abs().max().item() + 1e-3
    assert (out.float() - ref).abs().max().item() <= tol


@pytest.mark.parametrize("mode", ["mod", "idx"])
def test_pingpong_bias_residual(cuda_device, mode):
    from x_clip_b200 import kernels
    M, N, K = 133 * 128 - 5, 384, 256
    a, b = _mk(M, N, K, 0, 0, cuda_device, seed=7)
    bias = torch.randn(N, device=cuda_device)
    res = torch.randn(97, N, device=cuda_device).bfloat16()
    if mode == "mod":
        out = kernels.gemm(a, b, alpha=0.5, bias=bias, residual=res, res_row_mod=97)
        rows = torch.arange(M, device=cuda_device) % 97
    else:
        rows = torch.randint(0, 97, (M,), device=cuda_device, dtype=torch.int32)
        out = kernels.gemm(a, b, alpha=0.5, bias=bias, residual=res, res_row_idx=rows)
    torch.cuda.synchronize()
    ref = 0.5 * _ref(a, b, 0, 0) + bias + res.float()[rows.long()]
    assert (out.float() - ref).abs().max().item() <= 1e-2 * ref.abs().max().item()


@pytest.mark.parametrize("M,N,K", [(136, 264, 1000), (384, 384, 20000)])
def test_pingpong_splitk_accumulate(cuda_device, M, N, K):
    from x_clip_b200 import kernels
    a, b = _mk(M, N, K, 1, 1, cuda_device, seed=3)
    out = torch.ones(M, N, device=cuda_device)
    kernels.gemm(a, b, a_major=1, b_major=1, out=out, accumulate=True)
    torch.cuda.synchronize()
    ref = _ref(a, b, 1, 1) + 1.0
    assert (out - ref).abs().max().item() <= 2e-3 * ref.abs().max().item() + 1e-2


def test_pingpong_ff_epilogues_reproducible(cuda_device):
    """FF up / down / bwd twice on the same inputs, with an odd number of tiles per CTA."""
    from x_clip_b200 import kernels as K
    d = 256
    M = (3 * _sms() * 128) // (8 * d // 128) + 40     # up-projection: ~3 tiles per CTA
    g = torch.Generator().manual_seed(5)
    x = torch.randn(M, d, generator=g).to(cuda_device).bfloat16()
    w1 = ((torch.rand(8 * d, d, generator=g) * 2 - 1) / d ** 0.5).to(cuda_device)
    w2 = ((torch.rand(d, 4 * d, generator=g) * 2 - 1) / (4 * d) ** 0.5).to(cuda_device)
    g4 = torch.rand(4 * d, generator=g).to(cuda_device) + 0.5
    res = torch.randn(M, d, generator=g).to(cuda_device).bfloat16()
    dx = torch.randn(M, d, generator=g).to(cuda_device).bfloat16()
    w1p, w2g, colvec = K.ff_weights(w1, w2, g4)

    def run():
        u, hp, rowsum = K.ff_up(x, w1p)
        x2, acc, stats = K.ff_down(hp, w2g, colvec, rowsum, res, 1e-5)
        _, _, ab = K.ff_bwd_prep(dx, stats, acc, colvec)
        du = K.ff_bwd(dx, w2g, u, stats, ab)
        torch.cuda.synchronize()
        return [t.clone() for t in (u, hp, rowsum, x2, acc, stats, du)]

    first, second = run(), run()
    for p, q in zip(first, second):
        assert torch.equal(p, q)
    assert all(torch.isfinite(t.float()).all() for t in first)


@pytest.mark.parametrize("C", [72, 136, 200])
def test_pingpong_nce_simreg_reproducible_and_correct(cuda_device, C):
    """C < 256 runs the NCE / SIMREG epilogues on 128-wide tiles; with diag_offset 8 the positive of
    row 120 is the first column of the second column block."""
    from x_clip_b200 import kernels as K
    diag, D = 8, 64
    R = C - diag
    g = torch.Generator().manual_seed(C)
    a = (torch.randn(R, D, generator=g) * 0.3).to(cuda_device).bfloat16()
    b = (torch.randn(C, D, generator=g) * 0.3).to(cuda_device).bfloat16()
    temp = torch.tensor([3.0], device=cuda_device)

    def run():
        lse, pos = K.nce_fwd(a, b, temp, diag, 0)
        lse_col = torch.randn(C, generator=torch.Generator().manual_seed(1)).to(cuda_device)
        gq = K.nce_bwd(a, b, temp, diag, 0, lse, lse_col, 0.5, 0.5, 1.0,
                       torch.tensor([1.0], device=cuda_device))
        e2 = K.simreg_fwd(a, b, diag)
        ge = K.simreg_bwd(a, b, diag, torch.tensor([1.0], device=cuda_device))
        torch.cuda.synchronize()
        return [t.clone() for t in (lse, pos, gq, e2, ge)]

    first, second = run(), run()
    for p, q in zip(first, second):
        assert torch.equal(p, q)
    lse, pos = first[0], first[1]
    s = 3.0 * (a.double() @ b.double().t())
    ref_lse = torch.logsumexp(s, dim=1)
    ref_pos = s[torch.arange(R), torch.arange(R) + diag]
    assert (lse.double() - ref_lse).abs().max().item() <= 2e-3 * ref_lse.abs().max().item() + 1e-3
    assert (pos.double() - ref_pos).abs().max().item() <= 1e-3 * ref_pos.abs().max().item() + 1e-3
    E = a.double() @ b.double().t()
    E[torch.arange(R), torch.arange(R) + diag] = 0
    ref_e2 = (E ** 2).sum(1)
    assert (first[3].double() - ref_e2).abs().max().item() <= 1e-3 * ref_e2.abs().max().item() + 1e-3
