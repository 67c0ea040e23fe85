"""Data path of the fused feed-forward epilogues (csrc/gemm.cuh, EPI_FF_UP / EPI_FF_BWD): u, hp and du
move between shared memory and HBM as TMA boxes of 128 rows x 64 columns.  The values themselves are
checked against fp64 in test_gpu_ff.py; this file checks what the box path can break:

- output buffers with padded leading dimensions, sentinel rows past M and sentinel columns past
  8d / 4d: the stores must be clipped at the tensor's edges and leave the sentinels untouched, and
  the padding of the u read by the backward must not leak into du;
- the results must equal those of compact buffers bit for bit, with and without u (need_u=False);
- two identical runs give identical bits.

Tile counts (128 x 128 tiles, 132 CTAs; up N = 8d, backward N = 4d).  A CTA's warpgroups take its
tiles in turn, so a warpgroup reuses its activation buffer (tiles / CTA) / 2 times:
- M <= 129, d = 256: up 16 / 32 tiles, backward 8 / 16: one tile per CTA, warpgroup 1 idles;
- (1413, 512): up 384 tiles (3 or 2 per CTA), backward 192 (2 or 1);
- (8577, 256): up 1088 tiles (9 or 8 per CTA), backward 544 (5 or 4): odd and even counts per
  warpgroup, many buffer reuses.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

CASES = [(1, 256), (127, 256), (129, 256), (1413, 512), (8577, 256)]
SENTINEL = -7.75          # exact in bf16
PAD_ROWS, PAD_COLS = 3, 24


def _inputs(M, d, dev):
    from x_clip_b200 import kernels as K
    g = torch.Generator().manual_seed(1009 * M + d)
    x = torch.randn(M, d, generator=g).bfloat16().to(dev)
    w1 = ((torch.rand(8 * d, d, generator=g) * 2 - 1) / d ** 0.5).to(dev)
    w2 = ((torch.rand(d, 4 * d, generator=g) * 2 - 1) / (4 * d) ** 0.5).to(dev)
    g4 = (1 + 0.1 * torch.randn(4 * d, generator=g)).to(dev)
    res = torch.randn(M, d, generator=g).bfloat16().to(dev)
    dx = torch.randn(M, d, generator=g).bfloat16().to(dev)
    w1p, w2g, colvec = K.ff_weights(w1, w2, g4)
    return x, w1p, w2g, colvec, res, dx


def _padded(M, n, dev):
    return torch.full((M + PAD_ROWS, n + PAD_COLS), SENTINEL, device=dev, dtype=torch.bfloat16)


def _untouched(buf, M, n):
    return bool((buf[M:] == SENTINEL).all()) and bool((buf[:, n:] == SENTINEL).all())


def _ff_up_into(x, w1p, u, hp, M, d):
    from x_clip_b200 import _lib
    rowsum = torch.empty((M, d // 16, 2), device=x.device, dtype=torch.float32)
    _lib.call("xclip_ff_up", x.data_ptr(), x.stride(0), w1p.data_ptr(), None if u is None else u.data_ptr(),
              0 if u is None else u.stride(0), hp.data_ptr(), hp.stride(0), rowsum.data_ptr(), M, d,
              torch.cuda.current_stream(x.device).cuda_stream)
    return rowsum


def _ff_bwd_into(dx, w2g, u, stats, ab, du, M, d):
    from x_clip_b200 import _lib
    _lib.call("xclip_ff_bwd", dx.data_ptr(), dx.stride(0), w2g.data_ptr(), u.data_ptr(), u.stride(0),
              stats.data_ptr(), ab.data_ptr(), du.data_ptr(), du.stride(0), M, d,
              torch.cuda.current_stream(dx.device).cuda_stream)


@pytest.mark.parametrize("M,d", CASES)
def test_ff_box_path_padded_buffers(cuda_device, M, d):
    from x_clip_b200 import kernels as K
    x, w1p, w2g, colvec, res, dx = _inputs(M, d, cuda_device)
    u0, hp0, rowsum0 = K.ff_up(x, w1p)
    _, acc, stats = K.ff_down(hp0, w2g, colvec, rowsum0, res, 1e-5)
    _, _, ab = K.ff_bwd_prep(dx, stats, acc, colvec)
    du0 = K.ff_bwd(dx, w2g, u0, stats, ab)

    u, hp = _padded(M, 8 * d, cuda_device), _padded(M, 4 * d, cuda_device)
    rowsum = _ff_up_into(x, w1p, u, hp, M, d)
    hp_only = _padded(M, 4 * d, cuda_device)
    rowsum_only = _ff_up_into(x, w1p, None, hp_only, M, d)
    du = _padded(M, 8 * d, cuda_device)
    _ff_bwd_into(dx, w2g, u, stats, ab, du, M, d)      # u's sentinel padding is in the rows it reads
    torch.cuda.synchronize()

    assert torch.equal(u[:M, :8 * d], u0), "u"
    assert torch.equal(hp[:M, :4 * d], hp0), "hp"
    assert torch.equal(rowsum, rowsum0), "rowsum"
    assert torch.equal(hp_only[:M, :4 * d], hp0), "hp (need_u=False)"
    assert torch.equal(rowsum_only, rowsum0), "rowsum (need_u=False)"
    assert torch.equal(du[:M, :8 * d], du0), "du"
    for name, buf, n in (("u", u, 8 * d), ("hp", hp, 4 * d), ("hp (need_u=False)", hp_only, 4 * d),
                         ("du", du, 8 * d)):
        assert _untouched(buf, M, n), f"{name}: a store reached past row M or column {n}"


@pytest.mark.parametrize("M,d", [(129, 256), (8577, 256)])
def test_ff_box_path_is_deterministic(cuda_device, M, d):
    from x_clip_b200 import kernels as K
    x, w1p, w2g, colvec, res, dx = _inputs(M, d, cuda_device)
    runs = []
    for _ in range(2):
        u, hp, rowsum = K.ff_up(x, w1p)
        _, acc, stats = K.ff_down(hp, w2g, colvec, rowsum, res, 1e-5)
        _, _, ab = K.ff_bwd_prep(dx, stats, acc, colvec)
        du = K.ff_bwd(dx, w2g, u, stats, ab)
        torch.cuda.synchronize()
        runs.append((u, hp, rowsum, du))
    for name, a, b in zip(("u", "hp", "rowsum", "du"), *runs):
        assert torch.equal(a, b), f"{name} differs between two identical runs"
