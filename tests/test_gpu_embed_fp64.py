"""The embedding kernels against exact or fp64 references (csrc/embed.cu).  Worst gate ratios on an H100
80GB HBM3 (700 W power limit): reduction gates (dtok, dpos, dcls, d bias, d pos, scatter / colsum)
at most 0.008, patch dW 0.08, the bf16 patch-embedding output 0.995 (the bf16 rounding bound); the
file runs in about 14 s there.

- text embedding forward: out = bf16(fp32 tok[id] + fp32 pos) bit for bit, cls rows bf16(cls);
- text embedding backward: dtok with a vocabulary of 3 (every row hit hundreds of times) and a large one
  (most rows never hit, and those stay exactly 0), dpos / dcls with the column sums split over 1, some
  and all samples (bsplit), and the position rows past n exactly 0;
- the patch embedding (PatchEmbedFn) forward and backward, with dW under the GEMM gate and d bias /
  d pos per element under reduction gates, at rows <= 256 and > 256 and widths that use part of a
  512-column chunk; scatter_add_rows_ / colsum_rows_ on strided sources;
- patchify_gather exactly, and its refusal of patch * patch * channels % 8 != 0 before any launch.
Indices are always in range: an out-of-range index traps by design.
"""
import pytest
import torch

import block_oracle as BO
import gemm_oracle as GO

pytestmark = pytest.mark.gpu


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("d", [128, 384, 512, 640, 896, 1024])
def test_text_embed_forward_exact(cuda_device, d):
    from x_clip_b200 import kernels as K
    for n in (1, 16, 77, 255):
        B, vocab = 3, 1000
        ids, _ = GO.text_embed_case(B, n, d, vocab)
        g = torch.Generator().manual_seed(d + n)
        tok = torch.randn(vocab, d, generator=g)
        pos = torch.randn(n + 3, d, generator=g)
        cls = torch.randn(d, generator=g)
        out = K.text_embed_fwd(ids.to(cuda_device), tok.to(cuda_device), pos.to(cuda_device), cls.to(cuda_device))
        torch.cuda.synchronize()
        ref = torch.cat([cls.expand(B, 1, d), tok[ids] + pos[:n]], dim=1).bfloat16()
        assert torch.equal(out.cpu(), ref), (d, n)


def _text_bwd(dev, B, n, d, vocab, pos_extra=5):
    from x_clip_b200 import kernels as K
    ids, dx = GO.text_embed_case(B, n, d, vocab)
    dtok, dpos, dcls = K.text_embed_bwd(ids.to(dev), dx.to(dev), vocab, n + pos_extra)
    torch.cuda.synchronize()
    ref = GO.text_embed_bwd64(ids.to(dev), dx.to(dev), vocab, n + pos_extra)
    return ids, (dtok, dpos, dcls), ref


@pytest.mark.parametrize("vocab", [3, 49408])
@pytest.mark.parametrize("d", [128, 512, 896])
def test_text_embed_dtok(cuda_device, vocab, d):
    """Vocabulary 3: hundreds of red.add per table row; 49408: most rows never hit and exactly 0."""
    B, n = 16, 77
    ids, (dtok, _, _), ((ref, ab), _, _) = _text_bwd(cuda_device, B, n, d, vocab)
    BO.check(f"text_dtok_v{vocab}_d{d}", dtok, ref, GO.red_gate(ab))
    hit = torch.zeros(vocab, dtype=torch.bool)
    hit[ids.reshape(-1)] = True
    if vocab == 3:
        assert hit.all() and torch.bincount(ids.reshape(-1)).min() >= 300
    else:
        assert (~hit).sum() > vocab // 2
        assert torch.equal(dtok[~hit.to(cuda_device)], torch.zeros_like(dtok[~hit.to(cuda_device)]))


# (B, n, d) whose bsplit is 1, strictly between 1 and B, and B on an H100 SXM (132 SMs)
BSPLIT_CASES = {"one": (6, 255, 1024), "some": (64, 16, 512), "all": (8, 16, 512),
                "some_d640": (48, 33, 640), "all_d128": (5, 77, 128), "some_d384": (80, 9, 384)}


@pytest.mark.parametrize("name", list(BSPLIT_CASES))
def test_text_embed_dpos_dcls(cuda_device, name):
    B, n, d = BSPLIT_CASES[name]
    bs = GO.text_embed_bsplit(B, n, d, _sms())
    want = name.split("_")[0]
    assert {"one": bs == 1, "some": 1 < bs < B, "all": bs == B}[want], (name, bs)
    _, (_, dpos, dcls), (_, (rpos, apos), (rcls, acls)) = _text_bwd(cuda_device, B, n, d, vocab=100)
    BO.check(f"text_dpos_{name}", dpos[:n], rpos[:n], GO.red_gate(apos[:n]))
    BO.check(f"text_dcls_{name}", dcls, rcls, GO.red_gate(acls))
    assert torch.equal(dpos[n:], torch.zeros_like(dpos[n:]))


# (B, image size, patch, channels, keep per sample, d): rows = B * keep
PATCH_CASES = [(3, 64, 16, 3, 9, 384), (5, 224, 16, 3, 98, 768), (4, 240, 16, 3, 225, 896),
               (2, 256, 32, 3, 40, 1024), (6, 64, 8, 1, 30, 384)]


@pytest.mark.parametrize("B,S,p,C,k,d", PATCH_CASES)
def test_patch_embed_fp64(cuda_device, B, S, p, C, k, d):
    """PatchEmbedFn: y = patches W^T + bias + bf16(pos)[index] (bf16), dW = dy^T patches (split-K wgrad),
    d bias = column sums of dy, d pos = rows of dy scatter-added by index (repeated across samples)."""
    from x_clip_b200 import engine as E
    dev = cuda_device
    n = (S // p) ** 2
    t = GO.patch_embed_case(B, n, k, p * p * C, d)
    t = {key: v.to(dev) for key, v in t.items()}
    index = t["keep"].reshape(-1).to(torch.int32)
    assert torch.bincount(index.long()).max() > 1                   # some patch kept by several samples
    w = t["w"].clone().requires_grad_(True)
    bias = t["bias"].clone().requires_grad_(True)
    table = t["table"].clone().requires_grad_(True)
    y = E.PatchEmbedFn.apply(t["patches"], index, w, bias, table)
    y.backward(t["dy"])
    torch.cuda.synchronize()
    tb = t["table"].bfloat16()
    rows = index.long()
    ref = GO.gemm64(t["patches"], t["w"].bfloat16(), bias=t["bias"], residual=tb, res_rows=rows)
    gate = GO.gemm_gate(t["patches"], t["w"].bfloat16(), bias=t["bias"], residual=tb, res_rows=rows,
                        bf16_out=True, ref=ref)
    BO.check(f"patch_y_{S}_{p}_{d}", y, ref, gate)
    M = B * k
    plan = GO.split_plan(d, p * p * C, M, True, _sms())
    rdw = GO.gemm64(t["dy"], t["patches"], 1, 1)
    BO.check(f"patch_dW_{S}_{p}_{d}", w.grad, rdw,
             GO.gemm_gate(t["dy"], t["patches"], 1, 1, splits=plan["splits"]))
    dy = t["dy"].double()
    BO.check(f"patch_dbias_{S}_{p}_{d}_rows{M}", bias.grad, dy.sum(0), GO.red_gate(dy.abs().sum(0)))
    rpos = torch.zeros(n, d, dtype=torch.float64, device=dev).index_add_(0, rows, dy)
    apos = torch.zeros(n, d, dtype=torch.float64, device=dev).index_add_(0, rows, dy.abs())
    BO.check(f"patch_dpos_{S}_{p}_{d}", table.grad, rpos, GO.red_gate(apos))
    untouched = torch.ones(n, dtype=torch.bool, device=dev)
    untouched[rows] = False
    assert torch.equal(table.grad[untouched], torch.zeros_like(table.grad[untouched]))


@pytest.mark.parametrize("rows,d", [(1, 384), (200, 768), (257, 896), (3001, 1024)])
def test_scatter_colsum_strided(cuda_device, rows, d):
    """scatter_add_rows_ and colsum_rows_ into non-zero destinations from a source with lds = d + 24."""
    from x_clip_b200 import kernels as K
    dev = cuda_device
    g = torch.Generator().manual_seed(rows + d)
    big = (torch.randn(rows, d + 24, generator=g) * GO._scales(rows, g)).bfloat16().to(dev)
    src = big[:, :d]
    V = 37
    idx = torch.randint(0, V, (rows,), generator=g).to(dev, torch.int32)
    dst0 = torch.randn(V, d, generator=g).to(dev)
    col0 = torch.randn(d, generator=g).to(dev)
    dst = K.scatter_add_rows_(dst0.clone(), src, idx=idx)
    col = K.colsum_rows_(col0.clone(), src)
    torch.cuda.synchronize()
    s = src.double()
    rs = dst0.double().index_add(0, idx.long(), s)
    ra = dst0.double().abs().index_add(0, idx.long(), s.abs())
    BO.check(f"scatter_rows{rows}_d{d}", dst, rs, GO.red_gate(ra))
    BO.check(f"colsum_rows{rows}_d{d}", col, col0.double() + s.sum(0), GO.red_gate(col0.double().abs() + s.abs().sum(0)))


@pytest.mark.parametrize("B,C,S,p", [(2, 1, 64, 8), (3, 1, 48, 16), (2, 3, 64, 8), (2, 3, 224, 16)])
def test_patchify_gather_exact(cuda_device, B, C, S, p):
    from x_clip_b200 import kernels as K
    g = torch.Generator().manual_seed(B * S + C + p)
    img = torch.randn(B, C, S, S, generator=g)
    n = (S // p) ** 2
    ref = GO.patchify64(img, p)
    out = K.patchify_gather(img.to(cuda_device), p)
    keep = torch.stack([torch.randperm(n, generator=g)[: max(1, n // 2)] for _ in range(B)])
    outk = K.patchify_gather(img.to(cuda_device), p, keep.to(cuda_device))
    torch.cuda.synchronize()
    assert torch.equal(out.cpu(), ref.reshape(B * n, -1).bfloat16())
    refk = torch.stack([ref[b, keep[b]] for b in range(B)]).reshape(B * keep.shape[1], -1)
    assert torch.equal(outk.cpu(), refk.bfloat16())


def test_patchify_refuses_unaligned_patch_rows(cuda_device):
    """p = 14, C = 3: 588 values per patch, not a multiple of 8; refused before any launch."""
    from x_clip_b200 import _lib, kernels as K
    lib = _lib.load()
    img = torch.randn(2, 3, 56, 56, device=cuda_device)
    torch.cuda.synchronize()
    n0 = lib.xclip_launch_count()
    with pytest.raises(_lib.XClipB200Error):
        K.patchify_gather(img, 14)
    assert lib.xclip_launch_count() == n0
