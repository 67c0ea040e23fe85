"""The per-call fp64 checks of bench_call_oracle that the training-configuration workloads use, exercised
without a GPU:

- the torch restatement of the attention-dropout Philox mask equals dropout_oracle's numpy one bit for
  bit (seeds with the high word set, several layers, p of exactly 0 and exactly 1);
- augment_oracle.augment64, called with the arguments SimCLRAugmentation._apply_kernels passes to
  kernels.augment, equals the module's own reference SimCLRAugmentation.apply_torchvision in float64;
- the view-block column map of the multiview FILIP check equals filip.positive_column and is a
  permutation, rank-major and view-major;
- unpatchify64 inverts gemm_oracle.patchify64;
- accept / reject pairs: each check, fed the fp64 reference rounded to the kernel's output dtype, stays
  within its gates, and fed one plausible wrong output, exceeds them.
"""
import inspect

import numpy as np
import pytest
import torch

import augment_oracle as AU
import bench_call_oracle as BC
import dropout_oracle as DO
import gemm_oracle as GO

BF16, F32 = torch.bfloat16, torch.float32


def _args(name, *args, **kw):
    """The bound arguments (defaults applied) a spy on kernels.<name> would hand its check."""
    from x_clip_b200 import kernels as K
    ba = inspect.signature(getattr(K, name)).bind(*args, **kw)
    ba.apply_defaults()
    return dict(ba.arguments)


def _worst(ratios):
    return max(ratios.values())


# --------------------------------------------------------------------------- attention-dropout mask

@pytest.mark.parametrize("seed", [0, 1, 12345, -6917529027641081857, -1, (1 << 63) - 1])
def test_torch_philox_equals_numpy(seed):
    for p in (0.0, 0.1, 0.5, 0.9, 1.0):
        for layer in (0, 1, 11):
            want = DO.attn_keep(seed, 3, 2, 13, layer, p)
            got = DO.attn_keep_torch(seed, 0, 3, 2, 13, layer, p)
            assert np.array_equal(got.numpy(), want), (seed, p, layer)
    # a slice of batch items draws the counters of those items
    want = DO.attn_keep(seed, 5, 3, 6, 2, 0.3)[2:5]
    assert np.array_equal(DO.attn_keep_torch(seed, 2, 5, 3, 6, 2, 0.3).numpy(), want)
    raw = DO.philox4x32_10(np.array([[7, 8, 9, 10]], dtype=np.uint32), DO.seed_key(seed))
    c = [torch.tensor([v], dtype=torch.int64) for v in (7, 8, 9, 10)]
    assert [int(w) for w in DO.philox4x32_10_torch(*c, DO.seed_key(seed))] == [int(v) for v in raw[0]]


def test_torch_philox_extremes():
    """p = 0 keeps everything, p = 1 nothing; the multipliers match attn_drop_mul."""
    seed = -6917529027641081857
    assert bool(DO.attn_keep_torch(seed, 0, 2, 2, 9, 0, 0.0).all())
    assert not bool(DO.attn_keep_torch(seed, 0, 2, 2, 9, 0, 1.0).any())
    for p in (0.0, 0.1, 1.0):
        assert torch.equal(DO.attn_drop_mul_torch(seed, 0, 2, 2, 9, 4, p), DO.attn_drop_mul(seed, 2, 2, 9, 4, p))


# --------------------------------------------------------------------------- augmentation

def _kernel_args(monkeypatch, aug, x, params):
    """The keyword arguments SimCLRAugmentation._apply_kernels passes to kernels.augment."""
    from x_clip_b200 import kernels as K
    seen = []

    def capture(img, **kw):
        seen.append(kw)
        return AU.augment64(img, **kw)
    monkeypatch.setattr(K, "augment", capture)
    out = aug._apply_kernels(x, params)
    assert len(seen) == 1
    return seen[0], out


def test_augment64_equals_apply_torchvision(monkeypatch):
    """Over drawn parameters (every jitter op, grayscale, flip, blur, crops off the borders): the
    restatement from kernels.augment's arguments equals the module's torchvision reference in float64,
    up to the fp32 blur weights and Normalize constants the kernel is given."""
    from x_clip_b200.aux import SimCLRAugmentation
    aug = SimCLRAugmentation(40, 3)
    x = torch.rand(3, 3, 45, 38, generator=torch.Generator().manual_seed(0))
    seen = dict(jitter=0, gray=0, flip=0, blur=0, inner_crop=0)
    worst = 0.0
    for s in range(60):
        torch.manual_seed(s)
        p = aug.draw(x.shape)
        kw, got = _kernel_args(monkeypatch, aug, x, p)
        ref = aug.apply_torchvision(x.double(), p)
        err = ((got - ref).abs().max() / ref.abs().max().clamp(min=1.0)).item()
        worst = max(worst, err)
        assert err <= 1e-6, (s, p, err)
        seen["jitter"] += bool(kw["ops"])
        seen["gray"] += bool(kw["grayscale"])
        seen["flip"] += bool(kw["flip"])
        seen["blur"] += kw["blur_kernel"] is not None
        t, l, h, w = p.crop
        seen["inner_crop"] += t > 0 and l > 0 and t + h < 45 and l + w < 38
    print(f"augment64 vs apply_torchvision: worst {worst:.2e}, {seen}")
    assert min(seen.values()) > 0, seen


def test_augment_check_accepts_and_rejects():
    """The fp64 restatement in fp32 passes; the output with image 1 flipped the other way fails."""
    x = torch.rand(3, 3, 30, 34, generator=torch.Generator().manual_seed(1))
    kw = dict(ops=(2, 0, 3, 1), factor=(1.3, 0.7, 1.4, 0.1), one_minus=(-0.3, 0.3, -0.4, 0.9), grayscale=False,
              flip=True, blur_kernel=[0.07, 0.12, 0.07, 0.12, 0.24, 0.12, 0.07, 0.12, 0.07],
              normalize=((0.485, 0.456, 0.406), (0.229, 0.224, 0.225)), crop=(3, 5, 21, 17), out_size=(24, 24))
    A = _args("augment", x, **kw)
    good = AU.augment64(x, **kw).float()
    wrong = good.clone()
    wrong[1] = AU.augment64(x[1:2], **dict(kw, flip=False)).float()[0]
    assert _worst(BC.CHECKS["augment"].check(A, {}, good)) <= 1.0
    assert _worst(BC.CHECKS["augment"].check(A, {}, wrong)) > 1.0


# --------------------------------------------------------------------------- multiview FILIP

@pytest.mark.parametrize("n,b,B", [(2, 4, 12), (3, 5, 5), (2, 1, 3), (4, 2, 8)])
def test_filip_block_columns(n, b, B):
    from x_clip_b200.filip import positive_column
    for col_run in {b, B}:
        cols = torch.stack([BC.block_columns(n, b, B, col_run, j) for j in range(n)])
        assert sorted(cols.flatten().tolist()) == list(range(n * B)), (col_run, cols)
        for j in range(n):
            for rank in range(B // b):
                for x in range(b):
                    assert cols[j, rank * b + x].item() == positive_column(0, j, x, rank, b, n, col_run)


def _blocks_case(dcl, seed=0):
    """m = n = 2 views, b = 4 rows of rank 1 of 3 (B = 12), one row without valid tokens."""
    g = torch.Generator().manual_seed(seed)
    m, n, b, B, off = 2, 2, 4, 12, 4
    s = torch.randn(m * b, n * B, generator=g) * 3
    valid = torch.ones(m * b, dtype=torch.bool)
    valid[6] = False
    s[6] = -torch.finfo(F32).max
    block_w = torch.tensor([0.9, 0.1 / 3, 0.1 / 3, 0.1 / 3]) / (2 * B)
    return dict(s=s, m=m, n=n, diag_off=off, dcl=dcl, block_w=block_w, row_valid=valid, b=b, B=B)


def _blocks_outputs(c, col_run):
    """lse, loss and g of the block kernels in fp64 (the check's reference), rounded to fp32."""
    A = dict(c, col_run=col_run)
    lse, pos, bw, parts = BC._blocks_ref(A)
    valid = c["row_valid"]
    lse = torch.where(valid[:, None], lse, 0.0)
    loss = (bw * (lse - pos))[valid].sum()
    R = c["s"].shape[0]
    rows = torch.arange(R)
    g = torch.zeros(R, c["n"] * c["B"], dtype=torch.float64)
    for j, (cols, p) in enumerate(parts):
        gj = 0.7 * bw[:, j:j + 1] * p
        gj[rows, rows % c["b"] + c["diag_off"]] -= 0.7 * bw[:, j]
        g[:, cols] = gj
    g[~valid] = 0.0
    return lse.float(), loss.float().reshape(1), g.float()


@pytest.mark.parametrize("dcl", [False, True])
def test_filip_blocks_check_accepts_and_rejects(dcl):
    """The outputs of the rank-major map pass; those of the view-major map (col_run b and B swapped)
    fail both checks."""
    c = _blocks_case(dcl)
    b = c["b"]
    gs = torch.tensor([0.7])
    for out_run, ok in ((b, True), (c["B"], False)):
        lse, loss, g = _blocks_outputs(c, out_run)
        Af = _args("filip_nce_blocks_fwd", c["s"], c["m"], c["n"], b, c["diag_off"], dcl, c["block_w"], loss,
                   row_valid=c["row_valid"])
        rf = BC.CHECKS["filip_nce_blocks_fwd"].check(Af, {"loss_accum": torch.zeros(1)}, lse)
        Ab = _args("filip_nce_blocks_bwd", c["s"], lse, c["m"], c["n"], b, c["diag_off"], dcl, c["block_w"], gs,
                   row_valid=c["row_valid"])
        rb = BC.CHECKS["filip_nce_blocks_bwd"].check(Ab, {}, g)
        assert (_worst(rf) <= 1.0) == ok and (_worst(rb) <= 1.0) == ok, (out_run, rf, rb)


# --------------------------------------------------------------------------- sigmoid loss

def _split(p):
    z = torch.nn.functional.normalize(p, dim=-1)
    hi = z.to(BF16)
    lo = (z - hi.float()).to(BF16)
    return torch.cat([hi, lo, hi], 1), torch.cat([hi, hi, lo], 1)


def test_sigmoid_bwd_check_accepts_and_rejects():
    """g rounded to bf16 passes; g with the bias left out of the first 128 columns fails."""
    g0 = torch.Generator().manual_seed(3)
    R, C, D = 64, 203, 128
    a, _ = _split(torch.randn(R, D, generator=g0))
    _, b = _split(torch.randn(C, D, generator=g0))
    temp, bias, gs = torch.tensor([10.0]), torch.tensor([-10.0]), torch.tensor([1.0 / C])
    l = 10.0 * (a.double() @ b.double().t())
    from sigmoid_oracle import labels
    z = labels(R, C, 0, like=l)

    def g_of(lg):
        rg = gs.item() * -z * torch.sigmoid(-z * lg)
        g = torch.zeros(R, (C + 7) // 8 * 8, dtype=BF16)
        g[:, :C] = (10.0 * rg).to(BF16)
        return g, rg

    good, rg = g_of(l - 10.0)
    wrong_l = l - 10.0
    wrong_l[:, :128] += 10.0
    wrong, _ = g_of(wrong_l)
    dt, db = (rg * l).sum().float().reshape(1), rg.sum().float().reshape(1)
    before = {"dtemp": torch.zeros(1), "dbias": torch.zeros(1)}
    A = _args("sigmoid_bwd", a, b, temp, bias, 0, gs, dtemp=dt, dbias=db)
    assert _worst(BC.CHECKS["sigmoid_bwd"].check(A, before, good)) <= 1.0
    assert _worst(BC.CHECKS["sigmoid_bwd"].check(A, before, wrong)) > 1.0


# --------------------------------------------------------------------------- vocabulary cross-entropy

def _vce_case(n=300, V=1000, d=128, seed=4):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, d, generator=g).to(BF16)
    w = (torch.randn(V, d, generator=g) * d ** -0.5).to(BF16)
    bias = torch.randn(V, generator=g) * 0.5
    labels = torch.randint(0, V - 1, (n,), generator=g)
    l = x.double() @ w.double().t() + bias.double()
    return x, w, bias, labels, l


def test_vocab_ce_fwd_check_accepts_and_rejects():
    """lse and target logits in fp32 pass; target logits taken from label + 1 fail."""
    x, w, bias, labels, l = _vce_case()
    lse = torch.logsumexp(l, 1)
    A = _args("vocab_ce_fwd", x, w, bias, labels)
    good = (lse.float(), l.gather(1, labels[:, None])[:, 0].float())
    wrong = (good[0], l.gather(1, labels[:, None] + 1)[:, 0].float())
    assert _worst(BC.CHECKS["vocab_ce_fwd"].check(A, {}, good)) <= 1.0
    assert _worst(BC.CHECKS["vocab_ce_fwd"].check(A, {}, wrong)) > 1.0


def test_vocab_ce_bwd_check_accepts_and_rejects():
    """One backward window: g rounded to bf16 passes; g computed with the lse shifted by one row fails."""
    x, w, bias, labels, l = _vce_case()
    lse = torch.logsumexp(l, 1).float()
    gs = 1.0 / 300

    def g_of(lk):
        g = gs * torch.exp(l - lk.double()[:, None])
        g[torch.arange(300), labels] -= gs
        return g.to(BF16)

    A = _args("vocab_ce_bwd", x[100:250], w, bias, labels[100:250], lse[100:250], torch.tensor([gs]))
    good, wrong = g_of(lse)[100:250], g_of(lse.roll(1))[100:250]
    assert _worst(BC.CHECKS["vocab_ce_bwd"].check(A, {}, good)) <= 1.0
    assert _worst(BC.CHECKS["vocab_ce_bwd"].check(A, {}, wrong)) > 1.0


# --------------------------------------------------------------------------- similarity regularisation

def test_simreg_fwd_check_accepts_and_rejects():
    """Row sums of E^2 in fp32 pass; the row sums with the diagonal column left in fail.  The operands
    are not unit rows, so E's diagonal is not near 0 as it is for a training step's latents."""
    g = torch.Generator().manual_seed(5)
    t, v = torch.randn(40, 96, generator=g).to(BF16), torch.randn(40, 96, generator=g).to(BF16)
    a, b = torch.cat([t[8:24], v[8:24]], 1), torch.cat([t, -v], 1)
    e = a.double() @ b.double().t()
    full = (e * e).sum(1)
    r = torch.arange(16)
    good = (full - e[r, r + 8] ** 2).float()
    A = _args("simreg_fwd", a, b, 8)
    assert _worst(BC.CHECKS["simreg_fwd"].check(A, {}, good)) <= 1.0
    assert _worst(BC.CHECKS["simreg_fwd"].check(A, {}, full.float())) > 1.0


# --------------------------------------------------------------------------- attention with dropout

@pytest.mark.parametrize("causal", [False, True])
def test_attn_dropout_check_accepts_and_rejects(causal):
    """o, lse and dqkv from the fp64 reference with layer L's mask pass; with layer L + 1's mask fail."""
    import attn_oracle as AO
    B, n, H, p, layer, seed = 3, 17, 2, 0.2, 1, -6917529027641081857
    case = AO.attn_case("flat", B, n, H, causal=causal, seed=21)
    qkv, mask, d_o = case["qkv"], case["mask"], case["d_o"]
    seed_t = torch.tensor([seed], dtype=torch.int64)
    scale = 64 ** -0.5

    def outputs(L):
        drop = DO.attn_drop_mul(seed, B, H, n, L, p)
        f = DO._attn_chunk64(qkv, mask, B, n, H, scale, causal, None, None, drop)
        o = f["o"].to(BF16)
        r = DO._attn_chunk64(qkv, mask, B, n, H, scale, causal, o, d_o, drop)
        return o, f["lse"].float(), r["dqkv"].to(BF16)

    o, lse, dqkv = outputs(layer)
    ow, lsew, dqkvw = outputs(layer + 1)
    dr = (p, seed_t, layer)
    Af = _args("attn_fwd", qkv, mask, B, n, H, scale, causal, dropout=dr)
    assert _worst(BC.CHECKS["attn_fwd"].check(Af, {}, (o, lse))) <= 1.0
    assert _worst(BC.CHECKS["attn_fwd"].check(Af, {}, (ow, lsew))) > 1.0
    Ab = _args("attn_bwd", qkv, mask, o, d_o, lse, B, n, H, scale, causal, dropout=dr)
    assert _worst(BC.CHECKS["attn_bwd"].check(Ab, {}, dqkv)) <= 1.0
    assert _worst(BC.CHECKS["attn_bwd"].check(Ab, {}, dqkvw)) > 1.0


# --------------------------------------------------------------------------- image gradients

def test_unpatchify_inverts_patchify():
    img = torch.randn(2, 3, 28, 42, generator=torch.Generator().manual_seed(6))
    rows = GO.patchify64(img, 14).reshape(-1, 588)
    assert torch.equal(BC.unpatchify64(rows, img.shape, 14, None), img.double())


def test_patchify_scatter_check_accepts_and_rejects():
    """The image from the kept rows (588 values each, read from rows of stride 592) passes; the image
    with two patches of one sample swapped fails."""
    g = torch.Generator().manual_seed(7)
    B, k = 2, 3
    keep = torch.stack([torch.randperm(6, generator=g)[:k] for _ in range(B)])
    wide = torch.randn(B * k, 592, generator=g)
    src = wide[:, :588]
    shape = (B, 3, 28, 42)
    good = BC.unpatchify64(src, shape, 14, keep).float()
    swapped = BC.unpatchify64(src[[1, 0, 2, 3, 4, 5]], shape, 14, keep).float()
    A = _args("patchify_scatter", src, shape, 14, keep)
    assert _worst(BC.CHECKS["patchify_scatter"].check(A, {}, good)) <= 1.0
    assert _worst(BC.CHECKS["patchify_scatter"].check(A, {}, swapped)) > 1.0
    assert not bool(good.view(B, 3, 2, 14, 3, 14).permute(0, 2, 4, 1, 3, 5).reshape(B, 6, -1)
                    [torch.arange(B)[:, None], torch.tensor([[j for j in range(6) if j not in keep[b]]
                                                             for b in range(B)])].any()), "dropped patches are 0"


def test_cast_rows_check_accepts_and_rejects():
    src = torch.randn(5, 588, generator=torch.Generator().manual_seed(8))
    good = torch.zeros(5, 592, dtype=BF16)
    good[:, :588] = src.to(BF16)
    bad = good.clone()
    bad[2, 590] = 1.0
    A = _args("cast_bf16_rows", src, 592)
    assert _worst(BC.CHECKS["cast_bf16_rows"].check(A, {}, good)) <= 1.0
    assert _worst(BC.CHECKS["cast_bf16_rows"].check(A, {}, bad)) > 1.0
