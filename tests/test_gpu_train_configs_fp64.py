"""The training configurations bench.py does not time, checked kernel call by kernel call against fp64
(bench_call_oracle), at the shapes training sends.  Each workload is one forward and backward step under
the Recorder; every kernel call's first signature is checked, a call with no check fails the workload,
and each test asserts the signatures it exists to reach.

- sigmoid: cfg3 (ViT-B/16 + 77-token text tower, depth 2), CLIP(sigmoid_loss=True), 4096 pairs in
  micro-batches of 768: sigmoid_fwd / _bwd at a = b = (4096, 1536);
- simreg: cfg3 dcl_extra with sim_reg_loss_weight > 0, 4096 pairs in micro-batches of 768: simreg_fwd /
  _bwd at R = 4096;
- mlm_simclr: cfg3 with use_mlm and SimCLR, 4096 pairs in micro-batches of 768, CUDA images without
  grad so the augmentation kernels run: vocab_ce_fwd at V = 49 408 over about 47 k masked rows, a full
  10 752-row backward window and the ragged last one, augment at 224 px with contrast, the blur and a
  crop off the borders;
- simsiam: cfg2 (the README model), 1024 pairs: augment at 256 px from 256 px images;
- filip_multiview / filip_multiview_dcl: FILIP on the README model with aug_text and aug_image (m = n =
  2), 256 pairs, plain InfoNCE and dcl_extra, an empty caption in each text view (row_valid = False
  rows).  At one rank b == B, so col_run b and B name the same column map here; the self-test, at
  rank 1 of 3, is what tells the two maps apart;
- image_grad: ViT-L/14-shaped image tower (dim 1024, 16 heads, patch 14, depth 2) at 224 px with the
  cfg3 text tower at depth 2, patch dropout 0.5, image.requires_grad_(True), micro-batched; and one
  single-pass step at 336 px (576 patches): cast_bf16_rows (588 values in rows of 592) and
  patchify_scatter with keep;
- attn_dropout: cfg3 towers at depth 2 with attn_dropout = 0.1, 4096 pairs in micro-batches of 768:
  attn_fwd / _bwd with dropout at (768, 98, 12) and at (768, 78, 8) with a key mask.
A self-test feeds each new family's check the kernel's own output and one plausible wrong output.

The GEMM check's chain bound is four ulp per MMA of the running sum (gemm_oracle): one wgmma truncates
its 16 products two bits below the ulp of the largest term, all in one direction when they share a
sign.  test_one_mma_truncation_within_chain_bound pins that on the device: the MLM head's weight
gradient (168 k-blocks of small same-sign softmax terms) exceeded a two-ulp bound by 1.05 x.

Measured on an H100 80GB HBM3 (700 W power limit), each test with its fp64 references: run time and
peak allocated memory sigmoid 10.0 s / 44.6 GiB, simreg 8.3 s / 44.6 GiB, mlm_simclr 15.1 s / 51.7 GiB
(backward windows of 10 752 and 10 136 rows), simsiam 10.6 s / 47.7 GiB, filip_multiview 9.6 s / 23.4
GiB (dcl_extra 9.6 s / 24.6 GiB), image_grad 224 px 5.6 s / 18.7 GiB and 336 px 3.2 s / 5.6 GiB,
attn_dropout 12.8 s / 44.6 GiB, self-test 0.4 s / 1.8 GiB; the file runs in about 110 s.  NEED_GIB
holds each peak plus about 10 %: a test skips, naming both numbers, when less is free on the shared
device.  Worst gate ratios of the new families: sigmoid_fwd 0.010, sigmoid_bwd 0.487, simreg_fwd 0.081,
simreg_bwd 0.976, vocab_ce_fwd 0.013, vocab_ce_bwd 0.490, augment 0.440 (cfg3) and 0.127 (cfg2),
filip_nce_blocks_fwd 0.055, filip_nce_blocks_bwd 0.039, attention with dropout attn_fwd 0.693 and
attn_bwd 0.981; cast_bf16_rows, patchify_scatter and simreg_pack exact; gemm at most 0.988 (the bf16
outputs at their rounding bound).  Self-test: every wrong output at 17.9 gates or more (the lse shifted
by one row).  One MMA of 16 same-sign products lost up to 3.91 ulp of its running sum (2.12 on
average).
"""
import math

import pytest
import torch

import bench_call_oracle as BC
from test_gpu_bench_shapes_fp64 import _need, _report, _seen, _shape, _start, _verdict

pytestmark = pytest.mark.gpu

# free device memory (GiB) each test needs: its measured peak plus about 10 %
NEED_GIB = {"sigmoid": 49, "simreg": 49, "mlm_simclr": 57, "simsiam": 53, "filip_multiview": 27,
            "image_grad": 21, "attn_dropout": 49, "self_test": 2}

AUG_SEED_224 = 16      # torch seed whose two SimCLR draws at 224 px take contrast, the blur and an inner crop
AUG_SEED_256 = 13      # the same at 256 px


@pytest.fixture(autouse=True)
def _need_table(monkeypatch):
    import test_gpu_bench_shapes_fp64 as S
    monkeypatch.setattr(S, "NEED_GIB", {**S.NEED_GIB, **NEED_GIB})    # _need reads the sibling's table


def _data(cfg, batch, dev):
    gd = torch.Generator(device=dev).manual_seed(1)
    S, V, I = cfg["text_seq_len"], cfg["num_text_tokens"], cfg["visual_image_size"]
    text = torch.randint(1, V, (batch, S), generator=gd, device=dev)
    lens = torch.randint(S // 4, S + 1, (batch, 1), generator=gd, device=dev)
    text = text.masked_fill(torch.arange(S, device=dev)[None] >= lens, 0)      # right padding
    image = torch.randn(batch, 3, I, I, generator=gd, device=dev)
    return text, image


def _run(dev, monkeypatch, what, cfg, kw, batch, microbatch, drop=0.5, seed=None, image_grad=False,
         encoders=None, views=None, text_edit=None):
    import x_clip_b200
    from x_clip_b200 import kernels
    _need(what)
    t0 = _start()
    rec = BC.Recorder(kernels).install(monkeypatch)
    torch.manual_seed(0)
    clip = x_clip_b200.CLIP(**cfg, **kw, visual_patch_dropout=drop, microbatch=microbatch or None,
                            **(encoders or {})).to(dev)
    clip.train()
    text, image = _data(cfg, batch, dev)
    if text_edit is not None:
        text = text_edit(text)
    if image_grad:
        image.requires_grad_(True)
    extra = {}
    if views is not None:
        extra = views(text, image)
    if seed is not None:
        torch.manual_seed(seed)
    loss = clip(text, image, return_loss=True, **extra)
    loss.backward()
    _report(what, t0)
    assert math.isfinite(loss.item())
    if image_grad:
        assert image.grad is not None and bool(image.grad.abs().sum() > 0)
    return rec, clip


def _cfg3():
    import bench
    return dict(bench.VITB16_CFG, text_enc_depth=2, visual_enc_depth=2)


def test_sigmoid_cfg3(cuda_device, monkeypatch):
    rec, _ = _run(cuda_device, monkeypatch, "sigmoid", _cfg3(), dict(sigmoid_loss=True), 4096, 768)
    assert _seen(rec, "sigmoid_fwd", a=_shape(4096, 1536), b=_shape(4096, 1536))
    assert _seen(rec, "sigmoid_bwd", a=_shape(4096, 1536), b=_shape(4096, 1536),
                 dtemp=lambda t: t is not None)
    _verdict(rec, "sigmoid")


def test_simreg_cfg3(cuda_device, monkeypatch):
    import bench
    kw = dict(bench.LOSS_KW["dcl_extra"], sim_reg_loss_weight=1.0)
    rec, _ = _run(cuda_device, monkeypatch, "simreg", _cfg3(), kw, 4096, 768)
    rows = lambda t: t is not None and t.shape[0] == 4096          # noqa: E731
    assert _seen(rec, "simreg_fwd", a=rows) and _seen(rec, "simreg_bwd", a=rows) and _seen(rec, "simreg_pack")
    _verdict(rec, "simreg")


def _aug_seen(rec, size):
    sz = (size, size)
    assert _seen(rec, "augment", out_size=sz, ops=lambda o: 1 in o), "contrast"
    assert _seen(rec, "augment", out_size=sz, blur_kernel=lambda k: k is not None), "blur"
    inner = lambda A: A["crop"][0] > 0 and A["crop"][1] > 0                        # noqa: E731
    assert any(nm == "augment" and inner(A) for (nm, _), A in rec.arguments.items()), "crop off the borders"


def test_mlm_simclr_cfg3(cuda_device, monkeypatch):
    """MLM and SimCLR on cfg3, 4096 pairs of captions 19 to 77 tokens long: about 47 k masked rows, so
    the MLM backward runs four full windows of 10 752 rows and a ragged last one; both views of the 4096
    CUDA images are augmented by the kernels."""
    kw = dict(use_mlm=True, mlm_mask_token_id=2, use_visual_ssl=True, visual_ssl_type="simclr")
    rec, _ = _run(cuda_device, monkeypatch, "mlm_simclr", _cfg3(), kw, 4096, 768, seed=AUG_SEED_224)
    assert _seen(rec, "vocab_ce_fwd", w=lambda t: t is not None and t.shape[0] == 49408,
                 x=lambda t: t is not None and t.shape[0] > 2 * 10752)
    bwd_rows = sorted(A["x"].shape[0] for (nm, _), A in rec.arguments.items() if nm == "vocab_ce_bwd")
    print("vocab_ce_bwd windows", bwd_rows)
    assert 10752 in bwd_rows and any(r < 10752 for r in bwd_rows), bwd_rows
    assert _seen(rec, "augment", x=_shape(4096, 3, 224, 224))
    _aug_seen(rec, 224)
    _verdict(rec, "mlm_simclr")


def test_simsiam_cfg2(cuda_device, monkeypatch):
    import bench
    kw = dict(use_visual_ssl=True, visual_ssl_type="simsiam")
    rec, _ = _run(cuda_device, monkeypatch, "simsiam", bench.README_CFG, kw, 1024, 0, seed=AUG_SEED_256)
    assert _seen(rec, "augment", x=lambda t: t is not None and t.shape[-1] == 256)
    _aug_seen(rec, 256)
    _verdict(rec, "simsiam")


def _views(text, image):
    g = torch.Generator(device=text.device).manual_seed(2)
    t2 = text.roll(1, dims=1)
    t2[3] = 0                                         # an empty caption in the second view
    return dict(aug_text=[t2], aug_image=[image.flip(-1) + 0.1 * torch.randn(image.shape, generator=g,
                                                                               device=image.device)])


def _empty_caption(text):
    text = text.clone()
    text[5] = 0                                       # and one in the first
    return text


@pytest.mark.parametrize("loss", ["nce", "dcl_extra"])
def test_filip_multiview(cuda_device, monkeypatch, loss):
    import bench
    kw = dict(bench.LOSS_KW[loss], use_all_token_embeds=True)
    rec, _ = _run(cuda_device, monkeypatch, "filip_multiview", bench.README_CFG, kw, 256, 0, views=_views,
                  text_edit=_empty_caption)
    for name in ("filip_nce_blocks_fwd", "filip_nce_blocks_bwd"):
        assert _seen(rec, name, m=2, n=2), name
    # the empty captions' i2t rows reached both block kernels as row_valid = False rows: their checks
    # add the lse_invalid / g_invalid outputs only when such a row is present
    for out in ("filip_nce_blocks_fwd[", "filip_nce_blocks_bwd["):
        tail = "lse_invalid" if "fwd" in out else "g_invalid"
        assert any(lab.startswith(out) and lab.endswith(tail) for lab, _ in rec.results), out
    _verdict(rec, f"filip_multiview_{loss}")


def _vitl14():
    return dict(_cfg3(), dim_image=1024, visual_heads=16, visual_patch_size=14)


def test_image_grad_vitl14_224(cuda_device, monkeypatch):
    rec, _ = _run(cuda_device, monkeypatch, "image_grad", _vitl14(), {}, 1024, 256, image_grad=True)
    assert _seen(rec, "cast_bf16_rows", src=_shape(1024, 588), ld=592)
    assert _seen(rec, "patchify_scatter", keep=_shape(256, 128), patch=14)
    _verdict(rec, "image_grad_224")


def test_image_grad_vitl14_336(cuda_device, monkeypatch):
    cfg = dict(_vitl14(), visual_image_size=336)
    rec, _ = _run(cuda_device, monkeypatch, "image_grad", cfg, {}, 64, 0, image_grad=True)
    assert _seen(rec, "cast_bf16_rows", src=_shape(1024, 588), ld=592)
    assert _seen(rec, "patchify_scatter", keep=_shape(64, 288), image_shape=(64, 3, 336, 336))
    _verdict(rec, "image_grad_336")


def test_attn_dropout_cfg3(cuda_device, monkeypatch):
    import x_clip_b200
    cfg = _cfg3()

    def encoders():
        text = x_clip_b200.TextTransformer(512, num_tokens=49408, max_seq_len=77, dim_head=64, depth=2, heads=8,
                                           attn_dropout=0.1)
        image = x_clip_b200.VisionTransformer(768, image_size=224, patch_size=16, channels=3, dim_head=64, depth=2,
                                              heads=12, patch_dropout=0.5, attn_dropout=0.1)
        return dict(text_encoder=text, image_encoder=image)

    torch.manual_seed(0)
    rec, _ = _run(cuda_device, monkeypatch, "attn_dropout", cfg, {}, 4096, 768, encoders=encoders())
    dropped = lambda d: d is not None                                          # noqa: E731
    masked = lambda m: m is not None                                           # noqa: E731
    for name in ("attn_fwd", "attn_bwd"):
        assert _seen(rec, name, B=768, n=98, heads=12, dropout=dropped), name
        assert _seen(rec, name, B=768, n=78, heads=8, key_mask=masked, dropout=dropped), name
    _verdict(rec, "attn_dropout")


# --------------------------------------------------------------------------- the checks themselves

def _ratio(name, got, *args, before=None, **kw):
    import inspect
    from x_clip_b200 import kernels as K
    ba = inspect.signature(getattr(K, name)).bind(*args, **kw)
    ba.apply_defaults()
    return max(BC.CHECKS[name].check(dict(ba.arguments), before or {}, got).values())


def test_one_mma_truncation_within_chain_bound(cuda_device):
    """One MMA of 16 positive products 2^-12 to 2^-24 of a running sum of 1.0 (the first MMA of the
    k-block adds 1.0; the second the 16 products): the tensor cores lose up to 4 ulp of the running sum,
    more than 2^-22 of it, and the GEMM check's chain bound holds every element."""
    from x_clip_b200 import kernels as K
    _need("self_test")
    dev = cuda_device
    gen = torch.Generator(device=dev).manual_seed(11)
    M = N = 2048
    a = torch.zeros(M, 64, device=dev)
    b = torch.zeros(N, 64, device=dev)
    a[:, 0] = b[:, 0] = 1.0
    for t, n in ((a, M), (b, N)):
        e = torch.randint(6, 12, (n, 16), generator=gen, device=dev).float()
        t[:, 16:32] = (1 + torch.rand(n, 16, generator=gen, device=dev)) * 2.0 ** -e
    a, b = a.bfloat16(), b.bfloat16()
    out = K.gemm(a, b, accumulate=True)
    ref = a.double() @ b.double().t()
    lost = (ref - out.double()) / 2.0 ** -23              # in ulp of the running sum (1 <= ref < 2)
    ratio = _ratio("gemm", out, a, b, accumulate=True, before={"out": torch.zeros_like(out)})
    print(f"GATE one_mma_truncation lost ulp max {lost.max().item():.3f} mean {lost.mean().item():.3f}, "
          f"min {lost.min().item():.3f}; chain bound {ratio:.4f}")
    assert lost.min().item() >= 0.0                        # truncation: never above the exact sum
    assert lost.max().item() > 2.0                         # beyond two ulp, 2^-22 of a sum just above 1
    assert ratio <= 1.0


def test_checks_reject_wrong_outputs(cuda_device):
    """Each new family's check accepts the kernel's own output and rejects one plausible wrong one."""
    from x_clip_b200 import kernels as K
    _need("self_test")
    t0 = _start()
    dev = cuda_device
    gen = torch.Generator(device=dev).manual_seed(9)
    F32, BF16 = torch.float32, torch.bfloat16
    r = {}

    # vocabulary cross-entropy at V = 49 408, d = 512
    n, V, d = 1000, 49408, 512
    x = torch.randn(n, d, generator=gen, device=dev).to(BF16)
    w = (torch.randn(V, d, generator=gen, device=dev) * d ** -0.5).to(BF16)
    bias = torch.randn(V, generator=gen, device=dev) * 0.5
    labels = torch.randint(0, V - 1, (n,), generator=gen, device=dev)
    lse, pos = K.vocab_ce_fwd(x, w, bias, labels)
    _, pos1 = K.vocab_ce_fwd(x, w, bias, labels + 1)
    r["vocab_ce_fwd_good"] = _ratio("vocab_ce_fwd", (lse, pos), x, w, bias, labels)
    r["vocab_ce_fwd_label_plus_1"] = _ratio("vocab_ce_fwd", (lse, pos1), x, w, bias, labels)
    gs = torch.tensor([1.0 / n], device=dev)
    win = slice(200, 700)
    xs, ls, es = x[win].contiguous(), labels[win].contiguous(), lse[win].contiguous()
    g = K.vocab_ce_bwd(xs, w, bias, ls, es, gs)
    g_shift = K.vocab_ce_bwd(xs, w, bias, ls, es.roll(1), gs)
    r["vocab_ce_bwd_good"] = _ratio("vocab_ce_bwd", g, xs, w, bias, ls, es, gs)
    r["vocab_ce_bwd_lse_shifted"] = _ratio("vocab_ce_bwd", g_shift, xs, w, bias, ls, es, gs)
    del x, w, g, g_shift

    # sigmoid loss at (4096, 1536) split operands
    R, D = 4096, 512
    _, a, _, _ = K.l2norm_fwd(torch.randn(R, D, generator=gen, device=dev))
    _, _, b, _ = K.l2norm_fwd(torch.randn(R, D, generator=gen, device=dev))
    te, lb = torch.tensor([10.0], device=dev), torch.tensor([-10.0], device=dev)
    gs = torch.tensor([1.0 / R], device=dev)
    g = K.sigmoid_bwd(a, b, te, lb, 0, gs)
    g0 = K.sigmoid_bwd(a, b, te, torch.zeros(1, device=dev), 0, gs)
    wrong = g.clone()
    wrong[:, 1024:1152] = g0[:, 1024:1152]
    r["sigmoid_bwd_good"] = _ratio("sigmoid_bwd", g, a, b, te, lb, 0, gs)
    r["sigmoid_bwd_bias_left_out_of_a_block"] = _ratio("sigmoid_bwd", wrong, a, b, te, lb, 0, gs)

    # similarity regularisation on operands that are not unit rows (E's diagonal is not near 0)
    t, v = (torch.randn(R, 256, generator=gen, device=dev).to(BF16) for _ in range(2))
    sa, sb = K.simreg_pack(t, v, False), K.simreg_pack(t, v, True)
    rs = K.simreg_fwd(sa, sb, 0)
    diag = (sa.double() * sb.double()).sum(1) ** 2
    r["simreg_fwd_good"] = _ratio("simreg_fwd", rs, sa, sb, 0)
    r["simreg_fwd_diagonal_kept"] = _ratio("simreg_fwd", (rs.double() + diag).float(), sa, sb, 0)

    # multiview FILIP blocks: rank 1 of 3 (b = 64, B = 192), col_run b against B
    m = nv = 2
    bb, B = 64, 192
    s = torch.randn(m * bb, nv * B, generator=gen, device=dev) * 4
    bw = torch.tensor([0.9, 0.1 / 3, 0.1 / 3, 0.1 / 3], device=dev) / (2 * B)
    valid = torch.ones(m * bb, dtype=torch.bool, device=dev)
    valid[7] = False
    for dcl in (False, True):
        outs = {}
        for run in (bb, B):
            loss = torch.zeros(1, device=dev)
            lse_b = K.filip_nce_blocks_fwd(s, m, nv, run, bb, dcl, bw, loss, row_valid=valid)
            g_b = K.filip_nce_blocks_bwd(s, lse_b, m, nv, run, bb, dcl, bw, torch.ones(1, device=dev), row_valid=valid)
            outs[run] = (lse_b, loss, g_b)
        for run, tag in ((bb, "good"), (B, "col_run_swapped")):
            lse_b, loss, g_b = outs[run]
            r[f"filip_blocks_fwd_dcl{int(dcl)}_{tag}"] = _ratio(
                "filip_nce_blocks_fwd", lse_b, s, m, nv, bb, bb, dcl, bw, loss, row_valid=valid,
                before={"loss_accum": torch.zeros(1, device=dev)})
            r[f"filip_blocks_bwd_dcl{int(dcl)}_{tag}"] = _ratio(
                "filip_nce_blocks_bwd", g_b, s, outs[bb][0], m, nv, bb, bb, dcl, bw, torch.ones(1, device=dev),
                row_valid=valid)

    # attention with dropout at the cfg3 vision shape, 64 batch items: layer 1's mask against layer 2's
    import attn_oracle as AO
    Bn, n_, H = 64, 98, 12
    case = AO.attn_case("flat", Bn, n_, H, seed=3, device=dev)
    seed = torch.tensor([-6917529027641081857], dtype=torch.int64, device=dev)
    sc = 64 ** -0.5
    outs = {}
    for L in (1, 2):
        o, lse_a = K.attn_fwd(case["qkv"], None, Bn, n_, H, sc, dropout=(0.1, seed, L))
        outs[L] = (o, lse_a)
    o1, l1 = outs[1]
    dq1 = K.attn_bwd(case["qkv"], None, o1, case["d_o"], l1, Bn, n_, H, sc, dropout=(0.1, seed, 1))
    dq2 = K.attn_bwd(case["qkv"], None, o1, case["d_o"], l1, Bn, n_, H, sc, dropout=(0.1, seed, 2))
    fw = lambda got: _ratio("attn_fwd", got, case["qkv"], None, Bn, n_, H, sc, dropout=(0.1, seed, 1))  # noqa: E731
    bw_ = lambda got: _ratio("attn_bwd", got, case["qkv"], None, o1, case["d_o"], l1, Bn, n_, H, sc,    # noqa: E731
                             dropout=(0.1, seed, 1))
    r["attn_fwd_dropout_good"], r["attn_fwd_dropout_next_layer_mask"] = fw(outs[1]), fw(outs[2])
    r["attn_bwd_dropout_good"], r["attn_bwd_dropout_next_layer_mask"] = bw_(dq1), bw_(dq2)

    # patch scatter at ViT-L/14 (588 of 592 columns), two patches of sample 0 swapped
    Bi, k = 8, 128
    keep = torch.stack([torch.randperm(256, generator=gen, device=dev)[:k] for _ in range(Bi)])
    wide = torch.randn(Bi * k, 592, generator=gen, device=dev)
    src = wide[:, :588]
    img = K.patchify_scatter(src, (Bi, 3, 224, 224), 14, keep)
    keep_sw = keep.clone()
    keep_sw[0, [0, 1]] = keep[0, [1, 0]]
    img_sw = K.patchify_scatter(src, (Bi, 3, 224, 224), 14, keep_sw)
    r["patchify_scatter_good"] = _ratio("patchify_scatter", img, src, (Bi, 3, 224, 224), 14, keep)
    r["patchify_scatter_two_patches_swapped"] = _ratio("patchify_scatter", img_sw, src, (Bi, 3, 224, 224), 14, keep)

    # augmentation: image 1 of the batch without the flip the call asked for
    xa = torch.rand(4, 3, 224, 224, generator=gen, device=dev)
    kw = dict(ops=(0, 1, 2, 3), factor=(1.3, 0.7, 1.4, 0.1), one_minus=(-0.3, 0.3, -0.4, 0.9),
              blur_kernel=[0.07, 0.12, 0.07, 0.12, 0.24, 0.12, 0.07, 0.12, 0.07],
              normalize=((0.485, 0.456, 0.406), (0.229, 0.224, 0.225)), crop=(20, 31, 150, 170),
              out_size=(224, 224))
    out = K.augment(xa, flip=True, **kw)
    wrong = out.clone()
    wrong[1] = K.augment(xa[1:2], flip=False, **kw)[0]
    r["augment_good"] = _ratio("augment", out, xa, flip=True, **kw)
    r["augment_flip_on_the_wrong_image"] = _ratio("augment", wrong, xa, flip=True, **kw)
    _report("self_test", t0)
    for key, val in r.items():
        print(f"GATE selftest_{key} {val:.4f}")
    good = {k_: v_ for k_, v_ in r.items() if k_.endswith("good")}
    bad = {k_: v_ for k_, v_ in r.items() if not k_.endswith("good")}
    assert max(good.values()) <= 1.0, good
    assert min(bad.values()) > 1.0, bad
