"""Patch sizes whose rows are not a multiple of 8 values (ViT-L/14's 14 x 14 x 3 = 588, 14 x 14 x 1 = 196,
7 x 7 x 3 = 147, 10 x 10 x 3 = 300) on the GPU:

- xclip_patchify_gather_rows bit-exact against a torch patchify, zero columns past patch_dim included,
  and xclip_patchify_scatter_rows bit-exact against a torch scatter on its float2 (even patch) and
  scalar (odd patch, or more than 4 channels) variants; both refuse bad strides, alignment and k before
  any launch;
- PatchEmbedFn / PatchifyFn at patch_dim 588 (GEMM K = 592) against fp64 under the gates of
  test_gpu_embed_fp64.py;
- CLIP against the reference goldens of tests/golden/make_golden_patch14.py at the tolerances of
  test_gpu_clip_parity.py / test_gpu_image_grad.py, and the micro-batched step against the single pass.
"""
import json
from pathlib import Path

import pytest
import torch

import block_oracle as BO
import gemm_oracle as GO

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).parent / "golden"


def _r8(x):
    return -(-x // 8) * 8


def _torch_patchify(img, p):
    b, c, H, W = img.shape
    x = img.view(b, c, H // p, p, W // p, p).permute(0, 2, 4, 3, 5, 1)
    return x.reshape(b, (H // p) * (W // p), p * p * c)


PC = [(14, 3), (14, 1), (7, 3), (10, 3), (16, 3)]


@pytest.mark.parametrize("P,C", PC)
@pytest.mark.parametrize("with_keep", [False, True])
def test_padded_gather_is_an_exact_patchify(cuda_device, P, C, with_keep):
    from x_clip_b200 import kernels as K
    dev = cuda_device
    g = torch.Generator().manual_seed(P * 10 + C)
    B, H, W = 3, 4 * P, 5 * P
    n = (H // P) * (W // P)
    img = torch.randn(B, C, H, W, generator=g)
    ref = _torch_patchify(img, P)
    keep = torch.stack([torch.randperm(n, generator=g)[: n // 2] for _ in range(B)]) if with_keep else None
    if keep is not None:
        ref = torch.stack([ref[b, keep[b]] for b in range(B)])
    ref = ref.reshape(-1, P * P * C).bfloat16()
    pd = P * P * C
    for ld in (_r8(pd), _r8(pd) + 16):
        out = K.patchify_gather(img.to(dev), P, None if keep is None else keep.to(dev), ld=ld)
        assert out.shape == (ref.shape[0], ld)
        out = out.cpu()
        assert torch.equal(out[:, :pd], ref), (P, C, ld)
        assert torch.equal(out[:, pd:], torch.zeros_like(out[:, pd:])), (P, C, ld)
    if pd % 8 == 0:          # the unpadded entry point: the same rows
        assert torch.equal(K.patchify_gather(img.to(dev), P, None if keep is None else keep.to(dev)).cpu(), ref)


def test_padded_cast_is_an_exact_cast(cuda_device):
    from x_clip_b200 import kernels as K
    w = torch.randn(1024, 588, generator=torch.Generator().manual_seed(1)).to(cuda_device)
    wb = K.cast_bf16_rows(w, 592)
    assert wb.shape == (1024, 592)
    assert torch.equal(wb[:, :588], w.bfloat16()) and torch.equal(wb[:, 588:], torch.zeros_like(wb[:, 588:]))


# (P, C): float2 variant at even patches that are not a multiple of 4 (C <= 4), scalar variant at odd
# patches and at C > 4, and the float4 variant for comparison
SCATTER_PC = [(14, 3), (14, 1), (10, 3), (6, 2), (7, 3), (7, 1), (14, 5), (16, 3)]


@pytest.mark.parametrize("P,C", SCATTER_PC)
@pytest.mark.parametrize("kind", ["none", "subset", "perm", "k1"])
def test_padded_scatter_is_an_exact_torch_scatter(cuda_device, P, C, kind):
    from test_gpu_image_grad import _keep, torch_scatter
    from x_clip_b200 import _lib, kernels as K
    dev = cuda_device
    g = torch.Generator().manual_seed(P * 100 + C)
    B, H, W = 3, 3 * P, 5 * P
    n = (H // P) * (W // P)
    keep = _keep(kind, B, n, dev, g)
    k = n if keep is None else keep.shape[1]
    pd = P * P * C
    for lds in (_r8(pd), _r8(pd) + 12):
        buf = torch.randn(B * k, lds, generator=g).to(dev)
        src = buf[:, :pd]
        ref = torch_scatter(src.contiguous(), B, C, H, W, P, keep)
        out = torch.full((B, C, H, W), float("nan"), device=dev)
        _lib.call("xclip_patchify_scatter_rows", src.data_ptr(), lds, B, C, H, W, P, _lib_ptr(keep), k,
                  out.data_ptr(), torch.cuda.current_stream().cuda_stream)
        assert not torch.isnan(out).any()
        assert torch.equal(out, ref), (P, C, kind, lds)
        assert torch.equal(K.patchify_scatter(src, (B, C, H, W), P, keep), ref)


def _lib_ptr(t):
    return None if t is None else t.data_ptr()


def test_scatter_inverts_the_padded_gather(cuda_device):
    from x_clip_b200 import kernels as K
    dev = cuda_device
    img = torch.randn(4, 3, 56, 84, device=dev).bfloat16().float()
    keep = torch.rand(4, 24, device=dev).topk(12, dim=-1).indices
    rows = K.patchify_gather(img, 14, keep, ld=592).float()
    back = K.patchify_scatter(rows[:, :588], img.shape, 14, keep)
    mask = K.patchify_scatter(torch.ones(48, 588, device=dev), img.shape, 14, keep)
    assert torch.equal(back, img * mask)
    assert int(mask.sum().item()) == 4 * 12 * 588


def _refused(name, args):
    from x_clip_b200 import _lib
    lib = _lib.load()
    s = torch.cuda.current_stream().cuda_stream
    torch.cuda.synchronize()
    for a in args:
        before = lib.xclip_launch_count()
        with pytest.raises(_lib.XClipB200Error):
            _lib.call(name, *a, s)
        assert lib.xclip_launch_count() == before, (name, a)


def test_padded_gather_refusals_launch_nothing(cuda_device):
    from x_clip_b200 import _lib, kernels as K
    dev = cuda_device
    img = torch.randn(2, 3, 56, 56, device=dev)
    out = torch.zeros(2 * 16, 640, device=dev, dtype=torch.bfloat16)
    keep = torch.zeros(2, 1, dtype=torch.int64, device=dev)
    i, o = img.data_ptr(), out.data_ptr()
    _refused("xclip_patchify_gather_rows", [
        (i, 2, 3, 56, 56, 14, None, 16, o, 588),                 # ldo % 8
        (i, 2, 3, 56, 56, 14, None, 16, o, 584),                 # ldo < patch_dim
        (i, 2, 3, 56, 56, 14, None, 16, o + 8, 592),             # misaligned output
        (i, 2, 3, 56, 56, 14, None, 8, o, 592),                  # k != n without keep
        (i, 2, 3, 56, 56, 14, keep.data_ptr(), 0, o, 592),       # k = 0
        (i, 2, 3, 50, 56, 14, None, 16, o, 592),                 # H % patch
        (None, 2, 3, 56, 56, 14, None, 16, o, 592),              # null
        (i, 2, 3, 56, 56, 0, None, 16, o, 592),                  # patch 0
    ])
    lib = _lib.load()
    torch.cuda.synchronize()
    n0 = lib.xclip_launch_count()
    with pytest.raises(_lib.XClipB200Error):
        K.patchify_gather(img, 14, ld=596)
    with pytest.raises(_lib.XClipB200Error):
        K.patchify_gather(img, 14)                               # no padded layout asked for
    assert lib.xclip_launch_count() == n0


def test_padded_scatter_refusals_launch_nothing(cuda_device):
    dev = cuda_device
    src = torch.zeros(64, 800, device=dev)
    out = torch.zeros(2, 3, 56, 56, device=dev)
    keep = torch.zeros(2, 1, dtype=torch.int64, device=dev)
    s, o = src.data_ptr(), out.data_ptr()
    _refused("xclip_patchify_scatter_rows", [
        (s, 584, 2, 3, 56, 56, 14, None, 16, o),                 # lds < patch_dim
        (s, 590, 2, 3, 56, 56, 14, None, 16, o),                 # lds % 4
        (s + 4, 592, 2, 3, 56, 56, 14, None, 16, o),             # misaligned src
        (s, 592, 2, 3, 56, 56, 14, None, 16, o + 8),             # misaligned output
        (s, 592, 2, 3, 56, 56, 14, None, 8, o),                  # k != n without keep
        (s, 592, 2, 3, 56, 56, 14, keep.data_ptr(), 0, o),       # k = 0
        (s, 592, 2, 3, 56, 56, 14, keep.data_ptr(), 17, o),      # k > n
        (s, 592, 2, 3, 56, 50, 14, None, 16, o),                 # W % patch
        (None, 592, 2, 3, 56, 56, 14, None, 16, o),              # null
    ])


# ----------------------------------------------------------------------------- patch embedding vs fp64

# (B, image size, patch, channels, keep per sample, d)
PATCH_CASES = [(3, 56, 14, 3, 9, 384), (5, 224, 14, 3, 128, 1024), (4, 336, 14, 3, 288, 1024),
               (6, 56, 14, 1, 10, 384), (3, 70, 7, 3, 50, 768)]


def _pad(t, ld):
    return torch.nn.functional.pad(t, (0, ld - t.shape[1]))


@pytest.mark.parametrize("B,S,p,C,k,d", PATCH_CASES)
def test_padded_patch_embed_fp64(cuda_device, B, S, p, C, k, d):
    """PatchEmbedFn on [B*k, roundup8(patch_dim)] rows: y, dW (contiguous [d, patch_dim]), d bias and
    d pos under the gates of test_gpu_embed_fp64.test_patch_embed_fp64; d patches has zero columns past
    patch_dim."""
    from x_clip_b200 import engine as E
    dev = cuda_device
    n = (S // p) ** 2
    pd = p * p * C
    ld = _r8(pd)
    t = GO.patch_embed_case(B, n, k, pd, d)
    t = {key: v.to(dev) for key, v in t.items()}
    index = t["keep"].reshape(-1).to(torch.int32)
    w = t["w"].clone().requires_grad_(True)
    bias = t["bias"].clone().requires_grad_(True)
    table = t["table"].clone().requires_grad_(True)
    patches = _pad(t["patches"], ld).requires_grad_(True)
    y = E.PatchEmbedFn.apply(patches, index, w, bias, table)
    y.backward(t["dy"])
    torch.cuda.synchronize()
    tb = t["table"].bfloat16()
    rows = index.long()
    ref = GO.gemm64(t["patches"], t["w"].bfloat16(), bias=t["bias"], residual=tb, res_rows=rows)
    gate = GO.gemm_gate(t["patches"], t["w"].bfloat16(), bias=t["bias"], residual=tb, res_rows=rows,
                        bf16_out=True, ref=ref)
    BO.check(f"patch_y_{S}_{p}_{C}_{d}", y, ref, gate)
    M = B * k
    assert w.grad.shape == (d, pd) and w.grad.is_contiguous()
    plan = GO.split_plan(d, ld, M, True, torch.cuda.get_device_properties(0).multi_processor_count)
    BO.check(f"patch_dW_{S}_{p}_{C}_{d}", w.grad, GO.gemm64(t["dy"], t["patches"], 1, 1),
             GO.gemm_gate(t["dy"], t["patches"], 1, 1, splits=plan["splits"]))
    dy = t["dy"].double()
    BO.check(f"patch_dbias_{S}_{p}_{C}_{d}", bias.grad, dy.sum(0), GO.red_gate(dy.abs().sum(0)))
    rpos = torch.zeros(n, d, dtype=torch.float64, device=dev).index_add_(0, rows, dy)
    apos = torch.zeros(n, d, dtype=torch.float64, device=dev).index_add_(0, rows, dy.abs())
    BO.check(f"patch_dpos_{S}_{p}_{C}_{d}", table.grad, rpos, GO.red_gate(apos))
    dp = patches.grad
    assert dp.shape == (M, ld) and torch.equal(dp[:, pd:], torch.zeros_like(dp[:, pd:]))
    ref_dp = t["dy"].double() @ t["w"].bfloat16().double()
    assert (dp[:, :pd].double() - ref_dp).norm().item() <= 1e-2 * ref_dp.norm().item()


def test_patchify_fn_image_gradient_at_patch_14_fp64(cuda_device):
    """PatchifyFn at patch 14: d image = scatter(dy @ W) in f32, dW / d bias / d pos as PatchEmbedFn's."""
    from test_gpu_image_grad import torch_scatter
    from x_clip_b200 import engine as E
    dev = cuda_device
    g = torch.Generator().manual_seed(14)
    B, C, S, p, d = 6, 3, 56, 14, 384
    n, pd = (S // p) ** 2, p * p * C
    img = torch.randn(B, C, S, S, generator=g).to(dev).requires_grad_(True)
    keep = torch.rand(B, n, generator=g).topk(8, dim=-1).indices.to(dev)
    index = keep.reshape(-1).to(torch.int32)
    w = ((torch.rand(d, pd, generator=g) * 2 - 1) / pd ** 0.5).to(dev).requires_grad_(True)
    b = torch.randn(d, generator=g).to(dev).requires_grad_(True)
    tbl = torch.randn(n, d, generator=g).to(dev).requires_grad_(True)
    dy = torch.randn(B * 8, d, generator=g).to(dev)
    y = E.PatchifyFn.apply(img, p, keep, index, w, b, tbl)
    y.backward(dy)
    torch.cuda.synchronize()
    rows = torch.stack([_torch_patchify(img.detach(), p)[i, keep[i]] for i in range(B)]).reshape(-1, pd)
    ref_y = rows.bfloat16().double() @ w.detach().bfloat16().double().t() + b.detach().double() \
        + tbl.detach().bfloat16().double()[index.long()]
    assert (y.double() - ref_y).abs().max().item() <= 1e-2 * ref_y.abs().max().item()
    ref_i = torch_scatter((dy.bfloat16().double() @ w.detach().bfloat16().double()), B, C, S, S, p, keep)
    rel = (img.grad.double() - ref_i).norm().item() / ref_i.norm().item()
    assert rel <= 1e-2, rel
    ref_w = dy.bfloat16().double().t() @ rows.bfloat16().double()
    assert w.grad.shape == (d, pd) and w.grad.is_contiguous()
    assert (w.grad.double() - ref_w).norm().item() <= 1e-2 * ref_w.norm().item()
    assert torch.allclose(b.grad.double(), dy.bfloat16().double().sum(0), rtol=1e-3, atol=1e-3)


# ----------------------------------------------------------------------------- CLIP end to end

CLIP_CASES = ["tiny_p14", "tiny_p14_drop", "tiny_p14_c1", "tiny_p7", "vitl14_shaped", "vitl14_336_filip"]


@pytest.mark.parametrize("case", CLIP_CASES)
def test_clip_matches_reference_at_any_patch_size(cuda_device, case):
    import test_gpu_clip_parity as P
    P.test_clip_matches_reference(cuda_device, case)


def test_image_gradient_matches_the_reference_at_patch_14(cuda_device):
    import test_gpu_image_grad as IG
    IG.test_image_gradient_matches_the_reference(cuda_device, "imggrad_p14")


def _grads(clip):
    return {k: p.grad.clone() for k, p in clip.named_parameters() if p.grad is not None}


@pytest.mark.parametrize("case,kw", [("tiny_p14", {}), ("tiny_p7", {}),
                                     ("tiny_p14", dict(use_all_token_embeds=True)),
                                     ("tiny_p14", dict(use_visual_ssl=True))])
def test_microbatched_step_equals_single_pass_at_patch_14(cuda_device, case, kw):
    """The micro-batched step (chunks re-encoded or kept, FILIP, SimSiam views) goes through the same
    padded patch embedding as the single pass: same loss and gradients, and the image gradient too."""
    from oracle import clip_oracle as O
    import x_clip_b200
    gold = json.loads((GOLD / f"{case}.json").read_text())
    cfg_kw = dict(gold["cfg"], **kw)
    cfg = O.ClipConfig(**gold["cfg"])
    state = O.protocol_state_dict(cfg, gold["weight_seed"])
    text, image = O.protocol_inputs(cfg, 6, gold["input_seed"], 0.2)
    text, image = text.to(cuda_device), image.to(cuda_device)
    res = []
    for mb, keep in ((None, 0), (2, 0), (2, 1), (4, "auto")):
        clip = x_clip_b200.CLIP(**cfg_kw, visual_patch_dropout=0., microbatch=mb,
                                microbatch_retain=keep).to(cuda_device)
        clip.load_state_dict(state, strict=False)
        clip.train()
        if kw.get("use_visual_ssl"):     # the views of both steps must be the same images
            clip.visual_ssl.augment1 = clip.visual_ssl.augment2 = torch.nn.Identity()
        torch.manual_seed(5)
        loss = clip(text, image, return_loss=True)
        loss.backward()
        res.append((loss.item(), _grads(clip)))
    for loss, grads in res[1:]:
        assert abs(loss - res[0][0]) <= 1e-5 * max(1.0, abs(res[0][0])), (loss, res[0][0])
        assert grads.keys() == res[0][1].keys()
        for k, g in grads.items():
            ref = res[0][1][k]
            assert (g - ref).norm().item() <= 2e-2 * ref.norm().item() + 1e-6, k
    if kw:
        return
    # the image gradient, single pass against micro-batched
    dimg = []
    for mb in (None, 2):
        clip = x_clip_b200.CLIP(**cfg_kw, visual_patch_dropout=0., microbatch=mb).to(cuda_device)
        clip.load_state_dict(state, strict=False)
        clip.train()
        x = image.clone().requires_grad_(True)
        clip(text, x, return_loss=True).backward()
        dimg.append(x.grad)
    assert (dimg[1] - dimg[0]).norm().item() <= 2e-2 * dimg[0].norm().item()


def test_weight_scope_keeps_padded_and_plain_casts_apart(cuda_device):
    """Inside a weight_scope the padded patch-embedding cast is cached under its own key: a later
    weight_bf16 of the same parameter still gets the unpadded [dim, patch_dim] cast."""
    from x_clip_b200 import engine as E
    w = torch.randn(256, 588, device=cuda_device)
    with E.weight_scope():
        wp = E.patch_weight_bf16(w)
        wb = E.weight_bf16(w)
        assert wp.shape == (256, 592) and wb.shape == (256, 588)
        assert E.patch_weight_bf16(w) is wp and E.weight_bf16(w) is wb
    assert torch.equal(wp[:, :588], wb)


def test_frozen_image_tower_at_patch_14(cuda_device):
    """A frozen image tower at patch 14: no gradient reaches it, the text tower trains, and an image
    that requires grad still gets its gradient through the frozen tower (input-only backward)."""
    from oracle import clip_oracle as O
    import x_clip_b200
    gold = json.loads((GOLD / "tiny_p14.json").read_text())
    cfg = O.ClipConfig(**gold["cfg"])
    text, image = O.protocol_inputs(cfg, 4, gold["input_seed"], 0.2)
    text, image = text.to(cuda_device), image.to(cuda_device)
    clip = x_clip_b200.CLIP(**gold["cfg"], visual_patch_dropout=0.).to(cuda_device)
    clip.load_state_dict(O.protocol_state_dict(cfg, gold["weight_seed"]), strict=False)
    clip.train()
    clip(text, image, return_loss=True, freeze_image_encoder=True).backward()
    assert all(p.grad is None for p in clip.visual_transformer.parameters())
    assert clip.text_transformer.token_emb.weight.grad is not None
    for p in clip.parameters():
        p.grad = None
    clip.visual_transformer.requires_grad_(False)
    x = image.clone().requires_grad_(True)
    clip(text, x, return_loss=True).backward()
    assert all(p.grad is None for p in clip.visual_transformer.parameters())
    assert x.grad is not None and torch.isfinite(x.grad).all() and x.grad.abs().sum() > 0
