"""d loss / d image on the GPU: xclip_patchify_scatter against a torch scatter, the patch-embedding
input gradient against fp64, x_clip_b200.CLIP end to end against the oracle (pinned to the reference by
tests/golden/imggrad_*.json, see tests/test_image_grad.py), the launch budget of asking / not asking for
the image gradient, the input-only backward of a frozen model, the micro-batched step and two ranks."""
import json
import os
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).parent / "golden"


# ----------------------------------------------------------------------------- kernel

def torch_scatter(src, B, C, H, W, P, keep):
    """reference result: rows back to (b, patch), dropped patches 0, then '(p1 p2 c)' -> NCHW"""
    gh, gw = H // P, W // P
    n = gh * gw
    rows = src.view(B, -1, P, P, C)
    full = torch.zeros((B, n, P, P, C), device=src.device, dtype=src.dtype)
    idx = torch.arange(n, device=src.device).expand(B, n) if keep is None else keep
    full[torch.arange(B, device=src.device)[:, None], idx] = rows
    return full.view(B, gh, gw, P, P, C).permute(0, 5, 1, 3, 2, 4).reshape(B, C, H, W)


def run_scatter(src, B, C, H, W, P, keep, out):
    from x_clip_b200 import _lib
    _lib.call("xclip_patchify_scatter", src.data_ptr(), src.stride(0), B, C, H, W, P,
              None if keep is None else keep.data_ptr(), (H // P) * (W // P) if keep is None else keep.shape[1],
              out.data_ptr(), torch.cuda.current_stream().cuda_stream)


def _keep(kind, B, n, dev, g):
    if kind == "none":
        return None
    if kind == "subset":
        return torch.rand(B, n, generator=g).topk(max(1, n // 2), dim=-1).indices.to(dev)
    if kind == "perm":
        return torch.stack([torch.randperm(n, generator=g) for _ in range(B)]).to(dev)
    return torch.randint(0, n, (B, 1), generator=g).to(dev)              # k = 1


@pytest.mark.parametrize("P", [8, 16, 32])
@pytest.mark.parametrize("C", [3, 4])
@pytest.mark.parametrize("kind", ["none", "subset", "perm", "k1"])
def test_scatter_is_a_bit_exact_torch_scatter(cuda_device, P, C, kind):
    dev = cuda_device
    g = torch.Generator().manual_seed(P * 10 + C)
    B, H, W = 3, 3 * P, 5 * P                                           # H != W
    n = (H // P) * (W // P)
    keep = _keep(kind, B, n, dev, g)
    k = n if keep is None else keep.shape[1]
    pd = P * P * C
    for lds in (pd, pd + 12):                                           # packed and strided rows
        buf = torch.randn(B * k, lds, generator=g).to(dev)
        src = buf[:, :pd]
        out = torch.full((B, C, H, W), float("nan"), device=dev)
        run_scatter(src, B, C, H, W, P, keep, out)
        ref = torch_scatter(src.contiguous(), B, C, H, W, P, keep)
        assert not torch.isnan(out).any()
        assert torch.equal(out, ref)
    from x_clip_b200 import kernels as K
    assert torch.equal(K.patchify_scatter(src.contiguous(), (B, C, H, W), P, keep), ref)


@pytest.mark.parametrize("P,C", [(16, 1), (8, 2), (6, 2), (14, 4), (4, 8)])
def test_scatter_other_channel_counts_and_patch_sizes(cuda_device, P, C):
    """C outside 1..4 or patch % 4 != 0 run the scalar variant: same result"""
    dev = cuda_device
    g = torch.Generator().manual_seed(7)
    B, H, W = 2, 2 * P, 3 * P
    n = 6
    for kind in ("none", "subset"):
        keep = _keep(kind, B, n, dev, g)
        k = n if keep is None else keep.shape[1]
        src = torch.randn(B * k, P * P * C, generator=g).to(dev)
        out = torch.full((B, C, H, W), float("nan"), device=dev)
        run_scatter(src, B, C, H, W, P, keep, out)
        assert torch.equal(out, torch_scatter(src, B, C, H, W, P, keep))


def test_scatter_inverts_the_gather_on_kept_patches(cuda_device):
    from x_clip_b200 import kernels as K
    dev = cuda_device
    img = torch.randn(4, 3, 64, 96, device=dev).bfloat16().float()    # exact in bf16: the gather is lossless
    keep = torch.rand(4, 24, device=dev).topk(12, dim=-1).indices
    back = K.patchify_scatter(K.patchify_gather(img, 16, keep).float(), img.shape, 16, keep)
    mask = K.patchify_scatter(torch.ones(48, 768, device=dev), img.shape, 16, keep)
    assert torch.equal(back, img * mask)
    assert int(mask.sum().item()) == 4 * 12 * 768


def test_scatter_refusals_launch_nothing(cuda_device):
    from x_clip_b200 import _lib
    dev = cuda_device
    lib = _lib.load()
    src = torch.zeros(64, 800, device=dev)
    out = torch.zeros(2, 3, 64, 64, device=dev)
    keep = torch.zeros(2, 1, dtype=torch.int64, device=dev)
    s = torch.cuda.current_stream().cuda_stream
    bad = [
        (src.data_ptr(), 768, 2, 3, 60, 64, 16, None, 16, out.data_ptr()),        # H % patch
        (src.data_ptr(), 768, 2, 3, 64, 56, 16, None, 16, out.data_ptr()),        # W % patch
        (src.data_ptr(), 588, 2, 3, 56, 56, 14, None, 16, out.data_ptr()),        # patch*patch*C % 8
        (src.data_ptr(), 768, 2, 3, 64, 64, 16, None, 8, out.data_ptr()),         # k != n without keep
        (src.data_ptr(), 768, 2, 3, 64, 64, 16, keep.data_ptr(), 0, out.data_ptr()),   # k = 0
        (src.data_ptr(), 768, 2, 3, 64, 64, 16, keep.data_ptr(), 17, out.data_ptr()),  # k > n
        (src.data_ptr() + 4, 768, 2, 3, 64, 64, 16, None, 16, out.data_ptr()),    # misaligned src
        (src.data_ptr(), 770, 2, 3, 64, 64, 16, None, 16, out.data_ptr()),        # lds % 4
        (src.data_ptr(), 764, 2, 3, 64, 64, 16, None, 16, out.data_ptr()),        # lds < patch_dim
        (src.data_ptr(), 768, 2, 3, 64, 64, 16, None, 16, out.data_ptr() + 8),    # misaligned output
        (None, 768, 2, 3, 64, 64, 16, None, 16, out.data_ptr()),                  # null
    ]
    torch.cuda.synchronize()
    for args in bad:
        before = lib.xclip_launch_count()
        with pytest.raises(_lib.XClipB200Error):
            _lib.call("xclip_patchify_scatter", *args, s)
        assert lib.xclip_launch_count() == before, args


# ----------------------------------------------------------------------------- patch embedding

def test_patch_embed_input_gradient_against_fp64(cuda_device):
    from x_clip_b200 import engine as E
    dev = cuda_device
    g = torch.Generator().manual_seed(3)
    M, pd, d, n = 96, 768, 384, 16
    patches = torch.randn(M, pd, generator=g).to(dev).bfloat16().requires_grad_(True)
    index = (torch.arange(M) % n).to(torch.int32).to(dev)
    w = (torch.rand(d, pd, generator=g) * 2 - 1).mul(pd ** -0.5).to(dev).requires_grad_(True)
    b = torch.randn(d, generator=g).to(dev).requires_grad_(True)
    tbl = torch.randn(n, d, generator=g).to(dev).requires_grad_(True)
    dy = torch.randn(M, d, generator=g).to(dev)
    y = E.PatchEmbedFn.apply(patches, index, w, b, tbl)
    dp, = torch.autograd.grad(y, patches, dy)
    assert dp.dtype == torch.bfloat16                              # autograd: the dtype of `patches`
    ref = dy.bfloat16().double() @ w.detach().double()
    rel = (dp.double() - ref).norm().item() / ref.norm().item()
    assert rel <= 1e-2, rel
    # through PatchifyFn the f32 GEMM output reaches the pixels unrounded: d image = scatter(dy @ W)
    from x_clip_b200 import kernels as K
    img = torch.randn(6, 3, 64, 64, generator=g).to(dev).requires_grad_(True)     # 6 x 16 patches = M rows
    keep = torch.rand(6, 16, generator=g).argsort(dim=1).to(dev)                    # all 16, permuted
    y1 = E.PatchifyFn.apply(img, 16, keep, keep.reshape(-1).to(torch.int32), w, b, tbl)
    di, = torch.autograd.grad(y1, img, dy)
    ref_i = K.patchify_scatter((dy.bfloat16().double() @ w.detach().double()).float(), img.shape, 16, keep)
    rel = (di.double() - ref_i.double()).norm().item() / ref_i.double().norm().item()
    assert rel <= 1e-2, rel
    # frozen parameters: the same input gradient, and no weight-gradient launches
    from x_clip_b200 import _lib
    lib = _lib.load()
    for t in (w, b, tbl):
        t.requires_grad_(False)
    y2 = E.PatchEmbedFn.apply(patches, index, w, b, tbl)
    torch.cuda.synchronize()
    n0 = lib.xclip_launch_count()
    dp2, = torch.autograd.grad(y2, patches, dy)
    torch.cuda.synchronize()
    assert lib.xclip_launch_count() - n0 == 1                      # the dgrad GEMM alone
    assert torch.equal(dp2, dp)


# ----------------------------------------------------------------------------- end to end

def _model(gold, dev, **kw):
    from oracle import clip_oracle as O
    import x_clip_b200
    cfg = O.ClipConfig(**gold["cfg"])
    clip = x_clip_b200.CLIP(**gold["cfg"], visual_patch_dropout=gold["patch_dropout"], **kw).to(dev)
    clip.load_state_dict(O.protocol_state_dict(cfg, gold["weight_seed"]), strict=False)
    clip.train()
    if gold.get("keep") is not None:
        clip.visual_transformer.patch_dropout.forced_keep = torch.tensor(gold["keep"])
    return cfg, clip


def _inputs(gold, cfg, dev):
    from oracle import clip_oracle as O
    text, image = O.protocol_inputs(cfg, gold["batch"], gold["input_seed"], gold["pad_fraction"])
    images = [image]
    if gold["kind"] == "multiview":
        images += [O.protocol_inputs(cfg, gold["batch"], gold["input_seed"] + gold["aug_seed_stride"] * (v + 1), 0.2)[1]
                   for v in range(len(gold["images"]) - 1)]
    return text.to(dev), [im.to(dev) for im in images]


def _objective(clip, gold, cfg, text, ims):
    if gold["kind"] == "loss":
        return clip(text, ims[0], return_loss=True)
    if gold["kind"] == "multiview":
        return clip(text, ims[0], return_loss=True, aug_image=tuple(ims[1:]))
    clip.eval()
    zi = clip(text, ims[0], return_latents=True)[1]
    target = torch.randn(gold["batch"], cfg.dim_latent, generator=torch.Generator().manual_seed(gold["target_seed"]))
    return (zi * target.to(zi.device)).sum()


@pytest.mark.parametrize("case", ["imggrad_tiny", "imggrad_tiny_drop", "imggrad_vitb16_drop",
                                  "imggrad_tiny_filip_dcl_extra", "imggrad_tiny_multiview", "imggrad_tiny_guidance"])
def test_image_gradient_matches_the_reference(cuda_device, case):
    from test_image_grad import oracle_image_grads, patch_norms
    gold = json.loads((GOLD / f"{case}.json").read_text())
    cfg, clip = _model(gold, cuda_device)
    text, ims = _inputs(gold, cfg, cuda_device)
    ims = [im.clone().requires_grad_(True) for im in ims]
    obj = _objective(clip, gold, cfg, text, ims)
    obj.backward()
    if gold["kind"] == "guidance":
        # a sum of latent . target products: bf16 latents (cosine >= 0.999 to the reference) move it by
        # up to ~|dz| |target| per sample, whatever the size of the sum itself
        t = torch.randn(gold["batch"], cfg.dim_latent, generator=torch.Generator().manual_seed(gold["target_seed"]))
        tol = 2e-3 * t.norm(dim=1).sum().item()
    else:
        tol = 1e-3 * abs(gold["loss"])
    assert abs(obj.item() - gold["loss"]) <= tol, (obj.item(), gold["loss"], tol)
    o_obj, o_grads, keep, _ = oracle_image_grads(gold)
    assert abs(o_obj - gold["loss"]) <= 3e-6 * max(1.0, abs(gold["loss"]))      # oracle == reference
    for v, (im, og, rec) in enumerate(zip(ims, o_grads, gold["images"])):
        got = im.grad.detach().cpu().double()
        og = og.double()
        for b in range(got.shape[0]):
            cos = torch.nn.functional.cosine_similarity(got[b].flatten(), og[b].flatten(), dim=0).item()
            nrel = abs(got[b].norm().item() - og[b].norm().item()) / og[b].norm().item()
            assert cos >= 0.99 and nrel <= 5e-2, (v, b, cos, nrel)
        ref_pn = torch.tensor(rec["patch_norms"], dtype=torch.float64)
        pn = patch_norms(got, cfg.visual_patch_size)
        assert (pn[ref_pn == 0] == 0).all() and (pn[ref_pn > 0] > 0).all()     # dropped patches: exactly 0


def test_frozen_image_encoder_gives_no_image_gradient(cuda_device):
    gold = json.loads((GOLD / "imggrad_tiny.json").read_text())
    assert json.loads((GOLD / "imggrad_freeze.json").read_text())["image_grad_is_none"]
    cfg, clip = _model(gold, cuda_device)
    text, ims = _inputs(gold, cfg, cuda_device)
    img = ims[0].requires_grad_(True)
    clip(text, img, return_loss=True, freeze_image_encoder=True).backward()
    assert img.grad is None


def test_return_encodings_differentiate_to_the_image(cuda_device):
    gold = json.loads((GOLD / "imggrad_tiny.json").read_text())
    cfg, clip = _model(gold, cuda_device)
    clip.eval()
    text, ims = _inputs(gold, cfg, cuda_device)
    img = ims[0].requires_grad_(True)
    _, enc_i = clip(text, img, return_encodings=True)
    enc_i[:, 0].sum().backward()
    assert img.grad is not None and torch.isfinite(img.grad).all() and img.grad.abs().sum() > 0


def test_second_order_through_the_image_raises(cuda_device):
    gold = json.loads((GOLD / "imggrad_tiny.json").read_text())
    cfg, clip = _model(gold, cuda_device)
    text, ims = _inputs(gold, cfg, cuda_device)
    img = ims[0].requires_grad_(True)
    g, = torch.autograd.grad(clip(text, img, return_loss=True), img, create_graph=True)
    with pytest.raises(RuntimeError):
        g.square().sum().backward()


def _step(clip, text, img, want_image):
    from x_clip_b200 import _lib
    lib = _lib.load()
    for p in clip.parameters():
        p.grad = None
    x = img.clone().requires_grad_(want_image)
    torch.cuda.synchronize()
    n0 = lib.xclip_launch_count()
    loss = clip(text, x, return_loss=True)
    loss.backward()
    torch.cuda.synchronize()
    n = lib.xclip_launch_count() - n0
    return loss.item(), {k: p.grad.clone() for k, p in clip.named_parameters() if p.grad is not None}, x.grad, n


def _same_up_to_run_noise(got, ref, ref2):
    """bit-identical where the step itself is reproducible, up to the summation order of the fp32
    atomics that reduce gain gradients and column sums (vsum, d bias) across blocks: that order depends
    on block scheduling, so two runs of the SAME step may differ in the last bits (ref vs ref2)"""
    if torch.equal(got, ref):
        return True
    noise = (ref2 - ref).abs().max().item()
    return (got - ref).abs().max().item() <= 2 * noise + 1e-6 * ref.abs().max().item()


def test_asking_for_the_image_gradient_changes_nothing_else(cuda_device):
    gold = json.loads((GOLD / "imggrad_tiny_drop.json").read_text())
    cfg, clip = _model(gold, cuda_device)
    text, ims = _inputs(gold, cfg, cuda_device)
    l0, g0, none, n0 = _step(clip, text, ims[0], False)
    l1, g1, _, _ = _step(clip, text, ims[0], False)
    l2, g2, dimg, n2 = _step(clip, text, ims[0], True)
    assert none is None and dimg is not None
    assert l0 == l1 == l2                       # the forward is bit-reproducible and unchanged
    assert g0.keys() == g2.keys()
    exact = 0
    for k in g0:
        assert _same_up_to_run_noise(g2[k], g0[k], g1[k]), k
        exact += torch.equal(g2[k], g0[k])
    print(f"{exact} of {len(g0)} parameter gradients bit-identical with and without the image gradient")
    # one dgrad GEMM (d patches) and one patchify_scatter for the one vision-tower call
    assert n2 - n0 == 2, (n0, n2)


def test_input_only_backward_of_a_frozen_model(cuda_device):
    from x_clip_b200 import _lib
    lib = _lib.load()
    gold = json.loads((GOLD / "imggrad_tiny_drop.json").read_text())
    cfg, clip = _model(gold, cuda_device)
    text, ims = _inputs(gold, cfg, cuda_device)
    _, _, full, n_full = _step(clip, text, ims[0], True)
    _, _, full2, _ = _step(clip, text, ims[0], True)
    for p in clip.parameters():
        p.grad = None
    clip.requires_grad_(False)
    x = ims[0].clone().requires_grad_(True)
    torch.cuda.synchronize()
    n0 = lib.xclip_launch_count()
    loss = clip(text, x, return_loss=True)
    g, = torch.autograd.grad(loss, x)
    torch.cuda.synchronize()
    n_in = lib.xclip_launch_count() - n0
    assert _same_up_to_run_noise(g, full, full2)
    assert n_full - n_in >= 4 * cfg.visual_enc_depth, (n_full, n_in)
    assert all(p.grad is None for p in clip.parameters())
    # the same with only the image tower frozen: its wgrad GEMMs are gone, the text tower still trains
    clip.requires_grad_(True)
    clip.visual_transformer.requires_grad_(False)
    _, grads, g3, n3 = _step(clip, text, ims[0], True)
    assert _same_up_to_run_noise(g3, full, full2)
    assert n_full - n3 >= 4 * cfg.visual_enc_depth, (n_full, n3)
    assert all(p.grad is None for p in clip.visual_transformer.parameters())
    assert clip.text_transformer.token_emb.weight.grad is not None


@pytest.mark.parametrize("retain", [0, 1, "auto"])
def test_microbatched_step_image_gradient(cuda_device, retain):
    from oracle import clip_oracle as O
    import x_clip_b200
    dev = cuda_device
    gold = json.loads((GOLD / "tiny_dcl_extra.json").read_text())
    cfg = O.ClipConfig(**gold["cfg"])
    state = O.protocol_state_dict(cfg, 1234)
    text, image = O.protocol_inputs(cfg, 6, 4321, 0.2)
    text, image = text.to(dev), image.to(dev)
    res = []
    for mb in (None, 2):
        clip = x_clip_b200.CLIP(**gold["cfg"], visual_patch_dropout=0., microbatch=mb,
                                microbatch_retain=retain).to(dev)
        clip.load_state_dict(state)
        clip.train()
        base = image.clone().requires_grad_(True)
        img = base * 2.0 - 1.0                                 # a non-leaf image (a generator's output)
        loss = clip(text, img, return_loss=True)
        loss.backward()
        if mb is not None:
            assert clip.last_step_plan["chunks"] == 3
        res.append((loss.item(), base.grad.clone(), clip.to_visual_latent.weight.grad.clone()))
    (l0, d0, w0), (l1, d1, w1) = res
    assert abs(l0 - l1) < 1e-5
    for b in range(6):
        assert (d1[b] - d0[b]).norm().item() <= 1e-3 * d0[b].norm().item(), b
    assert (w1 - w0).norm().item() <= 2e-2 * w0.norm().item()


def test_microbatched_step_image_gradient_under_patch_dropout(cuda_device):
    """retained and re-encoded chunks replay the same PatchDropout draw: the same image gradient, zero on
    the dropped patches of every sample"""
    from oracle import clip_oracle as O
    import x_clip_b200
    dev = cuda_device
    gold = json.loads((GOLD / "tiny_plain.json").read_text())
    cfg = O.ClipConfig(**gold["cfg"])
    text, image = O.protocol_inputs(cfg, 6, 4321, 0.2)
    text, image = text.to(dev), image.to(dev)
    clip = x_clip_b200.CLIP(**gold["cfg"], visual_patch_dropout=0.5, microbatch=2).to(dev)
    clip.load_state_dict(O.protocol_state_dict(cfg, 1234))
    clip.train()
    out = []
    for retain in (0, "auto"):
        clip.microbatch_retain = retain
        torch.manual_seed(5)
        x = image.clone().requires_grad_(True)
        clip(text, x, return_loss=True).backward()
        out.append(x.grad.clone())
    a, b = out
    assert (a - b).abs().max().item() <= 1e-3 * a.abs().max().item()
    pn = O.patchify(a.cpu(), cfg.visual_patch_size).norm(dim=-1)
    assert ((pn > 0).sum(dim=1) == 8).all()                    # 8 of 16 patches kept per sample


# ----------------------------------------------------------------------------- two ranks

def _rank_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        from oracle import clip_oracle as O
        import x_clip_b200
        gold = json.loads((GOLD / "sharded_plain.json").read_text())
        cfg = O.ClipConfig(**gold["cfg"])
        state = O.protocol_state_dict(cfg, gold["weight_seed"])
        text, image = O.protocol_inputs(cfg, world * gold["per_rank"], gold["input_seed"], gold["pad_fraction"])
        text, image = text.to(dev), image.to(dev)
        grads = []
        for sharded in (True, False):
            clip = x_clip_b200.CLIP(**gold["cfg"], visual_patch_dropout=0.).to(dev)
            clip.requires_all_gather = sharded
            clip.load_state_dict(state)
            clip.train()
            t, im = (text.chunk(world)[rank], image.chunk(world)[rank]) if sharded else (text, image)
            x = im.clone().requires_grad_(True)
            clip(t, x, return_loss=True).backward()
            grads.append(x.grad.detach().cpu())
        mine = grads[1].chunk(world)[rank]
        worst = max((grads[0][b] - mine[b]).norm().item() / mine[b].norm().item() for b in range(mine.shape[0]))
        q.put((rank, worst))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def test_two_ranks_image_gradient_is_the_rows_of_the_single_process_one():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import queue as _q
    import time as _t
    import torch.multiprocessing as mp
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_rank_worker, args=(r, world, 29831, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = []
    t0 = _t.time()
    while len(res) < world and _t.time() - t0 < 300:
        try:
            res.append(q.get(timeout=2))
        except _q.Empty:
            if any(p.exitcode not in (None, 0) for p in procs):
                break
    for p in procs:
        p.join(timeout=60)
        if p.is_alive():
            p.terminate()
    assert len(res) == world, "a rank died"
    for rank, worst in res:
        assert worst <= 1e-2, (rank, worst)
