"""The SimCLR augmentation kernels (xclip_augment_mean / _apply through SimCLRAugmentation) against
torchvision's functional ops with the same forced parameters: in float64 (every stage, order, branch,
border and size), in fp32 on the GPU (the colour stages and Normalize bit for bit), past 2^31 elements,
in memory, synchronisation and RNG use, refusals, routing, and inside SimSiam / SimCLR training steps."""
import copy
import ctypes
import itertools

import pytest
import torch

import augment_oracle as AO
from x_clip_b200 import _lib
from x_clip_b200.aux import AugmentParams, SimCLRAugmentation

pytestmark = pytest.mark.gpu

FACTORS = (1.37, 0.61, 1.52, 0.13)          # brightness, contrast, saturation, hue
# max |kernel - fp64| over max(1, max |fp64|): augment_oracle.GATE, with what was measured against it
GATE = AO.GATE


@pytest.fixture(autouse=True)
def no_tf32():
    """cuDNN's fp32 convolution (torchvision's blur) uses TF32 by default."""
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32 = prev


def _params(order=(), factors=FACTORS, gray=False, flip=False, sigma=None, crop=None, shape=None):
    if crop is None:
        crop = (0, 0, shape[-2], shape[-1])
    return AugmentParams(tuple(order), tuple(factors) if order else (None,) * 4, gray, flip, sigma, tuple(crop))


def _input(kind, shape, dev, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    if kind == "unit":
        return torch.rand(shape, device=dev, generator=g)
    return torch.randn(shape, device=dev, generator=g)


def _err64(aug, x, p):
    out = aug.apply(x, p)
    ref = aug.apply_torchvision(x.double(), p)
    assert out.dtype == torch.float32 and out.shape == ref.shape
    return ((out.double() - ref).abs().max() / ref.abs().max().clamp(min=1.0)).item()


ORDERS = list(itertools.permutations(range(4)))


@pytest.mark.parametrize("kind", ["unit", "randn"])
def test_fp64_every_jitter_order(cuda_device, kind):
    """All 24 jitter orders, with the other branches on, a crop off the borders."""
    aug = SimCLRAugmentation(48, 3)
    x = _input(kind, (3, 3, 65, 33), cuda_device)
    worst = 0.0
    for order in ORDERS:
        p = _params(order, gray=False, flip=True, sigma=1.3, crop=(9, 4, 40, 21))
        worst = max(worst, _err64(aug, x, p))
    print(f"{kind}: worst over the 24 orders {worst:.2e}")
    assert worst <= GATE


@pytest.mark.parametrize("kind", ["unit", "randn"])
def test_fp64_every_branch(cuda_device, kind):
    """Jitter, grayscale, flip and blur each on and off (16 combinations), C = 3."""
    aug = SimCLRAugmentation(40, 3)
    x = _input(kind, (2, 3, 37, 40), cuda_device, seed=1)
    worst = 0.0
    for jit, gray, flip, blur in itertools.product([False, True], repeat=4):
        p = _params((2, 0, 3, 1) if jit else (), gray=gray, flip=flip, sigma=1.8 if blur else None,
                    crop=(3, 5, 30, 33))
        e = _err64(aug, x, p)
        worst = max(worst, e)
        assert e <= GATE, (jit, gray, flip, blur, e)
    print(f"{kind}: worst over the branches {worst:.2e}")


@pytest.mark.parametrize("channels", [1, 4])
def test_fp64_other_channel_counts(cuda_device, channels):
    """C = 1 (flip and crop only) and C = 4 (flip, blur, crop): no colour stages, no Normalize."""
    aug = SimCLRAugmentation(33, channels)
    x = _input("randn", (5, channels, 33, 30), cuda_device, seed=2)
    worst = 0.0
    for flip, sigma in itertools.product([False, True], [None, 1.1]):
        if channels == 1 and sigma is not None:
            continue
        e = _err64(aug, x, _params(flip=flip, sigma=sigma, crop=(2, 1, 27, 29)))
        worst = max(worst, e)
        assert e <= GATE, (flip, sigma, e)
    print(f"C={channels}: worst {worst:.2e}")


@pytest.mark.parametrize("flip", [False, True])
def test_fp64_crops_at_every_border(cuda_device, flip):
    """Crops touching the top, bottom, left and right borders (the blur reflects there, and reads the
    real neighbours at the crop's other edges), each corner, the full-image crop and tiny crops."""
    H, W, S = 41, 52, 56
    aug = SimCLRAugmentation(S, 3)
    x = _input("unit", (2, 3, H, W), cuda_device, seed=3)
    crops = [(0, 10, 20, 25), (H - 20, 10, 20, 25), (7, 0, 20, 25), (7, W - 25, 20, 25),
             (0, 0, 13, 17), (H - 13, W - 17, 13, 17), (0, 0, H, W), (0, W - 30, H, 30),
             (5, 6, 1, 1), (H - 2, W - 3, 2, 3), (0, 0, 3, 2), (17, 22, 4, 4)]
    worst = 0.0
    for crop in crops:
        for sigma in (None, 2.0):
            p = _params((1, 3, 0, 2), gray=False, flip=flip, sigma=sigma, crop=crop)
            e = _err64(aug, x, p)
            worst = max(worst, e)
            assert e <= GATE, (crop, sigma, e)
    print(f"flip={flip}: worst over the crops {worst:.2e}")


@pytest.mark.parametrize("B,H,W,S", [(1, 33, 33, 33), (7, 65, 33, 65), (300, 33, 65, 70), (2, 2, 2, 5),
                                     (3, 130, 97, 224)])
def test_fp64_sizes_and_batches(cuda_device, B, H, W, S):
    """Odd sizes, several output tiles, batches 1 to 300; parameters from `draw` over several seeds."""
    aug = SimCLRAugmentation(S, 3)
    x = _input("unit", (B, 3, H, W), cuda_device, seed=4)
    worst = 0.0
    for seed in range(6):
        torch.manual_seed(seed)
        p = aug.draw(x.shape)
        e = _err64(aug, x, p)
        assert e <= GATE, (seed, p, e)
        e2 = _err64(aug, x, p._replace(order=(3, 1, 2, 0), factors=FACTORS, sigma=1.5))
        assert e2 <= GATE, (seed, e2)
        worst = max(worst, e, e2)
    print(f"{B}x{H}x{W} -> {S}: worst {worst:.2e}")


def _rel_max(a, b):
    return ((a - b).abs().max() / b.abs().max()).item()


@pytest.mark.parametrize("kind", ["unit", "randn"])
def test_colour_stages_match_torchvision_fp32(cuda_device, kind):
    """Blur off and the identity crop: the jitter (every order), grayscale, flip and Normalize give
    torchvision's fp32 CUDA result bit for bit when the jitter has no contrast term; with contrast, the
    per-image mean is summed in another order than torch.mean, so the result differs by a few fp32
    roundings."""
    S = 40
    aug = SimCLRAugmentation(S, 3)
    x = _input(kind, (4, 3, S, S), cuda_device, seed=5)
    no_contrast = (FACTORS[0], None, FACTORS[2], FACTORS[3])
    worst = 0.0
    for order in ORDERS:
        for gray, flip in ((False, False), (True, True)):
            p = _params(order, no_contrast, gray=gray, flip=flip, shape=x.shape)
            out, ref = aug.apply(x, p), aug.apply_torchvision(x, p)
            assert torch.equal(out, ref), (order, gray, flip, _rel_max(out, ref))
            p = _params(order, FACTORS, gray=gray, flip=flip, shape=x.shape)
            worst = max(worst, _rel_max(aug.apply(x, p), aug.apply_torchvision(x, p)))
    print(f"{kind}: with contrast, at most {worst:.2e} of the largest value from torchvision fp32")
    assert worst <= 4e-6                                 # measured 1.9e-6


def test_past_2_31_elements(cuda_device):
    """4096 x 3 x 448^2 = 2.47e9 elements: the last images (offsets past 2^31) and the first, against the
    fp64 functional reference with the same parameters."""
    S = 448
    aug = SimCLRAugmentation(S, 3)
    x = torch.rand(4096, 3, S, S, device=cuda_device)
    assert x.numel() > 2 ** 31
    p = _params((3, 1, 0, 2), gray=False, flip=True, sigma=1.7, crop=(11, 20, 400, 411))
    out = aug.apply(x, p)
    for sl in (slice(0, 2), slice(4093, 4096)):
        ref = aug.apply_torchvision(x[sl].double(), p)
        e = ((out[sl].double() - ref).abs().max() / ref.abs().max().clamp(min=1.0)).item()
        print(f"images {sl.start}-{sl.stop - 1}: {e:.2e}")
        assert e <= GATE, (sl, e)
    del x, out
    torch.cuda.empty_cache()


def test_memory_sync_and_rng(cuda_device):
    """4096 x 3 x 256^2: the peak grows by the output and at most 1 MiB more; the call never
    synchronises the host and leaves the CUDA generator alone."""
    aug = SimCLRAugmentation(256, 3)
    x = torch.rand(4096, 3, 256, 256, device=cuda_device)
    p = _params((0, 1, 2, 3), gray=True, flip=True, sigma=1.2, crop=(0, 0, 256, 256))
    aug.apply(x, p)                                    # warm-up
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated(cuda_device)
    torch.cuda.reset_peak_memory_stats(cuda_device)
    out = aug.apply(x, p)
    torch.cuda.synchronize()
    grow = torch.cuda.max_memory_allocated(cuda_device) - base
    assert grow <= out.numel() * 4 + 2 ** 20, grow
    del out
    cuda_state = torch.cuda.get_rng_state()
    torch.cuda.set_sync_debug_mode("error")
    try:
        for seed in range(8):
            torch.random.default_generator.manual_seed(seed)    # the CPU generator only
            aug(x)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert torch.equal(torch.cuda.get_rng_state(), cuda_state)


def test_refusals_launch_nothing(cuda_device):
    from x_clip_b200 import kernels as K
    lib = _lib.load()
    x = torch.rand(2, 3, 40, 40, device=cuda_device)
    base = dict(ops=(1,), factor=FACTORS, one_minus=[1 - f for f in FACTORS], crop=(0, 0, 30, 30), out_size=(32, 32))
    bad = [dict(base, crop=(0, 0, 33, 30)),               # crop taller than the output
           dict(base, crop=(0, 0, 30, 33)),               # wider
           dict(base, crop=(20, 0, 30, 30)),              # outside the image
           dict(base, crop=(0, 0, 0, 30))]
    lib.xclip_launch_count_reset()
    for kw in bad:
        with pytest.raises(_lib.XClipB200Error):
            K.augment(x, **kw)
    with pytest.raises(_lib.XClipB200Error):
        K.augment(x.to(torch.bfloat16), **base)           # not fp32
    with pytest.raises(_lib.XClipB200Error):
        K.augment(torch.rand(2, 3, 1, 40, device=cuda_device), **dict(base, crop=(0, 0, 1, 30)))
    with pytest.raises(_lib.XClipB200Error):
        K.augment(torch.rand(2, 4, 40, 40, device=cuda_device), **base)   # colour stages need C = 3
    p = _lib.AugmentParams()
    p.ops[:] = [-1] * 4
    p.top, p.left, p.height, p.width, p.out_h, p.out_w = 0, 0, 30, 30, 32, 32
    out = torch.empty(2, 3, 32, 32, device=cuda_device)
    raw = torch.empty(2 * 3 * 40 * 40 * 4 + 16, dtype=torch.uint8, device=cuda_device)
    s = torch.cuda.current_stream().cuda_stream
    pa = ctypes.addressof(p)
    assert lib.xclip_augment_apply(None, 2, 3, 40, 40, pa, None, out.data_ptr(), s) != 0
    assert lib.xclip_augment_apply(x.data_ptr(), 2, 3, 40, 40, pa, None, None, s) != 0
    assert lib.xclip_augment_apply(x.data_ptr(), 2, 3, 40, 40, None, None, out.data_ptr(), s) != 0
    assert lib.xclip_augment_apply(raw.data_ptr() + 1, 2, 3, 40, 40, pa, None, out.data_ptr(), s) != 0
    assert lib.xclip_augment_apply(x.data_ptr(), 2, 3, 40, 40, pa, None, out.data_ptr() + 2, s) != 0
    assert lib.xclip_augment_mean(x.data_ptr(), 2, 3, 40, 40, pa, None, s) != 0
    p.ops[0] = 1                                          # contrast without the mean
    assert lib.xclip_augment_apply(x.data_ptr(), 2, 3, 40, 40, pa, None, out.data_ptr(), s) != 0
    assert lib.xclip_launch_count() == 0
    p.ops[0] = -1
    assert lib.xclip_augment_apply(x.data_ptr(), 2, 3, 40, 40, pa, None, out.data_ptr(), s) == 0
    assert lib.xclip_launch_count() == 1


def test_routing(cuda_device):
    """An input that requires grad gets torchvision's result and a gradient; under no_grad it takes
    the kernels."""
    aug = SimCLRAugmentation(32, 3)
    x = torch.rand(3, 3, 30, 30, device=cuda_device)
    p = _params((0, 1, 2, 3), gray=True, flip=True, sigma=1.4, crop=(2, 3, 25, 26))
    xg = x.clone().requires_grad_(True)
    lib = _lib.load()
    lib.xclip_launch_count_reset()
    y = aug.apply(xg, p)
    assert lib.xclip_launch_count() == 0
    assert torch.equal(y, aug.apply_torchvision(xg, p))
    y.square().sum().backward()
    assert xg.grad is not None and xg.grad.abs().sum() > 0
    with torch.no_grad():
        z = aug.apply(xg, p)
    assert lib.xclip_launch_count() == 2
    assert torch.equal(z, aug.apply(x, p))
    assert (z - y.detach()).abs().max() <= 1e-5


# --------------------------------------------------------------------------- training steps

TINY = dict(dim_text=256, dim_image=256, dim_latent=256, num_text_tokens=120, text_enc_depth=2,
            text_seq_len=16, text_heads=4, visual_enc_depth=2, visual_heads=4, visual_image_size=64,
            visual_patch_size=16, visual_patch_dropout=0.0, decoupled_contrastive_learning=True,
            extra_latent_projection=True, use_visual_ssl=True)
STEPS = {"simsiam": TINY, "simclr": dict(TINY, visual_ssl_type="simclr", simclr_temperature=0.5)}


def _rel(a, b):
    d = b.double().norm().item()
    return (a.double() - b.double()).norm().item() / (d if d > 0 else 1.0)


def _seed_with_every_branch(aug, shape):
    """A seed whose two views (augment1 then augment2) take the jitter, the grayscale and the blur."""
    for seed in range(1000):
        torch.manual_seed(seed)
        p1, p2 = aug.draw(shape), aug.draw(shape)
        if (p1.order or p2.order) and (p1.sigma or p2.sigma) and (p1.grayscale or p2.grayscale):
            return seed
    raise AssertionError("no seed")


def _models(kw, dev, batch=10):
    import x_clip_b200
    torch.manual_seed(0)
    a = x_clip_b200.CLIP(**kw).to(dev)
    b = copy.deepcopy(a)
    a.train(), b.train()
    text = torch.randint(3, 120, (batch, 16), device=dev)
    image = torch.rand(batch, 3, 64, 64, device=dev)
    return a, b, text, image


def _step(m, text, image, seed):
    torch.manual_seed(seed)
    loss = m(text, image, return_loss=True)
    loss.backward()
    torch.cuda.synchronize()
    return loss.item()


def _compare(a, b, tol_grad, skip=()):
    worst = 0.0
    for (name, p), q in zip(a.named_parameters(), b.parameters()):
        assert (p.grad is None) == (q.grad is None), name
        if p.grad is not None and not any(name.endswith(k) for k in skip):
            r = _rel(q.grad, p.grad)
            worst = max(worst, r)
            assert r <= tol_grad, (name, r)
    return worst


@pytest.mark.parametrize("ssl", sorted(STEPS))
@pytest.mark.parametrize("retain", [0, "auto"])
def test_microbatched_step_equals_single_pass(cuda_device, ssl, retain):
    """The default augmentation draws the same views in both steps (one decision per call, drawn
    before any chunk): the gates of the chunked-vs-single tests."""
    single, micro, text, image = _models(STEPS[ssl], cuda_device)
    micro.microbatch, micro.microbatch_retain = 4, retain
    seed = _seed_with_every_branch(single.visual_ssl.augment1, image.shape)
    l1 = _step(single, text, image, seed)
    l2 = _step(micro, text, image, seed)
    assert micro.last_step_plan is not None and micro.last_step_plan["chunks"] == 3
    assert abs(l2 - l1) <= 1e-5 * abs(l1), (l1, l2)
    worst = _compare(single, micro, 2e-3)
    print(f"{ssl} retain={retain}: loss {l1:.6f} / {l2:.6f}, worst gradient {worst:.2e}")


@pytest.mark.parametrize("ssl", sorted(STEPS))
def test_single_pass_equals_torchvision_sequential(cuda_device, ssl):
    """The same seed with the torchvision Sequential in place of the kernels: the two views the step
    makes agree to fp32 rounding.  The loss and gradients then agree only as far as this tiny random
    model lets them: its BatchNorm heads normalise ten nearly identical CLS representations, so a
    view difference of 5e-7 moves the loss by up to 9e-4 and some gradients by up to 17 % (measured on an
    H100); the gates are about twice that."""
    ours, tv, text, image = _models(STEPS[ssl], cuda_device)
    tv.visual_ssl.augment1 = tv.visual_ssl.augment2 = AO.torchvision_augmentation(64, 3)
    views = {"ours": [], "tv": []}
    ours.visual_ssl.augment1.register_forward_hook(lambda m, i, o: views["ours"].append(o.detach().clone()))
    tv.visual_ssl.augment1.register_forward_hook(lambda m, i, o: views["tv"].append(o.detach().clone()))
    seed = _seed_with_every_branch(ours.visual_ssl.augment1, image.shape)
    l1 = _step(ours, text, image, seed)
    l2 = _step(tv, text, image, seed)
    assert len(views["ours"]) == len(views["tv"]) == 2
    dv = [_rel_max(a, b) for a, b in zip(views["ours"], views["tv"])]
    print(f"{ssl}: views differ by {dv[0]:.2e} and {dv[1]:.2e} of their largest value")
    assert max(dv) <= 1e-6, dv                           # measured 4.5e-7
    assert abs(l2 - l1) <= 2e-3 * abs(l1), (l1, l2)
    # biases whose only way to the loss runs into a BatchNorm have a zero gradient up to rounding: the
    # Linear layers in front of BatchNorm, and SimSiam's projector output (it feeds the predictor only)
    skip = ("projector.0.bias", "online_predictor.0.bias") + (("projector.3.bias",) if ssl == "simsiam" else ())
    worst = _compare(tv, ours, 0.35, skip=skip)
    print(f"{ssl}: loss {l1:.6f} / torchvision {l2:.6f}, worst gradient {worst:.2e}")
