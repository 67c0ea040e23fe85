"""Attention dropout (xclip_attn_dropout_fwd / _bwd, engine.TransformerFn with `drop`) on the GPU.

- The kernels against attn_oracle's fp64 reference fed dropout_oracle's numpy mask, with attn_oracle's
  per-element gates (the multiplier M / (1 - p) enters wherever P meets V or dP).
- The mask itself read out exactly: with q = k = 0 every probability of an n = 64 row is 1/64, so with
  V = I the forward's o[i, j] = M_ij / (64 (1 - p)), and with dO = I the backward's dv[j, i] is the same.
- Statistics: the keep rate, the unbiased mean of o over 256 seeds, p = 1.
- Switched off: p = 0 through the dropout entry, and eval() / p = 0 modules, equal the plain path bit
  for bit.
- The encoder against block_oracle in fp64 with the masks, and whole CLIP steps: reproducibility
  under torch.manual_seed and the micro-batched step's RNG replay.
"""
import numpy as np
import pytest
import torch

import attn_oracle as AO
import block_oracle as BO
import dropout_oracle as DO

pytestmark = pytest.mark.gpu

ATTN_STREAM = 5     # XCLIP_TUNE_ATTN_STREAM (include/xclip_b200.h)
SCALE = 64 ** -0.5
SEED = -6917529027641081857     # a key with both 32-bit words non-zero


def _seed(seed, dev):
    return torch.tensor([seed], dtype=torch.int64, device=dev)


def _run(case, B, n, H, causal, p, seed, layer=0, bwd=True):
    from x_clip_b200 import kernels as K
    dr = None if p is None else (p, _seed(seed, case["qkv"].device), layer)
    o, lse = K.attn_fwd(case["qkv"], case["mask"], B, n, H, SCALE, causal, dropout=dr)
    dqkv = K.attn_bwd(case["qkv"], case["mask"], o, case["d_o"], lse, B, n, H, SCALE, causal, dropout=dr) \
        if bwd else None
    torch.cuda.synchronize()
    return o, lse, dqkv


def _forced(mode, fn):
    if mode != "forced":
        return fn()
    from x_clip_b200 import _lib
    lib = _lib.load()
    prev = lib.xclip_tune_set(ATTN_STREAM, 1)
    try:
        return fn()
    finally:
        lib.xclip_tune_set(ATTN_STREAM, prev)


def _check(tag, case, B, n, H, causal, o, lse, dqkv, drop):
    ref = DO.attn_dropout_ref64(case["qkv"], case["mask"], B, n, H, SCALE, causal, drop, o, case["d_o"])
    BO.check(f"drop o {tag}", o, ref["o"], ref["g_o"])
    BO.check(f"drop lse {tag}", lse, ref["lse"], ref["g_lse"])
    inner = H * 64
    for name, sl in (("dq", slice(0, inner)), ("dk", slice(inner, 2 * inner)), ("dv", slice(2 * inner, 3 * inner))):
        BO.check(f"drop {name} {tag}", dqkv[:, sl], ref["dqkv"][:, sl], ref["g_dqkv"][:, sl])


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("n", [1, 17, 64, 78, 99, 128, 320, 321, 577])
def test_attn_dropout_fp64(cuda_device, n, causal):
    """Every tail width and both schedules (n > 320 streams; n <= 320 also forced to), key-masked rows
    and rows with no visible key (no_visible recipe: the per-key dropped 1/n of their dv), p = 0.1 at
    layer 0 and p = 0.5 at layer 3."""
    B, H = 3, 2
    case = AO.attn_case("no_visible", B, n, H, causal=causal, seed=11, device=cuda_device)
    for p, layer in ((0.1, 0), (0.5, 3)):
        drop = DO.attn_drop_mul(SEED, B, H, n, layer, p, cuda_device)
        for mode in ("resident", "forced") if n <= 320 else ("streaming",):
            out = _forced(mode, lambda: _run(case, B, n, H, causal, p, SEED, layer))
            _check(f"n{n} causal{int(causal)} p{p} {mode}", case, B, n, H, causal, *out, drop)


@pytest.mark.parametrize("recipe", ["flat", "peaked", "block_masked"])
def test_attn_dropout_recipes(cuda_device, recipe):
    B, n, H = 3, 257, 2
    case = AO.attn_case(recipe, B, n, H, seed=12, device=cuda_device)
    drop = DO.attn_drop_mul(SEED + 1, B, H, n, 1, 0.2, cuda_device)
    _check(recipe, case, B, n, H, False, *_run(case, B, n, H, False, 0.2, SEED + 1, 1), drop)


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("n", [78, 257])
def test_attn_dropout_schedules_agree(cuda_device, n, causal):
    """Resident and streaming kernels give the same bits with dropout on."""
    B, H = 4, 3
    case = AO.attn_case("no_visible", B, n, H, causal=causal, seed=13, device=cuda_device)
    a = _run(case, B, n, H, causal, 0.3, SEED, 2)
    b = _forced("forced", lambda: _run(case, B, n, H, causal, 0.3, SEED, 2))
    for x, y in zip(a, b):
        assert torch.equal(x, y)


def _readout_case(B, H, dev):
    """q = k = 0, V = I per head (n = 64) and dO = I per head."""
    n = 64
    eye = torch.eye(64).repeat(1, H)                                   # [64, H 64]
    qkv = torch.zeros(B, n, 3 * H * 64)
    qkv[:, :, 2 * H * 64:] = eye
    d_o = eye.expand(B, n, H * 64).reshape(B * n, H * 64)
    return dict(qkv=qkv.reshape(B * n, -1).bfloat16().to(dev), mask=None, d_o=d_o.bfloat16().to(dev))


@pytest.mark.parametrize("p", [0.1, 0.5, 0.9])
def test_attn_dropout_mask_readout(cuda_device, p):
    """The kernels' masks equal the numpy restatement bit for bit (forward and dK / dV kernels, over
    12.6 M elements), the keep rate is within 5 sigma of 1 - p, and layers and seeds differ."""
    B, H, n = 256, 12, 64
    case = _readout_case(B, H, cuda_device)
    o, _, dqkv = _run(case, B, n, H, False, p, SEED, 0)
    fwd = (o.view(B, n, H, 64) != 0).permute(0, 2, 1, 3).cpu().numpy()         # [B, H, i, j]
    dv = dqkv[:, 2 * H * 64:].view(B, n, H, 64)                                 # [B, j, H, i]
    bwd = (dv != 0).permute(0, 2, 3, 1).cpu().numpy()                          # [B, H, i, j]
    want = DO.attn_keep(SEED, B, H, n, 0, p)
    assert np.array_equal(fwd, want)
    assert np.array_equal(bwd, want)
    kept = o.float().max().item() * 64 * (1 - np.float32(p))
    assert abs(kept - 1.0) < 1e-2, "kept probabilities carry 1 / (1 - p)"
    rate, N = fwd.mean(), fwd.size
    sd = (p * (1 - p) / N) ** 0.5
    print(f"GATE drop_keep_rate[p{p}] {abs(rate - (1 - p)) / (5 * sd):.4f}")
    assert N >= 1e7 and abs(rate - (1 - p)) <= 5 * sd
    for seed, layer in ((SEED, 1), (SEED + 1, 0)):
        o2, _, _ = _run(case, B, n, H, False, p, seed, layer, bwd=False)
        other = (o2.view(B, n, H, 64) != 0).permute(0, 2, 1, 3).cpu().numpy()
        assert np.array_equal(other, DO.attn_keep(seed, B, H, n, layer, p))
        assert (other != fwd).mean() > p * (1 - p)


def test_attn_dropout_unbiased(cuda_device):
    """The mean of o over 256 seeds lies within 6 standard errors (plus two bf16 roundings) of the p = 0
    kernel's o in every one of the 20 k elements: the kernel's dropout is unbiased."""
    B, n, H, p = 2, 78, 2, 0.1
    case = AO.attn_case("flat", B, n, H, seed=14, device=cuda_device)
    ref = _run(case, B, n, H, False, None, 0, bwd=False)[0].double()
    acc = torch.zeros_like(ref)
    acc2 = torch.zeros_like(ref)
    S = 256
    for s in range(S):
        o, _, _ = _run(case, B, n, H, False, p, 1000 + s, bwd=False)
        acc += o.double()
        acc2 += o.double() ** 2
    mean = acc / S
    se = ((acc2 / S - mean ** 2).clamp_min(0) / (S - 1)).sqrt()
    z = (mean - ref).abs() / (se + 2.0 ** -8 * ref.abs() + 1e-6)
    print(f"GATE drop_unbiased {z.max().item() / 6:.4f}")
    assert z.max().item() <= 6.0


def test_attn_dropout_p1_and_p0(cuda_device):
    """p = 1: o and every gradient are 0, lse is the undropped one.  p = 0 through the dropout entry
    gives the plain kernels' bits."""
    B, n, H = 3, 99, 4
    case = AO.attn_case("flat", B, n, H, seed=15, device=cuda_device)
    plain = _run(case, B, n, H, True, None, 0)
    o1, lse1, d1 = _run(case, B, n, H, True, 1.0, SEED)
    assert (o1 == 0).all() and (d1 == 0).all() and torch.equal(lse1, plain[1])
    for x, y in zip(_run(case, B, n, H, True, 0.0, SEED), plain):
        assert torch.equal(x, y)


def test_attn_dropout_refuses_bad_arguments(cuda_device):
    from x_clip_b200 import _lib
    lib = _lib.load()
    B, n, H = 2, 33, 2
    case = AO.attn_case("flat", B, n, H, device=cuda_device)
    o = torch.empty(B * n, H * 64, device=cuda_device, dtype=torch.bfloat16)
    lse = torch.empty(B, H, n, device=cuda_device)
    seed = torch.zeros(2, dtype=torch.int64, device=cuda_device)
    stream = torch.cuda.current_stream().cuda_stream
    args = (case["qkv"].data_ptr(), 3 * H * 64, None, o.data_ptr(), H * 64, lse.data_ptr(), B, n, H, SCALE, 0)
    for p, sp, layer in ((-0.1, seed.data_ptr(), 0), (1.5, seed.data_ptr(), 0), (float("nan"), seed.data_ptr(), 0),
                         (0.1, None, 0), (0.1, seed.data_ptr() + 4, 0), (0.1, seed.data_ptr(), -1)):
        n0 = lib.xclip_launch_count()
        assert lib.xclip_attn_dropout_fwd(*args, p, sp, layer, stream) == 1
        assert lib.xclip_launch_count() == n0
    assert lib.xclip_attn_dropout_fwd(*args, 0.1, seed.data_ptr(), 0, stream) == 0
    torch.cuda.synchronize()


@pytest.mark.parametrize("name", ["d512_mask_causal", "d768_n197"])
def test_transformer_dropout_fp64(cuda_device, name):
    """TransformerFn with dropout (depth 2, p = 0.1) against fp64 autograd of the reference block with the
    numpy masks of layers 0 and 1, under BLOCK_GATES."""
    from x_clip_b200 import engine as E
    case = BO.block_case(name, device=cuda_device)
    B, n, _ = case["x"].shape
    H = case["heads"]
    ws = [w.clone().requires_grad_(True) for w in case["weights"]]
    x = case["x"].clone().requires_grad_(True)
    cos, sin = case["rot"] if case["rot"] is not None else (None, None)
    drop = ((0.1, 0.1), _seed(SEED, cuda_device))
    out = E.TransformerFn.apply(x, case["mask"], H, BO.BLOCK_DEPTH, case["causal"], cos, sin, True, drop, *ws)
    out.backward(case["dout"])
    torch.cuda.synchronize()
    masks = [DO.attn_drop_mul(SEED, B, H, n, L, 0.1, cuda_device) for L in range(BO.BLOCK_DEPTH)]
    xr = case["x"].double().requires_grad_(True)
    wr = [w.double().requires_grad_(True) for w in case["weights"]]
    ref = DO.transformer_stack_dropout(xr, wr, BO.BLOCK_DEPTH, H, case["mask"], case["causal"], case["rot"], masks)
    ref.backward(case["dout"].double())
    undropped = BO.transformer_stack(case["x"].double(), [w.double() for w in case["weights"]], BO.BLOCK_DEPTH, H,
                                     case["mask"], case["causal"], case["rot"])
    assert BO.rel_fro(undropped, ref.detach()) > 5 * BO.BLOCK_GATES["out"], "the masks must matter"
    names = BO.flat_names(BO.BLOCK_DEPTH)
    pairs = [("out", out.detach(), ref.detach()), ("dx", x.grad, xr.grad)] + \
        list(zip(names, [w.grad for w in ws], [w.grad for w in wr]))
    for nm, got, want in pairs:
        gate = BO.BLOCK_GATES[nm.split(".")[0]]
        rel = BO.rel_fro(got, want)
        print(f"GATE drop_block_{nm}[{name}] {rel / gate:.4f}")
        assert rel <= gate, (nm, rel, gate)


# ---------------------------------------------------------------------------- whole CLIP steps

TINY = dict(dim_text=256, dim_image=256, dim_latent=256, num_text_tokens=128, text_enc_depth=2,
            text_seq_len=16, text_heads=4, visual_enc_depth=2, visual_heads=4,
            visual_image_size=64, visual_patch_size=16)


def _clip(dev, causal=False, p=0.1, microbatch=None, retain="auto"):
    import x_clip_b200
    torch.manual_seed(1)
    text = x_clip_b200.TextTransformer(256, num_tokens=128, max_seq_len=16, dim_head=64, depth=2, heads=4,
                                       causal=causal, attn_dropout=p, ff_dropout=p)
    image = x_clip_b200.VisionTransformer(256, image_size=64, patch_size=16, channels=3, dim_head=64, depth=2,
                                          heads=4, patch_dropout=0.5, attn_dropout=p, ff_dropout=p)
    clip = x_clip_b200.CLIP(**TINY, text_causal_mask=causal, text_eos_id=127 if causal else None, text_encoder=text,
                            image_encoder=image, microbatch=microbatch, microbatch_retain=retain).to(dev)
    clip.train()
    return clip


def _batch(dev, B=12):
    g = torch.Generator().manual_seed(5)
    text = torch.randint(1, 127, (B, 16), generator=g)
    text[:, -1] = 127                    # the EOS token of the causal configuration
    for b in range(B):
        text[b, :b % 5] = 0              # left padding: causal rows before the first token see no key
    return text.to(dev), torch.randn(B, 3, 64, 64, generator=g).to(dev)


def _step(clip, text, image, seed):
    clip.zero_grad(set_to_none=True)
    torch.manual_seed(seed)
    loss = clip(text, image, return_loss=True)
    loss.backward()
    torch.cuda.synchronize()
    return loss.detach().clone(), {k: p.grad.clone() for k, p in clip.named_parameters() if p.grad is not None}


def _grad_rel(a, b):
    return max(BO.rel_fro(a[k], b[k]) for k in a)


@pytest.mark.parametrize("causal", [False, True])
def test_clip_dropout_reproducible(cuda_device, causal):
    """Two steps after the same torch.manual_seed give the same loss bit for bit and the same gradients
    up to the run-to-run noise of the fp32 atomics; another seed draws other masks."""
    clip = _clip(cuda_device, causal)
    text, image = _batch(cuda_device)
    l1, g1 = _step(clip, text, image, 0)
    l2, g2 = _step(clip, text, image, 0)
    l3, g3 = _step(clip, text, image, 1)
    assert torch.equal(l1, l2) and set(g1) == set(g2)
    assert _grad_rel(g1, g2) <= 1e-5
    assert l1 != l3 and _grad_rel(g1, g3) > 1e-2


def test_clip_dropout_off_is_the_plain_path(cuda_device):
    """eval() with attn_dropout = 0.1, and train() with attn_dropout = 0, run the plain kernels: equal
    outputs bit for bit, and no draw from the CUDA generator."""
    a = _clip(cuda_device, p=0.1)
    b = _clip(cuda_device, p=0.0)
    b.load_state_dict(a.state_dict())
    text, image = _batch(cuda_device)
    mask = text != 0
    a.text_transformer.eval()
    b.text_transformer.train()
    with torch.no_grad():
        s0 = torch.cuda.get_rng_state()
        ea, eb = a.text_transformer(text, mask=mask), b.text_transformer(text, mask=mask)
        assert torch.equal(s0, torch.cuda.get_rng_state())
        a.text_transformer.train()
        ed = a.text_transformer(text, mask=mask)      # dropout on under no_grad, like nn.Dropout
    assert torch.equal(ea, eb)
    assert not torch.equal(ea, ed)


@pytest.mark.parametrize("causal", [False, True])
def test_clip_dropout_microbatch_replay(cuda_device, causal):
    """Micro-batched with no chunk retained (every chunk re-encoded in backward) and with every chunk
    retained: the same loss and gradients, so a re-encoded chunk draws its first-sweep masks."""
    text, image = _batch(cuda_device)
    runs = []
    for retain in (0, 3):
        clip = _clip(cuda_device, causal, microbatch=4, retain=retain)
        runs.append(_step(clip, text, image, 0))
        assert clip.last_step_plan["chunks"] == 3 and clip.last_step_plan["retained"] == retain
    (l0, g0), (l1, g1) = runs
    assert abs(l0.item() - l1.item()) <= 1e-6 * abs(l1.item())
    assert set(g0) == set(g1) and _grad_rel(g0, g1) <= 1e-5
    clip = _clip(cuda_device, causal, microbatch=4, retain=0)
    clip.text_transformer.transformer.forced_dropout_seed = 99    # the forward's and backward's masks now
    l2, g2 = _step(clip, text, image, 0)                          # differ from the drawn ones
    assert _grad_rel(g0, g2) > 1e-2
