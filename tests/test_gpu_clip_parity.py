"""End-to-end parity of x_clip_b200.CLIP on the GPU against (a) the committed golden values
produced by the reference and (b) the CPU oracle run live on the same protocol weights/inputs.

Tolerances (bf16 MMA operands/activations, fp32 accumulation/statistics/loss; compared with the
fp32 reference): loss rel-err <= 1e-3 (north star); latents cosine >= 0.999; d temperature within
1e-2 relative + 1e-3 absolute (d temperature = sum_rc g_rc*s_rc cancels O(1) terms - sum |g*s| ~
exp(temperature) ~ 2.7 - so bf16-level perturbations of the encoders move it by ~5e-4 absolute at
these 4-6 sample batches whatever its size; measured 2e-4..7e-4); global grad-norm rel <= 1e-2;
per-parameter gradient cosine >= 0.99 for every tensor with a non-negligible gradient."""
import json
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu
GOLD = Path(__file__).parent / "golden"

TINY_CASES = ["tiny_plain", "tiny_nomask", "tiny_dcl", "tiny_extra", "tiny_dcl_extra", "tiny_patchdrop",
              "tiny_filip", "tiny_filip_dcl_extra",
              # BASELINE cfg3-shaped towers at depth 2 (d_image 768, 12 heads, n = 196 / 98 image tokens,
              # 78 text tokens) and cfg4's FILIP token counts (T = 256, I = 64 / 32)
              "vitb16_shaped", "vitb16_shaped_drop", "filip_t256", "filip_t256_drop",
              # text-tower variants: rotary embedding (q, k and v), causal mask + EOS pooling
              "tiny_rotary", "tiny_causal", "text77_causal"]


def _run(case, dev):
    from oracle import clip_oracle as O
    import x_clip_b200
    gold = json.loads((GOLD / f"{case}.json").read_text())
    cfg = O.ClipConfig(**gold["cfg"])
    state = O.protocol_state_dict(cfg, gold["weight_seed"])
    text, image = O.protocol_inputs(cfg, gold["batch"], gold["input_seed"], gold["pad_fraction"])
    keep = None if gold["keep"] is None else torch.tensor(gold["keep"])

    clip = x_clip_b200.CLIP(**gold["cfg"], visual_patch_dropout=gold["patch_dropout"]).to(dev)
    missing = clip.load_state_dict(state, strict=False)
    assert not missing.unexpected_keys and all(k.endswith("inv_freq") for k in missing.missing_keys), missing
    clip.train()
    if keep is not None:
        clip.visual_transformer.patch_dropout.forced_keep = keep
    loss = clip(text.to(dev), image.to(dev), return_loss=True)
    loss.backward()
    torch.cuda.synchronize()
    grads = {k: p.grad.detach().float().cpu() for k, p in clip.named_parameters() if p.grad is not None}
    with torch.no_grad():
        lat = clip(text.to(dev), image.to(dev), return_latents=True)

    # oracle, live, fp32 CPU
    p = {k: v.clone().requires_grad_(True) for k, v in state.items()}
    o_loss = O.clip_forward(p, text, image, cfg, keep=keep)
    o_loss.backward()
    return gold, loss.item(), grads, [z.float().cpu() for z in lat], o_loss.item(), p


@pytest.mark.parametrize("case", TINY_CASES)
def test_clip_matches_reference(cuda_device, case):
    gold, loss, grads, lat, o_loss, p = _run(case, cuda_device)
    assert abs(o_loss - gold["loss"]) < 1e-5            # oracle == reference (pinned on CPU too)
    rel = abs(loss - gold["loss"]) / abs(gold["loss"])
    assert rel <= 1e-3, f"loss {loss} vs reference {gold['loss']} (rel {rel:.2e})"

    if "text_latents" in gold:
        zt_ref = torch.tensor(gold["text_latents"])
        zi_ref = torch.tensor(gold["image_latents"])
        for z, ref, name in ((lat[0], zt_ref, "text"), (lat[1], zi_ref, "image")):
            cos = torch.nn.functional.cosine_similarity(z, ref, dim=-1).min().item()
            assert cos >= 0.999, f"{name} latents cosine {cos}"
    else:       # FILIP: token-level latents [B, T, D]; the golden file keeps checksums only
        for z, ref in zip(lat, gold["latents"]):
            assert list(z.shape) == ref["shape"]
            assert abs(z.double().abs().sum().item() - ref["abs_sum"]) <= 5e-3 * ref["abs_sum"]
            head = torch.tensor(ref["head"])
            assert torch.allclose(z.flatten()[:8].double(), head.double(), atol=2e-2)

    dt = grads["temperature"].item()
    assert abs(dt - gold["dtemperature"]) <= 1e-2 * abs(gold["dtemperature"]) + 1e-3, (dt, gold["dtemperature"])
    gn = torch.sqrt(sum((g.double() ** 2).sum() for g in grads.values())).item()
    assert abs(gn - gold["grad_norm"]) <= 1e-2 * gold["grad_norm"], (gn, gold["grad_norm"])

    # a gradient the GPU step never produces (or produces where the reference has none) is a failure
    # of its own, before any per-parameter comparison below
    def has_grad(g):
        return g is not None and bool(g.ne(0).any())
    assert {k for k, g in grads.items() if has_grad(g)} == {k for k, q in p.items() if has_grad(q.grad)}

    bad = []
    for k, g in grads.items():
        og = p[k].grad
        if k == "temperature" or og is None or og.norm().item() < 1e-3 * gold["grad_norm"]:
            continue        # (temperature is a scalar: checked above with its own tolerance)
        cos = torch.nn.functional.cosine_similarity(g.flatten().double(), og.flatten().double(), dim=0).item()
        nrel = abs(g.norm().item() - og.norm().item()) / og.norm().item()
        if cos < 0.99 or nrel > 5e-2:
            bad.append((k, round(cos, 4), round(nrel, 4)))
    assert not bad, bad


def test_dtemperature_at_batch_64_meets_the_survey_gate(cuda_device):
    """SURVEY 8d gate: d loss / d temperature within 1e-2 RELATIVE, end to end.  At the 4-6 sample
    cases above the gradient is a cancellation of O(1) terms (see the module docstring); at batch 64
    it is not, and the plain relative gate holds."""
    gold, loss, grads, lat, o_loss, p = _run("tiny_b64", cuda_device)
    assert abs(loss - gold["loss"]) <= 1e-3 * abs(gold["loss"])
    dt = grads["temperature"].item()
    assert abs(dt - gold["dtemperature"]) <= 1e-2 * abs(gold["dtemperature"]), (dt, gold["dtemperature"])
    gn = torch.sqrt(sum((g.double() ** 2).sum() for g in grads.values())).item()
    assert abs(gn - gold["grad_norm"]) <= 1e-2 * gold["grad_norm"], (gn, gold["grad_norm"])


@pytest.mark.parametrize("case", ["tiny_plain", "tiny_dcl", "tiny_extra", "tiny_dcl_extra", "tiny_b64"])
def test_dtemperature_of_the_loss_kernels_in_isolation(cuda_device, case):
    """Feed the ORACLE the GPU's own latents: the similarity + InfoNCE/DCL forward/backward kernels
    (EPI_NCE_FWD / EPI_NCE_BWD) are then compared without any encoder noise.  Loss rel <= 1e-5,
    d temperature rel <= 1e-3 (+1e-6 abs; fp32 sum of g*s inside the kernel), latent gradients rel
    <= 1e-2 (they are dZ = bf16(g) @ bf16(Z): two bf16 operand roundings, ~2^-8 each)."""
    from oracle import clip_oracle as O
    import x_clip_b200
    gold = json.loads((GOLD / f"{case}.json").read_text())
    cfg = O.ClipConfig(**gold["cfg"])
    state = O.protocol_state_dict(cfg, gold["weight_seed"])
    text, image = O.protocol_inputs(cfg, gold["batch"], gold["input_seed"], gold["pad_fraction"])
    clip = x_clip_b200.CLIP(**gold["cfg"], visual_patch_dropout=0.).to(cuda_device)
    clip.load_state_dict(state)
    clip.train()
    lat = clip(text.to(cuda_device), image.to(cuda_device), return_latents=True)
    lat = [z.detach().requires_grad_(True) for z in lat]
    if len(lat) == 2:
        lat = lat + lat
    ops = []
    from x_clip_b200 import kernels as K
    for z in (lat if cfg.extra_latent_projection else lat[:2]):
        # the split-bf16 operands of exactly these fp32 latents (what ProjectL2NormFn hands the loss)
        hi = z.detach().to(torch.bfloat16)
        lo = (z.detach() - hi.float()).to(torch.bfloat16)
        ops.append((torch.cat([hi, lo, hi], 1).contiguous(), torch.cat([hi, hi, lo], 1).contiguous()))
    temp = clip.temperature.detach().clone().requires_grad_(True)
    from x_clip_b200 import engine as E
    loss = E.ContrastiveLossFn.apply(lat[0], lat[1], lat[2] if cfg.extra_latent_projection else None,
                                     lat[3] if cfg.extra_latent_projection else None, temp, tuple(ops),
                                     cfg.decoupled_contrastive_learning, False)
    loss.backward()
    zc = [z.detach().cpu().double().requires_grad_(True) for z in lat]
    tc = temp.detach().cpu().double().requires_grad_(True)
    ref = O.contrastive_loss(zc[0], zc[1], zc[2], zc[3], tc, cfg)
    ref.backward()
    assert abs(loss.item() - ref.item()) <= 1e-5 * abs(ref.item()), (loss.item(), ref.item())
    assert abs(temp.grad.item() - tc.grad.item()) <= 1e-3 * abs(tc.grad.item()) + 1e-6, (temp.grad.item(), tc.grad.item())
    n = 4 if cfg.extra_latent_projection else 2
    for j in range(n):
        g, r = lat[j].grad.cpu().double(), zc[j].grad
        if n == 2 and zc[j + 2].grad is not None:   # zt_x/zi_x ARE zt/zi here: gradients add up
            r = zc[j].grad + zc[j + 2].grad
        assert (g - r).norm().item() <= 1e-2 * r.norm().item() + 1e-9, (j, (g - r).norm().item(), r.norm().item())


def test_readme_config_matches_reference(cuda_device):
    """cfg1 (README model, B=4): the configuration the reference itself can run on CPU."""
    gold, loss, grads, lat, o_loss, p = _run("readme_plain", cuda_device)
    rel = abs(loss - gold["loss"]) / abs(gold["loss"])
    assert rel <= 1e-3, f"loss {loss} vs {gold['loss']} rel {rel:.2e}"
    gn = torch.sqrt(sum((g.double() ** 2).sum() for g in grads.values())).item()
    assert abs(gn - gold["grad_norm"]) <= 1e-2 * gold["grad_norm"], (gn, gold["grad_norm"])
    dt = grads["temperature"].item()
    assert abs(dt - gold["dtemperature"]) <= 1e-2 * abs(gold["dtemperature"]) + 1e-3   # see module docstring


def test_state_dict_roundtrip_and_early_returns(cuda_device):
    from oracle import clip_oracle as O
    import x_clip_b200
    gold = json.loads((GOLD / "tiny_extra.json").read_text())
    cfg = O.ClipConfig(**gold["cfg"])
    clip = x_clip_b200.CLIP(**gold["cfg"], visual_patch_dropout=0.).to(cuda_device)
    assert set(clip.state_dict().keys()) == set(O.param_shapes(cfg).keys())
    for k, v in clip.state_dict().items():
        assert tuple(v.shape) == O.param_shapes(cfg)[k], k
    clip.load_state_dict(O.protocol_state_dict(cfg, 1234))
    text, image = O.protocol_inputs(cfg, 4, 4321, 0.1)
    text, image = text.to(cuda_device), image.to(cuda_device)
    clip.eval()
    with torch.no_grad():
        et, ei = clip(text, image, return_encodings=True)
        assert et.shape == (4, cfg.text_seq_len + 1, cfg.dim_text) and ei.shape[0] == 4
        lat = clip(text, image, return_latents=True)
        assert len(lat) == 4 and lat[0].shape == (4, cfg.dim_latent)
        sim = clip(text, image)
        assert sim.shape == (4,)
        sim2 = clip(text, image, text_to_image=False)
        assert sim2.shape == (4,)
    with pytest.raises(AssertionError):
        clip(text, image, return_loss=True)        # loss while .eval(), reference x_clip.py:651


def test_weight_cache_not_confused_by_recycled_parameters(cuda_device):
    """Two models built one after the other with different weights must not share bf16 shadows
    (parameter ids / storage can be recycled by Python and the caching allocator)."""
    from oracle import clip_oracle as O
    import x_clip_b200
    gold = json.loads((GOLD / "tiny_plain.json").read_text())
    cfg = O.ClipConfig(**gold["cfg"])
    text, image = O.protocol_inputs(cfg, 4, 4321, 0.1)
    text, image = text.to(cuda_device), image.to(cuda_device)
    losses = []
    for seed in (1, 2, 1):
        clip = x_clip_b200.CLIP(**gold["cfg"], visual_patch_dropout=0.).to(cuda_device)
        clip.load_state_dict(O.protocol_state_dict(cfg, seed))
        clip.train()
        losses.append(clip(text, image, return_loss=True).item())
        del clip
    assert abs(losses[0] - losses[2]) < 1e-6
    assert abs(losses[0] - losses[1]) > 1e-4


def test_microbatched_step_equals_single_pass(cuda_device):
    """The GradCache-style chunked step (engine.ChunkedClipLossFn) is the same function as the
    single-pass step: identical loss and gradients (up to bf16 accumulation-order noise)."""
    from oracle import clip_oracle as O
    import x_clip_b200
    gold = json.loads((GOLD / "tiny_dcl_extra.json").read_text())
    cfg = O.ClipConfig(**gold["cfg"])
    state = O.protocol_state_dict(cfg, 1234)
    text, image = O.protocol_inputs(cfg, 6, 4321, 0.2)
    text, image = text.to(cuda_device), image.to(cuda_device)
    res = []
    # (micro-batch, retained chunks): none kept = pure two-pass step, some / all kept, planner
    for mb, keep in ((None, 0), (2, 0), (4, 0), (2, 1), (2, 3), (2, "auto")):
        clip = x_clip_b200.CLIP(**gold["cfg"], visual_patch_dropout=0., microbatch=mb,
                                microbatch_retain=keep).to(cuda_device)
        clip.load_state_dict(state)
        clip.train()
        loss = clip(text, image, return_loss=True)
        loss.backward()
        if mb is not None:
            plan = clip.last_step_plan
            want = {0: 0, 1: 1, 3: 3, "auto": plan["chunks"]}[keep]       # tiny model: everything fits
            assert plan["retained"] == want and plan["chunks"] == -(-6 // mb), plan
        res.append((loss.item(), {k: p.grad.clone() for k, p in clip.named_parameters() if p.grad is not None}))
    for loss, grads in res[1:]:
        assert abs(loss - res[0][0]) < 1e-5
        assert grads.keys() == res[0][1].keys()
        for k, g in grads.items():
            ref = res[0][1][k]
            assert (g - ref).norm().item() <= 2e-2 * ref.norm().item() + 1e-6, k

    # with patch dropout the per-chunk RNG is replayed in the recompute pass: deterministic, finite
    # (same draw whether a chunk's activations were kept or it is re-encoded: retain 0 / 1 / all agree)
    clip = x_clip_b200.CLIP(**gold["cfg"], visual_patch_dropout=0.5, microbatch=2).to(cuda_device)
    clip.load_state_dict(state)
    clip.train()
    out = []
    for keep in (0, 0, 1, "auto", "auto"):      # (the second "auto" step repeats the remembered plan)
        clip.microbatch_retain = keep
        torch.manual_seed(7)
        for p in clip.parameters():
            p.grad = None
        loss = clip(text, image, return_loss=True)
        loss.backward()
        out.append((loss.item(), clip.to_visual_latent.weight.grad.clone()))
    for o in out[1:]:
        assert out[0][0] == o[0] and torch.isfinite(o[1]).all()      # the forward is bit-reproducible
        assert (out[0][1] - o[1]).abs().max().item() <= 1e-3 * out[0][1].abs().max().item()


def test_microbatched_step_survives_an_out_of_memory_retained_chunk(cuda_device):
    """If keeping a chunk's activations runs out of memory (a fragmented allocator cache, memory taken by
    someone else since the plan was made) the step must fall back to re-encoding that chunk and the later
    ones - same loss, same gradients, same PatchDropout draw - and remember the smaller plan."""
    from oracle import clip_oracle as O
    import x_clip_b200
    gold = json.loads((GOLD / "tiny_dcl_extra.json").read_text())
    cfg = O.ClipConfig(**gold["cfg"])
    state = O.protocol_state_dict(cfg, 1234)
    text, image = O.protocol_inputs(cfg, 6, 4321, 0.2)
    text, image = text.to(cuda_device), image.to(cuda_device)
    clip = x_clip_b200.CLIP(**gold["cfg"], visual_patch_dropout=0.5, microbatch=2).to(cuda_device)
    clip.load_state_dict(state)
    clip.train()

    def step():
        torch.manual_seed(11)
        for p in clip.parameters():
            p.grad = None
        loss = clip(text, image, return_loss=True)
        loss.backward()
        return loss.item(), clip.to_visual_latent.weight.grad.clone(), clip.text_transformer.token_emb.weight.grad.clone()

    ref = step()                                       # all three chunks resident
    assert clip.last_step_plan["retained"] == 3 and clip.last_step_plan["oom_fallbacks"] == 0
    real = clip._encode_to_latents
    calls = {"n": 0}

    def flaky(*a, **k):
        calls["n"] += 1
        if calls["n"] == 2 and torch.is_grad_enabled():   # the second chunk's retained encode "runs out of memory"
            raise torch.OutOfMemoryError("injected by the test")
        return real(*a, **k)

    clip._encode_to_latents = flaky
    try:
        got = step()
    finally:
        clip._encode_to_latents = real
    plan = clip.last_step_plan
    assert plan["oom_fallbacks"] == 1 and plan["retained"] == 1, plan
    assert got[0] == ref[0]
    for a, b in zip(got[1:], ref[1:]):
        assert (a - b).abs().max().item() <= 1e-3 * b.abs().max().item() + 1e-7
    again = step()                                     # the smaller plan is remembered
    assert clip.last_step_plan["retained"] == 1 and clip.last_step_plan["oom_fallbacks"] == 0
    assert again[0] == ref[0]


def test_pluggable_encoders_freeze_and_maskless(cuda_device):
    """Hooks of the reference surface (x_clip.py:482-483, 501-502, 604-605, 659-660): foreign
    encoders returning [B,n,d] / [B,d], freeze_* flags, text_encode_without_mask."""
    from oracle import clip_oracle as O
    import x_clip_b200
    dev = cuda_device
    gold = json.loads((GOLD / "tiny_plain.json").read_text())
    cfg = O.ClipConfig(**gold["cfg"])
    text, image = O.protocol_inputs(cfg, 4, 4321, 0.2)
    text, image = text.to(dev), image.to(dev)

    class TextEnc(torch.nn.Module):                 # returns [B, 1+n, d], CLS at index 0
        def __init__(self):
            super().__init__()
            self.emb = torch.nn.Embedding(128, 256)
        def forward(self, ids, mask=None):
            h = self.emb(ids)
            return torch.cat((h.mean(1, keepdim=True), h), dim=1)

    class ImageEnc(torch.nn.Module):                # returns [B, d]
        def __init__(self):
            super().__init__()
            self.lin = torch.nn.Linear(3 * 64 * 64, 256)
        def forward(self, img):
            return self.lin(img.flatten(1))

    torch.manual_seed(0)
    clip = x_clip_b200.CLIP(**gold["cfg"], text_encoder=TextEnc(), image_encoder=ImageEnc()).to(dev)
    clip.train()
    loss = clip(text, image, return_loss=True)
    loss.backward()
    assert torch.isfinite(loss) and clip.text_transformer.emb.weight.grad.abs().sum() > 0
    assert clip.visual_transformer.lin.weight.grad.abs().sum() > 0
    # reference semantics of the same head on the same encodings (fp32 torch)
    with torch.no_grad():
        et, ei = clip(text, image, return_encodings=True)
        zt = torch.nn.functional.normalize(et[:, 0] @ clip.to_text_latent.weight.t(), dim=-1)
        zi = torch.nn.functional.normalize(ei @ clip.to_visual_latent.weight.t(), dim=-1)
        ref = O.contrastive_loss(zt.cpu(), zi.cpu(), zt.cpu(), zi.cpu(), clip.temperature.detach().cpu(), cfg)
    assert abs(loss.item() - ref.item()) <= 2e-3 * abs(ref.item())

    # freeze flags: no gradient reaches the frozen tower
    clip2 = x_clip_b200.CLIP(**gold["cfg"], visual_patch_dropout=0.).to(dev)
    clip2.load_state_dict(O.protocol_state_dict(cfg, 1234))
    clip2.train()
    l2 = clip2(text, image, return_loss=True, freeze_image_encoder=True)
    l2.backward()
    assert all(p.grad is None for p in clip2.visual_transformer.parameters())
    assert clip2.text_transformer.token_emb.weight.grad is not None
    assert clip2.to_visual_latent.weight.grad is not None

    # text_encode_without_mask: pads are attended like any token -> equals an all-True mask
    clip3 = x_clip_b200.CLIP(**gold["cfg"], visual_patch_dropout=0., text_encode_without_mask=True).to(dev)
    clip3.load_state_dict(O.protocol_state_dict(cfg, 1234))
    clip3.train()
    l3 = clip3(text, image, return_loss=True)
    p = {k: v.clone() for k, v in O.protocol_state_dict(cfg, 1234).items()}
    with torch.no_grad():
        tcpu, icpu = text.cpu(), image.cpu()
        enc_t = O.encode_text(tcpu, torch.ones_like(tcpu, dtype=torch.bool), p, cfg)
        enc_i = O.encode_image(icpu, p, cfg)
        z = O.project_latents(enc_t, enc_i, p, cfg)
        ref3 = O.contrastive_loss(*z, p["temperature"], cfg)
    assert abs(l3.item() - ref3.item()) <= 1e-3 * abs(ref3.item())
