"""FILIP models at token counts that are not multiples of 16, or exceed 256: cfg3's towers (77 text
tokens against 196 image tokens, 98 under patch dropout), 300 text tokens against 576 image tokens
(384 px / patch 16) and 7 text tokens against 9 image tokens (48 px / patch 16) at batch 33.  The
segment-max GEMMs then run xclip_filip_segmax_arg16.  Goldens: tests/golden/{vitb16_shaped_filip,
vitb16_shaped_filip_drop, vitb16_shaped_filip_dcl_extra, filip_t300_i576, filip_t7_i9}.json, written
by tests/golden/make_golden_filip_any.py."""
import json
from pathlib import Path

import pytest
import torch

import test_gpu_clip_parity
import test_gpu_multirank
import test_oracle_golden
from oracle import clip_oracle as O

GOLD = Path(__file__).parent / "golden"
FILIP_ANY_CASES = ["vitb16_shaped_filip", "vitb16_shaped_filip_drop", "vitb16_shaped_filip_dcl_extra",
                   "filip_t300_i576", "filip_t7_i9"]


@pytest.mark.parametrize("case", FILIP_ANY_CASES)
def test_filip_any_models_construct_with_the_reference_parameter_tree(case):
    import x_clip_b200
    gold = json.loads((GOLD / f"{case}.json").read_text())
    clip = x_clip_b200.CLIP(**gold["cfg"], visual_patch_dropout=gold["patch_dropout"])
    want = O.param_shapes(O.ClipConfig(**gold["cfg"]))
    got = {k: tuple(v.shape) for k, v in clip.state_dict().items()}
    assert got == want


@pytest.mark.parametrize("case", FILIP_ANY_CASES)
def test_oracle_reproduces_filip_any_goldens(case):
    test_oracle_golden.test_oracle_reproduces_reference(case)


# filip_t7_i9 takes a max over only 7 or 9 tokens for each of 33 x 33 pairs, and its parameter
# gradients follow which token wins.  Rounding the latents to bf16 inside the reference alone turns
# its per-parameter gradients by up to cosine 0.995 there, against 0.9995 at tiny_filip
# (test_filip_t7_i9_gradients_are_sensitive_to_latent_rounding).  The bf16 encoders perturb the
# latents more than that rounding; measured on an H100: worst per-parameter cosine 0.9877
# (visual pos_emb), while the FILIP kernels on identical latents stay within 3e-3 of fp64
# (test_gpu_filip_any).  That case is checked with the parity gates on loss, latents, d temperature
# and gradient norm, and per-parameter cosine 0.98.
T7_I9_COS = 0.98


@pytest.mark.gpu
@pytest.mark.parametrize("case", [c for c in FILIP_ANY_CASES if c != "filip_t7_i9"])
def test_filip_any_clip_matches_reference(cuda_device, case):
    """Loss, latent checksums, d temperature, gradient norm and per-parameter gradients against the
    reference, with the gates of test_gpu_clip_parity."""
    test_gpu_clip_parity.test_clip_matches_reference(cuda_device, case)


def _cosines(grads, ref_grads, grad_norm):
    out = {}
    for k, g in grads.items():
        og = ref_grads.get(k)
        if k == "temperature" or og is None or og.norm().item() < 1e-3 * grad_norm:
            continue
        out[k] = torch.nn.functional.cosine_similarity(g.flatten().double(), og.flatten().double(), dim=0).item()
    return out


@pytest.mark.gpu
def test_filip_t7_i9_clip_matches_reference(cuda_device):
    gold, loss, grads, lat, o_loss, p = test_gpu_clip_parity._run("filip_t7_i9", cuda_device)
    assert abs(o_loss - gold["loss"]) < 1e-5
    assert abs(loss - gold["loss"]) <= 1e-3 * abs(gold["loss"]), (loss, gold["loss"])
    for z, ref in zip(lat, gold["latents"]):
        assert list(z.shape) == ref["shape"]
        assert abs(z.double().abs().sum().item() - ref["abs_sum"]) <= 5e-3 * ref["abs_sum"]
    dt = grads["temperature"].item()
    assert abs(dt - gold["dtemperature"]) <= 1e-2 * abs(gold["dtemperature"]) + 1e-3, (dt, gold["dtemperature"])
    gn = torch.sqrt(sum((g.double() ** 2).sum() for g in grads.values())).item()
    assert abs(gn - gold["grad_norm"]) <= 1e-2 * gold["grad_norm"], (gn, gold["grad_norm"])
    cos = _cosines(grads, {k: v.grad for k, v in p.items() if v.grad is not None}, gold["grad_norm"])
    bad = {k: round(c, 4) for k, c in cos.items() if c < T7_I9_COS}
    print(f"filip_t7_i9: worst per-parameter cosine {min(cos.values()):.4f}")
    assert not bad, bad


class _RoundToBf16(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x):
        return x.to(torch.bfloat16).float()

    @staticmethod
    def backward(ctx, g):
        return g


def _worst_cos_under_latent_rounding(case):
    """worst per-parameter cosine between the oracle's gradients and the oracle's gradients with its
    latents rounded to bf16 on the way into the loss"""
    gold = json.loads((GOLD / f"{case}.json").read_text())
    cfg = O.ClipConfig(**gold["cfg"])
    state = O.protocol_state_dict(cfg, gold["weight_seed"])
    text, image = O.protocol_inputs(cfg, gold["batch"], gold["input_seed"], gold["pad_fraction"])
    loss_fn = O.contrastive_loss

    def grads(rounded):
        def cl(*zs_and_rest, **kw):
            zs, rest = zs_and_rest[:4], zs_and_rest[4:]
            if rounded:
                zs = [_RoundToBf16.apply(z) for z in zs]
            return loss_fn(*zs, *rest, **kw)
        p = {k: v.clone().requires_grad_(True) for k, v in state.items()}
        O.contrastive_loss = cl
        try:
            O.clip_forward(p, text, image, cfg).backward()
        finally:
            O.contrastive_loss = loss_fn
        return {k: v.grad for k, v in p.items() if v.grad is not None}

    g0, g1 = grads(False), grads(True)
    return min(_cosines(g1, g0, gold["grad_norm"]).values())


def test_filip_t7_i9_gradients_are_sensitive_to_latent_rounding():
    """The reason for T7_I9_COS, pinned on the CPU: the same bf16 rounding of the latents moves the
    reference's gradients ten times further at filip_t7_i9 than at tiny_filip."""
    worst_t7 = _worst_cos_under_latent_rounding("filip_t7_i9")
    worst_tiny = _worst_cos_under_latent_rounding("tiny_filip")
    assert worst_t7 < 0.997 and worst_tiny > 0.999, (worst_t7, worst_tiny)
    assert 1 - worst_t7 > 5 * (1 - worst_tiny), (worst_t7, worst_tiny)


@pytest.mark.gpu
@pytest.mark.parametrize("case,port", [("vitb16_shaped_filip", 29841), ("filip_t300_i576", 29851)])
def test_two_gpu_filip_any_matches_full_batch(case, port):
    """2 ranks x 2 pairs give the single-process loss of the 4-pair golden case and gradients that sum
    to its gradients (test_gpu_multirank's FILIP worker).  Skipped on boxes with < 2 GPUs."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import queue as _q
    import time as _t
    import torch.multiprocessing as mp
    gold = json.loads((GOLD / f"{case}.json").read_text())
    world = 2
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=test_gpu_multirank._filip_worker, args=(r, world, case, port, q))
             for r in range(world)]
    for p in procs:
        p.start()
    res = []
    t0 = _t.time()
    while len(res) < world + 1 and _t.time() - t0 < 600:
        try:
            res.append(q.get(timeout=2))
        except _q.Empty:
            if any(p.exitcode not in (None, 0) for p in procs):
                break
    for p in procs:
        p.join(timeout=60)
        if p.is_alive():
            p.terminate()
    assert len(res) == world + 1, "a rank died"
    ref = [r for r in res if r[0] == "ref"][0]
    ranks = sorted(r for r in res if r[0] != "ref")
    assert abs(ref[1] - gold["loss"]) < 1e-5
    for rank, loss, dtemp in ranks:
        assert abs(loss - gold["loss"]) <= 1e-3 * abs(gold["loss"]), (rank, loss, gold["loss"])
        assert abs(dtemp - gold["dtemperature"]) <= 1e-2 * abs(gold["dtemperature"]) + 1e-3
    assert abs(ranks[0][1] - ranks[1][1]) < 1e-6
    assert not ref[3], ref[3]
