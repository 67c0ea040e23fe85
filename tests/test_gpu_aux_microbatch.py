"""MLM and SimSiam / SimCLR through the micro-batched step (engine.ChunkedClipLossFn with the auxiliary
passes): against the fp64 whole-step reference, against the single pass on the same GPU, the
patch-dropout replay of re-encoded chunks, the memory of a step that keeps nothing, and which calls
take the micro-batched path."""
import copy

import pytest
import torch

import step_oracle as SO
from test_gpu_step_fp64 import _check, _grads, _model, _recorded_keeps

pytestmark = pytest.mark.gpu

AUX_KW = SO.CASES["aux"]["kw"]
TINY = dict(SO.TINY)


@pytest.mark.parametrize("retain", [0, 1, "auto"])
def test_aux_microbatched_step_fp64(cuda_device, monkeypatch, retain):
    """The step_oracle `aux` case (MLM with a pinned corruption, SimCLR with the identity augmentation)
    at batch 7 in chunks of 3, against the fp64 reference of the whole batch with the step gates."""
    name = f"aux_micro_{retain}"
    monkeypatch.setitem(SO.CASES, name, dict(kw=dict(AUX_KW, microbatch=3, microbatch_retain=retain),
                                             mlm=True, batch=7))
    monkeypatch.setitem(SO.GATE_SCALE, name, SO.GATE_SCALE["aux"])
    dev = cuda_device
    c = SO.make_case(name)
    clip = _model(c, dev)
    text, image = c["batches"][0]
    loss = clip(text.to(dev), image.to(dev), return_loss=True)
    loss.backward()
    torch.cuda.synchronize()
    plan = clip.last_step_plan
    retained = {0: 0, 1: 1, "auto": 3}[retain]                  # tiny model: "auto" keeps all
    assert plan["chunks"] == 3 and plan["retained"] == retained, plan
    assert plan["retained_chunks"] == list(range(retained))
    assert plan["passes"] == ["contrastive", "mlm", "view1", "view2"]
    ref = SO.reference(c, dev)
    _check(name, c, dict(loss=loss.item(), grads=_grads(clip), image_grads=None), ref)


# --------------------------------------------------------------------------- against the single pass

README = dict(TINY, num_text_tokens=120, decoupled_contrastive_learning=True, extra_latent_projection=True,
              use_visual_ssl=True)                                # SimSiam by default (README.md example)
CONFIGS = {
    "readme_simsiam": README,
    "mlm_simsiam": dict(README, use_mlm=True, mlm_mask_token_id=2),
    "filip_mlm": dict(TINY, num_text_tokens=120, use_all_token_embeds=True, use_mlm=True, mlm_mask_token_id=2),
    "simreg_simsiam": dict(README, decoupled_contrastive_learning=False, sim_reg_loss_weight=1.0),
    "mlm_simclr": dict(TINY, **dict(AUX_KW, simclr_temperature=0.5)),
}


def _pair(kw, dev, microbatch, retain, batch=10, seed=0):
    """The same model twice (single pass, micro-batched), identity augmentation, pinned corruption."""
    import x_clip_b200
    from oracle import clip_oracle as O
    torch.manual_seed(seed)
    single = x_clip_b200.CLIP(**kw).to(dev)
    micro = copy.deepcopy(single)
    micro.microbatch, micro.microbatch_retain = microbatch, retain
    cfg = O.ClipConfig(**{k: v for k, v in kw.items() if k in set(O.ClipConfig().__dict__)})
    text, image = O.protocol_inputs(cfg, batch, 4321, 0.2)
    text = text.clamp(max=kw["num_text_tokens"] - 1).to(dev)
    image = image.to(dev)
    pinned = None
    if kw.get("use_mlm"):
        torch.manual_seed(3)
        pinned = single.mlm.corrupt(text)
        assert (pinned[1] != 0).any()
    for m in (single, micro):
        m.train()
        if kw.get("use_visual_ssl"):
            m.visual_ssl.augment1 = m.visual_ssl.augment2 = torch.nn.Identity()
        if pinned is not None:
            m.mlm.corrupt = lambda seq, p=pinned: p
    return single, micro, text, image


def _rel(a, b):
    d = b.double().norm().item()
    return (a.double() - b.double()).norm().item() / (d if d > 0 else 1.0)


@pytest.mark.parametrize("config", sorted(CONFIGS))
@pytest.mark.parametrize("retain", [0, "auto"])
def test_microbatched_equals_single_pass(cuda_device, config, retain):
    """Loss, every parameter's gradient and every BatchNorm's running statistics after one step."""
    kw = CONFIGS[config]
    single, micro, text, image = _pair(kw, cuda_device, 4, retain)
    l1 = single(text, image, return_loss=True)
    l1.backward()
    micro.last_step_plan = None
    l2 = micro(text, image, return_loss=True)
    l2.backward()
    torch.cuda.synchronize()
    assert micro.last_step_plan is not None and micro.last_step_plan["chunks"] == 3
    assert abs(l2.item() - l1.item()) <= 1e-5 * abs(l1.item()), (l1.item(), l2.item())
    g1, g2 = dict(single.named_parameters()), dict(micro.named_parameters())
    worst = 0.0
    for name, p in g1.items():
        q = g2[name]
        assert (p.grad is None) == (q.grad is None), name
        if p.grad is not None:
            r = _rel(q.grad, p.grad)
            worst = max(worst, r)
            assert r <= 2e-3, (name, r)
    print(f"{config} retain={retain}: loss {l1.item():.6f} / {l2.item():.6f}, worst gradient {worst:.2e}")
    bn1 = {n: m for n, m in single.named_modules() if isinstance(m, torch.nn.BatchNorm1d)}
    bn2 = dict((n, m) for n, m in micro.named_modules() if isinstance(m, torch.nn.BatchNorm1d))
    assert bn1.keys() == bn2.keys()
    for n, m in bn1.items():
        assert m.num_batches_tracked.item() == bn2[n].num_batches_tracked.item() > 0, n
        assert torch.allclose(bn2[n].running_mean, m.running_mean, rtol=1e-4, atol=1e-6), n
        assert torch.allclose(bn2[n].running_var, m.running_var, rtol=1e-4, atol=1e-6), n


def test_reencoded_chunks_replay_their_patch_dropout(cuda_device):
    """Patch dropout 0.5, SimSiam + MLM, nothing retained: every chunk's forward draws the keeps of
    its contrastive pass, view 1, view 2 and then the two target passes; its re-encode in backward
    draws the first three again, in that order."""
    kw = dict(CONFIGS["mlm_simsiam"], visual_patch_dropout=0.5)
    _, micro, text, image = _pair(kw, cuda_device, 4, 0)
    rec = _recorded_keeps(micro)
    loss = micro(text, image, return_loss=True)
    rec["phase"] = "bwd"
    loss.backward()
    torch.cuda.synchronize()
    fwd, bwd = rec["fwd"], rec["bwd"]
    assert len(fwd) == 3 * 5 and len(bwd) == 3 * 3
    for k in range(3):
        f, b = fwd[5 * k: 5 * k + 5], bwd[3 * k: 3 * k + 3]
        for a, c in zip(b, f[:3]):
            assert torch.equal(a, c)
        assert not torch.equal(f[1], f[2]) and not torch.equal(f[1], f[3])


def test_memory_with_nothing_retained(cuda_device):
    """retain = 0 and chunks of 16: from B = 32 to B = 128 the peak grows by the full-batch leaves and
    heads, not by encoder activations.  Bound: 96 more rows of leaves, selected MLM rows and heads
    (well under 2 MB per row at these widths) - a fraction of the single pass's growth."""
    import x_clip_b200
    dev = cuda_device
    kw = dict(CONFIGS["mlm_simclr"], visual_image_size=128, text_seq_len=64)

    def peak(batch, microbatch):
        torch.manual_seed(0)
        m = x_clip_b200.CLIP(**kw, microbatch=microbatch, microbatch_retain=0).to(dev)
        m.train()
        m.visual_ssl.augment1 = m.visual_ssl.augment2 = torch.nn.Identity()
        text = torch.randint(3, 120, (batch, 64), device=dev)
        image = torch.randn(batch, 3, 128, 128, device=dev)
        m(text, image, return_loss=True).backward()        # warm-up: casts, plans, allocator
        m.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated(dev)
        torch.cuda.reset_peak_memory_stats(dev)
        m(text, image, return_loss=True).backward()
        torch.cuda.synchronize()
        out = torch.cuda.max_memory_allocated(dev) - base
        del m
        torch.cuda.empty_cache()
        return out

    grow_micro = peak(128, 16) - peak(32, 16)
    grow_single = peak(128, None) - peak(32, None)
    print(f"peak growth 32 -> 128: micro-batched {grow_micro / 2**20:.1f} MiB, single pass {grow_single / 2**20:.1f} MiB")
    assert grow_micro <= 96 * (2 << 20)
    assert grow_micro <= 0.25 * grow_single


def test_routing(cuda_device):
    """MLM and SSL calls with microbatch set take the micro-batched step; multiview, frozen towers and
    visual SSL on an image that requires grad keep the single pass."""
    dev = cuda_device
    _, mlm_only, text, image = _pair(dict(TINY, num_text_tokens=120, use_mlm=True, mlm_mask_token_id=2),
                                     dev, 4, "auto")
    mlm_only(text, image, return_loss=True).backward()
    assert mlm_only.last_step_plan["passes"] == ["contrastive", "mlm"]
    _, ssl, text, image = _pair(README, dev, 4, "auto")
    ssl(text, image, return_loss=True).backward()
    assert ssl.last_step_plan["passes"] == ["contrastive", "view1", "view2"]
    for call in (dict(aug_text=text.clone()), dict(freeze_image_encoder=True), dict(freeze_text_encoder=True)):
        ssl.last_step_plan = None
        ssl(text, image, return_loss=True, **call).backward()
        assert ssl.last_step_plan is None, call
    ssl.last_step_plan = None
    img = image.clone().requires_grad_(True)
    ssl(text, img, return_loss=True).backward()
    assert ssl.last_step_plan is None and img.grad is not None
