"""The pairwise sigmoid loss (CLIP(sigmoid_loss=True)) on the H100 against fp64:

- the kernels xclip_sigmoid_fwd / _bwd on split-bf16 operands, at row counts 1 to 4096, column counts
  that are not a multiple of 8 and rank blocks (C > R, diag_offset > 0), latent widths 72 / 256 / 512
  (K = 216 is not a whole 64-wide k-block), logit scales 10 and 100 and biases -10 and 0;
- engine.SigmoidLossFn against sigmoid_oracle.sigmoid_loss at global batches 1 to 4096;
- the whole step (single pass, augmented views, image gradient, MLM + SimCLR, the micro-batched step at
  microbatch_retain 0 and 1) against sigmoid_oracle.reference, with step_oracle's gates;
- the data-parallel step at W = 2 and 3 ranks on one GPU (gloo), rank by rank.
"""
import math
import os
import time
import traceback
from datetime import timedelta

import pytest
import torch

import sigmoid_oracle as SG
import step_oracle as SO
from test_gpu_step_fp64 import _recorded_keeps

pytestmark = pytest.mark.gpu

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64

# Gates: about 2x the largest error measured on an H100 80GB HBM3 at a 700 W power limit over the cases
# below.  Kernels: ROW_REL, LOSS_REL, G_REL and SUM_REL of sigmoid_oracle (shared with the per-call
# checks of bench_call_oracle.py).  SigmoidLossFn: loss 2.2e-5 (global batch 2), latent gradients 3.4e-3;
# its d temperature and d logit_bias gates are (as test_gpu_nce_loss.py) rel * |ref| + abs.
ROW_REL, LOSS_REL, G_REL, SUM_REL = SG.ROW_REL, SG.LOSS_REL, SG.G_REL, SG.SUM_REL
DSCALAR_REL, DSCALAR_ABS = 1e-4, 1e-7
FN_LOSS_REL = 5e-5      # SigmoidLossFn: loss, relative
FN_GRAD_REL = 8e-3      # SigmoidLossFn: latent gradients, relative Frobenius (two bf16 roundings)
# Whole steps: step_oracle's gates, the loss, d temperature and d logit_bias gates doubled.  Measured with
# step_oracle's own gates: d temperature 0.90 of its gate (single pass), the loss 0.77 (global batch 3 over
# 3 ranks); every gradient family at most 0.50 of its gate (the SimCLR head).  A logit scale of 10 (InfoNCE
# starts at e) carries the encoders' rounding of the latents into d temperature 3.7x as strongly.
STEP_SCALAR_SCALE = 2.0


# --------------------------------------------------------------------------- kernels

def _kernel_cases():
    cases = []
    for i, R in enumerate((1, 7, 129, 1000, 4096)):
        wide = 2 * R + 13 + (8 - (2 * R + 13) % 8) % 8 + 3          # not a multiple of 8
        for j, (C, off) in enumerate(((R, 0), (wide, R + 5 if R + 5 + R <= wide else wide - R))):
            D = (72, 256, 512)[(i + j) % 3]
            for te in (10.0, 100.0):
                for lb in (-10.0, 0.0):
                    cases.append((R, C, off, D, te, lb))
    return cases


KERNEL_CASES = _kernel_cases()


def _split_operands(p):
    """(unit rows z fp32, zrow = [hi | lo | hi], zcol = [hi | hi | lo]): xclip_l2norm_fwd's split-bf16
    operands, built here for any width (the kernel takes widths of 128 * k)"""
    z = torch.nn.functional.normalize(p.float(), dim=-1)
    hi = z.to(BF16)
    lo = (z - hi.float()).to(BF16)
    return z, torch.cat([hi, lo, hi], 1).contiguous(), torch.cat([hi, hi, lo], 1).contiguous()


@pytest.mark.parametrize("R,C,off,D,te,lb", KERNEL_CASES,
                         ids=[f"R{R}-C{C}-off{o}-D{D}-s{int(t)}-b{int(b)}" for R, C, o, D, t, b in KERNEL_CASES])
def test_sigmoid_kernels_match_fp64(cuda_device, R, C, off, D, te, lb):
    """Row losses, the summed loss, g (alpha * gscale * (sigmoid - [positive]) in bf16, zero pad columns),
    d temperature and d logit_bias.  Every second row's positive is its own latent, so at a logit scale of
    100 its logit (90 or 100) saturates: its g must be exactly 0."""
    from x_clip_b200 import kernels as K
    dev = cuda_device
    gen = torch.Generator(device=dev).manual_seed(R * 31 + C + D)
    pr = torch.randn((R, D), generator=gen, device=dev)
    pc = torch.randn((C, D), generator=gen, device=dev)
    pc[off:off + R:2] = pr[0::2]
    zr, ar, _ = _split_operands(pr)
    zc, _, bc = _split_operands(pc)
    te_d = torch.tensor([te], device=dev, dtype=F32)
    lb_d = torch.tensor([lb], device=dev, dtype=F32)
    gs = 0.37 / C
    gs_d = torch.tensor([gs], device=dev, dtype=F32)
    acc = torch.zeros(1, device=dev, dtype=F32)
    rowloss = K.sigmoid_fwd(ar, bc, te_d, lb_d, off, acc, 0.5)
    dsc = torch.zeros(2, device=dev, dtype=F32)
    g = K.sigmoid_bwd(ar, bc, te_d, lb_d, off, gs_d, dsc[0:1], dsc[1:2])
    torch.cuda.synchronize()

    s = zr.double() @ zc.double().t()
    l = te * s + lb
    z = SG.labels(R, C, off, like=l)
    r_rows = SG.softplus(-z * l).sum(1)
    r_g = gs * -z * torch.sigmoid(-z * l)                     # sigmoid(l) - [positive], no cancellation
    r_dt, r_db = (r_g * (l - lb)).sum().item(), r_g.sum().item()
    m_dt, m_db = (r_g * (l - lb)).abs().sum().item(), r_g.abs().sum().item()

    label = f"R={R} C={C} off={off} D={D} scale={te} bias={lb}"
    assert torch.isfinite(rowloss).all() and torch.isfinite(g.float()).all(), label
    # + 1e-30: a row made only of a saturated positive has a loss of e^-90, which fp32 flushes to 0
    e_row = ((rowloss.double() - r_rows).abs() / (r_rows + 1e-30)).max().item()
    e_loss = abs(acc.item() - 0.5 * r_rows.sum().item()) / (0.5 * r_rows.sum().item() + 1e-30)
    assert g.shape == (R, (C + 7) // 8 * 8)
    assert not g[:, C:].ne(0).any(), label
    gk = g[:, :C].double()
    want = te * r_g
    live = l.abs() < 80.0                                     # u = e^-|l| is a normal fp32 number
    e_g = ((gk - want).abs()[live] / want.abs()[live]).max().item() if live.any() else 0.0
    sat = l.abs() > 88.0
    assert not gk[sat].ne(0).any(), (label, "saturated logits must give g = 0 exactly")
    if te == 100.0:
        assert sat.any(), label
    dt, db = dsc.tolist()
    e_dt = abs(dt - r_dt) / (SUM_REL * m_dt + 1e-30)      # + 1e-30: every term saturated, as above
    e_db = abs(db - r_db) / (SUM_REL * m_db + 1e-30)
    print(f"GATE sigk[{label}] row {e_row:.2e} loss {e_loss:.2e} g {e_g:.2e} dtemp/gate {e_dt:.3f} "
          f"dbias/gate {e_db:.3f}")
    assert e_row <= ROW_REL, (label, e_row)
    assert e_loss <= LOSS_REL, (label, e_loss)
    assert e_g <= G_REL, (label, e_g)
    assert e_dt <= 1.0, (label, dt, r_dt)
    assert e_db <= 1.0, (label, db, r_db)


def test_sigmoid_refusals_launch_nothing(cuda_device):
    """Positives outside the columns and a missing bias scalar are refused without a launch."""
    from x_clip_b200 import _lib, kernels as K
    dev = cuda_device
    _, a, _ = _split_operands(torch.randn((8, 128), device=dev))
    _, _, b = _split_operands(torch.randn((12, 128), device=dev))
    one = torch.ones(1, device=dev, dtype=F32)
    n0 = _lib.load().xclip_launch_count()
    for off in (-1, 5):
        with pytest.raises(_lib.XClipB200Error):
            K.sigmoid_fwd(a, b, one, one, off)
        with pytest.raises(_lib.XClipB200Error):
            K.sigmoid_bwd(a, b, one, one, off, one)
    with pytest.raises(_lib.XClipB200Error):
        K.sigmoid_fwd(a, b, one, one.double(), 0)
    assert _lib.load().xclip_launch_count() == n0


# --------------------------------------------------------------------------- SigmoidLossFn

FN_BATCHES = [1, 2, 33, 127, 129, 1000, 4095, 4096]
FN_CASES = [(B, t, b) for B in FN_BATCHES for t, b in ((math.log(10.0), -10.0), (math.log(100.0), 0.0))]


@pytest.mark.parametrize("B,temperature,bias", FN_CASES,
                         ids=[f"B{B}-s{round(math.exp(t))}-b{int(b)}" for B, t, b in FN_CASES])
def test_sigmoid_loss_fn_matches_fp64_oracle(cuda_device, B, temperature, bias):
    from x_clip_b200 import engine as E
    dev = cuda_device
    gen = torch.Generator(device=dev).manual_seed(B)
    sets = []
    for _ in range(2):
        e = torch.randn((B, 256), generator=gen, device=dev).to(BF16)
        w = (torch.randn((512, 256), generator=gen, device=dev) / 16).requires_grad_(True)
        z, zrow, zcol = E.ProjectL2NormFn.apply(e, w)
        z.retain_grad()
        sets.append((z, zrow, zcol))
    t = torch.tensor(temperature, device=dev, dtype=F32, requires_grad=True)
    lb = torch.tensor(bias, device=dev, dtype=F32, requires_grad=True)
    loss = E.SigmoidLossFn.apply(sets[0][0], sets[1][0], t, lb, tuple((s[1], s[2]) for s in sets), False)
    loss.backward()

    zz = [s[0].detach().double().requires_grad_(True) for s in sets]
    t64 = t.detach().double().requires_grad_(True)
    b64 = lb.detach().double().requires_grad_(True)
    ref = SG.sigmoid_loss(zz[0], zz[1], t64, b64)
    ref.backward()
    label = f"B={B} scale={math.exp(temperature):.0f} bias={bias}"
    e_loss = abs(loss.item() - ref.item()) / abs(ref.item())
    e_dt = abs(t.grad.item() - t64.grad.item()) / (DSCALAR_REL * abs(t64.grad.item()) + DSCALAR_ABS)
    e_db = abs(lb.grad.item() - b64.grad.item()) / (DSCALAR_REL * abs(b64.grad.item()) + DSCALAR_ABS)
    rels = [(s[0].grad.double() - r.grad).norm().item() / r.grad.norm().item() for s, r in zip(sets, zz)]
    print(f"GATE sigfn[{label}] loss {e_loss:.2e} dtemp/gate {e_dt:.3f} dbias/gate {e_db:.3f} grad {max(rels):.2e}")
    assert e_loss <= FN_LOSS_REL, (label, loss.item(), ref.item())
    assert e_dt <= 1.0 and e_db <= 1.0, (label, t.grad.item(), t64.grad.item(), lb.grad.item(), b64.grad.item())
    assert max(rels) <= FN_GRAD_REL, (label, rels)


# --------------------------------------------------------------------------- whole step

MICRO = dict(microbatch=3, visual_patch_dropout=0.5)
AUX = dict(num_text_tokens=120, use_mlm=True, mlm_mask_token_id=2, use_visual_ssl=True, visual_ssl_type="simclr",
           simclr_temperature=10.0)
STEP_CASES = {
    "single": dict(kw={}, text_len=13),
    "multiview": dict(kw={}, aug=1),
    "imggrad": dict(kw=dict(visual_patch_dropout=0.5), keep="pinned", image_grad=True),
    "aux": dict(kw=AUX, mlm=True),
    "micro_r0": dict(kw=dict(MICRO, microbatch_retain=0), batch=7),
    "micro_r1": dict(kw=dict(MICRO, microbatch_retain=1), batch=7),
    "micro_aux": dict(kw=dict(AUX, microbatch=3, microbatch_retain=1), batch=7, mlm=True),
}


def _prepare(clip, c, dev):
    clip = clip.to(dev)
    clip.train()
    if c["mlm"] is not None:
        masked, labels = (t.to(dev) for t in c["mlm"])
        clip.mlm.corrupt = lambda seq: (masked, labels)
    if c["keep"] is not None:
        clip.visual_transformer.patch_dropout.forced_keep = c["keep"]
    return clip


def _ratios(label, c, got, ref, scale=1.0):
    """step_oracle's structural checks and gates, logit_bias gated like d temperature, the loss and both
    scalars at STEP_SCALAR_SCALE times their gates."""
    bad = SO.structural_errors(c["names"], got, ref)
    gb, rb = got["grads"]["logit_bias"], ref["grads"]["logit_bias"]
    strip = lambda d: dict(d, grads={k: v for k, v in d["grads"].items() if k != "logit_bias"})
    r = SO.ratios(strip(got), strip(ref), scale)
    r["dbias"] = abs(gb.item() - rb.item()) / (SO.DTEMP_REL * abs(rb.item()) + SO.DTEMP_ABS)
    for k in ("loss", "dtemp", "dbias"):
        r[k] /= STEP_SCALAR_SCALE
    for f, v in sorted(r.items()):
        print(f"GATE sigstep_{f}[{label}] {v:.4f}")
    return bad + [f"{f}: {v:.3f} x its gate" for f, v in r.items() if not v <= 1.0]


def _run(clip, c, dev, text, image):
    img = image.to(dev).requires_grad_(c["image_grad"])
    aug_t = tuple(t.to(dev) for t in c["aug_text"]) or None
    aug_i = tuple(t.to(dev) for t in c["aug_image"]) or None
    loss = clip(text.to(dev), img, return_loss=True, aug_text=aug_t, aug_image=aug_i)
    loss.backward()
    torch.cuda.synchronize()
    return dict(loss=loss.item(), grads={k: p.grad for k, p in clip.named_parameters()},
                image_grads=[img.grad] if c["image_grad"] else None)


@pytest.mark.parametrize("case", list(STEP_CASES))
def test_sigmoid_step_fp64(cuda_device, case):
    """One step of CLIP(sigmoid_loss=True) against the fp64 step.  A micro-batched case also runs the
    single pass on the same batch and patch-dropout keep: both must give the same loss and gradients up
    to the kernels' rounding."""
    import copy
    dev = cuda_device
    c = SG.make_case(case, STEP_CASES[case])
    micro = bool(c["kw"].get("microbatch"))
    single = copy.deepcopy(c["model"]) if micro else None
    clip = _prepare(c["model"], c, dev)
    text, image = c["batches"][0]
    keep = None
    if micro and c["kw"].get("visual_patch_dropout"):
        rec = _recorded_keeps(clip)
    torch.manual_seed(0)
    got = _run(clip, c, dev, text, image)
    if micro:
        plan = clip.last_step_plan
        assert plan["chunks"] == 3 and plan["retained"] == c["kw"]["microbatch_retain"], plan
        if c["kw"].get("visual_patch_dropout"):
            keep = torch.cat(rec["fwd"][:3])          # the forward's draws; a re-encoded chunk draws again
    ref = SG.reference(c, dev, keep)
    scale = SO.GATE_SCALE["aux"] if "aux" in case else 1.0
    bad = _ratios(case, c, got, ref, scale)
    if micro:
        single.microbatch = None
        single = _prepare(single, c, dev)
        if keep is not None:
            single.visual_transformer.patch_dropout.forced_keep = keep.to(dev)
        one = _run(single, c, dev, text, image)
        assert single.last_step_plan is None
        bad += _ratios(case + "_vs_single", c, got, one, scale)
    assert not bad, bad


def test_return_loss_false_is_scaled_similarity(cuda_device):
    """Without return_loss the sigmoid model returns exp(temperature) * <t_i, v_i>, without the bias."""
    dev = cuda_device
    c = SG.make_case("single", STEP_CASES["single"])
    clip = _prepare(c["model"], c, dev)
    text, image = (t.to(dev) for t in c["batches"][0])
    with torch.no_grad():
        sim = clip(text, image)
        zt, zi = clip(text, image, return_latents=True)
    assert torch.allclose(sim, (zt * zi).sum(-1) * 10.0, rtol=1e-5, atol=1e-6)


# --------------------------------------------------------------------------- data parallel

# (W, case) -> local batch b and the step spec
RANK_CASES = {
    (2, "single"): dict(b=3, spec=STEP_CASES["single"]),
    (2, "multiview"): dict(b=3, spec=STEP_CASES["multiview"]),
    (2, "micro_r1"): dict(b=7, spec=dict(kw=dict(microbatch=3, microbatch_retain=1))),
    (3, "single"): dict(b=3, spec=STEP_CASES["single"]),
    (3, "b1"): dict(b=1, spec=dict(kw={})),
}
GROUP_TIMEOUT = 200


def _rank_case(world, name):
    o = RANK_CASES[(world, name)]
    spec = dict(o["spec"])
    spec.pop("batch", None)
    return SG.make_case(name, spec, world, o["b"])


def _rank_worker(world, rank, rdzv, out, ppid):
    import test_gpu_multirank_fp64 as MRT
    MRT._exit_with_parent(ppid)
    os.environ["GLOO_SOCKET_IFNAME"] = "lo"
    import torch.distributed as dist
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    dist.init_process_group("gloo", init_method=f"file://{rdzv}", rank=rank, world_size=world,
                            timeout=timedelta(seconds=120))
    try:
        path = MRT._collectives(world, dev)
        for (w, name), o in RANK_CASES.items():
            if w != world:
                continue
            c = _rank_case(world, name)
            clip = c["model"].to(dev)
            clip.train()
            assert clip.requires_all_gather
            sl = slice(rank * o["b"], (rank + 1) * o["b"])
            text, image = c["batches"][0]
            aug_t = tuple(t[sl].to(dev) for t in c["aug_text"]) or None
            aug_i = tuple(t[sl].to(dev) for t in c["aug_image"]) or None
            loss = clip(text[sl].to(dev), image[sl].to(dev), return_loss=True, aug_text=aug_t, aug_image=aug_i)
            loss.backward()
            torch.cuda.synchronize()
            grads = {k: None if p.grad is None else p.grad.detach().cpu().clone() for k, p in clip.named_parameters()}
            torch.save(dict(loss=loss.detach().cpu(), grads=grads, plan=clip.last_step_plan, collectives=path),
                       os.path.join(out, f"{name}.r{rank}.pt"))
        dist.barrier()
    except BaseException:
        with open(os.path.join(out, f"error.r{rank}.txt"), "w") as f:
            f.write(traceback.format_exc())
        raise
    finally:
        dist.destroy_process_group()


def _rank_group(world, tmp_path_factory):
    import torch.multiprocessing as mp
    out = tmp_path_factory.mktemp(f"sig{world}")
    ctx = mp.get_context("spawn")
    procs = [ctx.Process(target=_rank_worker, args=(world, r, str(out / "rdzv"), str(out), os.getpid()), daemon=True)
             for r in range(world)]
    t0 = time.time()
    try:
        for p in procs:
            p.start()
        while time.time() - t0 < GROUP_TIMEOUT and any(p.is_alive() for p in procs):
            if any(p.exitcode not in (None, 0) for p in procs):
                break
            time.sleep(0.2)
        for p in procs:
            p.join(timeout=5)
    finally:
        for p in procs:
            if p.is_alive():
                p.terminate()
                p.join(timeout=10)
            if p.is_alive():
                p.kill()
                p.join(timeout=10)
    assert not any(p.is_alive() for p in procs), "a worker outlived its group"
    msg = "\n".join(e.read_text() for e in (out / f"error.r{r}.txt" for r in range(world)) if e.exists())
    assert all(p.exitcode == 0 for p in procs), f"exit codes {[p.exitcode for p in procs]}\n{msg}"
    print(f"\nWALL sig{world}: {world} ranks in {time.time() - t0:.1f} s")
    return out


@pytest.fixture(scope="module")
def sig_ranks2(tmp_path_factory):
    return _rank_group(2, tmp_path_factory)


@pytest.fixture(scope="module")
def sig_ranks3(tmp_path_factory):
    return _rank_group(3, tmp_path_factory)


@pytest.mark.parametrize("world,name,rank", [(w, n, r) for (w, n) in RANK_CASES for r in range(w)],
                         ids=[f"sig{w}-{n}-r{r}" for (w, n) in RANK_CASES for r in range(w)])
def test_sigmoid_rank_step_fp64(cuda_device, request, world, name, rank):
    """Rank r's gradients against the global step with gradients through its own latents; the loss,
    d temperature and d logit_bias against the single-process fp64 step of the global batch, and the loss
    bit-identical on every rank."""
    dev = cuda_device
    out = request.getfixturevalue(f"sig_ranks{world}")
    saved = [torch.load(out / f"{name}.r{r}.pt") for r in range(world)]
    c = _rank_case(world, name)
    full = SG.reference(c, dev)
    ref = SG.rank_reference(c, dev, world, rank)
    for k in ("temperature", "logit_bias"):
        ref["grads"][k] = full["grads"][k]
    ref["loss"] = full["loss"]
    got = saved[rank]
    if "micro" in name:
        assert (got["plan"]["chunks"], got["plan"]["retained"]) == (3, 1), got["plan"]
    mine = dict(loss=got["loss"].item(), grads={k: None if v is None else v.to(dev) for k, v in got["grads"].items()},
                image_grads=None)
    bad = _ratios(f"{name}.w{world}.r{rank}", c, mine, ref)
    losses = [s["loss"] for s in saved]
    if not all(torch.equal(x.view(torch.int32), losses[0].view(torch.int32)) for x in losses):
        bad.append(f"the ranks return different losses {[x.item() for x in losses]}")
    for k in ("temperature", "logit_bias"):
        if not all(torch.equal(s["grads"][k], saved[0]["grads"][k]) for s in saved):
            bad.append(f"the ranks hold different d {k} {[s['grads'][k].item() for s in saved]}")
    assert not bad, bad
