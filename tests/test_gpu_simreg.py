"""Similarity regularisation on the GPU (csrc/simreg.cu, ContrastiveLossFn with sim_reg_weight, CLIP with
sim_reg_loss_weight > 0), everything against fp64.

Kernels: the fp64 reference is built from the exact bf16 operands ([zrow_t | zrow_v], [zcol_t | -zcol_v]),
so it sees only the kernels' fp32 accumulation and the bf16 rounding of g.  The "aligned" cases draw
v = normalize(t + noise of norm 1e-3), so |E| ~ 1e-3: a difference of two separately rounded similarity
matrices would lose most of E's digits there.

Gates: see the constants below; the measured maxima next to them are from an H100 80GB HBM3 at a
700 W power limit."""
import json
import math
import multiprocessing as _mp
import os
import queue as _q
import time as _t
from pathlib import Path

import pytest
import torch

import simreg_oracle as SR
from test_gpu_filip import _report_peak, _start_peak
from test_gpu_nce_loss import _latents

pytestmark = pytest.mark.gpu

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
GOLD = Path(__file__).parent / "golden"

# The kernel gates E_ABS, ROWSUM_REL, LOSS_REL and G_REL live in simreg_oracle (shared with the per-call
# checks of bench_call_oracle.py), with what was measured against them.
E_ABS, ROWSUM_REL, LOSS_REL, G_REL = SR.E_ABS, SR.ROWSUM_REL, SR.LOSS_REL, SR.G_REL
# ContrastiveLossFn with the term (w = 300, B 2..4096) against fp64: loss rel measured at most 6.4e-6,
# latent gradient rel error norm 3.6e-3 (at B = 2; two bf16 roundings as in test_gpu_nce_loss), d
# temperature rel 7.7e-5
CL_LOSS_REL = 1.5e-5
GRAD_REL = 5e-3
DTEMP_REL = 2e-4


def _ops(rows, D, dev, seed, aligned=False):
    """(zrow_t, zcol_t, zrow_v, zcol_v) of unit latents from xclip_l2norm_fwd."""
    from x_clip_b200 import kernels as K
    gen = torch.Generator(device=dev).manual_seed(seed)
    pt = torch.randn((rows, D), generator=gen, device=dev)
    if aligned:
        tn = torch.nn.functional.normalize(pt, dim=-1)
        pv = tn + 1e-3 * D ** -0.5 * torch.randn((rows, D), generator=gen, device=dev)   # |v - t| ~ 1e-3
    else:
        pv = torch.randn((rows, D), generator=gen, device=dev)
    _, zrt, zct, _ = K.l2norm_fwd(pt)
    _, zrv, zcv, _ = K.l2norm_fwd(pv)
    return zrt, zct, zrv, zcv


def _e64(a, b, off):
    """fp64 E = a b^T of the packed operands, the diagonal column of each row zeroed."""
    e = a.double() @ b.double().t()
    r = torch.arange(a.shape[0], device=a.device)
    e[r, r + off] = 0.0
    return e


# (R, C, diag_offset, D, aligned): odd and even sizes, C from 2 to 32768, offsets on the 128 / 256
# column-block borders and rows straddling them, D from 256 to 1024
KERNEL_CASES = [
    (2, 2, 0, 256, False), (1, 3, 2, 512, False), (3, 5, 1, 768, False), (7, 7, 0, 1024, False),
    (64, 129, 65, 256, False), (128, 256, 128, 512, False), (129, 300, 127, 512, True),
    (255, 256, 1, 768, False), (33, 257, 224, 1024, True), (1000, 1000, 0, 512, False),
    (513, 4096, 3583, 256, True), (4096, 4096, 0, 512, True), (4095, 4097, 2, 1024, False),
    (4096, 32768, 0, 512, False), (4096, 32768, 28672, 512, True),
]


@pytest.mark.parametrize("R,C,off,D,aligned", KERNEL_CASES)
def test_simreg_kernels_against_fp64(cuda_device, R, C, off, D, aligned):
    from x_clip_b200 import kernels as K
    t0 = _start_peak()
    zrt, zct, zrv, zcv = _ops(C, D, cuda_device, seed=R * 7 + C, aligned=aligned)
    a = K.simreg_pack(zrt[off:off + R].contiguous(), zrv[off:off + R].contiguous(), False)
    b = K.simreg_pack(zct, zcv, True)
    assert torch.equal(a, torch.cat([zrt[off:off + R], zrv[off:off + R]], 1))
    assert torch.equal(b, torch.cat([zct, -zcv], 1))
    e = _e64(a, b, off)

    scale = 0.37
    acc = torch.zeros(1, device=cuda_device, dtype=F32)
    rs = K.simreg_fwd(a, b, off, acc, scale)
    ref_rs = (e * e).sum(1)
    bound = ROWSUM_REL * ref_rs + 2 * E_ABS * e.abs().sum(1)
    rs_err = ((rs.double() - ref_rs).abs() / bound).max().item()           # fraction of the gate
    loss_err = abs(acc.item() - scale * ref_rs.sum().item()) / (scale * ref_rs.sum().item())

    gs = torch.tensor([1.7], device=cuda_device, dtype=F32)
    g = K.simreg_bwd(a, b, off, gs)
    ldg = (C + 7) // 8 * 8
    assert g.shape == (R, ldg)
    assert not g[:, C:].any()                                         # zero padding
    r = torch.arange(R, device=cuda_device)
    assert not g[r, r + off].any()                                   # zero diagonal
    ref_g = 1.7 * e
    g_err = ((g[:, :C].double() - ref_g).abs() - G_REL * ref_g.abs()).max().item()
    print(f"simreg R={R} C={C} off={off} D={D} aligned={aligned}: rowsum {rs_err:.2e} of gate, "
          f"loss rel {loss_err:.2e}, g excess {g_err:.2e}")
    _report_peak("  case", t0)
    assert rs_err <= 1.0
    assert loss_err <= LOSS_REL
    assert g_err <= 1.7 * E_ABS                                       # beyond the rounding: E's fp32 error


def test_simreg_refuses_bad_calls_without_launching(cuda_device):
    from x_clip_b200 import _lib, kernels as K
    lib = _lib.load()
    zrt, zct, zrv, zcv = _ops(64, 256, cuda_device, seed=1)
    a = K.simreg_pack(zrt, zrv, False)
    b = K.simreg_pack(zct, zcv, True)
    ws = torch.empty(4 * 64, device=cuda_device, dtype=F32)
    gs = torch.ones(1, device=cuda_device, dtype=F32)
    g = torch.empty((64, 64), device=cuda_device, dtype=BF16)
    torch.cuda.synchronize()
    n0 = lib.xclip_launch_count()
    K_ = a.shape[1]
    bad = [
        ("xclip_simreg_fwd", (a.data_ptr(), b.data_ptr(), 64, 64, K_, 1, ws.data_ptr(), None, None, 0.0)),  # off+R > C
        ("xclip_simreg_fwd", (a.data_ptr(), b.data_ptr(), 64, 64, K_, -1, ws.data_ptr(), None, None, 0.0)),
        ("xclip_simreg_fwd", (a.data_ptr() + 2, b.data_ptr(), 64, 64, K_ - 8, 0, ws.data_ptr(), None, None, 0.0)),
        ("xclip_simreg_fwd", (a.data_ptr(), b.data_ptr(), 64, 64, K_ - 4, 0, ws.data_ptr(), None, None, 0.0)),
        ("xclip_simreg_fwd", (a.data_ptr(), b.data_ptr(), 0, 64, K_, 0, ws.data_ptr(), None, None, 0.0)),
        ("xclip_simreg_bwd", (a.data_ptr(), b.data_ptr(), 64, 64, K_, 1, gs.data_ptr(), g.data_ptr(), 64)),
        ("xclip_simreg_bwd", (a.data_ptr(), b.data_ptr(), 64, 64, K_, 0, gs.data_ptr(), g.data_ptr() + 2, 64)),
        ("xclip_simreg_bwd", (a.data_ptr(), b.data_ptr(), 64, 64, K_, 0, gs.data_ptr(), g.data_ptr(), 60)),
        ("xclip_simreg_bwd", (a.data_ptr(), b.data_ptr(), 64, 64, K_, 0, None, g.data_ptr(), 64)),
        ("xclip_simreg_pack", (zrt.data_ptr() + 2, zrv.data_ptr(), 64, 768, 0, a.data_ptr())),
        ("xclip_simreg_pack", (zrt.data_ptr(), zrv.data_ptr(), 64, 764, 0, a.data_ptr())),
    ]
    for name, args in bad:
        assert getattr(lib, name)(*args, None) != 0, (name, args)
    assert lib.xclip_launch_count() == n0


LOSS_BATCHES = [2, 3, 33, 65, 257, 1000, 4096]


@pytest.mark.parametrize("dcl", [False, True])
@pytest.mark.parametrize("B", LOSS_BATCHES)
def test_contrastive_loss_with_simreg_against_fp64(cuda_device, B, dcl):
    """ContrastiveLossFn(extra, sim_reg_weight w) = contrastive + w L_sim: loss and latent gradients."""
    from x_clip_b200 import engine as E
    from oracle import clip_oracle as O
    w = 300.0
    sets = _latents(B, 4, cuda_device, seed=B + 11 * dcl)
    z = [s[0] for s in sets]
    ops = tuple((s[1], s[2]) for s in sets)
    temp = torch.tensor(1.0, device=cuda_device, dtype=F32, requires_grad=True)
    loss = E.ContrastiveLossFn.apply(z[0], z[1], z[2], z[3], temp, ops, dcl, False, w, 1.0)
    loss.backward()
    grads = [t.grad for t in z]

    z64 = [t.detach().double().requires_grad_(True) for t in z]
    t64 = torch.tensor(1.0, dtype=F64, device=cuda_device, requires_grad=True)
    cfg = O.ClipConfig(decoupled_contrastive_learning=dcl, extra_latent_projection=True)
    ref = O.contrastive_loss(z64[0], z64[1], z64[2], z64[3], t64, cfg) + w * SR.sim_reg_loss(*z64)
    ref.backward()
    loss_rel = abs(loss.item() - ref.item()) / abs(ref.item())
    grad_rel = max(((g.double() - r.grad).norm() / r.grad.norm()).item() for g, r in zip(grads, z64))
    dt_rel = abs(temp.grad.item() - t64.grad.item()) / abs(t64.grad.item())
    print(f"B={B} dcl={dcl}: loss rel {loss_rel:.2e}, grad rel {grad_rel:.2e}, dtemp rel {dt_rel:.2e}")
    assert loss_rel <= CL_LOSS_REL
    assert grad_rel <= GRAD_REL
    assert dt_rel <= DTEMP_REL                             # the term does not involve the temperature


def test_simreg_batch_one_is_nan_without_gradient(cuda_device):
    """Global batch 1: the reference's mean over no entries is NaN and sends no gradient; the
    contrastive part (and d temperature) is what it is without the term."""
    from x_clip_b200 import engine as E
    res = []
    for w in (0.0, 5.0):
        sets = _latents(1, 4, cuda_device, seed=3)
        z = [s[0] for s in sets]
        ops = tuple((s[1], s[2]) for s in sets)
        temp = torch.tensor(1.0, device=cuda_device, dtype=F32, requires_grad=True)
        loss = E.ContrastiveLossFn.apply(z[0], z[1], z[2], z[3], temp, ops, True, False, w, 1.0)
        loss.backward()
        res.append((loss.item(), temp.grad.item(), [t.grad.clone() for t in z]))
    assert math.isfinite(res[0][0]) and math.isnan(res[1][0])
    assert res[1][1] == res[0][1]
    for g1, g0 in zip(res[1][2], res[0][2]):
        assert torch.equal(g1, g0)


@pytest.mark.parametrize("W,b", [(2, 3), (3, 33), (8, 512)])
def test_rank_emulation_matches_full_batch(cuda_device, W, b):
    """Row blocks with diag_offset = rank * b emulate W ranks: the row sums of all ranks are the full
    batch's (so every rank's gathered loss is the same), and each rank's latent gradients are its rows
    of the full gradients."""
    from x_clip_b200 import kernels as K
    B, D = W * b, 512
    zrt, zct, zrv, zcv = _ops(B, D, cuda_device, seed=W * 100 + b)
    bcol = K.simreg_pack(zct, zcv, True)
    afull = K.simreg_pack(zrt, zrv, False)
    gs = torch.tensor([0.01], device=cuda_device, dtype=F32)
    rs_full = K.simreg_fwd(afull, bcol, 0)
    gfull = K.simreg_bwd(afull, bcol, 0, gs)
    hi_t, hi_v = zct[:, :D].contiguous(), zcv[:, :D].contiguous()
    pad = gfull.shape[1]

    def padded(m):
        out = torch.zeros((pad, D), device=m.device, dtype=m.dtype)
        out[:B] = m
        return out

    dt_full = K.gemm(gfull, padded(hi_t), b_major=1, out_dtype=F32)
    dv_full = K.gemm(gfull, padded(hi_v), b_major=1, out_dtype=F32, alpha=-1.0)
    parts, losses = [], []
    for r in range(W):
        a = K.simreg_pack(zrt[r * b:(r + 1) * b].contiguous(), zrv[r * b:(r + 1) * b].contiguous(), False)
        rs = K.simreg_fwd(a, bcol, r * b)
        parts.append(rs)
        g = K.simreg_bwd(a, bcol, r * b, gs)
        assert torch.equal(g, gfull[r * b:(r + 1) * b])
        dt = K.gemm(g, padded(hi_t), b_major=1, out_dtype=F32)
        dv = K.gemm(g, padded(hi_v), b_major=1, out_dtype=F32, alpha=-1.0)
        assert torch.allclose(dt, dt_full[r * b:(r + 1) * b], rtol=1e-5, atol=1e-7)
        assert torch.allclose(dv, dv_full[r * b:(r + 1) * b], rtol=1e-5, atol=1e-7)
    gathered = torch.cat(parts)
    assert torch.equal(gathered, rs_full)
    e = _e64(afull, bcol, 0)
    assert abs(gathered.double().sum().item() - (e * e).sum().item()) <= LOSS_REL * (e * e).sum().item()


SIMREG_CASES = ["tiny_simreg_extra", "tiny_simreg_dcl_extra", "vitb16_shaped_simreg_extra"]


def _clip_step(gold, dev, microbatch=None, retain="auto", cfg_over=None):
    from oracle import clip_oracle as O
    import x_clip_b200
    cfg = O.ClipConfig(**gold["cfg"])
    state = O.protocol_state_dict(cfg, gold["weight_seed"])
    text, image = O.protocol_inputs(cfg, gold["batch"], gold["input_seed"], gold["pad_fraction"])
    clip = x_clip_b200.CLIP(**gold["cfg"], sim_reg_loss_weight=gold["sim_reg_loss_weight"],
                            visual_patch_dropout=gold["patch_dropout"], microbatch=microbatch,
                            microbatch_retain=retain).to(dev)
    clip.load_state_dict(state)
    clip.train()
    loss = clip(text.to(dev), image.to(dev), return_loss=True)
    loss.backward()
    torch.cuda.synchronize()
    grads = {k: p.grad.detach().float().cpu() for k, p in clip.named_parameters() if p.grad is not None}
    return clip, loss.item(), grads, (text, image, cfg, state)


@pytest.mark.parametrize("case", SIMREG_CASES)
def test_clip_with_simreg_matches_reference(cuda_device, case):
    """End to end against the reference's fixture.  The weights put w * L_sim at twice the contrastive
    loss, and d loss / d latents is ~80x that of the contrastive loss alone (gradient norm 163 against
    ~2), so the bf16 rounding of the encoders reaches the loss amplified: the loss and gradient-norm
    gates are 1e-2 / 2e-2 relative (measured at most 4.7e-3 loss rel on an H100) instead of
    test_gpu_clip_parity's 1e-3 / 1e-2.  That this is the encoders' rounding and not the loss is checked
    on the step's own latents: fp64 contrastive + w L_sim of them equals the GPU loss to 1e-4.  d
    temperature, per-parameter cosine / norm and latent summaries keep test_gpu_clip_parity's gates."""
    from oracle import clip_oracle as O
    gold = json.loads((GOLD / f"{case}.json").read_text())
    clip, loss, grads, (text, image, cfg, state) = _clip_step(gold, cuda_device)
    with torch.no_grad():
        lat = clip(text.to(cuda_device), image.to(cuda_device), return_latents=True)
    z64 = [z.double() for z in lat]
    own = O.contrastive_loss(*z64, clip.temperature.detach().double(), cfg) \
        + gold["sim_reg_loss_weight"] * SR.sim_reg_loss(*z64)
    rel = abs(loss - gold["loss"]) / abs(gold["loss"])
    gn = torch.sqrt(sum((g.double() ** 2).sum() for g in grads.values())).item()
    print(f"{case}: loss rel {rel:.2e}, own-latent loss rel {abs(loss - own.item()) / abs(own.item()):.2e}, "
          f"grad norm rel {abs(gn - gold['grad_norm']) / gold['grad_norm']:.2e}")
    assert abs(loss - own.item()) <= 1e-4 * abs(own.item()), (loss, own.item())
    assert rel <= 1e-2, (loss, gold["loss"])
    dt = grads["temperature"].item()
    assert abs(dt - gold["dtemperature"]) <= 1e-2 * abs(gold["dtemperature"]) + 1e-3, (dt, gold["dtemperature"])
    assert abs(gn - gold["grad_norm"]) <= 2e-2 * gold["grad_norm"], (gn, gold["grad_norm"])
    for z, ref in zip(lat, gold["latents"]):
        assert list(z.shape) == ref["shape"]
        assert abs(z.double().abs().sum().item() - ref["abs_sum"]) <= 5e-3 * ref["abs_sum"]
        assert torch.allclose(z.flatten()[:8].double().cpu(), torch.tensor(ref["head"], dtype=F64), atol=2e-2)
    p = {k: v.clone().requires_grad_(True) for k, v in state.items()}
    o_loss = SR.clip_forward(p, text, image, cfg, gold["sim_reg_loss_weight"])
    o_loss.backward()
    assert abs(o_loss.item() - gold["loss"]) < 1e-5 * abs(gold["loss"])
    bad = []
    for k, g in grads.items():
        og = p[k].grad
        if k == "temperature" or og is None or og.norm().item() < 1e-3 * gold["grad_norm"]:
            continue
        cos = torch.nn.functional.cosine_similarity(g.flatten().double(), og.flatten().double(), dim=0).item()
        nrel = abs(g.norm().item() - og.norm().item()) / og.norm().item()
        if cos < 0.99 or nrel > 5e-2:
            bad.append((k, round(cos, 4), round(nrel, 4)))
    assert not bad, bad


@pytest.mark.parametrize("retain", [0, "auto"])
def test_microbatched_simreg_equals_single_pass(cuda_device, retain):
    """B = 65 in micro-batches of 32 (chunks 32, 32, 1): the term joins the in-graph loss of the
    GradCache step, which equals the single pass (the gates of test_odd_batches)."""
    gold = dict(json.loads((GOLD / "tiny_simreg_dcl_extra.json").read_text()), batch=65)
    _, loss0, grads0, _ = _clip_step(gold, cuda_device)
    clip, loss1, grads1, _ = _clip_step(gold, cuda_device, microbatch=32, retain=retain)
    assert clip.last_step_plan["chunks"] == 3, clip.last_step_plan
    assert abs(loss1 - loss0) < 1e-5 * abs(loss0), (loss1, loss0)
    assert grads1.keys() == grads0.keys()
    for k, g in grads1.items():
        ref = grads0[k]
        assert (g - ref).norm().item() <= 2e-2 * ref.norm().item() + 1e-6, k


def test_simreg_on_the_aux_path_with_mlm(cuda_device):
    """use_mlm (auxiliary-loss path, one view): the loss is cl_w * contrastive + w_mlm * mlm + w * L_sim,
    so with the same MLM corruption (same RNG state) the loss with the term minus the loss without it is
    w * L_sim of the step's latents, checked against fp64."""
    from oracle import clip_oracle as O
    import x_clip_b200
    gold = json.loads((GOLD / "tiny_simreg_extra.json").read_text())
    kw = dict(gold["cfg"], num_text_tokens=120)      # + [MASK] -> 121 rows (as test_gpu_aux)
    text, image = O.protocol_inputs(O.ClipConfig(**dict(kw, num_text_tokens=121)), 6, 11, 0.2)
    text, image = text.clamp(max=119).to(cuda_device), image.to(cuda_device)
    w = gold["sim_reg_loss_weight"]
    out = []
    for weight in (0.0, w):
        torch.manual_seed(5)                         # the same initial weights for both models
        clip = x_clip_b200.CLIP(**kw, sim_reg_loss_weight=weight, use_mlm=True, mlm_mask_token_id=2,
                                visual_patch_dropout=0.).to(cuda_device)
        clip.train()
        torch.manual_seed(6)                         # the same MLM corruption
        loss = clip(text, image, return_loss=True)
        loss.backward()
        with torch.no_grad():
            lat = clip(text, image, return_latents=True)
        out.append((loss.item(), clip.to_text_latent_extra.weight.grad.norm().item(), lat))
    term = w * SR.sim_reg_loss(*[z.double() for z in out[1][2]]).item()
    assert abs((out[1][0] - out[0][0]) - term) <= 1e-3 * term, (out[1][0] - out[0][0], term)
    assert out[1][1] > out[0][1]                   # the term's gradient reaches the extra projections


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpu_simreg_matches_reference_ranks():
    """sharded_simreg_extra: two NCCL ranks against the two gloo ranks of the reference."""
    gold = json.loads((GOLD / "sharded_simreg_extra.json").read_text())
    ctx = _mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_rank_worker, args=(r, gold, 29841, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = []
    t0 = _t.time()
    while len(res) < 2 and _t.time() - t0 < 300:
        try:
            res.append(q.get(timeout=2))
        except _q.Empty:
            if any(p.exitcode not in (None, 0) for p in procs):
                break
    for p in procs:
        p.join(timeout=60)
        if p.is_alive():
            p.terminate()
    assert len(res) == 2, "a rank died"
    res.sort()
    for (rank, loss, gn, dtemp, norms), ref in zip(res, gold["ranks"]):
        assert abs(loss - ref["loss"]) <= 1e-3 * abs(ref["loss"]), (rank, loss, ref["loss"])
        assert abs(gn - ref["grad_norm"]) <= 1.5e-2 * ref["grad_norm"], (rank, gn, ref["grad_norm"])
        assert abs(dtemp - ref["dtemperature"]) <= 1e-2 * abs(ref["dtemperature"]) + 1e-3
        for k, v in ref["grad_norms"].items():
            if v > 1e-2 * ref["grad_norm"]:
                assert abs(norms[k] - v) <= 5e-2 * v, (rank, k, norms[k], v)
    assert res[0][1] == res[1][1]                  # the same global loss on both ranks
    assert abs(res[0][3] - res[1][3]) < 1e-6


def _rank_worker(rank, gold, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    world = gold["world"]
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        from oracle import clip_oracle as O
        import x_clip_b200
        cfg = O.ClipConfig(**gold["cfg"])
        state = O.protocol_state_dict(cfg, gold["weight_seed"])
        text, image = O.protocol_inputs(cfg, world * gold["per_rank"], gold["input_seed"], gold["pad_fraction"])
        t, im = text.chunk(world)[rank].to(dev), image.chunk(world)[rank].to(dev)
        clip = x_clip_b200.CLIP(**gold["cfg"], sim_reg_loss_weight=gold["sim_reg_loss_weight"],
                                visual_patch_dropout=0.).to(dev)
        assert clip.requires_all_gather
        clip.load_state_dict(state)
        clip.train()
        loss = clip(t, im, return_loss=True)
        loss.backward()
        torch.cuda.synchronize()
        norms = {k: p.grad.double().norm().item() for k, p in clip.named_parameters() if p.grad is not None}
        gn = sum(v * v for v in norms.values()) ** 0.5
        q.put((rank, loss.item(), gn, clip.temperature.grad.item(), norms))
        dist.barrier()
    finally:
        dist.destroy_process_group()
