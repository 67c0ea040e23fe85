"""FILIP with augmented views on the H100: the view-block InfoNCE / DCL kernels against fp64,
FilipLossFn with views against the fp64 restatement of every (text view, image view) pair under forced
save plans, CLIP against the reference's goldens (tests/golden/filip_mv_*.json), and W = 2 / 3 ranks on
one GPU over gloo against the single-process fp64 loss of the global batch.

Gates are those of test_gpu_filip: the block kernels take the row gates of test_nce_rows_match_fp64,
the loss function _compare_filip's (the loss gate with an absolute floor, see _compare_mv), the model
test_gpu_clip_parity's (loss rel 1e-3, d temperature 1e-2 rel + 1e-3, gradient norm 1e-2, per-parameter
cosine >= 0.99 and norm within 5 %, per-sample image gradient cosine >= 0.99 and norm within 5 %)."""
import json
import math
import os
import time
from datetime import timedelta
from pathlib import Path

import pytest
import torch

from test_gpu_filip import _gen, _split, _unit

pytestmark = pytest.mark.gpu

F32 = torch.float32
GOLD = Path(__file__).parent / "golden"
LOSS_ORDER_REL = 1e-6                     # fp32 atomics of the loss in another order, of max(1, |loss|)


def _compare_mv(got, ref, mask, label):
    """test_gpu_filip._compare_filip's gates, with an absolute floor of 2e-5 on the loss gate: under DCL at
    a small batch the weighted sum of terms of size up to the temperature can cancel to near 0 (or is
    exactly 0 at B = 1 without DCL), while the split-bf16 rounding of the similarities moves the loss by
    an amount set by the terms, not by the total (1.2e-5 at 4 x 4 views, B = 3, DCL, temperature 100)."""
    loss, dt, grads = got
    r_loss, r_dt, r_grads = ref
    assert abs(loss - r_loss) <= 1e-5 * abs(r_loss) + 2e-5, (label, loss, r_loss)
    assert math.isfinite(dt) and abs(dt - r_dt) <= 1e-3 * abs(r_dt) + 1e-5, (label, dt, r_dt)
    worst = 0.0
    for j, (g, r) in enumerate(zip(grads, r_grads)):
        assert g is not None and torch.isfinite(g).all(), (label, j)
        rel = (g.double() - r).norm().item() / (r.norm().item() + 1e-30)
        worst = max(worst, rel)
        assert rel <= 1e-2, (label, j, rel)
        if j % 2 == 0:                                  # text latents: padded tokens get nothing
            assert not bool(g[~mask].any()), (label, j, "gradient on padded text tokens")
    print(f"filip {label}: loss {loss:.7f} vs {r_loss:.7f} dtemp {dt:.6e} vs {r_dt:.6e} grad rel {worst:.2e}")


# --------------------------------------------------------------------------- block kernels

def _block_cols(n, B, run):
    return torch.tensor([[(k // run) * n * run + j * run + k % run for k in range(B)] for j in range(n)])


def _blocks_ref(s, m, n, b, B, run, off, dcl, w, gs):
    """fp64 (lse [m b, n], per-row loss terms [m b], g [m b, n B]) of the view-block loss."""
    dev = s.device
    cols = _block_cols(n, B, run).to(dev)
    s64 = s.double()
    blk = s64[:, cols]                                              # [m b, n, B]
    rows = torch.arange(m * b, device=dev)
    pos = rows % b + off
    onehot = torch.zeros_like(blk, dtype=torch.bool)
    onehot[rows, :, pos] = True
    lse_in = blk.masked_fill(onehot, -math.inf) if dcl else blk
    lse = torch.logsumexp(lse_in, dim=-1)
    lse = torch.where(torch.isinf(lse), math.log(1e-20), lse)      # dcl at B = 1: the empty denominator
    p = torch.exp(lse_in - lse[..., None])
    wr = w.double().view(m, n)[rows // b]                           # [m b, n]
    terms = (wr * (lse - blk[rows, :, pos])).sum(dim=1)
    gb = gs * wr[..., None] * (p - onehot.double())
    g = torch.zeros((m * b, n * B), dtype=torch.float64, device=dev)
    g[:, cols.reshape(-1)] = gb.reshape(m * b, n * B)
    return lse, terms, g, gs * wr[..., None] * (2e-5 * p + 2e-6)


BLOCK_CASES = [  # (m, n, b, W): B = W b
    (1, 1, 5, 1), (1, 2, 4, 2), (2, 1, 3, 3), (2, 2, 1, 1), (2, 3, 1, 3), (4, 4, 7, 2), (4, 4, 33, 4), (3, 2, 64, 8),
]


@pytest.mark.parametrize("strided", [False, True])
@pytest.mark.parametrize("order", ["rank_major", "view_major"])
@pytest.mark.parametrize("dcl", [False, True])
@pytest.mark.parametrize("m,n,b,W", BLOCK_CASES)
def test_block_kernels_match_fp64(cuda_device, m, n, b, W, dcl, order, strided):
    """Every rank's diag_off, with and without invalid rows; logits up to 100 in magnitude; a row stride
    wider than n B.  Gates of test_nce_rows_match_fp64: |lse - ref| <= 1e-6 |ref| + 4e-6, |g - ref| <=
    gscale w (2e-5 softmax + 2e-6), the loss within the summed lse gates plus one rounding per atomic."""
    from x_clip_b200 import kernels as K
    dev = cuda_device
    B = W * b
    run = b if order == "rank_major" else B
    gen = _gen(dev, 1000 * m + 100 * n + b + W)
    scale = torch.tensor([1.0, 10.0, 100.0], device=dev)[torch.arange(m * b, device=dev) % 3]
    wide = (2 * torch.rand((m * b, n * B + (5 if strided else 0)), generator=gen, device=dev) - 1) * scale[:, None]
    s = wide[:, :n * B]
    w = torch.rand((m * n,), generator=gen, device=dev, dtype=F32) + 0.1
    gs = 0.37
    gscale = torch.tensor([gs], device=dev, dtype=F32)
    worst = [0.0, 0.0]
    for rank in range(W):
        off = rank * b
        ref_lse, terms, ref_g, g_gate = _blocks_ref(s, m, n, b, B, run, off, dcl, w, gs)
        lse_gate = 1e-6 * ref_lse.abs() + 4e-6
        for row_valid in (None, torch.arange(m * b, device=dev) % 4 != 1):
            valid = torch.ones(m * b, dtype=torch.bool, device=dev) if row_valid is None else row_valid
            loss = torch.full((1,), 0.75, device=dev, dtype=F32)
            lse = K.filip_nce_blocks_fwd(s, m, n, run, off, dcl, w, loss, row_valid=row_valid)
            e_lse = ((lse.double() - ref_lse).abs() / lse_gate)[valid].max().item()
            assert e_lse <= 1.0, e_lse
            assert bool((lse[~valid] == 0).all())
            ref_loss = 0.75 + terms[valid].sum().item()
            w_max = w.max().item()
            loss_gate = w_max * lse_gate[valid].sum().item() + m * b * n * 2.0 ** -24 * (0.75 + terms.abs().sum().item())
            assert abs(loss.item() - ref_loss) <= loss_gate, (loss.item(), ref_loss, loss_gate)

            g = K.filip_nce_blocks_bwd(s, lse, m, n, run, off, dcl, w, gscale, row_valid=row_valid)
            cols = _block_cols(n, B, run).to(dev).reshape(-1)
            e_g = ((g.double() - ref_g)[:, cols].view(m * b, n, B).abs() / g_gate)[valid].max().item()
            assert e_g <= 1.0, e_g
            assert bool((g[~valid] == 0).all())
            worst = [max(worst[0], e_lse), max(worst[1], e_g)]
    print(f"nce_blocks m={m} n={n} b={b} W={W} dcl={dcl} {order} strided={strided}: "
          f"error/gate lse {worst[0]:.3f} g {worst[1]:.3f}")


@pytest.mark.parametrize("dcl", [False, True])
@pytest.mark.parametrize("R,C,where", [(5, 31, "first"), (13, 33, "middle"), (29, 256, "last"), (256, 2048, "last")])
def test_block_kernels_at_one_view_equal_the_single_view_kernels(cuda_device, R, C, where, dcl):
    """m = n = 1: lse and g bit for bit those of filip_nce_fwd / filip_nce_bwd (block weight 1 and the
    same gscale), the loss within the reordering of the fp32 atomics."""
    from x_clip_b200 import kernels as K
    from test_gpu_filip import _nce_case
    dev = cuda_device
    off = {"first": 0, "middle": (C - R) // 2, "last": C - R}[where]
    s = _nce_case(dev, R, C, R * 31 + C)
    s_blk = torch.zeros((R, C), device=dev, dtype=F32)
    s_blk[:, :] = s
    gscale = torch.tensor([0.37], device=dev, dtype=F32)
    one = torch.ones(1, device=dev, dtype=F32)
    for row_valid in (None, torch.arange(R, device=dev) % 3 != 2):
        l0 = torch.zeros(1, device=dev, dtype=F32)
        l1 = torch.zeros(1, device=dev, dtype=F32)
        lse0 = K.filip_nce_fwd(s, off, dcl, l0, 1.0, row_valid=row_valid)
        lse1 = K.filip_nce_blocks_fwd(s_blk, 1, 1, C, off, dcl, one, l1, row_valid=row_valid)
        assert torch.equal(lse0, lse1.view(-1))
        assert abs(l0.item() - l1.item()) <= 1e-6 * abs(l0.item()) + 1e-6
        g0 = K.filip_nce_bwd(s, lse0, off, dcl, gscale, row_valid=row_valid)
        g1 = K.filip_nce_blocks_bwd(s_blk, lse1, 1, 1, C, off, dcl, one, gscale, row_valid=row_valid)
        assert torch.equal(g0, g1)


# --------------------------------------------------------------------------- the loss function

def _views(dev, m, n, B, T, I, D, extra, seed, empty=()):
    """Per view fp32 unit latents and per text view masks of mixed lengths; `empty` = (view, row) pairs
    of captions made only of padding."""
    gen = _gen(dev, seed)
    zt = [_unit((B, T, D), gen, dev) for _ in range(m)]
    zi = [_unit((B, I, D), gen, dev) for _ in range(n)]
    ztx = [_unit((B, T, D), gen, dev) for _ in range(m)] if extra else None
    zix = [_unit((B, I, D), gen, dev) for _ in range(n)] if extra else None
    masks = []
    for i in range(m):
        lens = torch.randint(1, T + 1, (B,), generator=gen, device=dev)
        lens[i % B] = T
        masks.append(torch.arange(T, device=dev)[None, :] < lens[:, None])
    for v, row in empty:
        masks[v][row] = False
    return zt, zi, ztx, zix, masks


def _stack(views, rows):
    return None if views is None else torch.cat([v[rows] for v in views]).contiguous()


def _run_mv(zt, zi, ztx, zix, masks, temperature, dcl, weights, rows=slice(None), use_gather=False, stats=None):
    """FilipLossFn with views on rows `rows` of every view -> (loss, d temperature, [d zt, d zi(, d ztx, d zix)]
    each [views * rows, tokens, D])."""
    from x_clip_b200.filip import FilipLossFn
    lat = [_stack(zt, rows), _stack(zi, rows)]
    if ztx is not None:
        lat += [_stack(ztx, rows), _stack(zix, rows)]
    z = [t.clone().requires_grad_(True) for t in lat]
    ops = tuple(_split(t) for t in lat)
    temp = torch.tensor(temperature, device=lat[0].device, dtype=F32, requires_grad=True)
    mask = torch.cat([mk[rows] for mk in masks]).contiguous()
    extra = ztx is not None
    loss = FilipLossFn.apply(z[0], z[1], z[2] if extra else None, z[3] if extra else None, temp, ops, mask, dcl,
                             use_gather, stats, (len(zt), len(zi)), weights)
    loss.backward()
    return loss.item(), temp.grad.item(), [t.grad for t in z]


def _oracle_mv(zt, zi, ztx, zix, masks, temperature, dcl, weights):
    """fp64 autograd of cl_w L[0, 0] + mv_w mean(others) with oracle.contrastive_loss per pair; gradients
    stacked like _run_mv's."""
    from oracle import clip_oracle as O
    from test_gpu_filip import _oracle_cfg
    extra = ztx is not None
    d = lambda vs: None if vs is None else [v.detach().double().requires_grad_(True) for v in vs]
    zt, zi, ztx, zix = d(zt), d(zi), d(ztx), d(zix)
    t64 = torch.tensor(temperature, dtype=F32).double().to(zt[0].device).requires_grad_(True)
    cfg = _oracle_cfg(dcl, extra)
    losses = [O.contrastive_loss(zt[i], zi[j], ztx[i] if extra else zt[i], zix[j] if extra else zi[j], t64, cfg,
                                 masks[i]) for i in range(len(zt)) for j in range(len(zi))]
    loss = weights[0] * losses[0] + weights[1] * torch.stack(losses[1:]).mean()
    loss.backward()
    grads = [torch.cat([v.grad for v in zt]), torch.cat([v.grad for v in zi])]
    if extra:
        grads += [torch.cat([v.grad for v in ztx]), torch.cat([v.grad for v in zix])]
    return loss.item(), t64.grad.item(), grads


MV_SHAPES = [  # (m, n, B, T, I, D, empty)
    (1, 2, 5, 48, 144, 256, ()), (2, 1, 6, 16, 16, 256, ((1, 2),)), (2, 2, 5, 48, 144, 256, ((1, 0),)),
    (3, 2, 8, 80, 16, 128, ((2, 3), (2, 4))), (4, 4, 3, 7, 9, 128, ()), (2, 2, 1, 16, 16, 128, ()),
]


@pytest.mark.parametrize("extra", [False, True])
@pytest.mark.parametrize("dcl", [False, True])
@pytest.mark.parametrize("m,n,B,T,I,D,empty", MV_SHAPES)
def test_multiview_loss_matches_fp64(cuda_device, monkeypatch, m, n, B, T, I, D, empty, dcl, extra):
    """Nothing saved, everything saved and half saved, with a chunk budget that cuts each pass into
    several chunks: the same loss (up to the order of the fp32 atomics), and every plan within
    _compare_filip's gates of the fp64 restatement."""
    from x_clip_b200 import filip
    zt, zi, ztx, zix, masks = _views(cuda_device, m, n, B, T, I, D, extra, seed=m * 100 + n * 10 + B, empty=empty)
    weights = (0.9, 0.1)
    ref = _oracle_mv(zt, zi, ztx, zix, masks, math.log(100.0), dcl, weights)
    total = filip.saved_bytes(B, B, T, I, m, n)
    monkeypatch.setattr(filip, "FILIP_CHUNK_BYTES", 48 * max(T, I) * B * max(m, n))
    got = {}
    for plan, save in (("none", 0), ("part", total // 2), ("all", total)):
        monkeypatch.setattr(filip, "FILIP_SAVE_BYTES", save)
        stats = {}
        got[plan] = _run_mv(zt, zi, ztx, zix, masks, math.log(100.0), dcl, weights, stats=stats)
        assert stats["saved_bytes"] <= save and (plan != "all" or stats["saved_bytes"] == total), (plan, stats)
        assert stats["chunks"] > 2 or B == 1, stats
    for plan in ("none", "part"):
        assert abs(got[plan][0] - got["all"][0]) <= LOSS_ORDER_REL * max(1.0, abs(got["all"][0])), (plan, got[plan][0],
                                                                                          got["all"][0])
    mask = torch.cat(masks)
    for plan, g in got.items():
        _compare_mv(g, ref, mask, f"multiview plan={plan} m={m} n={n} {B}x{T}x{I}x{D} empty={empty} "
                       f"dcl={dcl} extra={extra}")


# --------------------------------------------------------------------------- CLIP against the reference

MV_GOLDEN = ["filip_mv_t1i2", "filip_mv_t2i1", "filip_mv_t2i2", "filip_mv_t2i2_dcl_extra", "filip_mv_t3i2_empty",
             "filip_mv_t48_i144_dcl_extra", "filip_mv_imggrad_dcl_extra"]


@pytest.mark.parametrize("case", MV_GOLDEN)
def test_clip_multiview_filip_matches_reference(cuda_device, case):
    from oracle import clip_oracle as O
    import x_clip_b200
    import filip_multiview_oracle as FMV
    from golden.make_golden_filip_multiview import view_inputs
    gold = json.loads((GOLD / f"{case}.json").read_text())
    cfg = O.ClipConfig(**gold["cfg"])
    state = O.protocol_state_dict(cfg, gold["weight_seed"])
    texts, images = view_inputs(cfg, gold["batch"], gold["pad_fraction"], gold["n_text_views"],
                                gold["n_image_views"], [tuple(e) for e in gold["empty"]])
    image_grad = "images" in gold
    clip = x_clip_b200.CLIP(**gold["cfg"], visual_patch_dropout=0.).to(cuda_device)
    clip.load_state_dict(state, strict=False)
    clip.train()
    ims = [im.to(cuda_device).requires_grad_(image_grad) for im in images]
    tx = [t.to(cuda_device) for t in texts]
    loss = clip(tx[0], ims[0], return_loss=True, aug_text=tuple(tx[1:]) or None, aug_image=tuple(ims[1:]) or None)
    loss.backward()
    torch.cuda.synchronize()
    grads = {k: q.grad.detach().double().cpu() for k, q in clip.named_parameters() if q.grad is not None}

    p = {k: v.clone().requires_grad_(True) for k, v in state.items()}
    o_ims = [im.clone().requires_grad_(image_grad) for im in images]
    o_loss = FMV.clip_forward_filip_multiview(p, texts, o_ims, cfg, gold["multiview_loss_weight"])
    o_loss.backward()
    assert abs(o_loss.item() - gold["loss"]) <= 3e-6 * max(1.0, abs(gold["loss"]))   # oracle == reference

    rel = abs(loss.item() - gold["loss"]) / abs(gold["loss"])
    assert rel <= 1e-3, (loss.item(), gold["loss"])
    dt = grads["temperature"].item()
    assert abs(dt - gold["dtemperature"]) <= 1e-2 * abs(gold["dtemperature"]) + 1e-3, (dt, gold["dtemperature"])
    gn = torch.sqrt(sum((g ** 2).sum() for g in grads.values())).item()
    assert abs(gn - gold["grad_norm"]) <= 1e-2 * gold["grad_norm"], (gn, gold["grad_norm"])
    has = lambda g: g is not None and bool(g.ne(0).any())
    assert {k for k, g in grads.items() if has(g)} == {k for k, q in p.items() if has(q.grad)}
    bad, worst = [], 1.0
    for k, g in grads.items():
        og = p[k].grad
        if k == "temperature" or og is None or og.norm().item() < 1e-3 * gold["grad_norm"]:
            continue
        cos = torch.nn.functional.cosine_similarity(g.flatten(), og.flatten().double(), dim=0).item()
        nrel = abs(g.norm().item() - og.norm().item()) / og.norm().item()
        worst = min(worst, cos)
        if cos < 0.99 or nrel > 5e-2:
            bad.append((k, round(cos, 4), round(nrel, 4)))
    assert not bad, bad
    if image_grad:
        for v, (im, og) in enumerate(zip(ims, o_ims)):
            got, ref = im.grad.detach().double().cpu(), og.grad.double()
            assert torch.allclose(ref.flatten(1).norm(dim=1), torch.tensor(gold["images"][v]["sample_norms"],
                                                                          dtype=torch.float64), rtol=2e-4)
            for b in range(got.shape[0]):
                cos = torch.nn.functional.cosine_similarity(got[b].flatten(), ref[b].flatten(), dim=0).item()
                nrel = abs(got[b].norm().item() - ref[b].norm().item()) / ref[b].norm().item()
                assert cos >= 0.99 and nrel <= 5e-2, (v, b, cos, nrel)
    print(f"{case}: loss rel {rel:.2e} dtemp {dt:.6f} vs {gold['dtemperature']:.6f} min cosine {worst:.5f}")


# --------------------------------------------------------------------------- W ranks on one GPU

RANK_CASES = {  # world -> (m, n, b, T, I, D, extra, dcl, empty (view, global row))
    2: (2, 2, 3, 48, 144, 256, True, True, ((1, 4),)),
    3: (2, 3, 2, 16, 16, 128, False, False, ((1, 1),)),
}
GROUP_TIMEOUT = 200


def _rank_inputs(world, dev):
    m, n, b, T, I, D, extra, dcl, empty = RANK_CASES[world]
    return _views(dev, m, n, world * b, T, I, D, extra, seed=4242 + world, empty=empty), (m, n, b, extra, dcl)


def _rank_worker(world, rank, rdzv, out, ppid):
    from test_gpu_multirank_fp64 import _collectives, _exit_with_parent
    _exit_with_parent(ppid)
    os.environ["GLOO_SOCKET_IFNAME"] = "lo"
    import torch.distributed as dist
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    dist.init_process_group("gloo", init_method=f"file://{rdzv}", rank=rank, world_size=world,
                            timeout=timedelta(seconds=120))
    try:
        path = _collectives(world, dev)
        (zt, zi, ztx, zix, masks), (m, n, b, extra, dcl) = _rank_inputs(world, dev)
        rows = slice(rank * b, (rank + 1) * b)
        got = _run_mv(zt, zi, ztx, zix, masks, math.log(100.0), dcl, (0.9, 0.1), rows=rows, use_gather=True)
        torch.save(dict(loss=got[0], dtemp=got[1], grads=[g.cpu() for g in got[2]], collectives=path),
                   os.path.join(out, f"r{rank}.pt"))
        dist.barrier()
    except BaseException:
        import traceback
        with open(os.path.join(out, f"error.r{rank}.txt"), "w") as f:
            f.write(traceback.format_exc())
        raise
    finally:
        dist.destroy_process_group()


def _run_ranks(world, out):
    """The W workers, always joined, terminated or killed (test_gpu_multirank_fp64's discipline)."""
    import torch.multiprocessing as mp
    procs = [mp.get_context("spawn").Process(target=_rank_worker, args=(world, r, str(out / "rdzv"), str(out),
                                                                        os.getpid()), daemon=True) for r in range(world)]
    t0 = time.time()
    try:
        for p in procs:
            p.start()
        while time.time() - t0 < GROUP_TIMEOUT and any(p.is_alive() for p in procs) \
                and not any(p.exitcode not in (None, 0) for p in procs):
            time.sleep(0.2)
    finally:
        for p in procs:
            for stop in (lambda: None, p.terminate, p.kill):
                if p.is_alive():
                    stop()
                    p.join(timeout=10)
    assert not any(p.is_alive() for p in procs), "a worker outlived its group"
    msg = "\n".join(f.read_text() for f in out.glob("error.r*.txt"))
    assert all(p.exitcode == 0 for p in procs), f"exit codes {[p.exitcode for p in procs]}\n{msg}"
    return [torch.load(out / f"r{r}.pt") for r in range(world)]


@pytest.mark.parametrize("world", sorted(RANK_CASES))
def test_ranks_match_the_single_process_fp64_loss(cuda_device, tmp_path, world):
    """Each rank holds rows [r b, (r+1) b) of every view: ONE all-gather of the n stacked image views,
    rank-major columns, positives at r n b + j b + x, one reduce-scatter of the image-token gradients.
    Every rank's loss and d temperature against the fp64 loss of the global batch (bit-identical loss
    on every rank), and its rows of every latent gradient against the fp64 gradient's."""
    saved = _run_ranks(world, tmp_path)
    (zt, zi, ztx, zix, masks), (m, n, b, extra, dcl) = _rank_inputs(world, cuda_device)
    loss, dt, grads = _oracle_mv(zt, zi, ztx, zix, masks, math.log(100.0), dcl, (0.9, 0.1))
    B = world * b
    for r, got in enumerate(saved):
        assert got["loss"] == saved[0]["loss"], (r, got["loss"], saved[0]["loss"])
        local = []
        for j, g in enumerate(grads):
            views = m if j % 2 == 0 else n
            local.append(torch.cat([g[v * B + r * b:v * B + (r + 1) * b] for v in range(views)]))
        mask = torch.cat([mk[r * b:(r + 1) * b] for mk in masks])
        _compare_mv((got["loss"], got["dtemp"], [g.to(cuda_device) for g in got["grads"]]),
                    (loss, dt, local), mask, f"W={world} rank {r} ({got['collectives']} collectives)")
