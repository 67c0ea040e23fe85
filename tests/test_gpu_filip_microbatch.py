"""FILIP at large batch: the compact (16-bit) argmax kernels, FilipLossFn under every save plan, its
peak memory with nothing saved, and the micro-batched CLIP step with use_all_token_embeds=True."""
import json
import math
import os
from pathlib import Path

import pytest
import torch

from test_gpu_filip import (_col_mask_tables, _compare_filip, _filip_inputs, _gen, _oracle_filip, _run_segmax,
                            _split, _unit, oracle_filip_chunked)

pytestmark = pytest.mark.gpu
BF16, F32 = torch.bfloat16, torch.float32
GOLD = Path(__file__).parent / "golden"


# --------------------------------------------------------------------------- kernels

@pytest.mark.parametrize("seg_len,nseg,masked", [(1, 300, False), (7, 40, True), (8, 33, False),
                                                 (98, 9, True), (256, 3, False), (577, 2, True)])
def test_segmax16_outputs_match_fp64_and_each_other(cuda_device, seg_len, nseg, masked):
    """The full call against fp64 (_run_segmax), then the partial calls: the argmax alone
    (want_max=False), the maximum alone (seg_arg=False) and the argmax written into a given buffer
    (seg_arg=into) equal the full call bit for bit."""
    from x_clip_b200 import kernels as K
    dev = cuda_device
    gen = _gen(dev, seg_len)
    R, D = 333, 128
    za, zb = _unit((R, D), gen, dev), _unit((nseg * seg_len, D), gen, dev)
    cm = ca = None
    if masked:
        mask = torch.rand(nseg * seg_len, generator=gen, device=dev) < 0.7
        mask.view(nseg, seg_len)[0] = False                  # a segment with every column masked
        cm, ca = _col_mask_tables(mask)
    m, arg, _, _ = _run_segmax(za, zb, 2.5, seg_len, cm, ca)
    a_row, _ = _split(za)
    _, b_col = _split(zb)
    t = torch.tensor([2.5], device=dev, dtype=F32)
    _, a_only = K.filip_segmax16(a_row, b_col, t, seg_len, cm, ca, want_max=False)
    m_only, none = K.filip_segmax16(a_row, b_col, t, seg_len, cm, ca, seg_arg=False)
    assert none is None and torch.equal(a_only.to(torch.int32) & 0xFFFF, arg)
    assert torch.equal(m_only.view(torch.int32), m.view(torch.int32))
    into = torch.full((R, nseg), -1, device=dev, dtype=torch.int16)
    K.filip_segmax16(a_row, b_col, t, seg_len, cm, ca, seg_arg=into)
    assert torch.equal(into, a_only)


@pytest.mark.parametrize("seg_len", [1, 7, 8, 98, 256, 577])
def test_expand16_window_matches_dense_construction(cuda_device, seg_len):
    """Random argmax, weights with zeros (masked rows and samples), windows at row0 > 0 and a row stride
    ldg > C, over a buffer of random bits: columns [0, C) equal G built densely in torch, the pad
    columns [C, roundup8(C)) are zero and columns [roundup8(C), ldg) keep their random bits."""
    from x_clip_b200 import _lib
    dev = cuda_device
    gen = _gen(dev, 100 + seg_len)
    samples, rps, nseg = 6, 13, 5
    R, C = samples * rps, nseg * seg_len
    arg16 = torch.randint(0, seg_len, (R, nseg), generator=gen, device=dev, dtype=torch.int16)
    wmat = torch.randn((samples, nseg), generator=gen, device=dev)
    wmat[1, 2] = 0.0
    rowscale = torch.rand(R, generator=gen, device=dev)
    rowscale[rps:2 * rps:3] = 0.0                             # masked text tokens
    t = torch.tensor([3.0], device=dev, dtype=F32)
    C8 = (C + 7) // 8 * 8
    ldg = C8 + 24
    for row0, rows in ((0, R), (5, 40), (R - 1, 1)):
        fill = torch.randint(-2 ** 15, 2 ** 15, (rows, ldg), generator=gen, device=dev, dtype=torch.int16)
        g = fill.clone().view(BF16)
        _lib.call("xclip_filip_expand16", arg16[row0:row0 + rows].data_ptr(), wmat.data_ptr(), rowscale.data_ptr(),
                  t.data_ptr(), row0, rows, rps, seg_len, nseg, g.data_ptr(), ldg, None)
        torch.cuda.synchronize()
        r = torch.arange(row0, row0 + rows, device=dev)
        w = wmat[r // rps] * rowscale[r, None]
        want = torch.zeros((rows, C), device=dev, dtype=BF16)
        cols = torch.arange(nseg, device=dev)[None, :] * seg_len + arg16[row0:row0 + rows].long()
        want.scatter_(1, cols, torch.where(w != 0, w * t, 0.0).to(BF16))     # a zero weight writes +0
        assert torch.equal(g[:, :C].view(torch.int16), want.view(torch.int16)), (seg_len, row0, rows)
        assert not bool(g[:, C:C8].view(torch.int16).any()), (seg_len, row0, rows)
        assert torch.equal(g[:, C8:].view(torch.int16), fill[:, C8:]), (seg_len, row0, rows)
        assert int((g[:, :C].float() != 0).sum()) > 0


# --------------------------------------------------------------------------- the loss under each plan

# The loss adds its rows with fp32 atomics (xclip_filip_nce_fwd), so two runs of one plan may differ in
# its last bits.  What the plan could change is upstream of that sum: the [b, B] similarity matrices and
# their row log-sum-exps, which are compared bit for bit; the loss itself within LOSS_ORDER_REL.
LOSS_ORDER_REL = 1e-6


def _recording_nce(monkeypatch):
    """Record (similarity matrix, lse) of every filip_nce_fwd call."""
    from x_clip_b200 import kernels as K
    seen, real = [], K.filip_nce_fwd

    def rec(s, *a, **kw):
        lse = real(s, *a, **kw)
        seen.append((s.clone(), lse.clone()))
        return lse
    monkeypatch.setattr(K, "filip_nce_fwd", rec)
    return seen


def _assert_same_matrices(a, b, label):
    assert len(a) == len(b), label
    for (s0, l0), (s1, l1) in zip(a, b):
        assert torch.equal(s0.view(torch.int32), s1.view(torch.int32)), label
        assert torch.equal(l0.view(torch.int32), l1.view(torch.int32)), label


def _loss_under_plans(monkeypatch, lat, mask, temperature, dcl, chunk_bytes):
    from x_clip_b200 import filip
    from test_gpu_filip import _run_filip_loss
    b, T = mask.shape
    I = lat[1].shape[1]
    total = filip.saved_bytes(b, b, T, I)
    monkeypatch.setattr(filip, "FILIP_CHUNK_BYTES", chunk_bytes)
    seen = _recording_nce(monkeypatch)
    out, mats = {}, {}
    for plan, save in (("none", 0), ("part", total // 2), ("all", total)):
        monkeypatch.setattr(filip, "FILIP_SAVE_BYTES", save)
        seen.clear()
        out[plan] = _run_filip_loss(lat, mask, temperature, dcl)
        mats[plan] = list(seen)
    _assert_same_matrices(mats["none"], mats["all"], "none vs all")
    _assert_same_matrices(mats["part"], mats["all"], "part vs all")
    return out


@pytest.mark.parametrize("extra", [False, True])
@pytest.mark.parametrize("dcl", [False, True])
@pytest.mark.parametrize("B,T,I,D,empty", [(9, 7, 9, 128, (4,)), (12, 77, 98, 256, (2,)), (5, 48, 144, 256, ())])
def test_loss_is_plan_independent_and_matches_fp64(cuda_device, monkeypatch, B, T, I, D, empty, dcl, extra):
    lat, mask = _filip_inputs(cuda_device, B, T, I, D, extra, seed=B + T + I, empty=empty)
    # a budget that cuts each pass into several chunks at these sizes
    res = _loss_under_plans(monkeypatch, lat, mask, math.log(100.0), dcl, chunk_bytes=48 * max(T, I) * B)
    ref = _oracle_filip(lat, mask, math.log(100.0), dcl)
    losses = {p: r[0] for p, r in res.items()}
    for p in ("none", "part"):
        assert abs(losses[p] - losses["all"]) <= LOSS_ORDER_REL * abs(losses["all"]), losses
    for plan, got in res.items():
        _compare_filip(got, ref, lat, mask, f"plan={plan} {B}x{T}x{I}x{D} empty={empty} dcl={dcl} extra={extra}")


def test_loss_cfg3_tokens_save_nothing_matches_fp64(cuda_device, monkeypatch):
    """cfg3's 77 x 196 token counts at b = 256 with nothing saved and a 32 MiB chunk budget, which cuts
    pass A into 4 and pass B into 7 chunks; against the chunked fp64 reference."""
    from x_clip_b200 import filip
    lat, mask = _filip_inputs(cuda_device, 256, 77, 196, 512, False, seed=777, empty=(5,))
    monkeypatch.setattr(filip, "FILIP_CHUNK_BYTES", 32 << 20)
    monkeypatch.setattr(filip, "FILIP_SAVE_BYTES", 0)
    from test_gpu_filip import _run_filip_loss
    seen = _recording_nce(monkeypatch)
    got = _run_filip_loss(lat, mask, math.log(100.0), False)
    none = list(seen)
    seen.clear()
    monkeypatch.setattr(filip, "FILIP_SAVE_BYTES", None)
    assert abs(_run_filip_loss(lat, mask, math.log(100.0), False)[0] - got[0]) <= LOSS_ORDER_REL * abs(got[0])
    _assert_same_matrices(none, seen, "nothing saved vs the free-HBM plan")
    ref = oracle_filip_chunked(lat, mask, math.log(100.0), False)
    _compare_filip(got, ref, lat, mask, "cfg3 tokens, nothing saved")


def test_peak_memory_with_nothing_saved(cuda_device, monkeypatch):
    """b = 256, 77 x 196, D = 512, nothing saved: the loss's peak allocation beyond its inputs stays under
    the chunk budget + the [b, B] matrices + the gradient outputs.  The unchunked schedule's figure,
    computed from shapes (8 B of saved max + argmax per entry, 8 B of keys per entry of the larger pass),
    is over that bound."""
    from x_clip_b200 import filip
    b, T, I, D = 256, 77, 196, 512
    budget = 32 << 20
    lat, mask = _filip_inputs(cuda_device, b, T, I, D, False, seed=5)
    z = [t.clone().requires_grad_(True) for t in lat]
    ops = tuple(_split(t) for t in lat)
    temp = torch.tensor(math.log(100.0), device=cuda_device, dtype=F32, requires_grad=True)
    monkeypatch.setattr(filip, "FILIP_CHUNK_BYTES", budget)
    monkeypatch.setattr(filip, "FILIP_SAVE_BYTES", 0)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    stats = {}
    loss = filip.FilipLossFn.apply(z[0], z[1], None, None, temp, ops, mask.contiguous(), False, False, stats)
    loss.backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    rows = b * T + b * I
    state = 8 * b * b * 4                                   # t2i, i2t, lse, g_t, g_i and its transpose
    grads = 2 * rows * D * 4                                 # d rows / d cols of both passes
    small = 4 * (4 * b * T + b * I) + (4 << 20)              # token weights, column masks, allocator rounding
    bound = budget + state + grads + small
    unchunked = 8 * (b * T * b + b * I * b) + 8 * b * I * b + state + grads
    print(f"peak {peak / 2**20:.1f} MiB, bound {bound / 2**20:.1f} MiB, unchunked {unchunked / 2**20:.1f} MiB, {stats}")
    assert stats["rows_saved"] == 0 and stats["rows_recomputed"] == rows
    assert peak <= bound
    assert unchunked > bound


# --------------------------------------------------------------------------- the micro-batched step

def _clip_case(case, dev, patch_dropout=0.0, **kw):
    from oracle import clip_oracle as O
    import x_clip_b200
    gold = json.loads((GOLD / f"{case}.json").read_text())
    cfg = O.ClipConfig(**gold["cfg"])
    state = O.protocol_state_dict(cfg, gold["weight_seed"])
    text, image = O.protocol_inputs(cfg, gold["batch"], gold["input_seed"], gold["pad_fraction"])
    clip = x_clip_b200.CLIP(**gold["cfg"], visual_patch_dropout=patch_dropout, **kw).to(dev)
    clip.load_state_dict(state, strict=False)
    clip.train()
    return gold, clip, text.to(dev), image.to(dev)


def _step(clip, text, image, image_grad=False, seed=None):
    for p in clip.parameters():
        p.grad = None
    if seed is not None:
        torch.manual_seed(seed)
    img = image.clone().requires_grad_(True) if image_grad else image
    loss = clip(text, img, return_loss=True)
    loss.backward()
    grads = {k: p.grad.clone() for k, p in clip.named_parameters() if p.grad is not None}
    return loss.item(), grads, (img.grad.clone() if image_grad else None)


def _assert_same_step(got, ref, label):
    """The gates of test_microbatched_step_equals_single_pass: loss within 1e-5, every parameter gradient
    (temperature included) within 2e-2 of its norm; the image gradient likewise."""
    assert abs(got[0] - ref[0]) < 1e-5, (label, got[0], ref[0])
    assert got[1].keys() == ref[1].keys(), label
    for k, g in got[1].items():
        r = ref[1][k]
        assert (g - r).norm().item() <= 2e-2 * r.norm().item() + 1e-6, (label, k)
    if ref[2] is not None:
        assert (got[2] - ref[2]).norm().item() <= 2e-2 * ref[2].norm().item() + 1e-6, label


@pytest.mark.parametrize("case", ["tiny_filip", "tiny_filip_dcl_extra", "vits16_filip", "filip_t48_i144_dcl_extra"])
def test_microbatched_filip_step_equals_single_pass(cuda_device, case):
    gold, clip, text, image = _clip_case(case, cuda_device, patch_dropout=gold_dropout(case))
    pd = clip.visual_transformer.patch_dropout
    if gold["keep"] is not None:
        # one kept set for every sample, so the same pin serves the whole batch and every chunk
        row = torch.tensor(gold["keep"])[:1]
        pd.forced_keep = row.repeat(text.shape[0], 1)
    single = _step(clip, text, image, image_grad=True)
    if gold["keep"] is None:
        assert abs(single[0] - gold["loss"]) <= 1e-3 * abs(gold["loss"]), (single[0], gold["loss"])
    clip.microbatch = 2
    for retain in (0, 1, "auto"):
        clip.microbatch_retain = retain
        if gold["keep"] is not None:
            pd.forced_keep = row.repeat(2, 1)
        got = _step(clip, text, image, image_grad=True)
        plan = clip.last_step_plan
        chunks = -(-text.shape[0] // 2)
        assert plan["chunks"] == chunks and plan["retained"] == {0: 0, 1: 1, "auto": chunks}[retain], plan
        assert plan["filip"]["rows_saved"] + plan["filip"]["rows_recomputed"] > 0, plan
        _assert_same_step(got, single, f"{case} retain={retain}")
        if gold["keep"] is None:
            assert abs(got[0] - gold["loss"]) <= 1e-3 * abs(gold["loss"]), (got[0], gold["loss"])


def gold_dropout(case):
    return json.loads((GOLD / f"{case}.json").read_text())["patch_dropout"]


def test_microbatched_filip_step_replays_patch_dropout(cuda_device, monkeypatch):
    """Patch dropout 0.5 drawn per chunk: retain 0 / 1 / auto (re-encoded or kept chunks) give the same
    similarity matrices bit for bit, the same loss and the same gradients, with nothing saved in the loss
    as with everything saved."""
    from x_clip_b200 import filip
    gold, clip, text, image = _clip_case("filip_t48_i144_dcl_extra", cuda_device, patch_dropout=0.5, microbatch=2)
    out, mats = [], []
    seen = _recording_nce(monkeypatch)
    for retain, save in ((0, None), (1, None), ("auto", None), ("auto", 0)):
        clip.microbatch_retain = retain
        monkeypatch.setattr(filip, "FILIP_SAVE_BYTES", save)
        seen.clear()
        out.append(_step(clip, text, image, image_grad=True, seed=11))
        mats.append(list(seen))
    for o, m in zip(out[1:], mats[1:]):
        _assert_same_matrices(m, mats[0], "patch dropout replay")
        _assert_same_step(o, out[0], "patch dropout replay")


def test_filip_microbatch_dispatch_fills_the_plan(cuda_device):
    """use_all_token_embeds=True with microbatch set takes the micro-batched step: its plan is filled in
    and covers every token row of both FILIP passes."""
    gold, clip, text, image = _clip_case("tiny_filip", cuda_device, microbatch=3)
    with torch.no_grad():
        zt, zi = clip(text, image, return_latents=True)
    clip.last_step_plan = None
    _step(clip, text, image)
    plan = clip.last_step_plan
    assert plan is not None and plan["chunks"] == 2 and plan["loss_reserve_bytes"] > 0, plan
    b, T, I = zt.shape[0], zt.shape[1], zi.shape[1]
    assert plan["filip"]["rows_saved"] + plan["filip"]["rows_recomputed"] == b * T + b * I, plan


def _mb_filip_worker(rank, world, case, port, q):
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        from oracle import clip_oracle as O
        import x_clip_b200
        gold = json.loads((GOLD / f"{case}.json").read_text())
        cfg = O.ClipConfig(**gold["cfg"])
        state = O.protocol_state_dict(cfg, gold["weight_seed"])
        text, image = O.protocol_inputs(cfg, gold["batch"], gold["input_seed"], gold["pad_fraction"])
        t, im = text.chunk(world)[rank].to(dev), image.chunk(world)[rank].to(dev)
        res = []
        for mb in (None, 1):
            clip = x_clip_b200.CLIP(**gold["cfg"], visual_patch_dropout=0., microbatch=mb).to(dev)
            clip.load_state_dict(state)
            clip.train()
            loss = clip(t, im, return_loss=True)
            loss.backward()
            res.append((loss.item(), {k: p.grad.cpu() for k, p in clip.named_parameters() if p.grad is not None},
                        mb is None or "filip" in clip.last_step_plan))
        q.put((rank, res[0][0], res[1][0], res[1][2], _max_rel(res[1][1], res[0][1])))
        dist.barrier()
    finally:
        dist.destroy_process_group()


def _max_rel(got, ref):
    """Largest |g - r| / (2e-2 |r| + 1e-6) over the parameters: <= 1 passes the step gate."""
    assert got.keys() == ref.keys()
    return max((got[k] - ref[k]).norm().item() / (2e-2 * ref[k].norm().item() + 1e-6) for k in ref)


@pytest.mark.parametrize("case", ["tiny_filip", "tiny_filip_dcl_extra"])
def test_two_gpu_microbatched_filip_equals_single_pass(case):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import queue as _q
    import time as _t
    import torch.multiprocessing as mp
    gold = json.loads((GOLD / f"{case}.json").read_text())
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_mb_filip_worker, args=(r, 2, case, 29831, q)) for r in range(2)]
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
    for rank, single, micro, ran_chunked, rel in res:
        assert ran_chunked, rank
        assert abs(micro - single) < 1e-5 and abs(micro - gold["loss"]) <= 1e-3 * abs(gold["loss"]), (rank, micro)
        assert rel <= 1.0, (rank, rel)
