"""Logits + InfoNCE/DCL kernels (csrc/nce.cu, EPI_NCE_FWD / EPI_NCE_BWD) against restatements of
x_clip/x_clip.py:813-847 in fp32 and in fp64.

The fp64 references start from the exact bf16 operands the kernels read: the split-bf16 row form
[hi|lo|hi] and column form [hi|hi|lo] that K.l2norm_fwd makes from fp32 latents (K = 3 * dim_latent),
or plain bf16 unit rows at D = 72 (K not a multiple of the 64-wide k-block):
s64 = temp * (rows64 @ cols64^T), computed on the GPU, in row chunks where it would not fit.

Error budget, with temp = exp(temperature) as the kernels receive it (fp32):
  - logits: temp * 2^-16 absolute (LOGIT_GATE; what the split-bf16 product keeps of fp32 latents;
    against the bf16 operands themselves only the fp32 accumulation remains);
  - lse / pos inherit it, plus the fp32 rounding and the approximate exp2 / log2 of the log-sum-exp;
  - g = bf16(temp * gscale * (...)): each exp term carries the logit error as a relative error, plus
    the exp2 argument's fp32 rounding and ex2.approx (nce_oracle.exp_rel), then one bf16 rounding (at most 2^-8
    relative; gated at BF16_REL = 2^-7);
  - d temperature = sum g * s is gated against the magnitudes of its terms, not against |d temperature|:
    the terms cancel.
Each test prints its largest error / gate; the largest over all cases, measured on an H100, is in
the test's docstring."""
import math

import pytest
import torch

from nce_oracle import LOGIT_GATE
from nce_oracle import check_bwd_rows as _check_bwd_rows
from nce_oracle import dtemp_gate as _dtemp_gate
from nce_oracle import lse_gate as _lse_gate
from nce_oracle import ref_rows as _ref_rows
from test_gpu_filip import _report_peak, _start_peak

pytestmark = pytest.mark.gpu

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
BLOCK_ELEMS = 1 << 24                   # fp64 elements per [rows, C] reference chunk (128 MiB)


def _unit(n, d, dev, seed):
    g = torch.Generator().manual_seed(seed)
    z = torch.nn.functional.normalize(torch.randn(n, d, generator=g), dim=-1)
    return z.to(dev).bfloat16()


@pytest.mark.parametrize("R,C,off,D,dcl,temp_exp", [
    (6, 6, 0, 256, False, 2.5), (128, 128, 0, 512, True, 2.5), (200, 1000, 300, 512, False, 2.5),
    (1024, 1024, 0, 512, True, 2.5), (384, 3000, 1500, 512, False, 2.5),
    # CLIP-style logit scale: exp(temperature) = 100.  A fixed shift exp(s - 100) underflows every
    # row whose cosines stay below ~0 (random latents!); the online row maximum must not.
    (300, 2000, 700, 512, False, 100.0), (128, 128, 0, 512, True, 100.0)])
def test_nce_fwd_bwd(cuda_device, R, C, off, D, dcl, temp_exp):
    from x_clip_b200 import kernels as K
    dev = cuda_device
    b = _unit(C, D, dev, 1)
    a = _unit(C, D, dev, 2)[off:off + R].contiguous()
    temp = torch.tensor([temp_exp], device=dev)
    lse, pos = K.nce_fwd(a, b, temp, off, dcl)
    s = (temp.double() * (a.double() @ b.double().t()))
    eye = torch.zeros(R, C, dtype=torch.bool, device=dev)
    eye[torch.arange(R), torch.arange(R) + off] = True
    ref_lse = torch.logsumexp(s.masked_fill(eye, -float("inf")) if dcl else s, dim=-1).float()
    s = s.float()
    assert torch.isfinite(lse).all()
    assert torch.allclose(lse, ref_lse, atol=2e-4 * max(1.0, temp_exp / 2.5), rtol=1e-5), (lse - ref_lse).abs().max()
    assert torch.allclose(pos, s[eye], atol=1e-4 * max(1.0, temp_exp / 2.5))

    # backward: g = gs*(w_row*exp(s-lse_row) + w_col*exp(s-lse_col) - w_diag*diag), out = temp*g
    lse_col = torch.randn(C, device=dev) * 0.1 + ref_lse.mean()
    gs = torch.tensor([0.37], device=dev)
    dtemp = torch.zeros(1, device=dev)
    g = K.nce_bwd(a, b, temp, off, dcl, lse, lse_col, 1.0, 0.5, 2.0, gs, dtemp)
    keep = ~eye if dcl else torch.ones_like(eye)
    ref_g = gs * ((torch.exp(s - ref_lse[:, None]) + 0.5 * torch.exp(s - lse_col[None, :])) * keep
                  - 2.0 * eye)
    got = g[:, :C].float()
    err = (got - temp * ref_g).abs().max().item()
    assert err <= 1e-2 * (temp * ref_g).abs().max().item(), err
    assert (g[:, C:] == 0).all()
    ref_dtemp = (ref_g * s).sum().item()
    assert abs(dtemp.item() - ref_dtemp) <= 2e-3 * max(1.0, abs(ref_dtemp)) + 1e-3 * ref_g.abs().sum().item() * 0.01


# --------------------------------------------------------------------------- fp64 references

def _ops(n, D, dev, seed):
    """(row operand, column operand) bf16 of n latents.  D a multiple of 256: K.l2norm_fwd of random
    fp32 projections (split-bf16, K = 3D), as ProjectL2NormFn hands them to the loss.  Otherwise plain
    bf16 unit rows used as both forms (K = D)."""
    from x_clip_b200 import kernels as K
    gen = torch.Generator(device=dev).manual_seed(seed)
    if D % 256:
        z = torch.nn.functional.normalize(torch.randn((n, D), generator=gen, device=dev), dim=-1).to(BF16)
        return z, z
    p = 3.0 * torch.randn((n, D), generator=gen, device=dev)
    _, zrow, zcol, _ = K.l2norm_fwd(p)
    return zrow, zcol


COLS = [1, 7, 31, 32, 33, 127, 128, 129, 255, 256, 257, 1000, 4095, 4096]
DIMS = [256, 512, 768, 1024, 72]
TEMPS = [0.1, 1.0, math.e, 1 / 0.07, 100.0]


def _offsets(R, C):
    """diag_offset 0 and C - R; one row: its positive on the first / last column of a 32-column chunk
    and of a 128 / 256 block; more rows: the middle (their positives then cross chunk borders)."""
    cand = [0, C - R] + ([31, 32, 127, 128, 255, 256] if R == 1 else [(C - R) // 2])
    return sorted({o for o in cand if 0 <= o <= C - R})


@pytest.mark.parametrize("dcl", [False, True])
@pytest.mark.parametrize("D", DIMS)
@pytest.mark.parametrize("C", COLS)
def test_nce_fwd_matches_fp64(cuda_device, C, D, dcl):
    """xclip_nce_fwd: lse, pos and loss_accum (from 0.75, loss_scale 0.3) for R in {1, 127, 128, 129, C}
    (those <= C), every offset of _offsets, exp(temperature) cycling over TEMPS.  C < 256 runs 128-wide
    column blocks, C >= 256 256-wide ones; 1000 / 4095 / 257 end in a ragged block.
    Gates: lse temp 2^-16 + 2^-20 (1 + |lse|); pos temp 2^-16; loss_accum 0.3 * the summed lse and pos
    gates + R 2^-24 (0.75 + 0.3 sum |lse - pos|).  Measured on an H100 over all 140 cases: lse at most
    0.14 of its gate, pos 0.05, loss_accum 0.14.  C = 1 under DCL (an empty denominator) gives
    lse = ln(1e-20), the reference's value."""
    from x_clip_b200 import kernels as K
    dev = cuda_device
    b_row, b_col = _ops(C, D, dev, seed=10 * C + D)
    del b_row
    k = 0
    worst = {"lse": 0.0, "pos": 0.0, "loss": 0.0}
    for R in sorted({r for r in (1, 127, 128, 129, C) if r <= C}):
        a_row, _ = _ops(R, D, dev, seed=10 * C + D + 7 * R + 1)
        s_unit = a_row.double() @ b_col.double().t()
        for off in _offsets(R, C):
            temp = TEMPS[k % len(TEMPS)]
            k += 1
            t = torch.tensor([temp], device=dev, dtype=F32)
            t64 = t.double()
            ref_lse, ref_pos = _ref_rows(t64 * s_unit, off, dcl)
            loss = torch.full((1,), 0.75, device=dev, dtype=F32)
            lse, pos = K.nce_fwd(a_row, b_col, t, off, dcl, loss_accum=loss, loss_scale=0.3)
            label = f"C={C} D={D} dcl={dcl} R={R} off={off} temp={temp:.4g}"
            lse_gate = _lse_gate(t64.item(), ref_lse)
            pos_gate = t64.item() * LOGIT_GATE
            e_lse = ((lse.double() - ref_lse).abs() / lse_gate).max().item()
            e_pos = (pos.double() - ref_pos).abs().max().item() / pos_gate
            assert e_lse <= 1.0, (label, e_lse)
            assert e_pos <= 1.0, (label, e_pos)
            terms = 0.3 * (ref_lse - ref_pos)
            ref_loss = 0.75 + terms.sum().item()
            loss_gate = (0.3 * (lse_gate.sum().item() + R * pos_gate)
                         + R * 2.0 ** -24 * (0.75 + terms.abs().sum().item()))
            e_loss = abs(loss.item() - ref_loss) / loss_gate
            assert e_loss <= 1.0, (label, loss.item(), ref_loss, loss_gate)
            for key, v in (("lse", e_lse), ("pos", e_pos), ("loss", e_loss)):
                worst[key] = max(worst[key], v)
        del s_unit
    print(f"nce_fwd C={C} D={D} dcl={dcl}: error/gate lse {worst['lse']:.3f} pos {worst['pos']:.3f} "
          f"loss {worst['loss']:.3f}")


WEIGHTS = [(1.0, 1.0, 2.0), (1.0, 0.0, 1.0), (0.0, 1.0, 1.0)]
BWD_SHAPES = [(1, 1, 0, 256), (1, 33, 32, 512), (33, 33, 0, 72), (127, 257, 130, 768),
              (129, 1000, 871, 1024), (256, 4095, 3839, 512), (300, 4096, 1000, 256)]


@pytest.mark.parametrize("dcl", [False, True])
@pytest.mark.parametrize("w", WEIGHTS, ids=["plain", "extra_rows", "extra_cols"])
@pytest.mark.parametrize("R,C,off,D", BWD_SHAPES)
def test_nce_bwd_matches_fp64(cuda_device, R, C, off, D, w, dcl):
    """xclip_nce_bwd with the three weight sets ContrastiveLossFn uses: (1, 1, 2) plain InfoNCE,
    (1, 0, 1) / (0, 1, 1) the row / column halves of the extra-latent loss.  lse_row is the kernel's
    own forward lse; lse_col the fp32 column log-sum-exp of the same logits (both what the loss passes:
    log-denominators of real logits).  g element by element within BF16_REL |ref| + temp gs ex EXP_REL;
    d temperature (from 0.5) within _dtemp_gate.  exp(temperature) = e and 100.  Measured on an H100
    over all 84 cases: g at most 0.50 of its gate (the bf16 rounding itself), d temperature 0.013."""
    from x_clip_b200 import kernels as K
    dev = cuda_device
    a_row, _ = _ops(R, D, dev, seed=R + 3 * C + D)
    _, b_col = _ops(C, D, dev, seed=R + 3 * C + D + 1)
    s_unit = a_row.double() @ b_col.double().t()
    gs = 0.37
    gscale = torch.tensor([gs], device=dev, dtype=F32)
    for temp in (math.e, 100.0):
        t = torch.tensor([temp], device=dev, dtype=F32)
        t64 = t.double().item()
        s = t64 * s_unit
        lse_row, _ = K.nce_fwd(a_row, b_col, t, off, dcl)
        lse_col = torch.logsumexp(s, dim=0).float().contiguous()
        dtemp = torch.full((1,), 0.5, device=dev, dtype=F32)
        g = K.nce_bwd(a_row, b_col, t, off, dcl, lse_row if w[0] else None, lse_col if w[1] else None,
                      *w, gscale, dtemp)
        assert g.shape == (R, (C + 7) // 8 * 8)
        err, sum_gs, abs_gs, abs_g = _check_bwd_rows(g, s, off, dcl, lse_row, lse_col, w, gs, t64)
        assert err <= 1.0, (R, C, off, D, w, dcl, temp, err)
        gate = _dtemp_gate(t64, abs_gs, abs_g, R, C)
        e_dt = abs(dtemp.item() - (0.5 + sum_gs)) / gate
        assert e_dt <= 1.0, (R, C, off, D, w, dcl, temp, dtemp.item(), 0.5 + sum_gs, gate)
        print(f"nce_bwd R={R} C={C} off={off} D={D} w={w} dcl={dcl} temp={temp:.4g}: error/gate g {err:.3f} "
              f"dtemp {e_dt:.3f}")


def test_nce_bwd_rejects_a_misaligned_lse_col(cuda_device):
    """lse_col is read with 16-byte loads.  An odd-length row of a stacked [4, B] tensor (row 2 starts
    8 B bytes in) and a view one float into its storage must be refused before any launch; a 16-byte
    aligned copy must give the same g as a fresh buffer, bit for bit."""
    from x_clip_b200 import _lib
    from x_clip_b200 import kernels as K
    dev = cuda_device
    B, D = 65, 256
    rows, _ = _ops(B, D, dev, seed=65)
    _, cols = _ops(B, D, dev, seed=66)
    t = torch.tensor([math.e], device=dev, dtype=F32)
    gs = torch.tensor([1.0 / (2 * B)], device=dev, dtype=F32)
    lse, pos = K.nce_fwd(rows, cols, t, 0, False)
    stats = torch.stack([lse, pos, lse, pos])
    spare = torch.empty(B + 1, device=dev, dtype=F32)
    spare[1:] = lse
    lib = _lib.load()
    for bad in (stats[2], spare[1:]):
        assert bad.data_ptr() % 16 != 0 and torch.equal(bad, lse)
        n0 = lib.xclip_launch_count()
        with pytest.raises(_lib.XClipB200Error, match="lse_col"):
            K.nce_bwd(rows, cols, t, 0, False, lse, bad, 1.0, 1.0, 2.0, gs)
        assert lib.xclip_launch_count() == n0, "a refused call launched a kernel"
    fresh = K.nce_bwd(rows, cols, t, 0, False, lse, lse.clone(), 1.0, 1.0, 2.0, gs)
    for good in (stats[0], stats[2].clone()):
        assert good.data_ptr() % 16 == 0
        assert torch.equal(K.nce_bwd(rows, cols, t, 0, False, lse, good, 1.0, 1.0, 2.0, gs), fresh)


def test_nce_fwd_rejects_a_misaligned_workspace(cuda_device):
    """part_ws holds float2 partials: a pointer 4 bytes into a buffer is refused before any launch."""
    from x_clip_b200 import _lib
    dev = cuda_device
    R, C, D = 40, 300, 256
    rows, _ = _ops(R, D, dev, seed=1)
    _, cols = _ops(C, D, dev, seed=2)
    t = torch.tensor([1.0], device=dev, dtype=F32)
    lib = _lib.load()
    part = torch.empty(2 * lib.xclip_nce_num_col_blocks(C) * R + 1, device=dev, dtype=F32)
    pos = torch.empty(R, device=dev, dtype=F32)
    lse = torch.empty(R, device=dev, dtype=F32)
    n0 = lib.xclip_launch_count()
    with pytest.raises(_lib.XClipB200Error, match="part_ws"):
        _lib.call("xclip_nce_fwd", rows.data_ptr(), cols.data_ptr(), R, C, rows.shape[1], t.data_ptr(), 0, 0,
                  part.data_ptr() + 4, pos.data_ptr(), lse.data_ptr(), None, 0.0, None)
    assert lib.xclip_launch_count() == n0


# --------------------------------------------------------------------------- one rank of W

@pytest.mark.parametrize("W,b,rank,dcl,temp", [
    (8, 4096, 0, False, 100.0), (8, 4096, 7, False, 100.0),      # cfg3 on 8 GPUs: 4096 x 32768
    (3, 33, 0, False, math.e), (3, 33, 1, True, math.e), (3, 33, 2, False, 1 / 0.07)])
def test_nce_one_rank_of_a_multi_gpu_step(cuda_device, W, b, rank, dcl, temp):
    """Rank `rank` of W: its b text rows against all W b image columns (diag_offset rank b); the image
    rows of every rank against all texts, their lse gathered in rank order as ContrastiveLossFn's
    gather_stats does, then the text-side backward with the gathered lse as lse_col.  Every lse / pos
    against fp64, g and d temperature with the gates above; the reference runs in row chunks of at most
    BLOCK_ELEMS fp64 elements per [rows, W b] block.  dim_latent 512 (cfg3).  Measured on an H100 at
    W = 8: lse at most 0.063 of its gate, pos 0.037, g 0.36, d temperature 0.009; each case with its
    reference takes 0.1-0.2 s and peaks at 2.5 GiB."""
    from x_clip_b200 import kernels as K
    dev = cuda_device
    t0 = _start_peak()
    D, Bg, off = 512, W * b, rank * b
    t_row, t_col = _ops(Bg, D, dev, seed=100 + W)
    i_row, i_col = _ops(Bg, D, dev, seed=200 + W)
    t = torch.tensor([temp], device=dev, dtype=F32)
    t64 = t.double().item()
    gs = 1.0 / (2 * Bg)
    gscale = torch.tensor([gs], device=dev, dtype=F32)

    mine = slice(off, off + b)
    lse_t, pos_t = K.nce_fwd(t_row[mine], i_col, t, off, dcl)
    per_rank = [K.nce_fwd(i_row[r * b:(r + 1) * b], t_col, t, r * b, dcl) for r in range(W)]
    stats = torch.stack([torch.stack([lse_t, pos_t, l, p]) for l, p in per_rank])     # [W, 4, b]
    gstats = stats.permute(1, 0, 2).reshape(4, Bg).contiguous()
    lse_i_all = gstats[2].clone()
    dtemp = torch.zeros(1, device=dev, dtype=F32)
    g = K.nce_bwd(t_row[mine], i_col, t, off, dcl, lse_t, lse_i_all, 1.0, 1.0, 2.0, gscale, dtemp)
    torch.cuda.synchronize()

    step = max(1, BLOCK_ELEMS // Bg)
    worst = {"lse_i": 0.0, "pos_i": 0.0, "lse_t": 0.0, "pos_t": 0.0, "g": 0.0}
    t_col64, i_col64 = t_col.double(), i_col.double()
    pos_gate = t64 * LOGIT_GATE
    for r0 in range(0, Bg, step):                      # image rows of every rank vs all texts
        s = t64 * (i_row[r0:r0 + step].double() @ t_col64.t())
        ref_lse, ref_pos = _ref_rows(s, r0, dcl)
        got_lse = lse_i_all[r0:r0 + step].double()
        got_pos = gstats[3, r0:r0 + step].double()
        worst["lse_i"] = max(worst["lse_i"], ((got_lse - ref_lse).abs() / _lse_gate(t64, ref_lse)).max().item())
        worst["pos_i"] = max(worst["pos_i"], (got_pos - ref_pos).abs().max().item() / pos_gate)
        del s
    sum_gs = abs_gs = abs_g = 0.0
    for r0 in range(0, b, step):                       # this rank's text rows vs all images
        r1 = min(b, r0 + step)
        s = t64 * (t_row[off + r0:off + r1].double() @ i_col64.t())
        ref_lse, ref_pos = _ref_rows(s, off + r0, dcl)
        rows_lse = lse_t[r0:r1]
        worst["lse_t"] = max(worst["lse_t"], ((rows_lse.double() - ref_lse).abs() / _lse_gate(t64, ref_lse)).max().item())
        worst["pos_t"] = max(worst["pos_t"], (pos_t[r0:r1].double() - ref_pos).abs().max().item() / pos_gate)
        err, a, b_abs, c_abs = _check_bwd_rows(g[r0:r1], s, off + r0, dcl, rows_lse, lse_i_all,
                                               (1.0, 1.0, 2.0), gs, t64)
        worst["g"] = max(worst["g"], err)
        sum_gs, abs_gs, abs_g = sum_gs + a, abs_gs + b_abs, abs_g + c_abs
        del s
    e_dt = abs(dtemp.item() - sum_gs) / _dtemp_gate(t64, abs_gs, abs_g, b, Bg)
    label = f"rank {rank} of W={W} b={b} dcl={dcl} temp={temp:.4g}"
    print(f"nce {label}: error/gate " + " ".join(f"{k} {v:.3f}" for k, v in worst.items()) + f" dtemp {e_dt:.3f}")
    for k_, v in worst.items():
        assert v <= 1.0, (label, k_, v)
    assert e_dt <= 1.0, (label, dtemp.item(), sum_gs)
    _report_peak(f"nce {label} with its fp64 reference", t0)
