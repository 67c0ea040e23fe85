"""Fused feed-forward (csrc/ff.cu: GEGLU in the up-projection epilogue, LayerNorm folded into the
down-projection and into the dgrad GEMM of the backward), stage by stage against fp64.

Every stage is fed the previous stage's actual outputs and compared with fp64 torch computed from
the exact operands it read (bf16 activations, bf16 weights, the kernel's own statistics), so the
gates sit at the stage's own rounding (block_oracle.py: 2^-8 |ref| + 2^-16 of the row's largest
|ref| per element).  Where an operation is exact by construction the check is bit for bit.  One
chained forward + backward check compares with an fp64 restatement of x_clip/x_clip.py:180-199.

Inputs (block_oracle.ff_case) make the LayerNorm-fold terms large: hp rows with |mean| ~ 0.5 std,
dx with a component along colvec (a = mean_k gdh large) and, on odd rows, along the block output
(b = mean_k gdh hn large).

Tile counts (128 x 128 tiles, 132 CTAs; up N = 8d, down N = d, backward N = 4d):
- M <= 129: at most 2 x 64 tiles, one per CTA, so ping-pong warpgroup 1 idles;
- (4000, 256):  up 512 tiles (CTAs get 4 or 3), down 64, backward 256 (2 or 1);
- (3000, 512):  up 768 (6 or 5), down 96, backward 384 (3 or 2);
- (1413, 768):  up 576 (5 or 4), down 72, backward 288 (3 or 2);
- (8577, 1024): up 4352 (33 or 32), down 544 (5 or 4), backward 2176 (17 or 16), and past the
  8448-row grid cap of ff_bwd_prep (132 x 4 blocks x 8 warps x 2 rows).

Largest error measured on an H100 80GB HBM3 at a 400 W power limit, as a fraction of its gate:
u, hp, x2, acc, du 0.991-0.992 (the bf16 rounding bound is tight by construction: a value just above
a power of two rounds by almost 2^-8 of itself); colvec 0.0004, rowsum 0.032, mean 0.016, rstd 0.036,
vsum 0.058, a 0.011, b 0.008, dg4 0.031.
"""
import pytest
import torch

import block_oracle as BO

pytestmark = pytest.mark.gpu

FF_CASES = [(M, d) for d in (256, 512, 768, 1024) for M in (1, 127, 128, 129)] + [
    (4000, 256), (3000, 512), (1413, 768), (8577, 1024)]


def _forward(t):
    from x_clip_b200 import kernels as K
    w1p, w2g, colvec = K.ff_weights(t["w1"], t["w2"], t["g4"])
    u, hp, rowsum = K.ff_up(t["x"], w1p)
    x2, acc, stats = K.ff_down(hp, w2g, colvec, rowsum, t["res"], BO.LN_EPS)
    torch.cuda.synchronize()
    return w1p, w2g, colvec, u, hp, rowsum, x2, acc, stats


@pytest.mark.parametrize("M,d", FF_CASES)
def test_ff_stages_fp64(cuda_device, M, d):
    from x_clip_b200 import kernels as K
    tag = f"{M}x{d}"
    t = BO.ff_case(M, d, cuda_device)
    w1p, w2g, colvec, u, hp, rowsum, x2, acc, stats = _forward(t)
    D4 = 4 * d

    # ff_weights: casts are exact, colvec is an fp32 row sum of the bf16 w2g
    assert torch.equal(w1p, BO.ff_permute(t["w1"].bfloat16())), "w1p"
    assert torch.equal(w2g, (t["w2"] * t["g4"]).bfloat16()), "w2g"
    BO.check(f"ff_colvec[{tag}]", colvec, w2g.double().sum(1), BO.RED_REL * w2g.double().abs().sum(1))

    # ff_up: u = x W1^T, hp = value * gelu(gate) of the fp32 accumulators, per-box sums of bf16 hp
    u_ref = t["x"].double() @ t["w1"].bfloat16().double().t()
    BO.check(f"ff_u[{tag}]", u.view(M, 2, D4), u_ref.view(M, 2, D4), BO.elem_gate(u_ref.view(M, 2, D4)))
    hp_ref = u_ref[:, :D4] * BO.gelu64(u_ref[:, D4:])
    BO.check(f"ff_hp[{tag}]", hp, hp_ref, BO.elem_gate(hp_ref))
    box = hp.double().view(M, -1, 64)
    box_abs = torch.stack([box.abs().sum(-1), (box * box).sum(-1)], -1)
    BO.check(f"ff_rowsum[{tag}]", rowsum, BO.ff_rowsum64(hp), BO.RED_REL * box_abs)
    _, hp2, rowsum2 = K.ff_up(t["x"], w1p, need_u=False)
    torch.cuda.synchronize()
    assert torch.equal(hp2, hp) and torch.equal(rowsum2, rowsum), "need_u=False changed hp / rowsum"

    # ff_down: statistics of the kernel's hp; x2 and acc at the kernel's statistics and colvec
    mean, rstd = BO.ln_stats64(hp)
    BO.check(f"ff_mean[{tag}]", stats[:, 0], mean, BO.STAT_REL * (mean.abs() + 1 / rstd))
    BO.check(f"ff_rstd[{tag}]", stats[:, 1], rstd, BO.STAT_REL * rstd)
    x2_ref, acc_ref, _ = BO.ff_down64(hp, w2g, colvec, stats[:, 0], stats[:, 1], t["res"])
    BO.check(f"ff_x2[{tag}]", x2, x2_ref, BO.elem_gate(x2_ref))
    BO.check(f"ff_acc[{tag}]", acc, acc_ref, BO.elem_gate(acc_ref))

    # ff_bwd_prep: dxs exact; vsum, ab from the kernel's dx, acc, colvec and statistics
    dx = t["dx"]
    dxs, vsum, ab = K.ff_bwd_prep(dx, stats, acc, colvec)
    torch.cuda.synchronize()
    assert torch.equal(dxs, (dx.float() * stats[:, 1:2]).bfloat16()), "dxs"
    terms = dxs.double() * stats[:, :1].double()
    BO.check(f"ff_vsum[{tag}]", vsum, terms.sum(0), BO.RED_REL * terms.abs().sum(0))
    a_ref, b_ref = BO.ff_ab64(dx, acc, colvec, stats[:, 0], stats[:, 1], D4)
    a_scale = (dx.double().abs() @ colvec.double().abs()) / D4
    b_scale = stats[:, 1].double() * ((dx.double() * acc.double()).abs().sum(1) / D4 + stats[:, 0].double().abs() * a_scale)
    BO.check(f"ff_a[{tag}]", ab[:, 0], a_ref, BO.RED_REL * a_scale)
    BO.check(f"ff_b[{tag}]", ab[:, 1], b_ref, BO.RED_REL * b_scale)

    # ff_bwd: LN(4d) + GEGLU backward in the dgrad epilogue, at the kernel's stats and ab
    du = K.ff_bwd(dx, w2g, u, stats, ab)
    torch.cuda.synchronize()
    du_ref = BO.ff_bwd64(dx, w2g, u, stats[:, 0], stats[:, 1], ab[:, 0], ab[:, 1]).view(M, 2, D4)
    BO.check(f"ff_du[{tag}]", du.view(M, 2, D4), du_ref, BO.elem_gate(du_ref))

    # ff_w2_grad_post_: dW2 = g4 (raw - vsum) exactly in fp32; dg4 accumulated onto a non-zero prefill
    raw = torch.zeros(d, D4, device=cuda_device)
    K.gemm(dxs, hp, a_major=1, b_major=1, out=raw, accumulate=True)
    raw0 = raw.clone()
    dg4 = t["dg0"].clone()
    dw2 = K.ff_w2_grad_post_(raw, vsum, t["g4"], t["w2"], dg4)
    torch.cuda.synchronize()
    assert torch.equal(dw2, t["g4"] * (raw0 - vsum[:, None])), "dW2"
    tt = (raw0.double() - vsum.double()[:, None]) * t["w2"].double()
    BO.check(f"ff_dg4[{tag}]", dg4, t["dg0"].double() + tt.sum(0),
             BO.RED_REL * (tt.abs().sum(0) + t["dg0"].double().abs()))


@pytest.mark.parametrize("M,d", [(129, 256), (1413, 768), (3000, 512)])
def test_ff_chained_fp64(cuda_device, M, d):
    """Forward + backward of the whole fused feed-forward against fp64 autograd of x_clip.py:180-199
    on the bf16 input and weights: bf16 roundings accumulate over the chain, so the gates are
    relative Frobenius errors.  Largest measured (H100 80GB HBM3, 400 W): x2 2.1e-3, du 3.9e-3,
    dW2 2.4e-3, dg4 1.3e-3."""
    from x_clip_b200 import kernels as K
    t = BO.ff_case(M, d, cuda_device)
    w1p, w2g, colvec, u, hp, rowsum, x2, acc, stats = _forward(t)
    dx = t["dx"]
    dxs, vsum, ab = K.ff_bwd_prep(dx, stats, acc, colvec)
    du = K.ff_bwd(dx, w2g, u, stats, ab)
    raw = torch.zeros(d, 4 * d, device=cuda_device)
    K.gemm(dxs, hp, a_major=1, b_major=1, out=raw, accumulate=True)
    dg4 = torch.zeros(4 * d, device=cuda_device)
    dw2 = K.ff_w2_grad_post_(raw, vsum, t["g4"], t["w2"], dg4)
    torch.cuda.synchronize()

    u_leaf = (t["x"].double() @ t["w1"].bfloat16().double().t()).requires_grad_(True)
    w2 = t["w2"].double().requires_grad_(True)
    g4 = t["g4"].double().requires_grad_(True)
    hp64 = u_leaf[:, :4 * d] * BO.gelu64(u_leaf[:, 4 * d:])
    mu = hp64.mean(-1, keepdim=True)
    hn = (hp64 - mu) / torch.sqrt(((hp64 - mu) ** 2).mean(-1, keepdim=True) + BO.LN_EPS)
    x2_ref = (hn * g4) @ w2.t()
    x2_ref.backward(dx.double())
    x2_ref = x2_ref.detach() + t["res"].double()
    for name, got, ref, gate in (("x2", x2, x2_ref, 4e-3), ("du", du, u_leaf.grad, 8e-3),
                                 ("dW2", dw2, w2.grad, 5e-3), ("dg4", dg4, g4.grad, 4e-3)):
        rel = BO.rel_fro(got, ref)
        print(f"GATE ff_chain_{name}[{M}x{d}] {rel / gate:.4f}")
        assert rel <= gate, (name, rel)


# Rows of hp with |mean| / std = r: E[hp^2] - mean^2 loses about log2(1 + r^2) bits of the fp32 sums.
VAR_RATIOS = (4, 16, 64, 256)


def test_ff_down_single_pass_variance(cuda_device):
    """ff_down derives the variance as E[hp^2] - mean^2 from fp32 per-box sums.  Pinned: at
    |mean| / std = 4 the saved rstd meets STAT_REL against fp64.  Larger ratios are measured and
    printed, not asserted: the formula is a documented bound, not a promise.  The rstd error grows
    as (|mean| / std)^2; on an H100 80GB HBM3 (400 W) it used 0.32 of the gate at 4, 3.6 x at 16,
    50 x at 64 and 650 x at 256, so the formula stops meeting the gate at about |mean| / std = 7.
    Random-weight blocks give hp rows with |mean| / std ~ 0.02."""
    from x_clip_b200 import kernels as K
    M, d = 256, 512
    gen = torch.Generator().manual_seed(5)
    t = BO.ff_case(129, d, cuda_device)
    _, w2g, colvec = K.ff_weights(t["w1"], t["w2"], t["g4"])
    res = torch.zeros(M, d, device=cuda_device, dtype=torch.bfloat16)
    z = torch.randn(M, 4 * d, generator=gen)
    sign = torch.where(torch.rand(M, 1, generator=gen) < 0.5, -1.0, 1.0)
    for r in VAR_RATIOS:
        hp = (z + sign * r).bfloat16().to(cuda_device)
        box = hp.float().view(M, -1, 64)
        rowsum = torch.stack([box.sum(-1), (box * box).sum(-1)], -1).contiguous()
        _, _, stats = K.ff_down(hp, w2g, colvec, rowsum, res, BO.LN_EPS)
        torch.cuda.synchronize()
        mean, rstd = BO.ln_stats64(hp)
        frac = BO.gate_ratio(stats[:, 1], rstd, BO.STAT_REL * rstd)
        print(f"GATE ff_var_ratio{r} {frac:.4f}")
        if r == 4:
            assert frac <= 1.0, f"rstd at |mean|/std = 4: {frac:.3f} x its gate"
