"""Row-wise kernels: LayerNorm against fp64 on the exact operands the kernel read; the other row-wise
kernels against fp32 torch autograd of the same (bf16-rounded) inputs."""
import pytest
import torch

import block_oracle as BO

pytestmark = pytest.mark.gpu


def _close(a, b, tol, what=""):
    err = (a.float() - b.float()).abs().max().item()
    ref = b.float().abs().max().item()
    assert err <= tol * max(ref, 1e-3), f"{what}: err {err} vs scale {ref}"


# LayerNorm forward / backward against fp64 on the exact operands the kernels read (block_oracle.py).
# Widths 256..1024 are NV = 1..4 vectors per lane: the forward software-pipelines the next row for
# d <= 768, the backward for d <= 512.  A warp gets a second row only past the grid cap:
# 132 SMs x 8 blocks x 8 warps = 8448 rows forward, 132 x 2 x 8 = 2112 rows backward.
LN_FWD_CAP, LN_BWD_CAP = 132 * 8 * 8, 132 * 2 * 8
LN_CASES = [(rows, d) for d in (256, 512, 768, 1024)
            for rows in (1, 7, 1003, LN_BWD_CAP + 37, LN_FWD_CAP + 37)] + [(768 * 197, 768)]


def _ln_fwd_bwd(t, x=None, dy=None):
    """All LayerNorm outputs of one case: (out, stats, out2, stats2, dx, dg accumulated onto dg0)."""
    from x_clip_b200 import kernels as K
    x = t["x"] if x is None else x
    dy = t["dy"] if dy is None else dy
    out, stats, out2, stats2 = K.layernorm_fwd(x, t["g"], res=t["res"], g2=t["g2"], eps=BO.LN_EPS)
    dg = t["dg0"].clone()
    dx = K.layernorm_bwd(dy, x, stats, t["g"], add=t["add"], dg=dg)
    torch.cuda.synchronize()
    return out, stats, out2, stats2, dx, dg


def _check_ln(tag, t, got):
    """Every output of _ln_fwd_bwd against fp64.  Statistics to STAT_REL; bf16 outputs per element to
    2^-8 |ref| + 2^-16 of the row's largest |ref|; dg to 2^-16 of the sum of |terms| and the prefill."""
    out, stats, out2, stats2, dx, dg = got
    x, g = t["x"], t["g"]
    mean, rstd = BO.ln_stats64(x)
    sd = 1 / rstd
    BO.check(f"ln_mean[{tag}]", stats[:, 0], mean, BO.STAT_REL * (mean.abs() + sd))
    BO.check(f"ln_rstd[{tag}]", stats[:, 1], rstd, BO.STAT_REL * rstd)
    ref = (x.double() - mean[:, None]) * rstd[:, None] * g.double() + t["res"].double()
    BO.check(f"ln_out[{tag}]", out, ref, BO.elem_gate(ref))
    # the second norm reads the bf16-rounded first output
    mean2, rstd2 = BO.ln_stats64(out)
    BO.check(f"ln_mean2[{tag}]", stats2[:, 0], mean2, BO.STAT_REL * (mean2.abs() + 1 / rstd2))
    BO.check(f"ln_rstd2[{tag}]", stats2[:, 1], rstd2, BO.STAT_REL * rstd2)
    ref2 = (out.double() - mean2[:, None]) * rstd2[:, None] * t["g2"].double()
    BO.check(f"ln_out2[{tag}]", out2, ref2, BO.elem_gate(ref2))
    # backward at the statistics the kernel saved and read
    dx_ref, dg_ref, _, _ = BO.ln_bwd64(t["dy"], x, stats[:, 0], stats[:, 1], g)
    dx_ref = dx_ref + t["add"].double()
    BO.check(f"ln_dx[{tag}]", dx, dx_ref, BO.elem_gate(dx_ref))
    xh = (x.double() - stats[:, 0].double()[:, None]) * stats[:, 1].double()[:, None]
    dg_scale = (t["dy"].double() * xh).abs().sum(0) + t["dg0"].double().abs()
    BO.check(f"ln_dg[{tag}]", dg, t["dg0"].double() + dg_ref, BO.RED_REL * dg_scale)


@pytest.mark.parametrize("rows,d", LN_CASES)
def test_layernorm_fp64(cuda_device, rows, d):
    """out = LN(x) g + res, out2 = LN(bf16 out) g2, both stats, dx = dLN(dy) + add and dg += ...,
    against fp64.  Inputs (block_oracle.ln_case) make the row terms large: x rows have a sizeable
    mean, dy has components along g and along xhat, so mean(g dy) and mean(g dy xhat) are O(1).
    Largest error measured on an H100 80GB HBM3 at a 400 W power limit, as a fraction of its gate:
    out, out2, dx 0.992 (the bf16 rounding bound is tight by construction: a value just above a
    power of two rounds by almost 2^-8 of itself); mean 0.011, rstd 0.029, mean2 0.001, rstd2 0.020,
    dg 0.042."""
    t = BO.ln_case(rows, d, cuda_device)
    _check_ln(f"{rows}x{d}", t, _ln_fwd_bwd(t))


def test_layernorm_chain(cuda_device):
    """out = LN(y) g + x ; out2 = LN(out) g2 in one pass (attention tail + next pre-norm), at the
    shape of one text-tower chunk's tail: both norms' outputs and statistics against fp64, the second
    norm on the bf16-rounded first output, and the backward of the first norm with the residual
    gradient added.  Largest error measured on an H100 80GB HBM3 at a 700 W power limit, as a
    fraction of its gate: out, out2, dx 0.988; mean 0.005, rstd 0.015, mean2 0.0003, rstd2 0.013,
    dg 0.017."""
    t = BO.ln_case(515, 512, cuda_device)
    _check_ln("chain515x512", t, _ln_fwd_bwd(t))


@pytest.mark.parametrize("d", [256, 512, 768, 1024])
def test_layernorm_strided(cuda_device, d):
    """x and dy as column slices of wider buffers (leading dimension > d)."""
    rows = 2149
    t = BO.ln_case(rows, d, cuda_device)
    xw = torch.zeros(rows, d + 264, device=cuda_device, dtype=torch.bfloat16)
    dyw = torch.zeros(rows, 2 * d + 8, device=cuda_device, dtype=torch.bfloat16)
    xw[:, 136:136 + d] = t["x"]
    dyw[:, 8:8 + d] = t["dy"]
    x, dy = xw[:, 136:136 + d], dyw[:, 8:8 + d]
    assert x.stride(0) > d and dy.stride(0) > d
    got = _ln_fwd_bwd(t, x=x, dy=dy)
    _check_ln(f"strided{d}", t, got)
    same = _ln_fwd_bwd(t)
    for name, a, b in zip(("out", "stats", "out2", "stats2", "dx"), got, same):
        assert torch.equal(a, b), name


@pytest.mark.parametrize("d", [256, 512, 768, 1024])
def test_layernorm_rows_per_warp_knobs(cuda_device, d):
    """XCLIP_TUNE_LN_FWD_BLOCKS / _BWD_BLOCKS = 1 cap the grid at one block per SM, so 3000 rows give
    warps two and three rows each (the pipelined next-row path).  The header promises identical
    results whatever the knob: every output but dg (atomics in another order) is bit-identical,
    and dg still meets its fp64 gate."""
    from x_clip_b200 import _lib
    FWD, BWD = 3, 4          # XCLIP_TUNE_LN_FWD_BLOCKS, XCLIP_TUNE_LN_BWD_BLOCKS (include/xclip_b200.h)
    t = BO.ln_case(3000, d, cuda_device)
    base = _ln_fwd_bwd(t)
    lib = _lib.load()
    prev_f = lib.xclip_tune_set(FWD, 1)
    try:
        prev_b = lib.xclip_tune_set(BWD, 1)
        try:
            capped = _ln_fwd_bwd(t)
        finally:
            lib.xclip_tune_set(BWD, prev_b)
    finally:
        lib.xclip_tune_set(FWD, prev_f)
    for name, a, b in zip(("out", "stats", "out2", "stats2", "dx"), base, capped):
        assert torch.equal(a, b), name
    _check_ln(f"knob{d}", t, capped)


def test_layernorm_without_res_or_g2(cuda_device):
    """The plain norm (no residual, no second norm, no add, no dg) gives the same out / stats / dx
    as the fused call minus the residual terms."""
    from x_clip_b200 import kernels as K
    t = BO.ln_case(1003, 512, cuda_device)
    out, stats, out2, stats2 = K.layernorm_fwd(t["x"], t["g"], eps=BO.LN_EPS)
    assert out2 is None and stats2 is None
    mean, rstd = BO.ln_stats64(t["x"])
    ref = (t["x"].double() - mean[:, None]) * rstd[:, None] * t["g"].double()
    BO.check("ln_plain_out", out, ref, BO.elem_gate(ref))
    BO.check("ln_plain_rstd", stats[:, 1], rstd, BO.STAT_REL * rstd)
    dx = K.layernorm_bwd(t["dy"], t["x"], stats, t["g"])
    dx_ref = BO.ln_bwd64(t["dy"], t["x"], stats[:, 0], stats[:, 1], t["g"])[0]
    BO.check("ln_plain_dx", dx, dx_ref, BO.elem_gate(dx_ref))


@pytest.mark.parametrize("rows,d", [(4, 256), (1024, 512)])
def test_l2norm(cuda_device, rows, d):
    from x_clip_b200 import kernels as K
    torch.manual_seed(3)
    p = torch.randn(rows, d, device=cuda_device)
    z, zrow, zcol, inv = K.l2norm_fwd(p)
    pf = p.clone().requires_grad_(True)
    ref = torch.nn.functional.normalize(pf, dim=-1)
    assert torch.allclose(z, ref, atol=1e-6)
    hi, lo = zrow[:, :d].float(), zrow[:, d:2 * d].float()
    assert torch.equal(zrow[:, 2 * d:], zrow[:, :d]) and torch.equal(zcol[:, :2 * d], zrow[:, :d].repeat(1, 2))
    assert torch.equal(zcol[:, 2 * d:], zrow[:, d:2 * d])
    assert (hi + lo - ref.detach()).abs().max().item() < 2e-5          # split-bf16 carries ~16 bits
    gram = zrow.float() @ zcol.float().t()
    assert (gram - ref.detach() @ ref.detach().t()).abs().max().item() < 1e-4
    dz = torch.randn(rows, d, device=cuda_device)
    dp = K.l2norm_bwd(dz, z, inv)
    ref.backward(dz)
    _close(dp, pf.grad, 1e-2, "l2norm dp")


def test_cast(cuda_device):
    from x_clip_b200 import kernels as K
    for n in (1, 7, 8, 1000003, 8 * 1024 * 1024):     # the last: an 8d x d weight at d = 1024, past the grid cap
        src = torch.randn(n, device=cuda_device)
        assert torch.equal(K.cast_bf16(src), src.bfloat16())


def test_text_embed_fwd_bwd(cuda_device):
    """[cls | tok[ids] + pos] and its backward (x_clip/x_clip.py:320-332) vs torch autograd."""
    from x_clip_b200 import engine as E
    torch.manual_seed(4)
    B, n, d, vocab = 37, 16, 512, 100
    ids = torch.randint(0, vocab, (B, n), device=cuda_device)
    tok = torch.randn(vocab, d, device=cuda_device, requires_grad=True)
    pos = torch.randn(n + 4, d, device=cuda_device, requires_grad=True)
    cls = torch.randn(d, device=cuda_device, requires_grad=True)
    out = E.TextEmbedFn.apply(ids, tok, pos, cls)
    ref = torch.cat((cls.expand(B, 1, d), tok[ids] + pos[:n]), dim=1)
    assert out.shape == (B, n + 1, d)
    _close(out, ref, 1e-2, "embed fwd")
    dx = torch.randn(B, n + 1, d, device=cuda_device).bfloat16()
    out.backward(dx)
    g = (tok.grad.clone(), pos.grad.clone(), cls.grad.clone())
    tok.grad = pos.grad = cls.grad = None
    ref.backward(dx.float())
    _close(g[0], tok.grad, 1e-5, "dtok")
    _close(g[1], pos.grad, 1e-5, "dpos")
    _close(g[2], cls.grad, 1e-5, "dcls")
