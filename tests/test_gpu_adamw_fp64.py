"""The fused AdamW (xclip_adamw_step, optim.FusedAdamW) against the fp64 update of its documented rule
(csrc/rowwise.cu:826-830), one step at a time from the kernel's own fp32 state, so that drift cannot
hide a wrong term.  Per-element gates: ADAM_ULP (eight fp32 ulp) of the sum of |terms| of each
of p, m and v, with step_size * |m| / denom as the size of the Adam term of p.  Worst gate ratios on an
H100 80GB HBM3 (700 W power limit): p 0.69, m 0.24, v 0.25; the file runs in about 20 s there.

- n from 1 to past the grid cap (num_sms * 16 blocks of 256 threads x 4 elements, so the grid-stride
  loop runs) with the scalar tail n % 4 != 0;
- grad_scale 1 and 2^-10, weight decay 0 and 0.05, betas (0.9, 0.999) and (0.9, 0.95), steps 1, 2
  and 10000, gradients with exact zeros and magnitudes near eps;
- FusedAdamW: parameters with numel % 4 != 0 leave the padding of the flat buffers exactly 0, a
  scaled step equals torch.optim.AdamW on the scaled gradient, and "no grad" equals a zero grad;
- the fp32 -> bf16 cast past its grid cap.
"""
import pytest
import torch

import block_oracle as BO
import gemm_oracle as GO

pytestmark = pytest.mark.gpu


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def grid_cap_elems(sms):
    return sms * 16 * 256 * 4               # elements one pass of the capped grid covers


def _sizes():
    return {"1": 1, "3": 3, "4": 4, "cap+3": grid_cap_elems(_sms()) + 3, "5M+3": 5 * 2 ** 20 + 3}


SMALL_CASES = [(betas, wd, gs, near) for betas in ((0.9, 0.999), (0.9, 0.95)) for wd in (0.0, 0.05)
               for gs in (1.0, 2.0 ** -10) for near in (False, True)]
LARGE_CASES = [((0.9, 0.999), 0.05, 1.0, True), ((0.9, 0.95), 0.0, 2.0 ** -10, False),
               ((0.9, 0.95), 0.05, 2.0 ** -10, True)]


def _step(dev, n, step, lr, betas, eps, wd, gs, near_eps, seed=0):
    from x_clip_b200 import kernels as K
    p, g, m, v = GO.adamw_state(n, seed, step, near_eps)
    P, G, Mo, V = (t.to(dev) for t in (p, g, m, v))
    K.adamw_step_(P, G, Mo, V, lr, betas[0], betas[1], eps, wd, step, gs)
    torch.cuda.synchronize()
    rp, rm, rv, gp, gm, gv = GO.adamw64(P.new_tensor(p), G.new_tensor(g), Mo.new_tensor(m), V.new_tensor(v),
                                        lr, betas[0], betas[1], eps, wd, step, gs)
    assert torch.equal(G.cpu(), g)
    return (P, rp, gp), (Mo, rm, gm), (V, rv, gv)


@pytest.mark.parametrize("size", ["1", "3", "4", "cap+3", "5M+3"])
@pytest.mark.parametrize("step", [1, 2, 10000])
def test_adamw_c_abi(cuda_device, size, step):
    n = _sizes()[size]
    worst = {}
    cases = LARGE_CASES if n > 10 ** 6 else SMALL_CASES     # large sizes: each knob value at least once
    for i, (betas, wd, gs, near) in enumerate(cases):
        res = _step(cuda_device, n, step, 1e-3, betas, 1e-8, wd, gs, near, seed=i)
        for nm, (got, ref, gate) in zip("pmv", res):
            r = BO.gate_ratio(got, ref, gate)
            assert r <= 1.0, (nm, betas, wd, gs, near, r)
            worst[nm] = max(worst.get(nm, 0.0), r)
    for nm, r in worst.items():
        print(f"GATE adamw_{nm}_n{size}_step{step} {r:.4f}")


def test_fused_adamw_padding_stays_zero_and_scale(cuda_device):
    """numel % 4 != 0 parameters: the padding slots of flat / grad / exp_avg / exp_avg_sq stay exactly 0
    over several steps (a scaled step among them), each step matches the fp64 rule from the optimizer's
    own state, and the result follows torch.optim.AdamW fed s * grad."""
    from x_clip_b200.optim import FusedAdamW
    torch.manual_seed(0)
    shapes = [(7,), (33, 5), (1,), (1000, 3), (6,)]
    ours = [torch.nn.Parameter(torch.randn(s, device=cuda_device)) for s in shapes]
    ref = [torch.nn.Parameter(p.detach().clone()) for p in ours]
    kw = dict(lr=3e-3, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.05)
    opt = FusedAdamW(ours, **kw)
    topt = torch.optim.AdamW(ref, **kw)
    pad = torch.ones_like(opt.flat, dtype=torch.bool)
    for p, off in zip(ours, opt.offsets):
        pad[off:off + p.numel()] = False
    assert pad.sum() > 0
    for step in range(1, 7):
        s = 2.0 ** -10 if step % 2 == 0 else 1.0
        for p, r in zip(ours, ref):
            g = torch.randn_like(r)
            p.grad = g.clone()
            r.grad = g * s
        before = [t.clone() for t in (opt.flat, opt.exp_avg, opt.exp_avg_sq)]
        opt.step(grad_scale=s)
        topt.step()
        torch.cuda.synchronize()
        for t in (opt.flat, opt.grad, opt.exp_avg, opt.exp_avg_sq):
            assert torch.equal(t[pad], torch.zeros_like(t[pad])), step
        rp, rm, rv, gp, gm, gv = GO.adamw64(*before[:1], opt.grad, *before[1:], kw["lr"], *kw["betas"], kw["eps"],
                                            kw["weight_decay"], step, s)
        BO.check(f"fused_adamw_p_step{step}", opt.flat, rp, gp)
        BO.check(f"fused_adamw_m_step{step}", opt.exp_avg, rm, gm)
        BO.check(f"fused_adamw_v_step{step}", opt.exp_avg_sq, rv, gv)
    for p, r in zip(ours, ref):
        assert torch.allclose(p, r, atol=2e-6, rtol=1e-5), (p - r).abs().max()


def test_fused_adamw_no_grad_is_zero_grad(cuda_device):
    """A parameter without .grad takes exactly the step of a zero gradient (decay and moment decay)."""
    from x_clip_b200.optim import FusedAdamW
    torch.manual_seed(1)
    a = [torch.nn.Parameter(torch.randn(s, device=cuda_device)) for s in ((5,), (3, 3))]
    b = [torch.nn.Parameter(p.detach().clone()) for p in a]
    oa, ob = FusedAdamW(a, lr=1e-2), FusedAdamW(b, lr=1e-2)
    for step in range(3):
        g = torch.randn(5, device=cuda_device)
        a[0].grad, b[0].grad = g.clone(), g.clone()
        if step == 1:
            a[1].grad, b[1].grad = None, torch.zeros_like(b[1])
        else:
            h = torch.randn(3, 3, device=cuda_device)
            a[1].grad, b[1].grad = h.clone(), h.clone()
        oa.step()
        ob.step()
    torch.cuda.synchronize()
    for t, u in ((oa.flat, ob.flat), (oa.exp_avg, ob.exp_avg), (oa.exp_avg_sq, ob.exp_avg_sq)):
        assert torch.equal(t, u)
