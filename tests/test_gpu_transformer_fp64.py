"""The encoder as a whole (engine.TransformerFn, depth 2) against fp64 autograd of the reference block
(block_oracle.transformer_stack, eps pinned to 1e-5), on bf16-rounded input and matmul weights,
fp32 gains and a fixed random bf16 cotangent of the output.

Each flat weight's gradient, the output and the input gradient are gated separately by relative
Frobenius error (BLOCK_GATES).  test_block_gates.py checks on the CPU that every gate is at most a
quarter of what a reference that skips the rotary inverse in the backward, or swaps value and gate,
changes.  The largest errors measured on an H100 80GB HBM3 at a 400 W power limit are listed
beside BLOCK_GATES: at most 0.55 of the output's gate and 0.6 of any gradient's.
"""
import pytest
import torch

import block_oracle as BO

pytestmark = pytest.mark.gpu


def _run(case, prefill=None):
    """TransformerFn forward + backward -> (out, dx, [flat-weight gradients])."""
    from x_clip_b200 import engine as E
    ws = [w.clone().requires_grad_(True) for w in case["weights"]]
    if prefill is not None:
        for w, p in zip(ws, prefill):
            w.grad = p.clone()
    x = case["x"].clone().requires_grad_(True)
    cos, sin = case["rot"] if case["rot"] is not None else (None, None)
    out = E.TransformerFn.apply(x, case["mask"], case["heads"], BO.BLOCK_DEPTH, case["causal"], cos, sin, True, None, *ws)
    out.backward(case["dout"])
    torch.cuda.synchronize()
    return out.detach(), x.grad, [w.grad for w in ws]


@pytest.mark.parametrize("name", list(BO.BLOCK_CASES))
def test_transformer_fp64(cuda_device, name):
    case = BO.block_case(name, device=cuda_device)
    out, dx, grads = _run(case)
    xr = case["x"].double().requires_grad_(True)
    ws = [w.double().requires_grad_(True) for w in case["weights"]]
    ref = BO.transformer_stack(xr, ws, BO.BLOCK_DEPTH, case["heads"], case["mask"], case["causal"], case["rot"])
    ref.backward(case["dout"].double())
    names = BO.flat_names(BO.BLOCK_DEPTH)
    for nm, got, want in [("out", out, ref.detach()), ("dx", dx, xr.grad)] + list(zip(names, grads, [w.grad for w in ws])):
        gate = BO.BLOCK_GATES[nm.split(".")[0]]
        rel = BO.rel_fro(got, want)
        print(f"GATE block_{nm}[{name}] {rel / gate:.4f}")
        assert rel <= gate, (nm, rel, gate)


def test_transformer_inplace_accumulation(cuda_device):
    """engine._accumulate_into_grad = True (the micro-batched step's mode for all but the last chunk):
    the kernels add into the prefilled .grad buffers; the result is prefill + the fresh gradient."""
    from x_clip_b200 import engine as E
    case = BO.block_case("d512_mask", device=cuda_device)
    _, dx0, fresh = _run(case)
    gen = torch.Generator().manual_seed(11)
    prefill = [torch.randn(w.shape, generator=gen).to(cuda_device) * g.abs().max() for w, g in zip(case["weights"], fresh)]
    prev = E._accumulate_into_grad
    E._accumulate_into_grad = True
    try:
        _, dx1, acc = _run(case, prefill)
    finally:
        E._accumulate_into_grad = prev
    assert torch.equal(dx0, dx1)
    for nm, a, p, f in zip(BO.flat_names(BO.BLOCK_DEPTH), acc, prefill, fresh):
        err = (a.double() - p.double() - f.double()).abs()
        scale = (p.double().abs() + f.double().abs()).max()
        assert err.max().item() <= 1e-5 * scale.item(), (nm, err.max().item(), scale.item())
