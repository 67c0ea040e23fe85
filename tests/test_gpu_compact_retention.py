"""Compact retention: the LayerNorm backward's rebuilt forward output, TransformerFn's compact save mode
against its full one, and the micro-batched step with its kept chunks in compact mode against the single
pass."""
import pytest
import torch

import block_oracle as BO
from test_gpu_aux_microbatch import CONFIGS, TINY, _pair, _rel

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("d", [128, 256, 384, 512, 640, 768, 896, 1024])
@pytest.mark.parametrize("rows", [1, 77, 1001])
def test_layernorm_bwd_emits_the_forward_output(cuda_device, d, rows):
    """xn of layernorm_bwd equals layernorm_fwd's output, with and without `add`, both for a plain
    LayerNorm (out) and for the chained second norm (out2 of bf16(out)); dx is unchanged by asking."""
    from x_clip_b200 import kernels as K
    gen = torch.Generator().manual_seed(d + rows)
    x = torch.randn(rows, d, generator=gen).bfloat16().to(cuda_device)
    g, g2 = [(1 + 0.3 * torch.randn(d, generator=gen)).to(cuda_device) for _ in range(2)]
    dy = torch.randn(rows, d, generator=gen).bfloat16().to(cuda_device)
    add = torch.randn(rows, d, generator=gen).bfloat16().to(cuda_device)
    out, st, out2, st2 = K.layernorm_fwd(x, g, g2=g2)
    for xin, stats, gain, want in ((x, st, g, out), (out, st2, g2, out2)):
        for a in (None, add):
            dx0 = K.layernorm_bwd(dy, xin, stats, gain, add=a)
            dx, xn = K.layernorm_bwd(dy, xin, stats, gain, add=a, want_xn=True)
            torch.cuda.synchronize()
            assert torch.equal(xn, want)
            assert torch.equal(dx, dx0)


def _transformer(case, compact, drop=None):
    from x_clip_b200 import engine as E
    ws = [w.clone().requires_grad_(True) for w in case["weights"]]
    x = case["x"].clone().requires_grad_(True)
    cos, sin = case["rot"] if case["rot"] is not None else (None, None)
    with E._scoped_global("_compact_save", compact):
        out = E.TransformerFn.apply(x, case["mask"], case["heads"], BO.BLOCK_DEPTH, case["causal"], cos, sin, True,
                                    drop, *ws)
    out.backward(case["dout"])
    torch.cuda.synchronize()
    return out.detach(), x.grad, [w.grad for w in ws]


@pytest.mark.parametrize("name", list(BO.BLOCK_CASES))
@pytest.mark.parametrize("dropout", [False, True])
def test_compact_transformer_matches_full(cuda_device, name, dropout):
    """Output and dx bit for bit the full mode's; every weight gradient within BLOCK_GATES of the fp64
    reference (without dropout) and within the wgrad GEMM's atomics of the full mode's."""
    case = BO.block_case(name, device=cuda_device)
    drop = ((0.1, 0.1), torch.tensor([4321], dtype=torch.int64, device=cuda_device)) if dropout else None
    out_f, dx_f, g_f = _transformer(case, False, drop)
    out_c, dx_c, g_c = _transformer(case, True, drop)
    assert torch.equal(out_c, out_f)
    assert torch.equal(dx_c, dx_f)
    names = BO.flat_names(BO.BLOCK_DEPTH)
    for nm, a, b in zip(names, g_c, g_f):
        assert _rel(a, b) <= 1e-5, (nm, _rel(a, b))
    if dropout:
        return
    xr = case["x"].double().requires_grad_(True)
    ws = [w.double().requires_grad_(True) for w in case["weights"]]
    ref = BO.transformer_stack(xr, ws, BO.BLOCK_DEPTH, case["heads"], case["mask"], case["causal"], case["rot"])
    ref.backward(case["dout"].double())
    for nm, got, w in zip(names, g_c, ws):
        gate = BO.BLOCK_GATES[nm.split(".")[0]]
        assert BO.rel_fro(got, w.grad) <= gate, (nm, BO.rel_fro(got, w.grad), gate)


STEP_CONFIGS = {"plain": dict(TINY, num_text_tokens=120), "filip_mlm": CONFIGS["filip_mlm"],
                "mlm_simsiam": CONFIGS["mlm_simsiam"], "image_grad": dict(TINY, num_text_tokens=120)}


@pytest.mark.parametrize("config", sorted(STEP_CONFIGS))
@pytest.mark.parametrize("retain", [0, 2, "auto"])
def test_compact_microbatched_step_equals_single_pass(cuda_device, monkeypatch, config, retain):
    """engine.RETAIN_MODE = "compact": the kept chunks are compact, the loss and every gradient (and the
    image's, for image_grad) those of the single pass."""
    from x_clip_b200 import engine as E
    monkeypatch.setattr(E, "RETAIN_MODE", "compact")
    single, micro, text, image = _pair(STEP_CONFIGS[config], cuda_device, 4, retain)
    images = [image, image]
    if config == "image_grad":
        images = [image.clone().requires_grad_(True), image.clone().requires_grad_(True)]
    l1 = single(text, images[0], return_loss=True)
    l1.backward()
    l2 = micro(text, images[1], return_loss=True)
    l2.backward()
    torch.cuda.synchronize()
    plan = micro.last_step_plan
    kept = {0: [], 2: [0, 1], "auto": [0, 1, 2]}[retain]          # tiny model: "auto" keeps all
    assert plan["chunks"] == 3 and plan["retained_chunks"] == kept and plan["compact_chunks"] == kept, plan
    assert abs(l2.item() - l1.item()) <= 1e-5 * abs(l1.item()), (l1.item(), l2.item())
    g1, g2 = dict(single.named_parameters()), dict(micro.named_parameters())
    for name, p in g1.items():
        q = g2[name]
        assert (p.grad is None) == (q.grad is None), name
        if p.grad is not None:
            assert _rel(q.grad, p.grad) <= 2e-3, (name, _rel(q.grad, p.grad))
    if config == "image_grad":
        assert _rel(images[1].grad, images[0].grad) <= 2e-3


def test_auto_plan_keeps_full_chunks_when_all_fit(cuda_device):
    """The tiny model fits: "auto" with the plan's own choice keeps every chunk in full mode, on the
    planning step and on the remembered plan."""
    single, micro, text, image = _pair(STEP_CONFIGS["plain"], cuda_device, 4, "auto")
    for _ in range(2):
        micro(text, image, return_loss=True).backward()
        assert micro.last_step_plan["retained_chunks"] == [0, 1, 2]
        assert micro.last_step_plan["compact_chunks"] == []
