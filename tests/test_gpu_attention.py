"""Fused attention fwd/bwd vs an fp32 torch restatement of the reference core
(x_clip/x_clip.py:217-244) on the same bf16-rounded q,k,v."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref_attention(qkv, mask, B, n, H, scale, causal=False):
    q, k, v = qkv.float().view(B, n, 3, H, 64).permute(2, 0, 3, 1, 4)
    s = (q * scale) @ k.transpose(-1, -2)
    if mask is not None:
        s = s.masked_fill(~mask[:, None, None, :], -torch.finfo(torch.float32).max)
    if causal:      # x_clip.py:233-236
        cm = torch.ones(n, n, dtype=torch.bool, device=s.device).triu(1)
        s = s.masked_fill(cm, -torch.finfo(torch.float32).max)
    p = s.softmax(-1)
    return (p @ v).permute(0, 2, 1, 3).reshape(B * n, H * 64), s


CASES = [(2, 33, 4, False), (3, 65, 8, False), (2, 128, 2, True), (2, 17, 4, True),
         (2, 197, 12, False), (2, 257, 8, True), (1, 320, 2, True), (5, 78, 8, True),
         # n = 64k+1: a last 64-row block with one row; 24*8 (b,h) items: many CTAs per SM
         (2, 129, 4, True), (3, 129, 2, False), (24, 257, 8, True), (20, 257, 8, False),
         # short sequences (attention_small.cu): ViT-B/16 with patch dropout (98), CLIP text (78),
         # README image tower (32); several items per CTA; every 16-key tail width
         (130, 98, 12, False), (90, 78, 8, True), (300, 32, 8, False), (3, 64, 4, True), (2, 112, 3, True),
         (2, 1, 2, False), (3, 16, 2, True), (2, 100, 4, True), (4, 128, 12, False), (2, 48, 2, False),
         (2, 81, 5, True),
         # batch x heads beyond 65535 CTAs in one grid dimension
         (16640, 16, 4, True)]
CAUSAL_CASES = [(3, 78, 8, True), (2, 33, 4, False), (2, 128, 2, True), (40, 64, 8, False)]


def _mk(B, n, H, masked, dev, seed=0):
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(B * n, 3 * H * 64, generator=g).to(dev).bfloat16()
    mask = None
    if masked:
        mask = (torch.rand(B, n, generator=g) > 0.3).to(dev)
        mask[:, 0] = True     # the CLS key is always attendable (x_clip.py:335)
    return qkv, mask


@pytest.mark.parametrize("B,n,H,masked", CASES)
def test_attn_fwd(cuda_device, B, n, H, masked):
    from x_clip_b200 import kernels as K
    qkv, mask = _mk(B, n, H, masked, cuda_device)
    scale = 64 ** -0.5
    o, lse = K.attn_fwd(qkv, mask, B, n, H, scale)
    torch.cuda.synchronize()
    ref, s = _ref_attention(qkv, mask, B, n, H, scale)
    err = (o.float() - ref).abs().max().item()
    assert err <= 2e-2 * ref.abs().max().item(), f"o err {err}"
    ref_lse = torch.logsumexp(s, dim=-1) / 0.6931471805599453
    assert torch.allclose(lse, ref_lse, atol=2e-2, rtol=1e-3)


@pytest.mark.parametrize("B,n,H,masked", CASES)
def test_attn_bwd(cuda_device, B, n, H, masked):
    from x_clip_b200 import kernels as K
    qkv, mask = _mk(B, n, H, masked, cuda_device, seed=1)
    scale = 64 ** -0.5
    o, lse = K.attn_fwd(qkv, mask, B, n, H, scale)
    d_o = torch.randn(B * n, H * 64, device=cuda_device).bfloat16()
    dqkv = K.attn_bwd(qkv, mask, o, d_o, lse, B, n, H, scale)
    torch.cuda.synchronize()
    qf = qkv.float().requires_grad_(True)
    ref, _ = _ref_attention(qf, mask, B, n, H, scale)
    ref.backward(d_o.float())
    g = qf.grad
    inner = H * 64
    for name, sl in (("dq", slice(0, inner)), ("dk", slice(inner, 2 * inner)), ("dv", slice(2 * inner, 3 * inner))):
        err = (dqkv[:, sl].float() - g[:, sl]).abs().max().item()
        sc = g[:, sl].abs().max().item()
        assert err <= 3e-2 * sc + 1e-5, f"{name}: err {err} vs scale {sc}"   # (n = 1: dq = dk = 0 up to fp32 rounding of p = 2^(s c - lse))
        rel = (dqkv[:, sl].float() - g[:, sl]).norm().item() / (g[:, sl].norm().item() + 1e-3)
        assert rel < 1e-2, f"{name}: rel fro err {rel}"


@pytest.mark.parametrize("B,n,H,masked", CAUSAL_CASES)
def test_attn_causal_fwd_bwd(cuda_device, B, n, H, masked):
    """Causal mask of the text tower (x_clip.py:233-236, text_causal_mask=True), n <= 128."""
    from x_clip_b200 import kernels as K
    qkv, mask = _mk(B, n, H, masked, cuda_device, seed=2)
    scale = 64 ** -0.5
    o, lse = K.attn_fwd(qkv, mask, B, n, H, scale, causal=True)
    d_o = torch.randn(B * n, H * 64, device=cuda_device).bfloat16()
    dqkv = K.attn_bwd(qkv, mask, o, d_o, lse, B, n, H, scale, causal=True)
    torch.cuda.synchronize()
    qf = qkv.float().requires_grad_(True)
    ref, s = _ref_attention(qf, mask, B, n, H, scale, causal=True)
    err = (o.float() - ref.detach()).abs().max().item()
    assert err <= 2e-2 * ref.abs().max().item(), f"o err {err}"
    ref.backward(d_o.float())
    rel = (dqkv.float() - qf.grad).norm().item() / qf.grad.norm().item()
    assert rel < 1e-2, f"rel fro err {rel}"
