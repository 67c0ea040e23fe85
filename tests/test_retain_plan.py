"""The micro-batched step's retention plan on the CPU: what TransformerFn saves per token and layer in
each save mode (its kernels replaced by shape-only stand-ins), and the plan's decisions at the cfg3 and
FILIP shapes from those figures."""
from types import SimpleNamespace

import pytest
import torch

from x_clip_b200 import engine as E
from x_clip_b200 import filip

BF16, F32 = torch.bfloat16, torch.float32
GiB = 1 << 30


class _ShapeKernels:
    """The kernels TransformerFn's forward calls, as outputs of the right shapes and dtypes."""

    @staticmethod
    def layernorm_fwd(x, g, res=None, g2=None, eps=None):
        M, d = x.shape
        two = (torch.empty(M, d, dtype=BF16), torch.empty(M, 2, dtype=F32)) if g2 is not None else (None, None)
        return (torch.empty(M, d, dtype=BF16), torch.empty(M, 2, dtype=F32)) + two

    @staticmethod
    def gemm(a, b):
        return torch.empty(a.shape[0], b.shape[0], dtype=BF16)

    @staticmethod
    def attn_fwd(qkv, mask, B, n, heads, scale, causal, dropout=None):
        return torch.empty(B * n, heads * 64, dtype=BF16), torch.empty(B, heads, n, dtype=F32)

    @staticmethod
    def ff_up(x, w1p, need_u=True):
        M, d = x.shape
        u = torch.empty(M, 8 * d, dtype=BF16) if need_u else None
        return u, torch.empty(M, 4 * d, dtype=BF16), torch.empty(M, d // 16, 2, dtype=F32)

    @staticmethod
    def ff_down(h, w2g, colvec, rowsum, res, eps):
        M, d = res.shape
        return torch.empty(M, d, dtype=BF16), torch.empty(M, d, dtype=BF16), torch.empty(M, 2, dtype=F32)


def _saved_activation_bytes(monkeypatch, B, n, d, heads, depth, compact):
    """Bytes of the per-layer activations one TransformerFn forward keeps for its backward."""
    monkeypatch.setattr(E, "K", _ShapeKernels)
    monkeypatch.setattr(E, "weight_bf16", lambda w: torch.empty(w.shape, dtype=BF16))
    monkeypatch.setattr(E, "ff_weights", lambda w1, w2, g4: (torch.empty(8 * d, d, dtype=BF16),
                                                             torch.empty(d, 4 * d, dtype=BF16),
                                                             torch.empty(d, dtype=F32)))
    weights = [torch.empty(d), torch.empty(d)]
    for _ in range(depth):
        weights += [torch.empty(d), torch.empty(3 * d, d), torch.empty(d, d), torch.empty(d), torch.empty(d),
                    torch.empty(8 * d, d), torch.empty(4 * d), torch.empty(d, 4 * d)]
    ctx = SimpleNamespace()
    with E._CompactSave(compact):
        E.TransformerFn._forward(ctx, torch.empty(B, n, d, dtype=BF16), None, heads, depth, False, None, None, True,
                                 None, weights)
    assert len(ctx.saved) == depth
    weight_shapes = {(8 * d, d), (d, 4 * d), (d,)}
    seen, total = set(), 0
    for layer in ctx.saved:
        flat = [t for x in layer for t in (x if isinstance(x, tuple) else (x,))]
        for t in flat:
            if t is None or tuple(t.shape) in weight_shapes or t.data_ptr() in seen:
                continue
            seen.add(t.data_ptr())
            total += t.numel() * t.element_size()
    return total


@pytest.mark.parametrize("d,heads", [(512, 8), (768, 12)])
def test_saved_bytes_per_token_and_layer(monkeypatch, d, heads):
    """Full: xcur, qkv, o, y, x1, xn2, u, h, acc = 21 d bf16; compact: xcur, qkv, o, y, acc = 7 d.  Row
    statistics: st1, st_y, st_v and the attention's lse in both, st_x1 in full mode only."""
    B, n, depth = 3, 5, 2
    tokens_layers = B * n * depth
    full = _saved_activation_bytes(monkeypatch, B, n, d, heads, depth, False)
    compact = _saved_activation_bytes(monkeypatch, B, n, d, heads, depth, True)
    assert full == tokens_layers * (2 * 21 * d + 4 * 8 + 4 * heads)
    assert compact == tokens_layers * (2 * 7 * d + 3 * 8 + 4 * heads)


def _cfg3_pair_bytes(saved_d):
    """Saved activation bytes per pair of the cfg3 towers: ViT-B/16 at patch dropout 0.5 (98 patches +
    CLS, d 768, 12 layers) and the 77-token text tower (+ CLS, d 512, 12 layers)."""
    return 2 * saved_d * 12 * (99 * 768 + 78 * 512)


def _plan(avail, foot_full, foot_compact, rows, chunk, reserve=0):
    """The "auto" plan of ChunkedClipLossFn on the planning step, for free HBM `avail` before the first
    chunk: -> the save mode of every chunk (None: re-encoded in backward)."""
    if len(rows) == 1 or E.fits_all_full(avail - foot_full, foot_full, rows, chunk, reserve):
        mode, foot = "full", foot_full
    else:
        mode, foot = "compact", foot_compact
    avail -= foot * rows[0] / chunk
    plan = [mode]
    for r in rows[1:]:
        keep = avail >= E.retain_need_bytes(foot, r, chunk, mode, reserve)
        plan.append(mode if keep else None)
        avail -= foot * r / chunk if keep else 0
    return plan


def test_cfg3_keeps_five_compact_chunks():
    """cfg3: 4096 pairs in chunks of 768 (5 x 768 + 256) on an 80 GB card with ~76 GiB free.  Full chunks
    (42 GiB) would keep two; compact chunks (14 GiB) keep four full-size chunks and the tail."""
    rows = [768] * 5 + [256]
    full, compact = 768 * _cfg3_pair_bytes(21), 768 * _cfg3_pair_bytes(7)
    assert round(full / GiB, 1) == 41.8 and round(compact / GiB, 1) == 13.9
    assert _plan(76 * GiB, full, compact, rows, 768) == ["compact"] * 4 + [None, "compact"]


def test_small_batches_keep_full_chunks():
    """Where every chunk fits in full mode the plan keeps them all in full mode: no rebuild work."""
    rows = [256] * 4
    full, compact = 256 * _cfg3_pair_bytes(21), 256 * _cfg3_pair_bytes(7)
    assert _plan(76 * GiB, full, compact, rows, 256) == ["full"] * 4
    assert _plan(76 * GiB, full, compact, [768], 768) == ["full"]


def test_filip_reserve_costs_compact_chunks():
    """FILIP at cfg3's shapes: the loss's reserve (saved argmax, chunk budget, token latents) is left free,
    so fewer compact chunks stay than without it, and still more than full chunks would."""
    rows = [768] * 5 + [256]
    full, compact = 768 * _cfg3_pair_bytes(21), 768 * _cfg3_pair_bytes(7)
    reserve = filip.step_reserve_bytes(4096, 4096, 78, 99, 512, False)
    plan = _plan(76 * GiB, full, compact, rows, 768, reserve)
    kept = sum(m is not None for m in plan)
    assert set(plan) <= {"compact", None} and plan[0] == "compact"
    assert 2 < kept < 5, (plan, reserve / GiB)
