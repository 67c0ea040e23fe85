"""The micro-batched step's retention plan on the CPU: what TransformerFn saves per token and layer in
each save mode (its kernels replaced by shape-only stand-ins), and the decisions of engine.RetainPlan,
driven as the step drives it on a simulated card, at the cfg3 and FILIP shapes from those figures."""
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
    with E._scoped_global("_compact_save", compact):
        E.TransformerFn.forward(ctx, torch.empty(B, n, d, dtype=BF16), None, heads, depth, False, None, None, True,
                                None, *weights)
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




def _step(plan, avail, foot, reserve=0, oom_at=None):
    """Drive `plan` through one step as ChunkedClipLossFn.forward calls it, on a simulated card with `avail`
    free bytes before the first chunk, where a full-size chunk holds foot[mode] bytes in each save mode and
    the kept encode of chunk `oom_at` runs out of memory (the card then holds what it held before).
    -> (the plan's modes, [(chunk, mode) of every kept encode], the free-HBM figures the plan was given)."""
    free, encodes, given = avail, [], []

    def measure():
        given.append(free)
        return free

    def encode(k, mode):
        nonlocal free
        encodes.append((k, mode))
        if k == oom_at:
            return None
        nbytes = foot[mode] * plan.rows[k] // plan.chunk
        free -= nbytes
        return nbytes

    for k in range(len(plan.rows)):
        mode = plan.mode_for(k, measure() if plan.weighs else None)
        got = None if mode is None else encode(k, mode)
        if got is not None and plan.foot is None:
            plan.measured(got, reserve)
            if plan.weighs_compact and plan.compact(measure()):
                free += got
                got = encode(k, plan.mode)
                if got is not None:
                    plan.measured(got, plan.reserve)
        if mode is not None and got is None:
            plan.out_of_memory()
        elif got is not None and plan.weighs_release(k) and plan.release(measure()):
            free += got
    return plan.modes, encodes, given


CFG3_ROWS = [768] * 5 + [256]
CFG3_FOOT = {"full": 768 * _cfg3_pair_bytes(21), "compact": 768 * _cfg3_pair_bytes(7)}


def _auto(rows=CFG3_ROWS, remembered=None, mode=None, retain="auto"):
    return E.RetainPlan(retain, remembered, mode, rows, rows[0])


def test_cfg3_keeps_five_compact_chunks():
    """cfg3: 4096 pairs in chunks of 768 (5 x 768 + 256) on an 80 GB card with ~76 GiB free.  Full chunks
    (42 GiB) would keep two; compact chunks (14 GiB) keep four full-size chunks and the tail.  The first
    chunk is measured in full mode, then again in compact mode, whose footprint the plan keeps."""
    assert round(CFG3_FOOT["full"] / GiB, 1) == 41.8 and round(CFG3_FOOT["compact"] / GiB, 1) == 13.9
    plan = _auto()
    modes, encodes, given = _step(plan, 76 * GiB, CFG3_FOOT)
    assert modes == ["compact"] * 4 + [None, "compact"]
    assert encodes[:2] == [(0, "full"), (0, "compact")] and plan.foot == CFG3_FOOT["compact"]
    assert len(given) == 2 + 5 and plan.remembers and plan.oom_fallbacks == 0


def test_small_batches_keep_full_chunks():
    """Where every chunk fits in full mode the plan keeps them all in full mode: no rebuild work."""
    foot = {m: b // 3 for m, b in CFG3_FOOT.items()}
    assert _step(_auto([256] * 4), 76 * GiB, foot)[0] == ["full"] * 4
    assert _step(_auto([768]), 76 * GiB, CFG3_FOOT)[0] == ["full"]


def test_single_chunk_is_never_measured_again():
    """One chunk: nothing else competes for the HBM, so the plan neither weighs compact mode nor lets the
    chunk go, however little is free - the free HBM is not even asked for."""
    plan = _auto([768])
    modes, encodes, given = _step(plan, 20 * GiB, CFG3_FOOT)
    assert modes == ["full"] and encodes == [(0, "full")] and given == []


def test_filip_reserve_costs_compact_chunks():
    """FILIP at cfg3's shapes: the loss's reserve (saved argmax, chunk budget, token latents) is left free,
    so fewer compact chunks stay than without it, and still more than full chunks would."""
    reserve = filip.step_reserve_bytes(4096, 4096, 78, 99, 512, False)
    plan = _auto()
    modes, _, _ = _step(plan, 76 * GiB, CFG3_FOOT, reserve)
    kept = sum(m is not None for m in modes)
    assert set(modes) <= {"compact", None} and modes[0] == "compact"
    assert 2 < kept < 5, (modes, reserve / GiB)
    assert plan.reserve == reserve


def test_first_chunk_is_released_when_no_second_fits():
    """On the planning step the first chunk is let go (re-encoded in backward) when the HBM left beside it
    would not hold a second full-size chunk; its memory then goes to the later chunks."""
    modes, encodes, given = _step(_auto(), 40 * GiB, CFG3_FOOT)
    assert encodes[:2] == [(0, "full"), (0, "compact")]
    assert modes == [None, "compact", None, None, None, "compact"]


def test_remembered_plan_is_replayed():
    """"auto" with a remembered plan repeats it chunk by chunk, measures nothing and stores nothing."""
    remembered = ["compact", None, "compact", "full", None, None]
    plan = _auto(remembered=remembered)
    modes, encodes, given = _step(plan, 1 * GiB, CFG3_FOOT)
    assert modes == remembered and given == []
    assert encodes == [(0, "compact"), (2, "compact"), (3, "full")]
    assert not plan.remembers


@pytest.mark.parametrize("mode", [None, "compact"])
def test_integer_plan_keeps_the_first_chunks(mode):
    """An int keeps the first `retain` chunks, in full mode unless RETAIN_MODE forces one; it measures no
    free HBM and is not remembered."""
    plan = _auto(retain=2, mode=mode)
    modes, encodes, given = _step(plan, 1 * GiB, CFG3_FOOT)
    want = mode or "full"
    assert modes == [want, want, None, None, None, None] and given == []
    assert encodes == [(0, want), (1, want)] and not plan.remembers


def test_forced_compact_mode_skips_the_full_measurement():
    """RETAIN_MODE = "compact": the first chunk is encoded and measured in compact mode once, and every
    kept chunk is compact."""
    plan = _auto(mode="compact")
    modes, encodes, _ = _step(plan, 76 * GiB, CFG3_FOOT)
    assert encodes[:2] == [(0, "compact"), (1, "compact")]
    assert modes == ["compact"] * 4 + [None, "compact"] and plan.foot == CFG3_FOOT["compact"]


@pytest.mark.parametrize("remembered", [None, ["full"] * 6])
def test_out_of_memory_ends_the_keeping(remembered):
    """A kept encode that runs out of memory at chunk 2 of 6: that chunk and every later one are re-encoded
    in backward, the fallback is counted, and the cut plan is remembered - by the planning step and in
    place of a remembered plan alike."""
    foot = {m: b // 10 for m, b in CFG3_FOOT.items()}
    plan = _auto(remembered=remembered)
    modes, encodes, _ = _step(plan, 76 * GiB, foot, oom_at=2)
    assert modes == ["full", "full", None, None, None, None]
    assert encodes[-1] == (2, "full")
    assert plan.oom_fallbacks == 1 and plan.remembers


def test_out_of_memory_of_an_integer_plan_is_not_remembered():
    """Nothing was remembered for the batch: an int plan cut by an out-of-memory stays this step's own."""
    plan = _auto(retain=4)
    modes, _, _ = _step(plan, 76 * GiB, CFG3_FOOT, oom_at=1)
    assert modes == ["full"] + [None] * 5 and plan.oom_fallbacks == 1 and not plan.remembers
