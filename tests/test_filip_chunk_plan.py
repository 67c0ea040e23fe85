"""The row-chunk plan of the FILIP loss (x_clip_b200/filip.py), on the CPU: chunk boundaries, the
transient byte bound, and the byte arithmetic of the plan against the tensors FilipLossFn allocates
(its kernels replaced by shape-only stand-ins that record what they allocate)."""
import pytest
import torch

from x_clip_b200 import _lib, filip
from x_clip_b200 import kernels as K

TOKENS = [1, 7, 77, 98, 576]


@pytest.mark.parametrize("rows_per_sample", TOKENS)
@pytest.mark.parametrize("seg_len", TOKENS)
@pytest.mark.parametrize("b,B", [(5, 5), (256, 2048), (4096, 4096), (4096, 32768)])
def test_chunks_fall_on_sample_boundaries_within_the_budget(rows_per_sample, seg_len, b, B):
    # pass A: rows = b captions, segments = B images; pass B: rows = B images, segments = b captions
    for samples, nseg in ((b, B), (B, b)):
        R = samples * rows_per_sample
        chunks = filip.chunk_bounds(rows_per_sample, samples, nseg)
        assert chunks[0][0] == 0 and chunks[-1][1] == R
        for (r0, r1), nxt in zip(chunks, chunks[1:] + [(R, R)]):
            assert r1 == nxt[0] and r1 > r0
            assert r0 % rows_per_sample == 0 and r1 % rows_per_sample == 0
            assert filip.chunk_transient_bytes(r1 - r0, R, nseg, seg_len) <= filip.FILIP_CHUNK_BYTES


def test_saved_state_figures():
    """2 bytes per (row, sample) of both passes: the cfg3 one-GPU figure, 5.9 GB instead of 23.5 GB."""
    n = filip.saved_bytes(4096, 4096, 77, 98)
    assert n == 2 * (4096 * 77 * 4096 + 4096 * 98 * 4096)
    assert round(n / 1e9, 1) == 5.9 and round(4 * n / 1e9, 1) == 23.5


class _ShapeKernels:
    """Stand-ins for the kernels FilipLossFn calls: outputs of the right shapes and dtypes, every
    allocation recorded as (kind, rows, bytes)."""

    check_arg16_seg_len = staticmethod(K.check_arg16_seg_len)

    def __init__(self):
        self.log = []

    def filip_segmax16(self, a, b, temp_exp, seg_len, col_mul, col_add, want_max=True, seg_arg=None):
        R, nseg = a.shape[0], b.shape[0] // seg_len
        keys = torch.empty((R, nseg), dtype=torch.int64)
        m = torch.zeros((R, nseg)) if want_max else None
        own = seg_arg is None
        arg = torch.zeros((R, nseg), dtype=torch.int16) if own else (None if seg_arg is False else seg_arg)
        if arg is not None:
            assert arg.shape == (R, nseg) and arg.dtype == torch.int16 and arg.is_contiguous()
        transient = keys.nbytes + (m.nbytes if m is not None else 0) + (arg.nbytes if own else 0)
        self.log.append(("segmax" if want_max else "recompute", R, transient))
        return m, arg

    def filip_reduce(self, m, w, samples, length, nseg, transpose):
        assert m.shape == (samples * length, nseg) and w.numel() == samples * length
        return torch.zeros((nseg, samples) if transpose else (samples, nseg))

    def filip_nce_fwd(self, s, off, dcl, loss, scale, row_valid=None):
        return torch.zeros(s.shape[0])

    def filip_nce_bwd(self, s, lse, off, dcl, gscale, row_valid=None):
        return torch.zeros_like(s)

    def filip_expand16(self, arg, wmat, rowscale, temp_exp, row0, rows_per_sample, seg_len, nseg):
        C = nseg * seg_len
        g = torch.zeros((arg.shape[0], (C + 7) // 8 * 8), dtype=torch.bfloat16)
        self.log.append(("expand", row0, arg.shape[0], g.nbytes))
        return g[:, :C]

    def gemm(self, a, b, **kw):
        pass


def _run_shape_only(monkeypatch, b, T, I, D, extra, save_bytes, chunk_bytes):
    fake = _ShapeKernels()
    monkeypatch.setattr(filip, "K", fake)
    monkeypatch.setattr(filip, "FILIP_SAVE_BYTES", save_bytes)
    monkeypatch.setattr(filip, "FILIP_CHUNK_BYTES", chunk_bytes)
    lat = [torch.zeros((b, T, D)), torch.zeros((b, I, D))]
    if extra:
        lat += [torch.zeros((b, T, D)), torch.zeros((b, I, D))]
    z = [t.requires_grad_(True) for t in lat]
    ops = tuple((torch.zeros((t.shape[0] * t.shape[1], 3 * D), dtype=torch.bfloat16),) * 2 for t in lat)
    mask = torch.ones((b, T), dtype=torch.bool)
    mask[0, 1:] = False
    temp = torch.zeros((), requires_grad=True)
    stats = {}
    loss = filip.FilipLossFn.apply(z[0], z[1], z[2] if extra else None, z[3] if extra else None, temp, ops,
                                   mask, False, False, stats)
    loss.backward()
    return fake.log, stats


@pytest.mark.parametrize("extra", [False, True])
@pytest.mark.parametrize("plan", ["none", "part", "all"])
@pytest.mark.parametrize("T,I", [(7, 9), (77, 98), (48, 144)])
def test_plan_bytes_match_what_the_loss_allocates(monkeypatch, T, I, extra, plan):
    b, D = 6, 8
    chunk_bytes = 24 * 1024                    # up to 6 chunks per pass at these sizes
    total = filip.saved_bytes(b, b, T, I)
    save = {"none": 0, "part": total // 2, "all": total}[plan]
    log, stats = _run_shape_only(monkeypatch, b, T, I, D, extra, save, chunk_bytes)

    passes = [(T, b, I), (I, b, T)]           # (rows per sample, segments, seg_len)
    rows_total = sum(rps * b for rps, _, _ in passes)
    assert stats["rows_saved"] + stats["rows_recomputed"] == rows_total
    assert stats["saved_bytes"] <= save
    if plan == "all":
        assert stats["saved_bytes"] == total and stats["rows_recomputed"] == 0
    if plan == "none":
        assert stats["saved_bytes"] == 0 and stats["rows_saved"] == 0
    if plan == "part":
        assert 0 < stats["rows_saved"] < rows_total

    fwd = [e for e in log if e[0] == "segmax"]
    rec = [e for e in log if e[0] == "recompute"]
    exp = [e for e in log if e[0] == "expand"]
    # forward: every row once, in the planned chunks, each with 12 B of keys + maxima per entry
    k = 0
    for rps, nseg, seg_len in passes:
        chunks = filip.chunk_bounds(rps, b, nseg, chunk_bytes)
        for r0, r1 in chunks:
            kind, rows, nbytes = fwd[k]
            assert rows == r1 - r0 and nbytes == rows * nseg * (filip.KEY_BYTES + filip.MAX_BYTES)
            assert filip.chunk_transient_bytes(rows, b * rps, nseg, seg_len, chunk_bytes) <= chunk_bytes
            k += 1
    assert k == len(fwd)
    # backward: recomputed rows = rows not saved, with keys + argmax transient per entry
    assert sum(e[1] for e in rec) == stats["rows_recomputed"]
    # every row of both passes is expanded exactly once, in windows whose G stays in the budget
    covered = sum(e[2] for e in exp)
    assert covered == rows_total
    for _, row0, rows, nbytes in exp:
        assert nbytes <= chunk_bytes // 2 + rows * 16


def test_seg_len_over_65535_is_refused_before_any_launch(monkeypatch):
    with pytest.raises(_lib.XClipB200Error, match="65535"):
        K.check_arg16_seg_len(65536)
    K.check_arg16_seg_len(65535)
    # the kernels' wrappers refuse before touching their operands (these are not even CUDA tensors)
    with pytest.raises(_lib.XClipB200Error, match="65535"):
        K.filip_segmax16(torch.zeros(8, 24), torch.zeros(65536, 24), torch.ones(1), 65536, None, None)
    with pytest.raises(_lib.XClipB200Error, match="65535"):
        K.filip_expand16(torch.zeros((1, 1), dtype=torch.int16), None, None, None, 0, 1, 65536, 1)

    # and so does the loss: an image of 65536 tokens stops it before its first kernel
    class _NoKernels(_ShapeKernels):
        def __getattribute__(self, name):
            if name.startswith("filip_") or name == "gemm":
                raise AssertionError(f"{name} called")
            return object.__getattribute__(self, name)

    monkeypatch.setattr(filip, "K", _NoKernels())
    monkeypatch.setattr(filip, "FILIP_SAVE_BYTES", 0)
    b, T, I, D = 1, 2, 65536, 8
    zt, zi = torch.zeros((b, T, D), requires_grad=True), torch.zeros((b, I, D), requires_grad=True)
    ops = ((torch.zeros((T, 3 * D)),) * 2, (torch.zeros((I, 3 * D)),) * 2)
    with pytest.raises(_lib.XClipB200Error, match="65535"):
        filip.FilipLossFn.apply(zt, zi, None, None, torch.zeros(()), ops, torch.ones((b, T), dtype=torch.bool),
                                False, False)
