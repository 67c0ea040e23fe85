"""FILIP at any token count: the segment max at lengths that are not multiples of 16 or exceed a
256-column tile (segments cut by one or more tile edges, merged through 64-bit keys), filip_expand16
at segment lengths that are not multiples of 8, and FilipLossFn at cfg3's 77 x 98 / 77 x 196, at
300 x 576 and at 7 x 9 tokens, against the fp64 references and gates of test_gpu_filip."""
import math

import pytest
import torch

from test_gpu_filip import (_check_expand, _col_mask_tables, _compare_filip, _filip_inputs,
                            _gen, _oracle_filip, _report_peak, _run_filip_loss, _run_segmax,
                            _start_peak, _unit, oracle_filip_chunked)

pytestmark = pytest.mark.gpu

BF16, F32 = torch.bfloat16, torch.float32
FMAX = torch.finfo(F32).max
TILE = 256                                     # columns per output tile of the segment-max GEMM


def _nseg_any(seg_len):
    """At least three tiles' worth of columns and at least three segments, with a partial last tile:
    short segments sit inside a tile or cross one edge, segments longer than a tile cross two or
    more."""
    nseg = max(3, -(-3 * TILE // seg_len) + 1)
    if (nseg * seg_len) % TILE == 0:
        nseg += 1
    return nseg


def _edges_crossed(seg_len, nseg):
    """{number of tile edges strictly inside a segment} over the segments"""
    out = set()
    for s in range(nseg):
        lo, hi = s * seg_len, (s + 1) * seg_len
        out.add(sum(1 for e in range(TILE, hi, TILE) if e > lo))
    return out


# --------------------------------------------------------------------------- segment max

SEG_LENS_ANY = [1, 2, 7, 9, 15, 17, 77, 98, 196, 255, 257, 300, 512, 513, 576, 1000]


def test_segment_counts_cover_the_tile_cases():
    """The cases below see segments inside a tile, across one edge and across two, and partial last
    tiles (wherever the segment length allows one: 512 tokens always end on a tile edge)."""
    seen = set()
    for L in SEG_LENS_ANY:
        nseg = _nseg_any(L)
        assert (nseg * L) % TILE != 0 or L % TILE == 0
        seen |= _edges_crossed(L, nseg)
    assert {0, 1, 2} <= seen


@pytest.mark.parametrize("D", [256, 72])               # K = 3D = 216: not a multiple of the 64-wide k-block
@pytest.mark.parametrize("seg_len", SEG_LENS_ANY)
def test_segmax_any_matches_fp64(cuda_device, seg_len, D):
    """R = 1 / 129 / 1100: ragged last row tile; m-fastest and n-fastest rasters."""
    gen = _gen(cuda_device, 5000 + 7 * seg_len + D)
    C = _nseg_any(seg_len) * seg_len
    zb = _unit((C, D), gen, cuda_device)
    for i, R in enumerate((1, 129, 1100)):
        za = _unit((R, D), gen, cuda_device)
        temp = math.e if i % 2 == 0 else 100.0
        _, _, ev, ea = _run_segmax(za, zb, temp, seg_len)
        print(f"segmax_any seg_len={seg_len} D={D} R={R} C={C}: error/gate value {ev:.3f} arg {ea:.3f}")


def _straddling(seg_len, nseg, edge):
    """index of the segment that contains tile edge `edge` strictly inside, or None"""
    s = edge // seg_len
    return s if s < nseg and s * seg_len < edge else None


@pytest.mark.parametrize("seg_len", [7, 9, 77, 98, 300, 513])
def test_segmax_any_masked_columns(cuda_device, seg_len):
    """Padded text tokens (col_mul 0 / col_add -FLT_MAX): a masked column is never returned while its
    segment has a valid one; a fully masked segment that straddles a tile edge gives exactly -FLT_MAX
    at index 0, and one whose only valid token sits past the edge returns that token."""
    gen = _gen(cuda_device, 11 + seg_len)
    D, nseg = 256, _nseg_any(seg_len)
    C = nseg * seg_len
    zb = _unit((C, D), gen, cuda_device)
    mask = torch.rand((nseg, seg_len), generator=gen, device=cuda_device) < 0.5
    s_empty = _straddling(seg_len, nseg, TILE)
    s_last = next(s for k in range(2, nseg * seg_len // TILE + 1)
                  for s in [_straddling(seg_len, nseg, k * TILE)] if s not in (None, s_empty))
    mask[s_empty] = False
    mask[s_last] = False
    mask[s_last, -1] = True
    for R in (129, 1100):
        za = _unit((R, D), gen, cuda_device)
        col_mul, col_add = _col_mask_tables(mask)
        m, arg, ev, ea = _run_segmax(za, zb, 100.0, seg_len, col_mul, col_add)
        empty = ~mask.any(1)
        assert bool(empty[s_empty])
        assert bool((m[:, empty] == -FMAX).all()) and bool((arg[:, empty] == 0).all())
        picked = mask[torch.arange(nseg, device=cuda_device)[None, :], arg.long()]
        assert bool(picked[:, ~empty].all()), "a padded token won the segment maximum"
        assert bool((arg[:, s_last] == seg_len - 1).all())
        print(f"segmax_any masked seg_len={seg_len} R={R}: error/gate value {ev:.3f} arg {ea:.3f}")


@pytest.mark.parametrize("seg_len", [7, 9, 77, 300, 513, 1000])
def test_segmax_any_ties_across_a_tile_edge_go_to_the_lowest_index(cuda_device, seg_len):
    """Two identical tokens p < q, both the segment's maximum.  In a segment that contains a tile edge
    e they sit at columns e - 1 and e, computed by two CTAs and merged through the keys; elsewhere at
    (s mod (seg_len - 1), seg_len - 1).  The lower index p must win everywhere."""
    gen = _gen(cuda_device, 333 + seg_len)
    D, nseg, R = 256, _nseg_any(seg_len), 300
    u = _unit((D,), gen, cuda_device)
    za = torch.nn.functional.normalize(u + 0.02 * torch.randn((R, D), generator=gen, device=cuda_device), dim=-1)
    zb = _unit((nseg, seg_len, D), gen, cuda_device)
    p = torch.empty(nseg, dtype=torch.long)
    crossing = 0
    for s in range(nseg):
        lo, hi = s * seg_len, (s + 1) * seg_len
        edges = [e for e in range(TILE, hi, TILE) if e > lo]
        if edges:
            p[s], q = edges[0] - 1 - lo, edges[0] - lo
            crossing += 1
        else:
            p[s], q = s % (seg_len - 1), seg_len - 1
        zb[s, p[s]] = u
        zb[s, q] = u
    assert crossing > 0
    _, arg, _, _ = _run_segmax(za, zb.reshape(-1, D), 100.0, seg_len)
    assert torch.equal(arg.long().cpu(), p[None, :].expand(R, nseg))


# --------------------------------------------------------------------------- expand

@pytest.mark.parametrize("seg_len", [7, 9, 77, 300])
def test_expand_any_matches_dense_construction(cuda_device, seg_len):
    samples, rows_per_sample, nseg = 6, 40, 5
    R = samples * rows_per_sample
    _check_expand(cuda_device, samples, rows_per_sample, nseg, seg_len,
                  [(0, R), (37, 150), (R - 1, 1)], seed=seg_len)


@pytest.mark.parametrize("seg_len", [7, 77])
def test_expand_pad_columns_are_never_read(cuda_device, seg_len):
    """G is [rows, roundup8(C)] behind a [:, :C] view.  Its pad columns are written as zeros, and with
    NaN written into them both gradient GEMMs (d rows = G @ cols, d cols = G^T @ rows) stay finite and
    equal to the fp64 products of the view."""
    from x_clip_b200 import kernels as K
    dev = cuda_device
    gen = _gen(dev, 21 + seg_len)
    samples, rows_per_sample, nseg, D = 6, 40, 5, 128
    R, C = samples * rows_per_sample, nseg * seg_len
    seg_arg = torch.randint(0, seg_len, (R, nseg), generator=gen, device=dev, dtype=torch.int16)
    wmat = torch.randn((samples, nseg), generator=gen, device=dev)
    rowscale = torch.rand((R,), generator=gen, device=dev) + 0.5
    alpha = torch.tensor([3.0], device=dev, dtype=F32)
    g = K.filip_expand16(seg_arg, wmat, rowscale, alpha, 0, rows_per_sample, seg_len, nseg)
    ld = g.stride(0)
    assert g.shape == (R, C) and ld % 8 == 0 and ld >= C and ld > C
    full = g.as_strided((R, ld), (ld, 1))
    assert not bool(full[:, C:].any())
    full[:, C:] = float("nan")
    cols = _unit((C, D), gen, dev).to(BF16)
    rows = _unit((R, D), gen, dev).to(BF16)
    d_rows = K.gemm(g, cols, b_major=1, out_dtype=F32)
    d_cols = K.gemm(g, rows, a_major=1, b_major=1, out_dtype=F32)
    g64 = g.double()
    for got, ref in ((d_rows, g64 @ cols.double()), (d_cols, g64.t() @ rows.double())):
        assert torch.isfinite(got).all()
        rel = (got.double() - ref).norm().item() / ref.norm().item()
        assert rel <= 1e-5, rel


# --------------------------------------------------------------------------- FilipLossFn vs the oracle

FILIP_ANY_SHAPES = [(5, 77, 98, 256), (4, 77, 196, 512), (4, 300, 576, 256), (33, 7, 9, 128)]


@pytest.mark.parametrize("temperature", [1.0, math.log(100.0)])
@pytest.mark.parametrize("extra", [False, True])
@pytest.mark.parametrize("dcl", [False, True])
@pytest.mark.parametrize("B,T,I,D", FILIP_ANY_SHAPES)
def test_filip_any_loss_fn_matches_fp64_oracle(cuda_device, B, T, I, D, dcl, extra, temperature):
    lat, mask = _filip_inputs(cuda_device, B, T, I, D, extra, seed=B * T + I + D)
    got = _run_filip_loss(lat, mask, temperature, dcl)
    ref = _oracle_filip(lat, mask, temperature, dcl)
    _compare_filip(got, ref, lat, mask, f"{B}x{T}x{I}x{D} dcl={dcl} extra={extra} temp={temperature:.3f}")


@pytest.mark.parametrize("dcl,extra", [(False, False), (True, True)])
@pytest.mark.parametrize("B,T,I,D", FILIP_ANY_SHAPES)
def test_filip_any_empty_captions_match_fp64_oracle(cuda_device, B, T, I, D, dcl, extra):
    lat, mask = _filip_inputs(cuda_device, B, T, I, D, extra, seed=29 + B, empty=(1,))
    got = _run_filip_loss(lat, mask, 1.0, dcl)
    ref = _oracle_filip(lat, mask, 1.0, dcl)
    _compare_filip(got, ref, lat, mask, f"empty (1,) {B}x{T}x{I}x{D} dcl={dcl} extra={extra}")


def test_filip_loss_fn_cfg3_single_gpu(cuda_device):
    """cfg3 FILIP on one GPU: 256 pairs of 77 text tokens against 98 kept image tokens, D = 512.
    Text 3 is an empty caption.  The reference is chunked over texts."""
    t0 = _start_peak()
    lat, mask = _filip_inputs(cuda_device, 256, 77, 98, 512, False, seed=77, empty=(3,))
    got = _run_filip_loss(lat, mask, math.log(100.0), False)
    _report_peak("FilipLossFn cfg3", t0)
    ref = oracle_filip_chunked(lat, mask, math.log(100.0), False)
    _compare_filip(got, ref, lat, mask, "cfg3 256x77x98x512")
    _report_peak("FilipLossFn cfg3 with its fp64 reference", t0)


# --------------------------------------------------------------------------- refusals

def test_segmax_any_and_expand_refuse_bad_arguments_without_launching(cuda_device):
    """xclip_filip_segmax_arg16 and xclip_filip_expand16 refuse bad arguments before any launch; either
    output of the segment max may be null, not both."""
    from x_clip_b200 import _lib
    lib = _lib.load()
    dev = cuda_device
    R, C, D, L = 64, 77 * 3, 96, 77
    nseg = C // L
    a = torch.zeros((R, D), device=dev, dtype=BF16)
    b = torch.zeros((C + 8, D), device=dev, dtype=BF16)
    t = torch.ones(2, device=dev, dtype=F32)
    m = torch.empty(R * nseg + 1, device=dev, dtype=F32)
    arg = torch.empty(R * nseg + 1, device=dev, dtype=torch.int16)
    keys = torch.empty(R * nseg + 1, device=dev, dtype=torch.int64)
    cm = torch.ones(C, device=dev, dtype=F32)
    good = dict(a=a.data_ptr(), b=b.data_ptr(), R=R, C=C, D=D, t=t.data_ptr(), L=L, cm=None, ca=None,
                m=m.data_ptr(), arg=arg.data_ptr(), keys=keys.data_ptr())

    def call(**kw):
        v = dict(good, **kw)
        _lib.call("xclip_filip_segmax_arg16", v["a"], v["b"], v["R"], v["C"], v["D"], v["t"], v["L"], v["cm"],
                  v["ca"], v["m"], v["arg"], v["keys"], None)

    bad = [dict(L=0), dict(L=-3), dict(L=76), dict(L=65536, C=65536 * nseg), dict(C=C + 1), dict(a=None),
           dict(b=None), dict(keys=None), dict(m=None, arg=None), dict(a=a.data_ptr() + 2),
           dict(b=b.data_ptr() + 8), dict(keys=keys.data_ptr() + 4), dict(m=m.data_ptr() + 2),
           dict(arg=arg.data_ptr() + 1), dict(cm=cm.data_ptr()), dict(ca=cm.data_ptr()), dict(D=100)]
    torch.cuda.synchronize()
    for kw in bad:
        n0 = lib.xclip_launch_count()
        with pytest.raises(_lib.XClipB200Error, match="filip_segmax_arg16"):
            call(**kw)
        assert lib.xclip_launch_count() == n0, f"a refused call launched a kernel: {kw}"
    n0 = lib.xclip_launch_count()
    call(m=m[1:].data_ptr(), arg=arg[1:].data_ptr(), keys=keys[1:].data_ptr())    # 4 / 2 / 8-byte aligned
    call(m=None)
    call(arg=None)
    torch.cuda.synchronize()
    assert lib.xclip_launch_count() == n0 + 6

    g = torch.empty((R, 240), device=dev, dtype=BF16)
    w = torch.zeros((1, nseg), device=dev, dtype=F32)
    rs = torch.zeros(R, device=dev, dtype=F32)
    eg = dict(arg=arg.data_ptr(), L=L, ldg=240, g=g.data_ptr(), row0=0)

    def expand(**kw):
        v = dict(eg, **kw)
        _lib.call("xclip_filip_expand16", v["arg"], w.data_ptr(), rs.data_ptr(), t.data_ptr(), v["row0"], R, R,
                  v["L"], nseg, v["g"], v["ldg"], None)

    for kw in [dict(L=0), dict(L=65536), dict(ldg=236), dict(ldg=224), dict(g=g.data_ptr() + 2),
               dict(arg=None), dict(arg=arg.data_ptr() + 1), dict(row0=-1)]:
        n0 = lib.xclip_launch_count()
        with pytest.raises(_lib.XClipB200Error, match="filip_expand16"):
            expand(**kw)
        assert lib.xclip_launch_count() == n0, f"a refused call launched a kernel: {kw}"
    n0 = lib.xclip_launch_count()
    expand()
    torch.cuda.synchronize()
    assert lib.xclip_launch_count() == n0 + 1
