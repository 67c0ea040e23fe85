"""The FILIP loss kernels (csrc/filip.cu) one by one, and FilipLossFn as a whole, against plain fp64
torch references.

Operands are built as the model builds them (engine.ProjectL2NormFn): fp32 unit latents z,
hi = bf16(z), lo = bf16(z - hi), row form [hi|lo|hi] and column form [hi|hi|lo].  The references are
computed in fp64 from the fp32 latents, on the GPU (the cfg4-sized ones are out of a CPU's reach), in
row blocks of at most ~1 GB.

cfg4 on 8 GPUs has, per rank, 256 local texts of T = 256 tokens against 2048 images of I = 32 kept
tokens: both segment-max passes are 65536 x 65536 with K = 3 * 512."""
import math
import time

import pytest
import torch

pytestmark = pytest.mark.gpu

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
FMAX = torch.finfo(F32).max
BLOCK_ELEMS = 1 << 27                   # fp64 elements per reference block (1 GB)


def _gen(dev, seed):
    return torch.Generator(device=dev).manual_seed(seed)


def _unit(shape, gen, dev):
    return torch.nn.functional.normalize(torch.randn(shape, generator=gen, device=dev), dim=-1)


def _split(z):
    """(row form [hi|lo|hi], column form [hi|hi|lo]) of fp32 latents z [..., D] -> bf16 [rows, 3D]."""
    z = z.reshape(-1, z.shape[-1])
    hi = z.to(BF16)
    lo = (z - hi.float()).to(BF16)
    return torch.cat([hi, lo, hi], 1).contiguous(), torch.cat([hi, hi, lo], 1).contiguous()


def _start_peak():
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    return time.perf_counter()


def _report_peak(label, t0):
    torch.cuda.synchronize()
    print(f"{label}: {time.perf_counter() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2**30:.1f} GiB")


def _col_mask_tables(mask):
    """col_mul / col_add of a flattened token mask: padded tokens -> 0 * s - FLT_MAX (filip.py)."""
    mask = mask.reshape(-1)
    return mask.float().contiguous(), torch.where(mask, 0.0, -FMAX).to(F32).contiguous()


# --------------------------------------------------------------------------- segment max

# The split-bf16 product drops lo*lo and rounds lo to bf16: both ~2^-18 of |a||b| = 1 per element
# pair, plus fp32 accumulation over K = 3D.  Gate: 2^-16 * temp absolute on a similarity of at most
# temp.  Measured on an H100 over every case below, cfg4 included: seg_max within 0.22 of the gate
# (3.4e-6 * temp; an fp32 restatement of the same split product on the CPU errs as much), the fp64
# similarity at seg_arg within 0.06 of it.
SEGMAX_GATE = 2.0 ** -16


def _run_segmax(za, zb, temp, seg_len, col_mul=None, col_add=None):
    """kernels.filip_segmax16 on the split operands of za [R, D] x zb [C, D], checked against fp64:
    seg_max elementwise, seg_arg by value (the fp64 similarity at the returned column must be within
    the gate of the fp64 maximum: near-ties may legitimately pick the other index).
    Returns (seg_max, seg_arg as int32, max value error / gate, max arg error / gate)."""
    from x_clip_b200 import kernels as K
    a_row, _ = _split(za)
    _, b_col = _split(zb)
    t = torch.tensor([temp], device=za.device, dtype=F32)
    m, arg16 = K.filip_segmax16(a_row, b_col, t, seg_len, col_mul, col_add)
    arg = arg16.to(torch.int32) & 0xFFFF                # the int16 holds an unsigned 16-bit index
    R, C = za.shape[0], zb.shape[0]
    nseg = C // seg_len
    assert m.shape == (R, nseg) and arg.shape == (R, nseg)
    assert bool(((arg >= 0) & (arg < seg_len)).all())
    gate = SEGMAX_GATE * t.item()
    zb64, t64 = zb.double(), t.double()
    step = max(1, BLOCK_ELEMS // C)
    e_val = e_arg = 0.0
    for r0 in range(0, R, step):
        s = t64 * (za[r0:r0 + step].double() @ zb64.t())
        if col_mul is not None:
            s = s * col_mul.double() + col_add.double()
        s = s.view(s.shape[0], nseg, seg_len)
        ref = s.amax(-1)
        at = s.gather(-1, arg[r0:r0 + step].long().unsqueeze(-1)).squeeze(-1)
        e_val = max(e_val, (m[r0:r0 + step].double() - ref).abs().max().item())
        e_arg = max(e_arg, (ref - at).abs().max().item())
        del s, ref, at
    assert e_val <= gate, f"seg_max error {e_val:.3e} > {gate:.3e}"
    assert e_arg <= gate, f"similarity at seg_arg is {e_arg:.3e} below the maximum (gate {gate:.3e})"
    return m, arg, e_val / gate, e_arg / gate


def _nseg_for(seg_len):
    """3 * (256 // seg_len) + 1 segments: two to four 256-column output tiles, most of them ending in
    a partial one.  Lengths that do not divide 256 have segments cut by a tile edge."""
    return 3 * (256 // seg_len) + 1


SEG_LENS = list(range(16, 257, 16))


@pytest.mark.parametrize("D", [256, 512, 72])          # K = 3D = 216: not a multiple of the 64-wide k-block
@pytest.mark.parametrize("seg_len", SEG_LENS)
def test_segmax_matches_fp64(cuda_device, seg_len, D):
    """Every token count from 16 to 256: segments wholly inside a tile where seg_len divides 256, cut by
    a tile edge elsewhere (48, 80, 144...), segments that restart inside a 128-column staging pass.
    R = 1 / 127 / 129 / 1100: ragged last row tile; 129 < C (m-fastest raster), 1100 > C (n-fastest)."""
    gen = _gen(cuda_device, 1000 * seg_len + D)
    C = _nseg_for(seg_len) * seg_len
    zb = _unit((C, D), gen, cuda_device)
    for i, R in enumerate((1, 127, 129, 1100)):
        za = _unit((R, D), gen, cuda_device)
        temp = math.e if i % 2 == 0 else 100.0
        _, _, ev, ea = _run_segmax(za, zb, temp, seg_len)
        print(f"segmax seg_len={seg_len} D={D} R={R} C={C}: error/gate value {ev:.3f} arg {ea:.3f}")


@pytest.mark.parametrize("seg_len", SEG_LENS)
def test_segmax_masked_columns(cuda_device, seg_len):
    """Padded text tokens (col_mul 0 / col_add -FLT_MAX): a masked column is never returned while its
    segment has a valid one; a fully masked segment gives exactly -FLT_MAX at index 0."""
    gen = _gen(cuda_device, 7 + seg_len)
    D, nseg = 256, _nseg_for(seg_len)
    C = nseg * seg_len
    zb = _unit((C, D), gen, cuda_device)
    mask = torch.rand((nseg, seg_len), generator=gen, device=cuda_device) < 0.5
    mask[0] = False                         # an empty caption
    mask[1] = False
    mask[1, -1] = True                      # a single valid token, the segment's last
    mask[2] = True
    col_mul, col_add = _col_mask_tables(mask)
    for R in (129, 1100):
        za = _unit((R, D), gen, cuda_device)
        m, arg, ev, ea = _run_segmax(za, zb, 100.0, seg_len, col_mul, col_add)
        empty = ~mask.any(1)
        assert bool((m[:, empty] == -FMAX).all()) and bool((arg[:, empty] == 0).all())
        picked = mask[torch.arange(nseg, device=cuda_device)[None, :], arg.long()]
        assert bool(picked[:, ~empty].all()), "a padded token won the segment maximum"
        assert bool((arg[:, 1] == seg_len - 1).all())
        print(f"segmax masked seg_len={seg_len} R={R}: error/gate value {ev:.3f} arg {ea:.3f}")


@pytest.mark.parametrize("seg_len", [16, 48, 144, 256])
def test_segmax_ties_go_to_the_lowest_index(cuda_device, seg_len):
    """Two identical tokens p < q in a segment, both the segment's maximum: the kernel keeps the first
    (strict '>' scan), p.  In segment 0 every token is the same: index 0."""
    gen = _gen(cuda_device, 99 + seg_len)
    D, nseg, R = 256, _nseg_for(seg_len), 300
    u = _unit((D,), gen, cuda_device)
    za = torch.nn.functional.normalize(u + 0.02 * torch.randn((R, D), generator=gen, device=cuda_device), dim=-1)
    zb = _unit((nseg, seg_len, D), gen, cuda_device)
    segs = torch.arange(nseg, device=cuda_device)
    p = segs % (seg_len - 1)
    zb[segs, p] = u
    zb[segs, seg_len - 1] = u
    zb[0] = u
    _, arg, _, _ = _run_segmax(za, zb.reshape(-1, D), 100.0, seg_len)
    assert torch.equal(arg.long(), p[None, :].expand(R, nseg))


def test_segmax_cfg4_text_rows(cuda_device):
    """cfg4 pass A: 65536 local text tokens x 65536 image tokens (2048 images x 32), D = 512."""
    t0 = _start_peak()
    gen = _gen(cuda_device, 4)
    za = _unit((65536, 512), gen, cuda_device)
    zb = _unit((65536, 512), gen, cuda_device)
    _, _, ev, ea = _run_segmax(za, zb, 100.0, 32)
    print(f"segmax cfg4 pass A: error/gate value {ev:.3f} arg {ea:.3f}")
    _report_peak("segmax cfg4 pass A", t0)


def test_segmax_cfg4_image_rows_with_text_mask(cuda_device):
    """cfg4 pass B: 65536 image tokens x 65536 local text tokens (256 texts x 256), padded text tokens
    masked; text 0 is an empty caption."""
    t0 = _start_peak()
    gen = _gen(cuda_device, 5)
    za = _unit((65536, 512), gen, cuda_device)
    zb = _unit((65536, 512), gen, cuda_device)
    lens = torch.randint(1, 257, (256,), generator=gen, device=cuda_device)
    lens[0] = 0
    mask = torch.arange(256, device=cuda_device)[None, :] < lens[:, None]
    col_mul, col_add = _col_mask_tables(mask)
    m, arg, ev, ea = _run_segmax(za, zb, 100.0, 256, col_mul, col_add)
    assert bool((m[:, 0] == -FMAX).all()) and bool((arg[:, 0] == 0).all())
    assert bool((arg[:, 1:].long() < lens[None, 1:]).all()), "a padded token won the segment maximum"
    print(f"segmax cfg4 pass B: error/gate value {ev:.3f} arg {ea:.3f}")
    _report_peak("segmax cfg4 pass B", t0)


# --------------------------------------------------------------------------- reduce

@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("samples,length,nseg", [(5, 48, 7), (16, 256, 300), (256, 256, 2048), (2048, 32, 256)])
def test_reduce_matches_fp64_sums(cuda_device, samples, length, nseg, transpose):
    """out[a, b] = sum_k w[a, k] m[a, k, b] (masked mean weights 1 / count, zero on padded tokens).
    Rows of zero weight hold -FLT_MAX or -inf (a multiplied -inf would give NaN): they must be skipped.
    Gate 1e-6 * sum_k |w m| (fp32 sequential sum of up to 256 terms); measured on an H100: at most
    2.4e-7 * sum_k |w m|."""
    from x_clip_b200 import kernels as K
    gen = _gen(cuda_device, samples + length + nseg)
    m = 50.0 * torch.randn((samples, length, nseg), generator=gen, device=cuda_device)
    lens = torch.randint(1, length + 1, (samples,), generator=gen, device=cuda_device)
    lens[0] = 0                                     # all weights zero: out row is exactly 0
    lens[1] = 1
    valid = torch.arange(length, device=cuda_device)[None, :] < lens[:, None]
    w = (valid.float() / lens.clamp(min=1)[:, None].float()).reshape(-1).contiguous()
    pad_val = torch.where(torch.arange(length, device=cuda_device) % 3 == 0, -math.inf, -FMAX)
    m = torch.where(valid[:, :, None], m, pad_val[None, :, None]).reshape(samples * length, nseg).contiguous()
    out = K.filip_reduce(m, w, samples, length, nseg, transpose)
    mv = torch.where(valid.reshape(-1)[:, None], m, 0.0).double()
    terms = (w.double()[:, None] * mv).view(samples, length, nseg)
    ref, scale = terms.sum(1), terms.abs().sum(1)
    if transpose:
        ref, scale = ref.t(), scale.t()
    assert out.shape == ref.shape
    err = ((out.double() - ref).abs() / (scale + 1e-300)).max().item()
    assert torch.isfinite(out).all() and err <= 1e-6, err
    zero_row = out[:, 0] if transpose else out[0]
    assert bool((zero_row == 0).all())
    print(f"reduce {samples}x{length}x{nseg} t={transpose}: error / sum|w m| = {err:.3e}")


# --------------------------------------------------------------------------- InfoNCE / DCL rows

def _nce_case(dev, R, C, seed):
    gen = _gen(dev, seed)
    scale = torch.tensor([1.0, 10.0, 100.0], device=dev)[torch.arange(R, device=dev) % 3]
    return ((2 * torch.rand((R, C), generator=gen, device=dev) - 1) * scale[:, None]).contiguous()


@pytest.mark.parametrize("dcl", [False, True])
@pytest.mark.parametrize("where", ["first", "middle", "last"])
@pytest.mark.parametrize("R,C", [(5, 31), (7, 32), (13, 33), (29, 256), (251, 2048), (256, 2048)])
def test_nce_rows_match_fp64(cuda_device, R, C, where, dcl):
    """filip_nce_fwd: lse = logsumexp of the row (the positive x + diag_off removed under DCL), loss_accum
    += loss_scale * sum_x (lse_x - s[x, pos]) onto a non-zero start; filip_nce_bwd: g = gscale *
    (softmax - onehot), the DCL positive exactly -gscale.  Logits up to 100 in magnitude (the max shift
    matters).  diag_off 0, middle, C - R (cfg4 rank 7: R 256, C 2048, offset 1792).  Then again with a
    row_valid mask: invalid rows add no loss and get g = 0.
    Gates: |lse - ref| <= 1e-6 |ref| + 4e-6; |g - ref| <= gscale (2e-5 softmax + 2e-6); loss within the
    summed lse gates plus one fp32 rounding per atomic add.  Measured on an H100: lse at most 0.05 of
    its gate, g at most 0.17."""
    from x_clip_b200 import kernels as K
    dev = cuda_device
    off = {"first": 0, "middle": (C - R) // 2, "last": C - R}[where]
    s = _nce_case(dev, R, C, R * 7919 + C)
    rows = torch.arange(R, device=dev)
    pos = rows + off
    s64 = s.double()
    lse_in = s64.clone()
    if dcl:
        lse_in[rows, pos] = -math.inf
    ref_lse = torch.logsumexp(lse_in, dim=1)
    p = torch.exp(lse_in - ref_lse[:, None])
    onehot = torch.zeros_like(s64)
    onehot[rows, pos] = 1.0
    gs = 0.37
    ref_g = gs * (p - onehot)
    lse_gate = 1e-6 * ref_lse.abs() + 4e-6

    for row_valid in (None, torch.arange(R, device=dev) % 4 != 1):
        valid = torch.ones(R, dtype=torch.bool, device=dev) if row_valid is None else row_valid
        loss = torch.full((1,), 0.75, device=dev, dtype=F32)
        lse = K.filip_nce_fwd(s, off, dcl, loss, 0.3, row_valid=row_valid)
        e_lse = ((lse.double() - ref_lse).abs() / lse_gate)[valid].max().item()
        assert e_lse <= 1.0, e_lse
        assert bool((lse[~valid] == 0).all())
        terms = 0.3 * (ref_lse - s64[rows, pos])[valid]
        ref_loss = 0.75 + terms.sum().item()
        # the lse gates, plus one fp32 rounding of the running sum per atomic add
        loss_gate = 0.3 * lse_gate[valid].sum().item() + R * 2.0 ** -24 * (0.75 + terms.abs().sum().item())
        assert abs(loss.item() - ref_loss) <= loss_gate, (loss.item(), ref_loss, loss_gate)

        gscale = torch.tensor([gs], device=dev, dtype=F32)
        g = K.filip_nce_bwd(s, lse, off, dcl, gscale, row_valid=row_valid)
        g_gate = gs * (2e-5 * p + 2e-6)
        e_g = ((g.double() - ref_g).abs() / g_gate)[valid].max().item()
        assert e_g <= 1.0, e_g
        assert bool((g[~valid] == 0).all())
        if dcl:
            assert bool((g[rows, pos][valid] == -gscale).all())
        print(f"nce R={R} C={C} off={off} dcl={dcl} masked={row_valid is not None}: "
              f"error/gate lse {e_lse:.3f} g {e_g:.3f}")


# --------------------------------------------------------------------------- expand

def _expand_case(dev, samples, rows_per_sample, nseg, seg_len, seed):
    gen = _gen(dev, seed)
    R = samples * rows_per_sample
    seg_arg = torch.randint(0, seg_len, (R, nseg), generator=gen, device=dev, dtype=torch.int32)
    wmat = torch.randn((samples, nseg), generator=gen, device=dev) * 1e-3
    wmat[:, 1] = 0.0                                       # e.g. the row of an empty caption
    rowscale = torch.rand((R,), generator=gen, device=dev) + 0.5
    rowscale[torch.arange(R, device=dev) % rows_per_sample >= rows_per_sample - 3] = 0.0   # padded tokens
    w = wmat[torch.arange(R, device=dev) // rows_per_sample] * rowscale[:, None]
    return seg_arg, wmat.contiguous(), rowscale.contiguous(), w


def _check_expand(dev, samples, rows_per_sample, nseg, seg_len, chunks, seed):
    """filip_expand16 over row chunks [row0, row0 + rows), each given the argmax of its rows only,
    against G built densely in torch: bf16(alpha * wmat[r // rows_per_sample, seg] * rowscale[r]) at
    seg * seg_len + seg_arg[r, seg].  G must be bit-identical (the same two fp32 products and one
    rounding)."""
    from x_clip_b200 import kernels as K
    seg_arg, wmat, rowscale, w = _expand_case(dev, samples, rows_per_sample, nseg, seg_len, seed)
    alpha = torch.tensor([42.5], device=dev, dtype=F32)
    for row0, rows in chunks:
        sl = slice(row0, row0 + rows)
        g = K.filip_expand16(seg_arg[sl].to(torch.int16), wmat, rowscale, alpha, row0, rows_per_sample,
                             seg_len, nseg)
        want = torch.zeros((rows, nseg * seg_len), device=dev, dtype=BF16)
        cols = torch.arange(nseg, device=dev)[None, :] * seg_len + seg_arg[sl].long()
        want.scatter_(1, cols, (w[sl] * alpha).to(BF16))
        assert torch.equal(g, want), (row0, rows)
        assert not bool(g[rowscale[sl] == 0].any())        # padded tokens: all-zero rows


@pytest.mark.parametrize("seg_len", [16, 48, 144, 256])
def test_expand_matches_dense_construction(cuda_device, seg_len):
    samples, rows_per_sample, nseg = 6, 40, 5
    R = samples * rows_per_sample
    _check_expand(cuda_device, samples, rows_per_sample, nseg, seg_len,
                  [(0, R), (37, 150), (R - 1, 1)], seed=seg_len)


def test_expand_cfg4_chunk(cuda_device):
    """The last of cfg4's pass-A backward chunks: rows [57344, 65536) of 256 texts x 256 tokens, against
    2048 images of 32 tokens."""
    t0 = _start_peak()
    _check_expand(cuda_device, 256, 256, 2048, 32, [(57344, 8192)], seed=4)
    _report_peak("expand cfg4 chunk", t0)


# --------------------------------------------------------------------------- FilipLossFn vs the oracle

def _filip_inputs(dev, B, T, I, D, extra, seed, empty=()):
    """fp32 unit latents [zt, zi(, zt_x, zi_x)] and a text mask of mixed lengths: text 0 has exactly one
    token, the last text all T, the texts in `empty` none."""
    gen = _gen(dev, seed)
    lat = [_unit((B, T, D), gen, dev), _unit((B, I, D), gen, dev)]
    if extra:
        lat += [_unit((B, T, D), gen, dev), _unit((B, I, D), gen, dev)]
    lens = torch.randint(1, T + 1, (B,), generator=gen, device=dev)
    lens[0], lens[-1] = 1, T
    for e in empty:
        lens[e] = 0
    return lat, torch.arange(T, device=dev)[None, :] < lens[:, None]


def _run_filip_loss(lat, mask, temperature, dcl):
    """FilipLossFn on the latents' split-bf16 operands -> (loss, d temperature, latent gradients)."""
    from x_clip_b200.filip import FilipLossFn
    extra = len(lat) == 4
    z = [t.clone().requires_grad_(True) for t in lat]
    ops = tuple(_split(t) for t in lat)
    temp = torch.tensor(temperature, device=lat[0].device, dtype=F32, requires_grad=True)
    loss = FilipLossFn.apply(z[0], z[1], z[2] if extra else None, z[3] if extra else None, temp, ops,
                             mask.contiguous(), dcl, False)
    loss.backward()
    return loss.item(), temp.grad.item(), [t.grad for t in z]


def _oracle_cfg(dcl, extra):
    from oracle import clip_oracle as O
    return O.ClipConfig(use_all_token_embeds=True, decoupled_contrastive_learning=dcl, extra_latent_projection=extra)


def _oracle_filip(lat, mask, temperature, dcl):
    """oracle.clip_oracle.contrastive_loss in fp64 autograd -> (loss, d temperature, latent gradients)."""
    from oracle import clip_oracle as O
    extra = len(lat) == 4
    z = [t.detach().double().requires_grad_(True) for t in lat]
    t64 = torch.tensor(temperature, dtype=F32).double().to(lat[0].device).requires_grad_(True)
    zt_x, zi_x = (z[2], z[3]) if extra else (z[0], z[1])
    loss = O.contrastive_loss(z[0], z[1], zt_x, zi_x, t64, _oracle_cfg(dcl, extra), mask)
    loss.backward()
    return loss.item(), t64.grad.item(), [t.grad for t in z]


def oracle_filip_chunked(lat, mask, temperature, dcl, block=8):
    """_oracle_filip for batches whose 6-D similarity does not fit: the lines of
    oracle.clip_oracle.contrastive_loss restated per block of texts.  (1) t2i / i2t rows in fp64
    without grad; (2) autograd of _nce_from_logits on those [B, B] leaves; (3) each block recomputed
    with grad and back-propagated with its rows of the leaves' gradients, accumulating into the
    latents and the temperature."""
    from oracle import clip_oracle as O
    extra = len(lat) == 4
    z = [t.detach().double().requires_grad_(True) for t in lat]
    t64 = torch.tensor(temperature, dtype=F32).double().to(lat[0].device).requires_grad_(True)
    zt, zi = z[0], z[1]
    zt_x, zi_x = (z[2], z[3]) if extra else (zt, zi)
    B = zt.shape[0]

    def rows(x0, x1):                                   # oracle.contrastive_loss, FILIP branch
        temp = t64.exp()
        sim = temp * torch.einsum("xtd,yid->xyti", zt[x0:x1], zi)
        sim_x = temp * torch.einsum("xtd,yid->xyti", zt_x[x0:x1], zi_x) if extra else sim
        tm = mask[x0:x1]
        m = tm[:, None, :]
        t2i = sim.amax(dim=-1).masked_fill(~m, 0.0).sum(-1) / m.sum(-1).clamp_min(1e-6)
        fill = -torch.finfo(sim_x.dtype).max
        i2t = sim_x.masked_fill(~tm[:, None, :, None], fill).amax(dim=-2).mean(dim=-1)
        return t2i, i2t

    blocks = [(x0, min(B, x0 + block)) for x0 in range(0, B, block)]
    with torch.no_grad():
        parts = [rows(*b) for b in blocks]
    t2i = torch.cat([p[0] for p in parts]).requires_grad_(True)
    i2t = torch.cat([p[1] for p in parts]).requires_grad_(True)
    del parts
    loss = O._nce_from_logits(t2i, i2t, dcl)
    loss.backward()
    for x0, x1 in blocks:
        torch.autograd.backward(rows(x0, x1), (t2i.grad[x0:x1], i2t.grad[x0:x1]))
    return loss.item(), t64.grad.item(), [t.grad for t in z]


def _compare_filip(got, ref, lat, mask, label):
    """Gates of test_dtemperature_of_the_loss_kernels_in_isolation: loss rel 1e-5; d temperature rel
    1e-3 + 1e-5 absolute (fp32 sums over the [B, B] matrices); latent gradients relative
    error norm 1e-2 (G and the hi operands are bf16).  Gradients of padded text tokens exactly 0.
    Measured on an H100 over all cases of this file: loss rel at most 6.0e-6 (B = 5 at temperature
    log 100, where the loss is small), d temperature within 0.04 of its gate (rel 6.5e-5), gradients
    rel at most 4.0e-3 (cfg4)."""
    loss, dt, grads = got
    r_loss, r_dt, r_grads = ref
    assert abs(loss - r_loss) <= 1e-5 * abs(r_loss), (label, loss, r_loss)
    assert math.isfinite(dt) and abs(dt - r_dt) <= 1e-3 * abs(r_dt) + 1e-5, (label, dt, r_dt)
    worst = 0.0
    for j, (g, r) in enumerate(zip(grads, r_grads)):
        assert g is not None and torch.isfinite(g).all(), (label, j)
        rel = (g.double() - r).norm().item() / (r.norm().item() + 1e-30)
        worst = max(worst, rel)
        assert rel <= 1e-2, (label, j, rel)
        if j % 2 == 0:                                  # text latents: padded tokens get nothing
            assert not bool(g[~mask].any()), (label, j, "gradient on padded text tokens")
    print(f"filip {label}: loss rel {abs(loss - r_loss) / abs(r_loss):.2e} dtemp {dt:.6e} vs {r_dt:.6e} "
          f"grad rel {worst:.2e}")


FILIP_SHAPES = [(5, 48, 144, 256), (8, 80, 16, 128), (16, 256, 64, 512)]


@pytest.mark.parametrize("temperature", [1.0, math.log(100.0)])
@pytest.mark.parametrize("extra", [False, True])
@pytest.mark.parametrize("dcl", [False, True])
@pytest.mark.parametrize("B,T,I,D", FILIP_SHAPES)
def test_filip_loss_fn_matches_fp64_oracle(cuda_device, B, T, I, D, dcl, extra, temperature):
    """FilipLossFn (both segment-max passes, reduce, InfoNCE / DCL, expand + the gradient GEMMs) on the
    split operands of fp32 latents against the oracle in fp64, no encoder in between."""
    lat, mask = _filip_inputs(cuda_device, B, T, I, D, extra, seed=B * T + I + D)
    got = _run_filip_loss(lat, mask, temperature, dcl)
    ref = _oracle_filip(lat, mask, temperature, dcl)
    _compare_filip(got, ref, lat, mask, f"{B}x{T}x{I}x{D} dcl={dcl} extra={extra} temp={temperature:.3f}")


@pytest.mark.parametrize("extra", [False, True])
@pytest.mark.parametrize("dcl", [False, True])
@pytest.mark.parametrize("B,T,I,D,empty", [(5, 48, 144, 256, (1,)), (8, 80, 16, 128, (2, 5))])
def test_filip_empty_captions_match_fp64_oracle(cuda_device, B, T, I, D, empty, dcl, extra):
    """Captions made only of padding: the reference's image-to-text row is -inf (a mean of -max fills)
    and adds neither loss nor gradient; the text-to-image row is 0.  Loss, a finite d temperature and the
    latent gradients must match, and the empty captions' tokens get exactly zero gradient."""
    lat, mask = _filip_inputs(cuda_device, B, T, I, D, extra, seed=17 + B, empty=empty)
    got = _run_filip_loss(lat, mask, 1.0, dcl)
    ref = _oracle_filip(lat, mask, 1.0, dcl)
    _compare_filip(got, ref, lat, mask, f"empty {empty} {B}x{T}x{I}x{D} dcl={dcl} extra={extra}")


def test_filip_loss_fn_cfg4_single_gpu(cuda_device):
    """cfg4 on one GPU: B = 256, T = 256, I = 64, D = 512 - both backward passes run in 2 row chunks
    (filip_expand16 with row0 > 0).  Text 3 is an empty caption.  The reference is chunked over texts."""
    t0 = _start_peak()
    lat, mask = _filip_inputs(cuda_device, 256, 256, 64, 512, False, seed=256, empty=(3,))
    got = _run_filip_loss(lat, mask, math.log(100.0), False)
    _report_peak("FilipLossFn cfg4", t0)
    ref = oracle_filip_chunked(lat, mask, math.log(100.0), False)
    _compare_filip(got, ref, lat, mask, "cfg4 256x256x64x512")
    _report_peak("FilipLossFn cfg4 with its fp64 reference", t0)
