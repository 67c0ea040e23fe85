"""FILIP fine-grained loss (reference x_clip/x_clip.py:799-811 + :821-847) on the CUDA kernels.

Schedule (see csrc/filip.cu): two segment-max GEMM passes (text tokens x image tokens and the
transposed orientation, fp32-accurate through the split-bf16 operands), each in row chunks of whole
samples reduced straight into the [B,B] similarity matrices, row-wise InfoNCE/DCL; backward
re-expands each chunk's argmax (saved in 16 bits, or recomputed by its segment-max GEMM) into a
one-hot weighted bf16 operand window by window and runs two plain wgmma GEMMs per window.
The 6-D similarity tensor of the reference is never materialised.  Under data parallelism the
image-token operands are all-gathered and each rank owns the rows of its local texts (the
reference itself cannot all-gather FILIP latents, SURVEY.md 8c - what W ranks must reproduce is
the single-process loss on the concatenated batch)."""
from __future__ import annotations

import torch

from . import kernels as K
from . import distributed as D_
from .engine import _avail_bytes

F32 = torch.float32

# Bytes of transient working set one row chunk may use, whatever b, B and the token counts are.  Half
# goes to the forward's 64-bit keys + f32 maxima (12 B per (row, sample)), the other half to one
# backward window of the bf16 one-hot operand G.  A chunk holds at least one whole sample, so the bound
# holds while one sample's keys fit: tokens x samples x 12 B <= 1 GiB (155 k samples at 576 tokens).
FILIP_CHUNK_BYTES = 2 << 30
# Bytes of compact argmax (2 B per (row, sample)) the loss may keep from forward to backward.  None:
# decide from the free HBM when the loss is called; 0 recomputes every chunk in backward, a value at
# least the total saves every chunk.  Tests set it to force a plan.
FILIP_SAVE_BYTES = None
# HBM the save plan leaves free beside the chunk budget: the gradient outputs, the NCE matrices and
# the encoders' backward that follows
FILIP_SAVE_MARGIN_BYTES = 10 << 30

KEY_BYTES, MAX_BYTES, ARG_BYTES = 8, 4, 2


def chunk_bounds(rows_per_sample: int, samples: int, nseg: int, budget: int = None):
    """Row chunks [r0, r1) of one pass, each a whole number of samples, whose keys and maxima
    (12 B per (row, segment)) fit in half the budget."""
    budget = FILIP_CHUNK_BYTES if budget is None else budget
    per_sample = rows_per_sample * nseg * (KEY_BYTES + MAX_BYTES)
    step = max(1, (budget // 2) // per_sample)
    return [(s * rows_per_sample, min(s + step, samples) * rows_per_sample) for s in range(0, samples, step)]


def window_rows(R: int, C: int, budget: int = None) -> int:
    """Rows of one backward window of G [rows, roundup8(C)] bf16: budget / 4 elements, a multiple of 128
    rows where that many fit."""
    budget = FILIP_CHUNK_BYTES if budget is None else budget
    n = min(R, (budget // 4) // max(C, 1))
    return n // 128 * 128 if n >= 128 else max(n, 1)


def chunk_transient_bytes(rows: int, R: int, nseg: int, seg_len: int, budget: int = None) -> int:
    """Peak transient bytes of one chunk of `rows` rows (of R in its pass): forward keys + maxima;
    backward recompute keys + argmax; then argmax + one G window (the saved argmax is not transient)."""
    e = rows * nseg
    C = nseg * seg_len
    g = min(rows, window_rows(R, C, budget)) * ((C + 7) // 8 * 8) * 2
    return max(e * (KEY_BYTES + MAX_BYTES), e * (KEY_BYTES + ARG_BYTES), e * ARG_BYTES + g)


def saved_bytes(b: int, B: int, T: int, I: int, m: int = 1, n: int = 1) -> int:
    """Compact argmax of both passes when every chunk is saved: [m b T, n B] + [n B I, m b] at 2 B
    (m text views, n image views; one view each is the single-view loss)."""
    return ARG_BYTES * (m * b * T * n * B + n * B * I * m * b)


def step_reserve_bytes(b: int, B: int, T: int, I: int, D: int, extra: bool, m: int = 1, n: int = 1) -> int:
    """HBM the micro-batched step leaves to the loss when it plans which encoder chunks to keep: the
    saved argmax of both passes, the chunk budget, and per token row and latent pair 24 D bytes (the
    fp32 leaf and its gradient, the two split-bf16 operands)."""
    pairs = 2 if extra else 1
    return saved_bytes(b, B, T, I, m, n) + FILIP_CHUNK_BYTES + 24 * D * (m * b * T + n * B * I) * pairs


class _Pass:
    """One segment-max pass: rows (tokens of one modality, rows_per_sample per sample) against the
    segments of the columns; chunks [r0, r1) and the prefix [0, saved_rows) whose argmax is kept."""

    def __init__(self, rows_op, cols_op, seg_len, col_mul, col_add, rows_per_sample):
        K.check_arg16_seg_len(seg_len)
        self.rows_op, self.cols_op = rows_op, cols_op
        self.seg_len, self.col_mul, self.col_add = seg_len, col_mul, col_add
        self.rows_per_sample = rows_per_sample
        self.R = rows_op.shape[0]
        self.nseg = cols_op.shape[0] // seg_len
        self.chunks = chunk_bounds(rows_per_sample, self.R // rows_per_sample, self.nseg)
        self.saved_rows, self.saved = 0, None

    def plan(self, budget_bytes: int) -> int:
        """Keep the argmax of the longest chunk prefix within budget_bytes; returns the bytes kept."""
        per_row = ARG_BYTES * self.nseg
        for r0, r1 in self.chunks:
            if r1 * per_row > budget_bytes:
                break
            self.saved_rows = r1
        if self.saved_rows:
            self.saved = torch.empty((self.saved_rows, self.nseg), device=self.rows_op.device, dtype=torch.int16)
        return self.saved_rows * per_row

    def forward(self, temp_exp, weights, out, transpose):
        """segment-max -> filip_reduce per chunk, into rows (or columns) [r0, r1) / rows_per_sample of out."""
        for r0, r1 in self.chunks:
            arg = self.saved[r0:r1] if r1 <= self.saved_rows else False
            m, _ = K.filip_segmax16(self.rows_op[r0:r1], self.cols_op, temp_exp, self.seg_len, self.col_mul,
                                    self.col_add, want_max=True, seg_arg=arg)
            s0, s1 = r0 // self.rows_per_sample, r1 // self.rows_per_sample
            part = K.filip_reduce(m, weights[r0:r1], s1 - s0, self.rows_per_sample, self.nseg, transpose)
            del m
            if transpose:
                out[:, s0:s1] = part
            else:
                out[s0:s1] = part

    def backward(self, temp_exp, wmat, rowscale, row_hi, col_hi, D):
        """-> (d rows [R, D], d cols [C, D]) fp32.  Saved rows run in windows of window_rows from row 0
        (the accumulation order of d cols does not depend on the plan's chunks when everything is
        saved); each recomputed chunk re-runs its segment-max GEMM for the argmax, then its windows."""
        dev = self.rows_op.device
        C = self.nseg * self.seg_len
        d_rows = torch.empty((self.R, D), device=dev, dtype=F32)
        d_cols = torch.zeros((C, D), device=dev, dtype=F32)
        gr = window_rows(self.R, C)

        def windows(lo, hi, arg):
            for r0 in range(lo, hi, gr):
                rows = min(gr, hi - r0)
                g = K.filip_expand16(arg[r0 - lo:r0 - lo + rows], wmat, rowscale, temp_exp, r0,
                                     self.rows_per_sample, self.seg_len, self.nseg)
                K.gemm(g, col_hi, b_major=1, out=d_rows[r0:r0 + rows])
                K.gemm(g, row_hi[r0:r0 + rows], a_major=1, b_major=1, out=d_cols, accumulate=True)
                del g

        if self.saved_rows:
            windows(0, self.saved_rows, self.saved)
        self.saved = None
        for r0, r1 in self.chunks:
            if r1 <= self.saved_rows:
                continue
            _, arg = K.filip_segmax16(self.rows_op[r0:r1], self.cols_op, temp_exp, self.seg_len, self.col_mul,
                                      self.col_add, want_max=False)
            windows(r0, r1, arg)
            del arg
        return d_rows, d_cols


class FilipLossFn(torch.autograd.Function):
    """Rows of both [texts, images] similarity matrices are the LOCAL texts; columns are the images
    of ALL ranks (image-token operands are all-gathered once).  Backward returns
    d loss / d(local latents): text gradients are local, image-token gradients are summed over
    ranks with one reduce-scatter - the same per-rank contract as the CLS path.

    Both passes run in row chunks of whole samples (pass A: captions of T rows; pass B: images of I
    rows), bounded by FILIP_CHUNK_BYTES.  The argmax of a chunk prefix is saved in 16 bits (the plan:
    FILIP_SAVE_BYTES, or the free HBM); the other chunks keep nothing and re-run their segment-max GEMM
    in backward.  The loss does not depend on the plan.  `stats`, a dict, receives the plan's rows.

    Augmented views (x_clip.py:625-650, :821-868): views = (m, n) with zt / text_mask holding m text
    views and zi n image views of the same b pairs, stacked along the batch; weights = (cl_w, mv_w).
    Every (text view i, image view j) pair is a FILIP loss of its own, text view i masked by its own
    rows of text_mask, and the result is cl_w L[0, 0] + mv_w mean(the other m n - 1 pairs).  The two
    passes simply grow: pass A's rows are the m views' text tokens [m b T] against the n views' image
    tokens of every rank [n B I], pass B the reverse; t2i and i2t become [m b, n B] and the block
    kernels (xclip_filip_nce_blocks_fwd / _bwd) run the InfoNCE / DCL of all m n blocks in one launch
    per direction.  Image columns are rank-major - rank r's n views in turn, the order the one
    all-gather of the stacked local views gives and the reduce-scatter takes back - so image view j's
    sample r b + y is column r n b + j b + y (positive_column).  views = (1, 1) is the single-view
    loss, on the single-view kernels."""

    @staticmethod
    def forward(ctx, zt, zi, zt_x, zi_x, temperature, ops, text_mask, dcl: bool, use_gather: bool,
                stats=None, views=(1, 1), weights=None):
        m, n = views
        extra = len(ops) == 4
        rank, world = D_.world() if use_gather else (0, 1)
        T, D = zt.shape[1], zt.shape[2]
        b = zt.shape[0] // m
        I = zi.shape[1]
        B, off = world * b, rank * b
        dev = zt.device
        temp_exp = temperature.detach().float().exp().reshape(1)
        mask = text_mask.reshape(m * b * T)
        cnt = text_mask.sum(dim=1).clamp(min=1e-6).float()                       # x_clip.py:40-44
        w_t = (text_mask.float() / cnt[:, None]).reshape(m * b * T).contiguous()
        w_i = torch.full((n * B * I,), 1.0 / I, device=dev, dtype=F32)
        col_mul = mask.float().contiguous()
        col_add = torch.where(mask, torch.zeros((), device=dev),
                              torch.full((), -torch.finfo(F32).max, device=dev)).contiguous()

        img = list(ops[1]) + (list(ops[3]) if extra else [])       # (row, col) forms of image tokens
        img_all = D_.gather_rows(img) if world > 1 else img        # ONE all-gather: [n*B*I, 3D] each
        irow_all, icol_all = img_all[0], img_all[1]
        trow, tcol = ops[0]
        if extra:
            rows_i, cols_t = img_all[2], ops[2][1]
        else:
            rows_i, cols_t = irow_all, tcol
        pa = _Pass(trow, icol_all, I, None, None, T)                              # [m*b*T, n*B]
        pb = _Pass(rows_i, cols_t, T, col_mul, col_add, I)                        # [n*B*I, m*b]
        budget = FILIP_SAVE_BYTES
        if budget is None:
            budget = max(0, _avail_bytes(dev) - FILIP_SAVE_MARGIN_BYTES - FILIP_CHUNK_BYTES)
        budget -= pa.plan(budget)
        pb.plan(budget)
        t2i = torch.empty((m * b, n * B), device=dev, dtype=F32)
        i2t = torch.empty((m * b, n * B), device=dev, dtype=F32)                  # (text, image)
        pa.forward(temp_exp, w_t, t2i, transpose=False)
        pb.forward(temp_exp, w_i, i2t, transpose=True)

        # A caption without any valid token (an empty string) has every i2t similarity at the
        # -FLT_MAX fill: the reference's mean overflows to -inf and that row adds neither loss nor
        # gradient.  Its t2i row is 0 (the masked mean of nothing) and is an ordinary row.
        has_tokens = text_mask.any(dim=1).contiguous()

        loss = torch.zeros(1, device=dev, dtype=F32)
        block_w = None
        if m * n == 1:
            lse_t = K.filip_nce_fwd(t2i, off, dcl, loss, 1.0 / (2 * B))
            lse_i = K.filip_nce_fwd(i2t, off, dcl, loss, 1.0 / (2 * B), row_valid=has_tokens)
        else:
            block_w = torch.tensor(view_block_weights(m, n, weights[0], weights[1], B), device=dev, dtype=F32)
            lse_t = K.filip_nce_blocks_fwd(t2i, m, n, b, off, dcl, block_w, loss)
            lse_i = K.filip_nce_blocks_fwd(i2t, m, n, b, off, dcl, block_w, loss, row_valid=has_tokens)
        if world > 1:
            D_.all_reduce_sum_(loss)

        if stats is not None:
            stats.update(rows_saved=pa.saved_rows + pb.saved_rows,
                         rows_recomputed=(pa.R - pa.saved_rows) + (pb.R - pb.saved_rows),
                         saved_bytes=ARG_BYTES * (pa.saved_rows * pa.nseg + pb.saved_rows * pb.nseg),
                         chunks=len(pa.chunks) + len(pb.chunks))
        ctx.cfg = (dcl, extra, rank, world, m, n, b, B, T, I, D, off)
        ctx.stuff = (temp_exp, ops, img_all, w_t, w_i, pa, pb, t2i, i2t, lse_t, lse_i, has_tokens, block_w)
        return loss.reshape(())

    @staticmethod
    def backward(ctx, gloss):
        dcl, extra, rank, world, m, n, b, B, T, I, D, off = ctx.cfg
        temp_exp, ops, img_all, w_t, w_i, pa, pb, t2i, i2t, lse_t, lse_i, has_tokens, block_w = ctx.stuff
        if block_w is None:
            gscale = (gloss.detach().float() / (2.0 * B)).reshape(1)
            g_t = K.filip_nce_bwd(t2i, lse_t, off, dcl, gscale)                      # [x local, y all]
            g_i = K.filip_nce_bwd(i2t, lse_i, off, dcl, gscale, row_valid=has_tokens)  # [x local, y all]
        else:                                            # the block weights carry 1 / (2 B)
            gscale = gloss.detach().float().reshape(1)
            g_t = K.filip_nce_blocks_bwd(t2i, lse_t, m, n, b, off, dcl, block_w, gscale)
            g_i = K.filip_nce_blocks_bwd(i2t, lse_i, m, n, b, off, dcl, block_w, gscale, row_valid=has_tokens)
        # t2i and i2t are exp(temperature) times a function of the latents alone, so
        # d loss / d temperature = sum g_t * t2i + sum g_i * i2t.  An empty caption's i2t row (the
        # -FLT_MAX fill, possibly -inf) has g_i = 0 and is left out rather than multiplied.
        dtemp = ((g_t * t2i).sum() + (g_i * torch.where(has_tokens[:, None], i2t, 0.0)).sum()).reshape(1)
        g_i = g_i.t().contiguous()                                               # -> [y all, x local]

        hi = lambda t: t[:, :D]
        # pass A: rows = local text tokens, columns = image tokens of all ranks
        dzt, dzi_all = pa.backward(temp_exp, g_t, w_t, hi(ops[0][0]), hi(img_all[1]), D)
        # pass B: rows = image tokens of all ranks, columns = local text tokens
        if extra:
            dzi_x_all, dzt_x = pb.backward(temp_exp, g_i, w_i, hi(img_all[2]), hi(ops[2][1]), D)
            dzi_x = D_.reduce_scatter_rows(dzi_x_all)
        else:
            dzi_b, dzt_b = pb.backward(temp_exp, g_i, w_i, hi(img_all[0]), hi(ops[0][1]), D)
            dzt += dzt_b
            dzi_all += dzi_b
            dzt_x = dzi_x = None
        dzi = D_.reduce_scatter_rows(dzi_all)
        if world > 1:
            D_.all_reduce_sum_(dtemp)
        ctx.stuff = None
        shp_t, shp_i = (m * b, T, D), (n * b, I, D)
        grads = (dzt.view(shp_t), dzi.view(shp_i),
                 None if dzt_x is None else dzt_x.view(shp_t),
                 None if dzi_x is None else dzi_x.view(shp_i),
                 dtemp.reshape(()))
        return grads + (None,) * (len(ctx.needs_input_grad) - len(grads))


def view_block_weights(m: int, n: int, cl_w: float, mv_w: float, B: int) -> list:
    """Loss weight of each (text view i, image view j) block, i * n + j, scale 1 / (2 B) included:
    cl_w on the (0, 0) pair, mv_w / (m n - 1) on every other (x_clip.py:851-868)."""
    other = mv_w / (m * n - 1) if m * n > 1 else 0.0
    return [(cl_w if k == 0 else other) / (2 * B) for k in range(m * n)]


def positive_column(i: int, j: int, x: int, rank: int, b: int, n: int, col_run: int) -> int:
    """Column of the positive of text view i's local row x in image view j's block, in a view-block
    matrix with runs of col_run samples (col_run = b: rank-major, FilipLossFn's order; col_run = W b:
    view-major); the arithmetic of xclip_filip_nce_blocks_fwd.  i does not move it."""
    k = rank * b + x
    return (k // col_run) * n * col_run + j * col_run + k % col_run

