"""FILIP fine-grained loss (reference x_clip/x_clip.py:799-811 + :821-847) on the CUDA kernels.

Schedule (see csrc/filip.cu): two segment-max GEMM passes (text tokens x image tokens and the
transposed orientation, fp32-accurate through the split-bf16 operands), two tiny reductions to the
[B,B] similarity matrices, row-wise InfoNCE/DCL; backward re-expands the saved argmax into a
one-hot weighted bf16 operand chunk by chunk and runs two plain wgmma GEMMs per chunk.
The 6-D similarity tensor of the reference is never materialised.  Under data parallelism the
image-token operands are all-gathered and each rank owns the rows of its local texts (the
reference itself cannot all-gather FILIP latents, SURVEY.md 8c - what W ranks must reproduce is
the single-process loss on the concatenated batch)."""
from __future__ import annotations

import torch

from . import kernels as K
from . import distributed as D_

F32 = torch.float32


class FilipLossFn(torch.autograd.Function):
    """Rows of both [texts, images] similarity matrices are the LOCAL texts; columns are the images
    of ALL ranks (image-token operands are all-gathered once).  Backward returns
    d loss / d(local latents): text gradients are local, image-token gradients are summed over
    ranks with one reduce-scatter - the same per-rank contract as the CLS path."""

    @staticmethod
    def forward(ctx, zt, zi, zt_x, zi_x, temperature, ops, text_mask, dcl: bool, use_gather: bool):
        extra = len(ops) == 4
        rank, world = D_.world() if use_gather else (0, 1)
        b, T, D = zt.shape
        I = zi.shape[1]
        B, off = world * b, rank * b
        dev = zt.device
        temp_exp = temperature.detach().float().exp().reshape(1)
        mask = text_mask.reshape(b * T)
        cnt = text_mask.sum(dim=1).clamp(min=1e-6).float()                       # x_clip.py:40-44
        w_t = (text_mask.float() / cnt[:, None]).reshape(b * T).contiguous()
        w_i = torch.full((B * I,), 1.0 / I, device=dev, dtype=F32)
        col_mul = mask.float().contiguous()
        col_add = torch.where(mask, torch.zeros((), device=dev),
                              torch.full((), -torch.finfo(F32).max, device=dev)).contiguous()

        img = list(ops[1]) + (list(ops[3]) if extra else [])       # (row, col) forms of image tokens
        img_all = D_.gather_rows(img) if world > 1 else img        # ONE all-gather: [B*I, 3D] each
        irow_all, icol_all = img_all[0], img_all[1]
        trow, tcol = ops[0]
        m1, a1 = K.filip_segmax(trow, icol_all, temp_exp, I, None, None)         # [b*T, B]
        t2i = K.filip_reduce(m1, w_t, b, T, B, transpose=False)                  # [b, B]
        if extra:
            rows_i, cols_t = img_all[2], ops[2][1]
        else:
            rows_i, cols_t = irow_all, tcol
        m2, a2 = K.filip_segmax(rows_i, cols_t, temp_exp, T, col_mul, col_add)   # [B*I, b]
        i2t = K.filip_reduce(m2, w_i, B, I, b, transpose=True)                   # [b, B] (text, image)

        # A caption without any valid token (an empty string) has every i2t similarity at the
        # -FLT_MAX fill: the reference's mean overflows to -inf and that row adds neither loss nor
        # gradient.  Its t2i row is 0 (the masked mean of nothing) and is an ordinary row.
        has_tokens = text_mask.any(dim=1).contiguous()

        loss = torch.zeros(1, device=dev, dtype=F32)
        lse_t = K.filip_nce_fwd(t2i, off, dcl, loss, 1.0 / (2 * B))
        lse_i = K.filip_nce_fwd(i2t, off, dcl, loss, 1.0 / (2 * B), row_valid=has_tokens)
        if world > 1:
            D_.all_reduce_sum_(loss)

        ctx.cfg = (dcl, extra, rank, world, b, B, T, I, D, off)
        ctx.stuff = (temp_exp, ops, img_all, w_t, w_i, m1, a1, m2, a2, t2i, i2t, lse_t, lse_i, has_tokens)
        return loss.reshape(())

    @staticmethod
    def backward(ctx, gloss):
        dcl, extra, rank, world, b, B, T, I, D, off = ctx.cfg
        temp_exp, ops, img_all, w_t, w_i, m1, a1, m2, a2, t2i, i2t, lse_t, lse_i, has_tokens = ctx.stuff
        dev = gloss.device
        gscale = (gloss.detach().float() / (2.0 * B)).reshape(1)
        g_t = K.filip_nce_bwd(t2i, lse_t, off, dcl, gscale)                      # [x local, y all]
        g_i = K.filip_nce_bwd(i2t, lse_i, off, dcl, gscale,                      # -> [y all, x local]
                              row_valid=has_tokens).t().contiguous()
        dtemp = torch.zeros(1, device=dev, dtype=F32)

        def one_pass(seg_arg, seg_max, wmat, rowscale, rows_per_sample, seg_len, nseg, row_hi, col_hi):
            """rows x cols pass: returns (d rows [R, D], d cols [C, D]) in fp32."""
            R = seg_arg.shape[0]
            C = nseg * seg_len
            d_rows = torch.empty((R, D), device=dev, dtype=F32)
            d_cols = torch.zeros((C, D), device=dev, dtype=F32)
            chunk = max(128, min(R, (1 << 29) // max(C, 1)) // 128 * 128)
            for r0 in range(0, R, chunk):
                rows = min(chunk, R - r0)
                g = K.filip_expand(seg_arg, seg_max, wmat, rowscale, temp_exp, r0, rows,
                                   rows_per_sample, seg_len, nseg, dtemp)
                K.gemm(g, col_hi, b_major=1, out=d_rows[r0:r0 + rows])
                K.gemm(g, row_hi[r0:r0 + rows], a_major=1, b_major=1, out=d_cols, accumulate=True)
            return d_rows, d_cols

        hi = lambda t: t[:, :D]
        # pass A: rows = local text tokens, columns = image tokens of all ranks
        dzt, dzi_all = one_pass(a1, m1, g_t, w_t, T, I, B, hi(ops[0][0]), hi(img_all[1]))
        # pass B: rows = image tokens of all ranks, columns = local text tokens
        if extra:
            dzi_x_all, dzt_x = one_pass(a2, m2, g_i, w_i, I, T, b, hi(img_all[2]), hi(ops[2][1]))
            dzi_x = D_.reduce_scatter_rows(dzi_x_all)
        else:
            dzi_b, dzt_b = one_pass(a2, m2, g_i, w_i, I, T, b, hi(img_all[0]), hi(ops[0][1]))
            dzt += dzt_b
            dzi_all += dzi_b
            dzt_x = dzi_x = None
        dzi = D_.reduce_scatter_rows(dzi_all)
        if world > 1:
            D_.all_reduce_sum_(dtemp)
        ctx.stuff = None
        shp_t, shp_i = (b, T, D), (b, I, D)
        return (dzt.view(shp_t), dzi.view(shp_i),
                None if dzt_x is None else dzt_x.view(shp_t),
                None if dzi_x is None else dzi_x.view(shp_i),
                dtemp.reshape(()), None, None, None, None)


def filip_loss(clip, zt, zi, zt_x, zi_x, ops, text_mask):
    extra = clip.extra_latent_projection
    return FilipLossFn.apply(zt, zi, zt_x if extra else None, zi_x if extra else None,
                             clip.temperature, tuple(ops), text_mask.contiguous(),
                             clip.decoupled_contrastive_learning, clip.requires_all_gather)
