"""Forward/backward schedules of the hot path as torch.autograd.Functions.

Each Function is a hand-written schedule of C-ABI kernel calls (x_clip_b200.kernels);
autograd only stitches them to the few torch ops left around them (embedding gather,
patchify, patch-dropout gather).  Activations are bf16, accumulation/statistics fp32,
parameters stay fp32 in the modules (state_dict compatible with the reference) and are
cast to bf16 once per step.

Reference call sites: Transformer.forward x_clip/x_clip.py:274-291 (TransformerFn),
nn.Linear :358,:368 (LinearFn), :713-724 (ProjectL2NormFn), :759-769 + :797-847
(ContrastiveLossFn, with x_clip/distributed.py:41-56 for the gather contract).  SigmoidLossFn is
SigLIP's pairwise sigmoid loss (not in the reference) on the same operands and gather contract.
"""
from __future__ import annotations

from typing import List, Optional

import torch
from torch.autograd.function import once_differentiable

from . import kernels as K
from . import distributed as D_

BF16 = torch.bfloat16
F32 = torch.float32
LN_EPS = 1e-5   # the reference's fp32 branch (x_clip.py:118); parameters/outputs are fp32-facing

_scope_cache = None     # dict while a weight_scope() is active, else None


def ff_weights(w1: torch.Tensor, w2: torch.Tensor, g4: torch.Tensor):
    """(w1 permuted bf16, w2*g4 bf16, row sums) for the fused feed-forward; shared inside a
    weight_scope() like weight_bf16."""
    key = ("ff", id(w1), id(w2), id(g4))
    if _scope_cache is not None:
        hit = _scope_cache.get(key)
        if hit is not None and hit[0] is w1:
            return hit[1]
    out = K.ff_weights(w1.detach(), w2.detach(), g4.detach())
    if _scope_cache is not None:
        _scope_cache[key] = (w1, out)
    return out


def weight_bf16(p: torch.Tensor) -> torch.Tensor:
    """bf16 copy of an fp32 parameter (the MMA operand).

    Cast afresh on every call: a cache validated by `p._version` goes stale under `p.data.add_()`
    style updates (Lion/LARS-type optimizers, EMA swaps, clamping), which do not bump the version
    counter - the kernels would silently keep training on old weights.  Forward schedules keep
    the casts they used in `ctx` for their backward (autograd semantics: backward sees the weights
    of its forward).  Only inside an explicit `weight_scope()` - one micro-batched forward or
    backward sweep, during which no optimizer can run - are casts shared between calls."""
    if _scope_cache is not None:
        hit = _scope_cache.get(id(p))
        if hit is not None and hit[0] is p:
            return hit[1]
    w = K.cast_bf16(p.detach())
    if _scope_cache is not None:
        _scope_cache[id(p)] = (p, w)     # holds p: ids cannot be recycled inside the scope
    return w


class weight_scope:
    """Share bf16 weight casts between the encoder calls of ONE sweep over micro-batches.
    `cache`: continue with the casts of an earlier scope (the backward sweep of a step reuses the
    forward sweep's - autograd semantics: backward sees the weights of its forward)."""

    def __init__(self, cache=None):
        self.given = cache

    def __enter__(self):
        global _scope_cache
        self.prev = _scope_cache
        if self.given is not None:
            _scope_cache = self.given
        elif _scope_cache is None:
            _scope_cache = {}
        self.cache = _scope_cache
        return self

    def __exit__(self, *exc):
        global _scope_cache
        _scope_cache = self.prev
        return False


def _wgrad(dy: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """dW[out,in] = dy^T @ x in fp32: both operands consumed MN-major, split-K + atomics."""
    out = torch.zeros((dy.shape[1], x.shape[1]), device=dy.device, dtype=F32)
    K.gemm(dy, x, a_major=1, b_major=1, out=out, accumulate=True)
    return out


# Set by the micro-batched step for every chunk but the last one it back-propagates: transformer
# weight gradients are then accumulated by the kernels straight INTO the existing `.grad` buffers
# (split-K wgrad GEMM with accumulate, gain gradients by atomics) and `None` is returned to autograd -
# no zero-filled temporary, no `grad += new` pass per parameter and chunk.  The last chunk returns
# ordinary gradient tensors, so post-accumulate hooks (GradSync) fire exactly once per step.
_accumulate_into_grad = False
INPLACE_GRAD_ACCUMULATION = True     # module switch for A/B measurements (tools/ab_step.py)


def _grad_target(param: torch.Tensor):
    """`param.grad` when this backward may accumulate into it in place, else None."""
    if not _accumulate_into_grad:
        return None
    g = getattr(param, "grad", None)
    if g is None or g.dtype != F32 or not g.is_contiguous() or g.shape != param.shape or not param.is_leaf:
        return None
    return g


class TransformerFn(torch.autograd.Function):
    """x[B,n,d] (bf16) -> norm_out(blocks(norm_in(x))) (bf16); mask: bool [B,n] or None.

    flat weights = [norm_in.g, norm_out.g] + depth * [g1, wqkv, wo, go, g2, w1, g4, w2].
    causal: the reference's causal mask (x_clip.py:233-236); rot_cos / rot_sin: f32 [n, 16] tables of
    the rotary embedding applied to q, k and v (x_clip.py:221-223) or None.
    TransformerDropoutFn is the same encoder with attention dropout.
    """

    @staticmethod
    def forward(ctx, x, mask, heads: int, depth: int, causal: bool, rot_cos, rot_sin, need_bwd: bool,
                *weights):
        return TransformerFn._forward(ctx, x, mask, heads, depth, causal, rot_cos, rot_sin, need_bwd, None, weights)

    @staticmethod
    def backward(ctx, dout):
        return TransformerFn._backward(ctx, dout, 8)

    @staticmethod
    def _forward(ctx, x, mask, heads, depth, causal, rot_cos, rot_sin, need_bwd, drop, weights):
        B, n, d = x.shape
        M = B * n
        scale = 64 ** -0.5
        g_in, g_out = weights[0], weights[1]
        layers = [weights[2 + 8 * L: 2 + 8 * (L + 1)] for L in range(depth)]
        x_in = x.reshape(M, d)
        if x_in.dtype != BF16:
            x_in = x_in.to(BF16)
        x_in = x_in.contiguous()
        mask_c = None if mask is None else mask.contiguous()

        saved = []
        # need_bwd = torch.is_grad_enabled() at the call site (inside forward() it is always off and
        # needs_input_grad ignores no_grad): in the first sweep of the micro-batched step and in
        # inference nothing is kept for a backward, and the 8d-wide u = [value | gate] is not written
        # bf16 MMA operands of this call's weights; backward reuses exactly these (ctx.wb)
        wb = [tuple(weight_bf16(w) for w in (l[1], l[2], l[5])) for l in layers]
        # norm_in fused with the first pre-norm
        xcur, st_in, xn, st1 = K.layernorm_fwd(x_in, g_in, g2=layers[0][0], eps=LN_EPS)
        for L, (g1, wqkv, wo, go, g2, w1, g4, w2) in enumerate(layers):
            bqkv, bo, _ = wb[L]
            qkv = K.gemm(xn, bqkv)
            if rot_cos is not None:
                K.rotary_(qkv, n, 3 * heads, rot_cos, rot_sin)
            o, lse = K.attn_fwd(qkv, mask_c, B, n, heads, scale, causal, dropout=_attn_dropout(drop, L))
            y = K.gemm(o, bo)
            # x1 = LN(y)*go + x ; xn2 = LN(x1)*g2   (attention tail + feed-forward pre-norm)
            x1, st_y, xn2, st_x1 = K.layernorm_fwd(y, go, res=xcur, g2=g2, eps=LN_EPS)
            # fused feed-forward (csrc/ff.cu): GEGLU in the up-projection's epilogue, LayerNorm(4d)
            # folded into the down-projection.  h is hp = value*gelu(gate) BEFORE the LayerNorm.
            w1p, w2g, colvec = ff_weights(w1, w2, g4)
            u, h, rowsum = K.ff_up(xn2, w1p, need_u=need_bwd)
            x2, acc, st_v = K.ff_down(h, w2g, colvec, rowsum, x1, LN_EPS)
            # forward-only sweeps keep NOTHING alive beyond the layer (the list below would otherwise hold
            # every layer's activations until the call returns: ~14 of the 22 d per token-layer)
            if need_bwd:
                saved.append((xcur, st1, xn, qkv, o, lse, y, st_y, x1, st_x1, xn2, u, st_v, h,
                              w2g, colvec, acc))
            del qkv, o, lse, y, x1, xn2, u, h
            xcur = x2
            if L + 1 < depth:
                xn, st1, _, _ = K.layernorm_fwd(xcur, layers[L + 1][0], eps=LN_EPS)
        out, st_out, _, _ = K.layernorm_fwd(xcur, g_out, eps=LN_EPS)

        ctx.saved = saved
        ctx.tail = (x_in, st_in, xcur, st_out) if need_bwd else None
        ctx.mask = mask_c
        ctx.dims = (B, n, d, heads, depth, scale, causal)
        ctx.rot = (rot_cos, rot_sin)
        ctx.weights = weights
        ctx.wb = wb
        ctx.drop = drop
        return out.view(B, n, d)

    @staticmethod
    def _backward(ctx, dout, n_args: int):
        """-> gradients of the n_args leading arguments (dx and Nones) + the weights' gradients"""
        B, n, d, heads, depth, scale, causal = ctx.dims
        rot_cos, rot_sin = ctx.rot
        M = B * n
        weights = ctx.weights
        g_in, g_out = weights[0], weights[1]
        layers = [weights[2 + 8 * L: 2 + 8 * (L + 1)] for L in range(depth)]
        x_in, st_in, x_last, st_out = ctx.tail
        dev = dout.device
        dout = dout.reshape(M, d)
        if dout.dtype != BF16:
            dout = dout.to(BF16)
        dout = dout.contiguous()

        grads: List[Optional[torch.Tensor]] = [None] * len(weights)
        # parameters with requires_grad=False (a frozen tower: adversarial / guidance use) cost no
        # weight-gradient work: their wgrad GEMMs and gain reductions are skipped and None returned.
        # The data-gradient chain reads none of them, so dx is the same either way.
        wneed = ctx.needs_input_grad[n_args:]

        def gain_grad(idx):
            """fp32 accumulator for the gain gradient of weights[idx]: its .grad (in-place mode) or
            zeros; (None, None) when the gain needs no gradient"""
            if not wneed[idx]:
                return None, None
            tgt = _grad_target(weights[idx])
            if tgt is not None:
                return tgt, None
            z = torch.zeros(weights[idx].shape[0], device=dev, dtype=F32)
            return z, z

        def weight_grad(idx, dy_, x_):
            if not wneed[idx]:
                return None
            tgt = _grad_target(weights[idx])
            if tgt is not None:
                K.gemm(dy_, x_, a_major=1, b_major=1, out=tgt, accumulate=True)
                return None
            return _wgrad(dy_, x_)

        dg_out, grads[1] = gain_grad(1)
        dx = K.layernorm_bwd(dout, x_last, st_out, g_out, dg=dg_out)
        for L in reversed(range(depth)):
            g1, wqkv, wo, go, g2, w1, g4, w2 = layers[L]
            (xcur, st1, xn, qkv, o, lse, y, st_y, x1, st_x1, xn2, u, st_v, h,
             w2g, colvec, acc) = ctx.saved[L]
            ctx.saved[L] = None
            bqkv, bo, b1 = ctx.wb[L]
            base = 2 + 8 * L
            # feed-forward: x2 = LN(hp) g4 @ w2^T + x1, h the pre-norm hp.  Row means of the LayerNorm
            # backward from d-wide data, the LN + GEGLU backward inside the dgrad GEMM, dW2 / dg4 from
            # dW2g = dxs^T hp - vsum
            dg4, grads[base + 6] = gain_grad(base + 6)
            dxs, vsum, ab = K.ff_bwd_prep(dx, st_v, acc, colvec)     # dxs / vsum: dW2 / dg4 only
            du = K.ff_bwd(dx, w2g, u, st_v, ab)
            dw2 = None
            if wneed[base + 7] or wneed[base + 6]:     # dg4 comes out of dW2g as well
                dw2 = K.ff_w2_grad_post_(_wgrad(dxs, h), vsum, g4.detach(),
                                         *((w2.detach(), dg4) if dg4 is not None else ()))
                tgt = _grad_target(w2) if wneed[base + 7] else None
                if tgt is not None:
                    tgt.add_(dw2)
                if tgt is not None or not wneed[base + 7]:
                    dw2 = None
            grads[base + 7] = dw2
            dxn2 = K.gemm(du, b1, b_major=1)
            grads[base + 5] = weight_grad(base + 5, du, xn2)
            del du
            dg2, grads[base + 4] = gain_grad(base + 4)
            dx1 = K.layernorm_bwd(dxn2, x1, st_x1, g2, add=dx, dg=dg2)
            # attention: x1 = LN(o @ wo^T) * go + x
            dgo, grads[base + 3] = gain_grad(base + 3)
            dy = K.layernorm_bwd(dx1, y, st_y, go, dg=dgo)
            d_o = K.gemm(dy, bo, b_major=1)
            grads[base + 2] = weight_grad(base + 2, dy, o)
            dqkv = K.attn_bwd(qkv, ctx.mask, o, d_o, lse, B, n, heads, scale, causal,
                              dropout=_attn_dropout(ctx.drop, L))
            if rot_cos is not None:      # back through the rotation (its transpose)
                K.rotary_(dqkv, n, 3 * heads, rot_cos, rot_sin, inverse=True)
            dxn = K.gemm(dqkv, bqkv, b_major=1)
            grads[base + 1] = weight_grad(base + 1, dqkv, xn)
            dg1, grads[base + 0] = gain_grad(base + 0)
            dx = K.layernorm_bwd(dxn, xcur, st1, g1, add=dx1, dg=dg1)
        dg_in, grads[0] = gain_grad(0)
        dx_in = K.layernorm_bwd(dx, x_in, st_in, g_in, dg=dg_in)
        ctx.saved = ctx.wb = ctx.drop = None
        return (dx_in.view(B, n, d),) + (None,) * (n_args - 1) + tuple(grads)


def _attn_dropout(drop, L: int):
    """The (p, seed, layer) argument of K.attn_fwd / attn_bwd for layer L, or None (no dropout)."""
    if drop is None or drop[0][L] == 0.0:
        return None
    return drop[0][L], drop[1], L


class TransformerDropoutFn(torch.autograd.Function):
    """TransformerFn with dropout on the attention probabilities (x_clip.py:211, :241-243).

    drop = (p per layer, seed): seed is an int64 [1] device tensor, the Philox key of every layer's
    mask (xclip_attn_dropout_fwd; layer L draws with counter word L).  The backward reuses the seed
    kept in ctx, so it sees the forward's masks; a second forward with the same seed (the re-encode of
    a micro-batched step, or a forward-only sweep) draws the same masks as well.  A layer with p = 0
    runs the plain kernels."""

    @staticmethod
    def forward(ctx, x, mask, heads: int, depth: int, causal: bool, rot_cos, rot_sin, need_bwd: bool, drop,
                *weights):
        return TransformerFn._forward(ctx, x, mask, heads, depth, causal, rot_cos, rot_sin, need_bwd, drop, weights)

    @staticmethod
    def backward(ctx, dout):
        return TransformerFn._backward(ctx, dout, 9)


class TextEmbedFn(torch.autograd.Function):
    """[cls | token_emb[ids] + abs_pos_emb] -> bf16 [B, n+1, d] (x_clip.py:320-332), one pass."""

    @staticmethod
    def forward(ctx, ids, tok, pos, cls):
        out = K.text_embed_fwd(ids, tok.detach(), pos.detach(), cls.detach())
        ctx.save_for_backward(ids)
        ctx.shapes = (tok.shape[0], pos.shape[0])
        return out

    @staticmethod
    def backward(ctx, dx):
        (ids,) = ctx.saved_tensors
        vocab, pos_rows = ctx.shapes
        if dx.dtype != BF16:
            dx = dx.to(BF16)
        dtok, dpos, dcls = K.text_embed_bwd(ids, dx, vocab, pos_rows)
        return None, dtok, dpos, dcls


class LinearFn(torch.autograd.Function):
    """y = x @ W^T (+ bias) (+ table[row % period])  - x bf16 [M,K], W fp32 [N,K].

    `table` is a positional-embedding table added per row modulo `period` (the vision
    transformer's pos_emb, x_clip.py:382-383) fused in the GEMM epilogue."""

    @staticmethod
    def forward(ctx, x, weight, bias, table):
        x = x.contiguous()
        tbl16 = None if table is None else K.cast_bf16(table.detach())
        wb = weight_bf16(weight)
        y = K.gemm(x, wb, bias=None if bias is None else bias.detach(),
                   residual=tbl16, res_row_mod=0 if table is None else table.shape[0])
        ctx.save_for_backward(x, wb)
        ctx.has_bias = bias is not None
        ctx.period = None if table is None else table.shape[0]
        return y

    @staticmethod
    def backward(ctx, dy):
        x, wb = ctx.saved_tensors
        dy = dy.contiguous()
        if dy.dtype != BF16:
            dy = dy.to(BF16)
        dx = K.gemm(dy, wb, b_major=1) if ctx.needs_input_grad[0] else None
        dw = _wgrad(dy, x) if ctx.needs_input_grad[1] else None
        db = dy.float().sum(dim=0) if ctx.has_bias and ctx.needs_input_grad[2] else None
        dt = None
        if ctx.period is not None and ctx.needs_input_grad[3]:
            dt = dy.float().view(-1, ctx.period, dy.shape[1]).sum(dim=0)
        return dx, dw, db, dt


def patch_rows(img, patch: int, keep):
    """bf16 patch rows of `img` (the kept patches, K.patchify_gather) in the layout PatchEmbedFn
    takes: [B*k, K.patch_row_stride(patch_dim)], zero columns after patch_dim."""
    return K.patchify_gather(img, patch, keep, ld=K.patch_row_stride(patch * patch * img.shape[1]))


def patch_weight_bf16(weight: torch.Tensor) -> torch.Tensor:
    """bf16 patch-embedding weight [dim, K.patch_row_stride(patch_dim)] with zero columns after
    patch_dim: the operand that meets patch_rows() in a GEMM with K = row stride (the zero columns add
    exact zeros).  weight_bf16 itself when patch_dim is a multiple of 8; otherwise shared inside a
    weight_scope() under a key of its own, apart from weight_bf16's unpadded casts."""
    ld = K.patch_row_stride(weight.shape[1])
    if ld == weight.shape[1]:
        return weight_bf16(weight)
    key = ("patch_rows", id(weight))
    if _scope_cache is not None:
        hit = _scope_cache.get(key)
        if hit is not None and hit[0] is weight:
            return hit[1]
    w = K.cast_bf16_rows(weight.detach(), ld)
    if _scope_cache is not None:
        _scope_cache[key] = (weight, w)
    return w


def _patch_embed_fwd(ctx, patches, index, weight, bias, table, keep_wb: bool):
    wb = patch_weight_bf16(weight)
    tbl16 = K.cast_bf16(table.detach())
    y = K.gemm(patches, wb, bias=bias.detach(), residual=tbl16, res_row_idx=index)
    ctx.save_for_backward(patches, index)
    ctx.wb = wb if keep_wb else None          # the dgrad operand, kept only when d patches is wanted
    ctx.table_rows = table.shape[0]
    ctx.patch_dim = weight.shape[1]
    return y


def _patch_embed_bwd(ctx, dy, need_dp: bool, need_w: bool, need_b: bool, need_t: bool):
    """(d patches f32 [M, row stride], dW [dim, patch_dim], d bias, d pos), each None unless asked for"""
    patches, index = ctx.saved_tensors
    dy = dy.contiguous()
    if dy.dtype != BF16:
        dy = dy.to(BF16)
    dp = K.gemm(dy, ctx.wb, b_major=1, out_dtype=F32) if need_dp else None
    dw = None
    if need_w:
        # N = row stride; the columns past patch_dim are dropped into a contiguous [dim, patch_dim]
        # gradient (GradSync / FusedAdamW flatten .grad, which would copy a strided view every step)
        dw = _wgrad(dy, patches)
        if dw.shape[1] != ctx.patch_dim:
            dw = dw[:, :ctx.patch_dim].contiguous()
    db = K.colsum_rows_(torch.zeros(dy.shape[1], device=dy.device, dtype=F32), dy) if need_b else None
    dt = None
    if need_t:
        dt = K.scatter_add_rows_(torch.zeros((ctx.table_rows, dy.shape[1]), device=dy.device, dtype=F32),
                                 dy, idx=index)
    ctx.wb = None
    return dp, dw, db, dt


class PatchEmbedFn(torch.autograd.Function):
    """tokens = patches @ W^T + bias + pos[index]  (x_clip.py:356-359, :382-383, with the
    PatchDropout selection :134-151 already applied to `patches` and `index`).

    patches bf16 [B*k, K.patch_row_stride(patch_dim)] come from patch_rows() (only the kept patches are
    read from the image; zero columns after patch_dim, so any patch size runs on the GEMM); `index`
    int32 [B*k] is the patch index of every row = the row of the position table the GEMM epilogue
    adds.  Backward: d patches = dy @ W (f32 GEMM output; autograd hands it back in
    the dtype of `patches`), dW by the wgrad GEMM, d bias = column sums, d pos = rows of dy
    scatter-added by `index`; each only for inputs that need a gradient.  An image that wants a
    gradient goes through PatchifyFn instead, which keeps d patches in f32 up to the pixels."""

    @staticmethod
    def forward(ctx, patches, index, weight, bias, table):
        return _patch_embed_fwd(ctx, patches, index, weight, bias, table, ctx.needs_input_grad[0])

    @staticmethod
    def backward(ctx, dy):
        n = ctx.needs_input_grad
        dp, dw, db, dt = _patch_embed_bwd(ctx, dy, n[0], n[2], n[3], n[4])
        return dp, None, dw, db, dt


class PatchifyFn(torch.autograd.Function):
    """tokens of an image that wants a gradient: patchify + PatchDropout selection (x_clip.py:356-359,
    :134-151; forward K.patchify_gather) and the patch embedding of PatchEmbedFn in one Function.
    Backward: d patches = dy @ W in f32, then K.patchify_scatter - the kept patches' rows go back to
    their pixels, dropped patches get 0, as the reference's gather `x[batch_indices, keep]` gives.  One
    Function, so that d patches reaches the scatter in f32 (autograd would round a gradient flowing
    between two Functions to the bf16 of the patches).  once_differentiable: a double backward through
    the image raises instead of returning zero curvature."""

    @staticmethod
    def forward(ctx, img, patch: int, keep, index, weight, bias, table):
        patches = patch_rows(img, patch, keep)
        ctx.shape, ctx.patch, ctx.keep = tuple(img.shape), patch, keep
        return _patch_embed_fwd(ctx, patches, index, weight, bias, table, ctx.needs_input_grad[0])

    @staticmethod
    @once_differentiable
    def backward(ctx, dy):
        n = ctx.needs_input_grad
        dp, dw, db, dt = _patch_embed_bwd(ctx, dy, n[0], n[4], n[5], n[6])
        dimg = None
        if dp is not None:
            dimg = K.patchify_scatter(dp[:, :ctx.patch_dim], ctx.shape, ctx.patch, ctx.keep)
        ctx.keep = None
        return dimg, None, None, None, dw, db, dt


class ProjectL2NormFn(torch.autograd.Function):
    """z = normalize(e @ W^T) (x_clip.py:713-715).  Returns (z fp32, zrow, zcol): the last two
    are the split-bf16 MMA operands of the logits contraction (no grad), see xclip_l2norm_fwd."""

    @staticmethod
    def forward(ctx, e, weight):
        e = e.contiguous()
        wb = weight_bf16(weight)
        p = K.gemm(e, wb, out_dtype=F32)
        z, zrow, zcol, inv = K.l2norm_fwd(p)
        ctx.save_for_backward(e, wb, z, inv)
        ctx.mark_non_differentiable(zrow, zcol)
        return z, zrow, zcol

    @staticmethod
    def backward(ctx, dz, _a, _b):
        e, wb, z, inv = ctx.saved_tensors
        dp = K.l2norm_bwd(dz.contiguous().float(), z, inv)
        de = K.gemm(dp, wb, b_major=1) if ctx.needs_input_grad[0] else None
        dw = _wgrad(dp, e) if ctx.needs_input_grad[1] else None
        return de, dw


class ContrastiveLossFn(torch.autograd.Function):
    """InfoNCE / DCL over all pairs of the GLOBAL batch (x_clip.py:759-769, :813-847).

    Inputs: local unit-norm latents zt, zi [b, D] (fp32, carry the graph), optional extra pair,
    the temperature parameter, and `ops`: per latent set the (zrow, zcol) split-bf16 operands.
    With world size W > 1 one all-gather exchanges the column operands of every set (replacing
    x_clip/distributed.py:14-39), each rank evaluates only its own row blocks, and a second tiny
    all-gather exchanges (lse, pos) so every rank returns the same global loss.  Backward
    reproduces AllGather.backward's contract (distributed.py:50-54): latent grads are
    d loss / d(local latents); d temperature is the full-batch gradient on every rank.

    sim_reg_weight w > 0 (extra latents only) adds the similarity regularisation (x_clip.py:771-784,
    :870-873): w/2 * (mean_{i!=j} E_ij^2 + mean_{i!=j} E'_ij^2), E = T T^T - V V^T over the global
    batch, E' the same over the extra pair (xclip_simreg_*).  It reuses the gathered column operands and
    rides in the statistics gather, so a step still makes one latent all-gather.  The returned value
    is then cl_weight * contrastive + w * L_sim (cl_weight lets the auxiliary-loss path weigh the two
    terms as the reference does).  Global batch 1 gives NaN, the mean of nothing, and no gradient from
    the term - the reference's behaviour."""

    @staticmethod
    def forward(ctx, zt, zi, zt_x, zi_x, temperature, ops, dcl: bool, use_gather: bool,
                sim_reg_weight: float = 0.0, cl_weight: float = 1.0):
        extra = len(ops) == 4
        sim_w = float(sim_reg_weight)
        if sim_w != 0.0 and not extra:
            raise ValueError("the similarity regularisation needs the extra latent pair")
        rank, world = D_.world() if use_gather else (0, 1)
        b = ops[0][0].shape[0]
        D = ops[0][0].shape[1] // 3
        temp_exp = temperature.detach().float().exp().reshape(1)

        rows = [o[0] for o in ops]                                  # local [b, 3D], [hi|lo|hi]
        cols = D_.gather_rows([o[1] for o in ops]) if world > 1 else [o[1] for o in ops]
        Bg = world * b
        off = rank * b

        # forward row blocks: texts vs all images; images vs all texts (extra latents if any)
        T, I, TX, IX = 0, 1, 2, 3
        lse_t, pos_t = K.nce_fwd(rows[T], cols[I], temp_exp, off, dcl)
        if extra:
            lse_i, pos_i = K.nce_fwd(rows[IX], cols[TX], temp_exp, off, dcl)
        else:
            lse_i, pos_i = K.nce_fwd(rows[I], cols[T], temp_exp, off, dcl)

        sim_ops = None
        if sim_w != 0.0:
            # E = [T | V] . [T | -V]^T per pair: the difference forms inside the fp32 accumulator
            sim_ops = [(K.simreg_pack(rows[t], rows[v], False), K.simreg_pack(cols[t], cols[v], True))
                       for t, v in ((T, I), (TX, IX))]
            sim_rows = [K.simreg_fwd(a, c, off) for a, c in sim_ops]

        stats = torch.stack([lse_t, pos_t, lse_i, pos_i] + (sim_rows if sim_ops else []))   # [4 or 6, b]
        gstats = D_.gather_stats(stats) if world > 1 else stats
        loss = ((gstats[0] - gstats[1]).sum() + (gstats[2] - gstats[3]).sum()) / (2.0 * Bg)
        if sim_ops:
            # mean over the Bg (Bg - 1) off-diagonal entries; 0 / 0 = NaN at Bg = 1 like the reference
            loss = cl_weight * loss + sim_w * ((gstats[4].sum() + gstats[5].sum()) / (2.0 * Bg * (Bg - 1)))
        elif cl_weight != 1.0:
            loss = cl_weight * loss

        ctx.cfg = (dcl, extra, rank, world, b, D, Bg, off)
        ctx.sim = (sim_w, float(cl_weight), sim_ops)
        ctx.temp_exp = temp_exp
        ctx.rows, ctx.cols = rows, cols
        # xclip_nce_bwd reads lse_col with 16-byte vector loads.  Row k of the [4, Bg] stats starts
        # 4*k*Bg bytes in, so row 2 is misaligned for odd Bg: clone the rows into storage of their own.
        ctx.lse = (lse_t, lse_i, gstats[0].clone(), gstats[2].clone())
        return loss

    @staticmethod
    def backward(ctx, gloss):
        dcl, extra, rank, world, b, D, Bg, off = ctx.cfg
        temp_exp = ctx.temp_exp
        rows, cols = ctx.rows, ctx.cols
        lse_t, lse_i, lse_t_all, lse_i_all = ctx.lse
        sim_w, cl_weight, sim_ops = ctx.sim
        gl = gloss.detach().float()
        gscale = ((gl if cl_weight == 1.0 else gl * cl_weight) / (2.0 * Bg)).reshape(1)
        dtemp = torch.zeros(1, device=gloss.device, dtype=F32)
        T, I, TX, IX = 0, 1, 2, 3

        def latent_grad(r, c, lse_row, lse_col, w_row, w_col, w_diag, want_dtemp):
            g = K.nce_bwd(rows[r], cols[c], temp_exp, off, dcl, lse_row, lse_col, w_row, w_col,
                          w_diag, gscale, dtemp if want_dtemp else None)
            # d rows = (temp * g) @ cols_hi ; g is zero-padded to a multiple of 8 columns
            return K.gemm(g, _pad_rows(cols[c][:, :D], g.shape[1]), b_major=1, out_dtype=F32)

        if not extra:
            dzt = latent_grad(T, I, lse_t, lse_i_all, 1.0, 1.0, 2.0, True)
            dzi = latent_grad(I, T, lse_i, lse_t_all, 1.0, 1.0, 2.0, False)
            dzt_x = dzi_x = None
        else:
            dzt = latent_grad(T, I, lse_t, None, 1.0, 0.0, 1.0, True)
            dzi = latent_grad(I, T, None, lse_t_all, 0.0, 1.0, 1.0, False)
            dzi_x = latent_grad(IX, TX, lse_i, None, 1.0, 0.0, 1.0, True)
            dzt_x = latent_grad(TX, IX, None, lse_i_all, 0.0, 1.0, 1.0, False)
        if sim_ops and Bg > 1:
            # d(w L_sim)/dt_r = (2w/N) sum_j E_rj t_j, d/dv_r = -(2w/N) sum_j E_rj v_j over the global j
            sgs = (gloss.detach().float() * (2.0 * sim_w / (Bg * (Bg - 1.0)))).reshape(1)
            for (a, c), t, v, dt_, dv_ in zip(sim_ops, (T, TX), (I, IX), (dzt, dzt_x), (dzi, dzi_x)):
                g = K.simreg_bwd(a, c, off, sgs)
                K.gemm(g, _pad_rows(cols[t][:, :D], g.shape[1]), b_major=1, out=dt_, accumulate=True)
                K.gemm(g, _pad_rows(cols[v][:, :D], g.shape[1]), b_major=1, out=dv_, alpha=-1.0,
                       accumulate=True)
                del g
        if world > 1:
            D_.all_reduce_sum_(dtemp)       # every rank holds the full-batch d loss / d temperature
        ctx.rows = ctx.cols = ctx.sim = None
        grads = (dzt, dzi, dzt_x, dzi_x, dtemp.reshape(()))
        return grads + (None,) * (len(ctx.needs_input_grad) - len(grads))


class SigmoidLossFn(torch.autograd.Function):
    """The pairwise sigmoid loss of SigLIP (Zhai et al., ICCV 2023) over all pairs of the GLOBAL batch:

        l_ij = exp(temperature) <t_i, v_j> + logit_bias,   z_ij = +1 if i == j else -1
        L = (1/B) sum_ij softplus(-z_ij l_ij)

    Inputs as ContrastiveLossFn without the extra pair: local unit latents zt, zi [b, D] (fp32, carry the
    graph), the temperature and logit_bias parameters (scalars) and `ops`, the (zrow, zcol) split-bf16
    operands of texts and images.  The forward runs one row block, the local texts against all
    (gathered) images at diag_offset = rank * b; the per-row losses ride in one statistics gather, so every
    rank returns the same global loss.  Backward: the texts x images block gives d zt and the images x
    texts block d zi, each through the plain dgrad GEMM; d temperature and d logit_bias come from the
    first block and are all-reduced, so every rank holds their full-batch gradients (the contract of
    d temperature in ContrastiveLossFn)."""

    @staticmethod
    def forward(ctx, zt, zi, temperature, logit_bias, ops, use_gather: bool):
        rank, world = D_.world() if use_gather else (0, 1)
        b = ops[0][0].shape[0]
        D = ops[0][0].shape[1] // 3
        temp_exp = temperature.detach().float().exp().reshape(1)
        bias = logit_bias.detach().float().reshape(1).contiguous()
        rows = [o[0] for o in ops]
        cols = D_.gather_rows([o[1] for o in ops]) if world > 1 else [o[1] for o in ops]
        Bg = world * b
        off = rank * b
        rowloss = K.sigmoid_fwd(rows[0], cols[1], temp_exp, bias, off)
        stats = D_.gather_stats(rowloss[None]) if world > 1 else rowloss[None]
        ctx.cfg = (world, D, Bg, off)
        ctx.scalars = (temp_exp, bias)
        ctx.rows, ctx.cols = rows, cols
        return stats.sum() / Bg

    @staticmethod
    def backward(ctx, gloss):
        world, D, Bg, off = ctx.cfg
        temp_exp, bias = ctx.scalars
        rows, cols = ctx.rows, ctx.cols
        gscale = (gloss.detach().float() / Bg).reshape(1)
        dscalars = torch.zeros(2, device=gloss.device, dtype=F32)     # d temperature, d logit_bias

        def latent_grad(r, c, want_scalars):
            g = K.sigmoid_bwd(rows[r], cols[c], temp_exp, bias, off, gscale,
                              dscalars[0:1] if want_scalars else None, dscalars[1:2] if want_scalars else None)
            # d rows = (temp * g) @ cols_hi ; g is zero-padded to a multiple of 8 columns
            return K.gemm(g, _pad_rows(cols[c][:, :D], g.shape[1]), b_major=1, out_dtype=F32)

        dzt = latent_grad(0, 1, True)
        dzi = latent_grad(1, 0, False)
        if world > 1:
            D_.all_reduce_sum_(dscalars)
        ctx.rows = ctx.cols = None
        # two tensors of their own: .grad buffers must not share storage
        return dzt, dzi, dscalars[0].clone(), dscalars[1].clone(), None, None


# bytes of one backward window of the vocabulary cross-entropy's g [rows, roundup8(V)] bf16: at the
# CLIP BPE vocabulary (V = 49408) that is 10752 rows, against 2.4 G logits for 49 k selected rows
VOCAB_CE_WINDOW_BYTES = 1 << 30


def vocab_window_rows(n: int, V: int, budget: int = None) -> int:
    """Rows of one backward window of g [rows, roundup8(V)] bf16 within `budget` bytes: all n rows
    when they fit, else a multiple of 128 rows where that many fit, else at least 1."""
    budget = VOCAB_CE_WINDOW_BYTES if budget is None else budget
    rows = budget // (2 * ((V + 7) // 8 * 8))
    if rows >= n:
        return n
    return rows // 128 * 128 if rows >= 128 else max(rows, 1)


def check_labels(labels: torch.Tensor, V: int) -> None:
    """Raise, as F.cross_entropy does, on a target outside [0, V).  The comparison stays on the
    device: for CUDA labels the error is a device-side assert, reported by the next synchronising
    call, and no host synchronisation is added to the step; for CPU labels it raises here."""
    torch._assert_async(((labels >= 0) & (labels < V)).all(), "x_clip_b200: cross-entropy target out of bounds")


class VocabCrossEntropyFn(torch.autograd.Function):
    """F.cross_entropy(rows @ weight^T + bias, labels): the mean over the n rows of lse - target
    logit (reference mlm.py:105-107 on the selected positions).

    rows bf16 [n, d] (n >= 1), weight fp32 [V, d], bias fp32 [V] or None, labels int64 [n] in
    [0, V) for any V >= 1.  Forward: xclip_vocab_ce_fwd, the softmax reduced inside the GEMM
    epilogue, so no [n, V] logits exist.  Backward: g = gscale (softmax - onehot) in row windows
    of VOCAB_CE_WINDOW_BYTES (xclip_vocab_ce_bwd recomputes the logits), then d rows = g W,
    d weight = g^T rows and d bias = column sums of g - each only when its input needs a gradient.
    A label outside [0, V) raises as in torch, through a device-side assert (no host sync)."""

    @staticmethod
    def forward(ctx, rows, weight, bias, labels):
        rows = rows.contiguous()
        if rows.dtype != BF16:
            rows = rows.to(BF16)
        labels = labels.contiguous()
        n, V = rows.shape[0], weight.shape[0]
        check_labels(labels, V)
        wb = weight_bf16(weight)
        b = None if bias is None else bias.detach().contiguous()
        loss = torch.zeros(1, device=rows.device, dtype=F32)
        lse, _ = K.vocab_ce_fwd(rows, wb, b, labels, loss, 1.0 / n)
        # the bias as given: autograd's version check refuses a backward after an in-place update
        # (wb is already this call's own copy of the weight)
        ctx.save_for_backward(rows, wb, labels, lse, bias)
        return loss.reshape(())

    @staticmethod
    @once_differentiable
    def backward(ctx, gloss):
        rows, wb, labels, lse, bias = ctx.saved_tensors
        b = None if bias is None else bias.detach().contiguous()
        need_x, need_w, need_b = ctx.needs_input_grad[:3]
        n, d = rows.shape
        V = wb.shape[0]
        dev = rows.device
        gscale = (gloss.detach().float() / n).reshape(1)
        dx = torch.empty((n, d), device=dev, dtype=BF16) if need_x else None
        dw = torch.zeros((V, d), device=dev, dtype=F32) if need_w else None
        db = torch.zeros(((V + 7) // 8 * 8,), device=dev, dtype=F32) if need_b else None
        if need_x or need_w or need_b:
            win = vocab_window_rows(n, V)
            gbuf = torch.empty((win, (V + 7) // 8 * 8), device=dev, dtype=BF16)
            for r0 in range(0, n, win):
                r1 = min(r0 + win, n)
                x = rows[r0:r1]
                g = K.vocab_ce_bwd(x, wb, b, labels[r0:r1], lse[r0:r1], gscale, out=gbuf[: r1 - r0])
                gv = g[:, :V]
                if need_x:
                    K.gemm(gv, wb, b_major=1, out=dx[r0:r1])
                if need_w:
                    K.gemm(gv, x, a_major=1, b_major=1, out=dw, accumulate=True)
                if need_b:
                    K.colsum_rows_(db, g)                 # the pad columns of g are zero
            del gbuf
        return dx, dw, None if db is None else db[:V], None


def _pad_rows(m: torch.Tensor, rows: int) -> torch.Tensor:
    """g has roundup8(C) columns; the matching operand needs that many rows (zeros beyond C)."""
    if m.shape[0] == rows:
        return m
    out = torch.zeros((rows, m.shape[1]), device=m.device, dtype=m.dtype)
    out[: m.shape[0]] = m
    return out


def _avail_bytes(dev) -> int:
    """HBM a further allocation can draw on: free device memory + the cached-but-unused part of
    torch's pool (counted at 80 %: cached blocks are not one contiguous range)."""
    free, _ = torch.cuda.mem_get_info(dev)
    cached = torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev)
    return int(free + 0.8 * max(cached, 0))


# HBM head-room the retention planner leaves untouched: contrastive-loss workspace (g[b, B_g] bf16
# per direction, gathered operands), gradient buckets, allocator slack.  The similarity
# regularisation adds its packed operands, 24 (b + B_g) D bytes for the two latent pairs, and one
# more transient g[b, B_g] bf16 at a time: 0.72 GB at b = 4096, B_g = 32768, D = 512 - inside the margin.
RETAIN_MARGIN_BYTES = 10 << 30
# transient buffers of one chunk's backward (du 8d + a few d-wide rows of one layer) relative to
# the chunk's saved activations (22 d per token-layer x depth)
RETAIN_TRANSIENT_FRAC = 0.15


class _InPlaceGradAccumulation:
    def __init__(self, flag: bool):
        self.flag = flag

    def __enter__(self):
        global _accumulate_into_grad
        self.prev = _accumulate_into_grad
        _accumulate_into_grad = self.flag
        return self

    def __exit__(self, *exc):
        global _accumulate_into_grad
        _accumulate_into_grad = self.prev
        return False


def _chunk_passes(clip, text, image, text_mask, aux, s: int, e: int, img_k=None):
    """The gradient passes of chunk [s, e), in a fixed order: contrastive encoders, then the MLM text
    pass on the corrupted rows, then the two augmented image views.  Each image pass draws its
    patch-dropout keep from the RNG stream in that order, so a re-encode from the chunk's saved RNG
    state draws the keeps of the forward.  -> (outputs, ops): the latents, then the encodings of the
    chunk's MLM-selected positions [n_sel, d] and the CLS representations of both views [e - s, rep]."""
    z, ops = clip._encode_to_latents(text[s:e], image[s:e] if img_k is None else img_k, text_mask[s:e])
    outs = list(z)
    if aux is not None:
        if aux["mlm"] is not None:
            masked, sel, _ = aux["mlm"]
            enc = clip.mlm.transformer(masked[s:e], mask=text_mask[s:e])[:, 1:]
            outs.append(enc[sel[s:e]])
        if aux["ssl"] is not None:
            one, two = aux["ssl"]
            outs += [aux["ssl_encoder"].rep(one[s:e]), aux["ssl_encoder"].rep(two[s:e])]
    return outs, ops


def _chunk_targets(aux, s: int, e: int):
    """SimSiam's target passes of chunk [s, e): both views encoded again without gradient (their own
    patch-dropout draws, after the gradient passes), never kept for backward."""
    one, two = aux["ssl"]
    enc = aux["ssl_encoder"]
    with torch.no_grad():
        return enc.rep(one[s:e]), enc.rep(two[s:e])


def _aux_losses(clip, aux, leaves, targets):
    """(MLM loss, visual SSL loss) on the full-batch leaves, each None when off."""
    mlm = ssl = None
    i = 0
    if aux["mlm"] is not None:
        rows, labels = leaves[i], aux["mlm"][2]
        i += 1
        head = clip.mlm.to_logits
        # no selected position: the single pass's enc.sum() * 0
        mlm = VocabCrossEntropyFn.apply(rows, head.weight, head.bias, labels) if rows.shape[0] else \
            rows.sum() * 0.
    if aux["ssl"] is not None:
        r1, r2 = leaves[i], leaves[i + 1]
        if aux["ssl_targets"]:
            t1 = torch.cat([t[0] for t in targets])
            t2 = torch.cat([t[1] for t in targets])
            ssl = clip.visual_ssl.loss_from_reps(r1, r2, t1, t2)
        else:
            ssl = clip.visual_ssl.loss_from_reps(r1, r2)
    return mlm, ssl


class ChunkedClipLossFn(torch.autograd.Function):
    """Full-batch contrastive loss with micro-batched encoders.

    The reference offers `checkpoint_during_training` (x_clip.py:280-286) to fit large batches;
    here the same need (4096 pairs per GPU for a 32768 global batch) is met by a GradCache-style
    schedule that is mathematically identical to the single-pass step:
      1. encode every chunk -> latents of the whole local batch
      2. one contrastive loss over ALL latents (with the usual cross-rank all-gather); with
         `use_all_token_embeds` the FILIP loss (filip.FilipLossFn) over all token latents, which
         works in row chunks of its own and is left `filip.step_reserve_bytes` of HBM by the plan;
         with `logit_bias` given (CLIP(sigmoid_loss=True)) the sigmoid loss, SigmoidLossFn, with
         logit_bias as one more leaf beside the temperature
      3. in backward: d loss / d latents, then back-propagate the matching slice of the latent
         gradient through every chunk's encoders.
    Memory plan: a chunk's saved activations are KEPT from step 1 for as many chunks as
    the GPU's HBM holds (80 GB on an H100) (`retain`: "auto" measures the first chunk's footprint and plans against
    the free memory; an int fixes the count; 0 = none); only the remaining chunks are encoded
    without saving anything and re-encoded in step 3 (RNG replayed for PatchDropout).  Retained
    chunks cost no extra flops; each re-encoded chunk costs one extra encoder forward.
    An image that wants a gradient enters every chunk's encoder as a detached per-chunk leaf; backward
    collects the leaves' gradients into d loss / d image, so the outer graph (a generator, an
    augmentation) is only ever entered by autograd itself, after this backward returns.

    `aux` (CLIP._aux_inputs) adds the auxiliary losses: the corruption (MLM) and both augmented views
    (SimSiam / SimCLR) of the whole batch, drawn once before any chunk.  Every chunk runs its gradient
    passes in one fixed order (_chunk_passes); the MLM encodings of the selected positions and the
    views' CLS representations become full-batch leaves like the latents, and the heads (vocabulary
    cross-entropy, projector / predictor with BatchNorm over the whole batch, NT-Xent) run once on
    them.  SimSiam's target passes run chunk by chunk without gradient and are never kept.  The step
    returns cl_w * contrastive + w_t * MLM + w_i * SSL, as the single pass does.  Retention keeps or
    re-encodes a chunk with all of its gradient passes."""

    @staticmethod
    def forward(ctx, clip, text, image, text_mask, chunk, temperature, retain="auto", aux=None, logit_bias=None):
        B = text.shape[0]
        dev = text.device
        bounds = [(s, min(s + chunk, B)) for s in range(0, B, chunk)]
        rng_states, zs, opss, kept, targets = [], [], [], [], []
        want_dimage = image.requires_grad
        img_leaves = []                               # per retained chunk: its image leaf (or None)

        def chunk_image(s, e):
            if not want_dimage:
                return image[s:e]
            return image[s:e].detach().requires_grad_(True)

        foot = None                                   # bytes of one retained chunk's activations
        reserve = 0                                   # HBM left to the loss (FILIP: filip.step_reserve_bytes)
        filip = clip.use_all_token_embeds
        # "auto" plans ONCE per (batch, chunk size): the first step measures and decides, later steps
        # repeat its decision - the same tensors are then allocated in the same order every step, which
        # is what keeps torch's caching allocator free of fragmentation this close to the HBM limit
        plans = clip.__dict__.setdefault("_retain_plans", {})
        plan_key = (B, chunk, str(dev))
        planned = retain == "auto" and plan_key not in plans
        keep_mask = None                              # a remembered plan: which chunks stay resident
        if retain == "auto" and not planned:
            keep_mask = plans[plan_key]
        oom_fallbacks = 0
        with torch.no_grad(), weight_scope() as wscope:
            for k, (s, e) in enumerate(bounds):
                rng_states.append(torch.cuda.get_rng_state(dev))
                if keep_mask is not None:
                    keep_it = keep_mask[k]
                elif retain == "auto":
                    scale = (e - s) / float(chunk)
                    if foot is None:                  # first chunk: keep it, measure it
                        keep_it = True
                    else:
                        need = foot * scale * (1.0 + RETAIN_TRANSIENT_FRAC) + RETAIN_MARGIN_BYTES + reserve
                        keep_it = _avail_bytes(dev) >= need
                else:
                    keep_it = k < int(retain)
                if keep_it:
                    before = torch.cuda.memory_allocated(dev)
                    z = ops = None
                    img_k = chunk_image(s, e)
                    try:
                        with torch.enable_grad():
                            z, ops = _chunk_passes(clip, text, image, text_mask, aux, s, e, img_k)
                    except torch.OutOfMemoryError:
                        # the plan was too optimistic (a fragmented cache, memory taken by someone else
                        # since the estimate): this chunk and all later ones are re-encoded in backward
                        z = ops = None
                        retain, keep_mask = 0, None   # (an int plan: nothing further is kept)
                        oom_fallbacks += 1
                    if z is None:
                        torch.cuda.empty_cache()
                        torch.cuda.set_rng_state(rng_states[-1], dev)
                        z, ops = _chunk_passes(clip, text, image, text_mask, aux, s, e)
                        kept.append(None)
                        img_leaves.append(None)
                        zs.append(z)
                        opss.append(ops)
                        if aux is not None and aux["ssl_targets"]:
                            targets.append(_chunk_targets(aux, s, e))
                        continue
                    kept.append(list(z))
                    img_leaves.append(img_k if want_dimage else None)
                    if foot is None:
                        foot = max(torch.cuda.memory_allocated(dev) - before, 1)
                        if filip:
                            from .filip import step_reserve_bytes
                            world = D_.world()[1] if clip.requires_all_gather else 1
                            reserve = step_reserve_bytes(B, world * B, z[0].shape[1], z[1].shape[1],
                                                         z[0].shape[2], len(z) == 4)
                        if planned and len(bounds) > 1 and _avail_bytes(dev) < \
                                foot * (1.0 + RETAIN_TRANSIENT_FRAC) + RETAIN_MARGIN_BYTES + reserve:
                            kept[-1] = None           # not even a second live chunk fits beside it: let it go
                            img_leaves[-1] = None
                    z = [t.detach() for t in z]
                else:
                    z, ops = _chunk_passes(clip, text, image, text_mask, aux, s, e)
                    kept.append(None)
                    img_leaves.append(None)
                zs.append(z)
                opss.append(ops)
                if aux is not None and aux["ssl_targets"]:
                    targets.append(_chunk_targets(aux, s, e))
        # rows [start, end) of every chunk in each full-batch leaf (the MLM leaf has n_sel rows)
        row_bounds, offs = [], [0] * len(zs[0])
        for z in zs:
            row_bounds.append([(offs[j], offs[j] + t.shape[0]) for j, t in enumerate(z)])
            offs = [b for _, b in row_bounds[-1]]
        nleaves = len(zs[0])
        nsets = len(opss[0])
        leaves = [torch.cat([z[j] for z in zs]).detach().requires_grad_(True) for j in range(nleaves)]
        ops_all = tuple((torch.cat([o[j][0] for o in opss]), torch.cat([o[j][1] for o in opss]))
                        for j in range(nsets))
        del zs, opss
        temp_leaf = temperature.detach().requires_grad_(True)
        bias_leaf = None if logit_bias is None else logit_bias.detach().requires_grad_(True)
        cl_w = 1.0
        if aux is not None:
            cl_w = 1 - (clip.text_ssl_loss_weight + clip.image_ssl_loss_weight)
        filip_stats = {} if filip else None
        with torch.enable_grad():
            if filip:
                from .filip import FilipLossFn
                loss = FilipLossFn.apply(
                    leaves[0], leaves[1], leaves[2] if nsets == 4 else None,
                    leaves[3] if nsets == 4 else None, temp_leaf, ops_all, text_mask.contiguous(),
                    clip.decoupled_contrastive_learning, clip.requires_all_gather, filip_stats)
            elif bias_leaf is not None:
                loss = SigmoidLossFn.apply(leaves[0], leaves[1], temp_leaf, bias_leaf, ops_all,
                                           clip.requires_all_gather)
            else:
                loss = ContrastiveLossFn.apply(
                    leaves[0], leaves[1], leaves[2] if nsets == 4 else None,
                    leaves[3] if nsets == 4 else None, temp_leaf, ops_all,
                    clip.decoupled_contrastive_learning, clip.requires_all_gather,
                    *((clip.sim_reg_loss_weight, cl_w) if clip.has_sim_reg_loss else ()))
            if aux is not None:
                if not (clip.has_sim_reg_loss and not filip):      # sim-reg weighs its contrastive term itself
                    loss = loss * cl_w
                mlm_loss, ssl_loss = _aux_losses(clip, aux, leaves[nsets:], targets)
                if mlm_loss is not None:
                    loss = loss + mlm_loss * clip.text_ssl_loss_weight
                if ssl_loss is not None:
                    loss = loss + ssl_loss * clip.image_ssl_loss_weight
        del targets
        ctx.clip, ctx.inputs = clip, (text, image, text_mask)
        ctx.bounds, ctx.rng_states, ctx.kept = bounds, rng_states, kept
        ctx.aux, ctx.row_bounds = aux, row_bounds
        ctx.img_leaves = img_leaves if want_dimage else None
        ctx.graph = (loss, leaves, temp_leaf, bias_leaf)
        ctx.weight_casts = wscope.cache
        n_kept = sum(z is not None for z in kept)
        if planned or (oom_fallbacks and plan_key in plans):
            plans[plan_key] = [z is not None for z in kept]    # WHICH chunks stay resident
        passes = ["contrastive"]
        if aux is not None:
            passes += (["mlm"] if aux["mlm"] is not None else []) + (["view1", "view2"] if aux["ssl"] is not None else [])
        clip.last_step_plan = dict(chunks=len(bounds), retained=n_kept, chunk_activation_bytes=foot,
                                   oom_fallbacks=oom_fallbacks, passes=passes,
                                   retained_chunks=[k for k, z in enumerate(kept) if z is not None])
        if filip:
            # rows of both FILIP passes whose argmax was saved / will be recomputed in backward
            clip.last_step_plan.update(filip=filip_stats, loss_reserve_bytes=reserve)
        return loss.detach()

    @staticmethod
    def backward(ctx, g):
        clip = ctx.clip
        text, image, text_mask = ctx.inputs
        loss, leaves, temp_leaf, bias_leaf = ctx.graph
        with torch.enable_grad():
            torch.autograd.backward(loss, g)
        dz = [l.grad for l in leaves]
        dev = text.device
        keep_state = torch.cuda.get_rng_state(dev)
        kept = ctx.kept
        dimage = torch.empty_like(image) if ctx.img_leaves is not None else None
        # retained chunks first: their backward releases HBM before any chunk is re-encoded
        order = [k for k in range(len(ctx.bounds)) if kept[k] is not None] + \
                [k for k in range(len(ctx.bounds)) if kept[k] is None]
        with weight_scope(ctx.weight_casts):
            for pos, k in enumerate(order):
                s, e = ctx.bounds[k]
                # parameter gradients accumulate over the chunks; gradient-sync hooks (GradSync)
                # must see a parameter ONCE per step, with its complete gradient: every chunk but
                # the last one processed runs with the hooks deferred (the DDP no_sync convention)
                with torch.enable_grad(), D_.defer_grad_sync(pos != len(order) - 1), \
                        _InPlaceGradAccumulation(INPLACE_GRAD_ACCUMULATION and pos != len(order) - 1):
                    img_k = None
                    if kept[k] is not None:
                        z, kept[k] = kept[k], None
                        if dimage is not None:
                            img_k, ctx.img_leaves[k] = ctx.img_leaves[k], None
                    else:
                        torch.cuda.set_rng_state(ctx.rng_states[k], dev)
                        if dimage is not None:
                            img_k = image[s:e].detach().requires_grad_(True)
                        z, _ = _chunk_passes(clip, text, image, text_mask, ctx.aux, s, e, img_k)
                    # accumulates into .grad; an output with no gradient or no rows in this chunk is skipped
                    pairs = [(t, dz[j][a:b]) for j, (t, (a, b)) in enumerate(zip(z, ctx.row_bounds[k]))
                             if dz[j] is not None and b > a and t.requires_grad]
                    if pairs:
                        torch.autograd.backward([t for t, _ in pairs], [d for _, d in pairs])
                    del z, pairs
                    if img_k is not None:
                        if img_k.grad is None:
                            dimage[s:e].zero_()
                        else:
                            dimage[s:e].copy_(img_k.grad)
                        del img_k
        torch.cuda.set_rng_state(keep_state, dev)
        ctx.graph = ctx.inputs = ctx.kept = ctx.weight_casts = ctx.img_leaves = ctx.aux = None
        grads = (None, None, dimage, None, None, temp_leaf.grad, None, None,
                 None if bias_leaf is None else bias_leaf.grad)
        return grads[:len(ctx.needs_input_grad)]
