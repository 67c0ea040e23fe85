"""Per-call fp64 checks of the kernel wrappers (x_clip_b200.kernels) at the shapes a whole training step
really runs.  TEST INFRASTRUCTURE ONLY.

`Recorder` replaces every public wrapper of `kernels` by a spy.  The first call of each distinct
signature (the wrapper's name plus the shape, dtype and strides of every tensor argument and the value
of every other argument: majors, accumulate, bias / residual mode, causal, mask, dropout, want_xn,
need_u, ...) runs the real call, is checked against an fp64 reference computed on the GPU in row
chunks, and prints `GATE <wrapper>[<signature>]<output> <ratio>`; later calls of the signature run
unchecked.  Buffers a call writes in place or accumulates into are cloned before it runs, so the
reference starts from what the kernel started from.  Every wrapper that launches a kernel has an entry
in CHECKS and every variant of it is checked; a call of a wrapper with no entry is counted in
`unchecked`.

The references are the existing oracles: gemm_oracle (gemm64, gemm_gate, text_embed_bwd64,
patchify64, adamw64), block_oracle (LayerNorm and feed-forward stages, rotate64), attn_oracle
(attn_ref64) with dropout_oracle's masks (drawn on the device), nce_oracle, sigmoid_oracle,
simreg_oracle and augment_oracle (augment64).  The per-element gates are theirs; the vocabulary
cross-entropy's are derived below from what its kernels compute.  Sums over the rows of a call - the
LayerNorm gain gradient dg, the feed-forward's vsum and dg4, the column sums (d bias, dpos, dcls) and
the scatter-adds (dtok, d pos table) - are gated at `n_add * 2^-24 * sum |terms|`, n_add the longest
chain of fp32 additions any term goes through in the kernel's launch: the sequential rows of one
thread or warp, the shared-memory and global atomics after it, and the prefill.  That gate grows
with the rows the way the kernel's error does, and stays far below what a dropped or doubled row
block would add.
"""
from __future__ import annotations

import inspect
import math
from collections import Counter

import torch

import attn_oracle as AO
import augment_oracle as AU
import block_oracle as BO
import dropout_oracle as DO
import gemm_oracle as GO
import nce_oracle as NO
import sigmoid_oracle as SG
import simreg_oracle as SR

U24 = 2.0 ** -24          # one fp32 addition, relative to the sum of |terms| it adds
ROWS = 4096               # rows per fp64 reference chunk
K_CHUNK = 8192            # columns of K converted to fp64 at a time by the GEMM reference
ATTN_TOKENS = 8192        # tokens per fp64 attention reference chunk
FLAT_CHUNK = 1 << 24      # elements per fp64 AdamW reference chunk
EXACT_FAIL = math.inf     # the ratio of a bit-exact output that differs

# host helpers of kernels.py: they compute a size or check an argument and launch nothing
HOST_HELPERS = {
    "patch_row_stride": "row stride arithmetic, no launch",
    "check_arg16_seg_len": "argument check, no launch",
}


def sms() -> int:
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def public_wrappers(K) -> list:
    """Names of the public functions defined in the kernels module (host helpers included)."""
    return sorted(n for n, f in vars(K).items()
                  if inspect.isfunction(f) and f.__module__ == K.__name__ and not n.startswith("_"))


# --------------------------------------------------------------------------- reduction gates

def red_gate(abs_terms, n_add):
    """n_add fp32 additions in the longest chain, relative to the sum of |terms| (prefill included)."""
    return n_add * U24 * abs_terms


def adds_row_grid(rows: int, cap_blocks: int, warps: int = 8) -> int:
    """Column sums of a grid-stride row kernel (LayerNorm backward dg, ff_bwd_prep vsum): each lane adds
    its rows in sequence, then one shared-memory atomic per warp of the block, one global atomic per
    block, onto the prefill.  grid = min(ceil(rows / warps), cap_blocks)."""
    grid = max(1, min(-(-rows // warps), cap_blocks))
    return -(-rows // (grid * warps)) + warps + grid + 1


def adds_ln_dg(rows: int) -> int:
    return adds_row_grid(rows, 2 * sms())          # xclip_layernorm_bwd_xn: 2 blocks per SM


def adds_vsum(rows: int) -> int:
    return adds_row_grid(rows, 4 * sms())          # xclip_ff_bwd_prep: 4 blocks per SM


def adds_colsum(rows: int) -> int:
    """colsum_rows_: min(rows, 256) row slices summed in sequence, one atomic per slice."""
    slices = max(1, min(rows, 256))
    return -(-rows // slices) + slices + 1


def adds_text_colsum(B: int, n: int, d: int) -> int:
    """text_embed_bwd dpos / dcls: bsplit batch slices summed in sequence, one atomic per slice."""
    bs = GO.text_embed_bsplit(B, n, d, sms())
    return -(-B // bs) + bs + 1


def adds_scatter(rows_idx: torch.Tensor, V: int) -> torch.Tensor:
    """Scatter-adds (red.add per source row): a table row hit h times adds h terms onto its prefill."""
    return (torch.bincount(rows_idx, minlength=V) + 1).double()[:, None]


def adds_dg4(d: int) -> int:
    """ff_w2_grad_post_ dg: 8 rows of W2 per thread in sequence, one atomic per 8-row block."""
    return 8 + -(-d // 8) + 1


# --------------------------------------------------------------------------- helpers

class Worst(dict):
    def add(self, key, ratio):
        self[key] = max(self.get(key, 0.0), float(ratio))


def exact(got, ref) -> float:
    return 0.0 if torch.equal(got, ref) else EXACT_FAIL


def _chunks(n, step=ROWS):
    for r0 in range(0, n, step):
        yield r0, min(n, r0 + step)


# --------------------------------------------------------------------------- GEMM

def gemm_rows(a, b, a_major, b_major):
    M, K = a.shape if a_major == 0 else a.shape[::-1]
    N = b.shape[0] if b_major == 0 else b.shape[1]
    return M, N, K


def gemm_ratio(a, b, a_major, b_major, got, alpha=1.0, bias=None, residual=None, res_rows=None, prefill=None,
               plan=None) -> float:
    """Largest |got - ref| / gemm_gate over the output, the fp64 reference in row chunks, the
    accumulation term the larger of GAMMA S and the chain bound of the split plan's k-block chains."""
    M, N, K = gemm_rows(a, b, a_major, b_major)
    splits, ranges = (1, None) if plan is None else (plan["splits"], GO.split_ranges(plan))
    ratio = 0.0
    for r0, r1 in _chunks(M):
        ac = a[r0:r1] if a_major == 0 else a[:, r0:r1]
        acc, S, P = GO.chain_sums64(ac, b, a_major, b_major, ranges, K_CHUNK)
        sl = dict(bias=bias, residual=residual, res_rows=None if res_rows is None else res_rows[r0:r1],
                  prefill=None if prefill is None else prefill[r0:r1])
        ref = alpha * acc
        del acc
        if bias is not None:
            ref = ref + bias.double()
        if residual is not None:
            ref = ref + residual.double()[sl["res_rows"]]
        if prefill is not None:
            ref = ref + sl["prefill"].double()
        gate = GO.gemm_gate(ac, b, a_major, b_major, alpha, **sl, bf16_out=got.dtype == torch.bfloat16,
                            splits=splits, ref=ref, S=S, P=P)
        ratio = max(ratio, BO.gate_ratio(got[r0:r1], ref, gate))
    return ratio


def _res_rows(A, M, dev):
    if A["residual"] is None:
        return None
    if A["res_row_idx"] is not None:
        return A["res_row_idx"].long()
    if A["res_row_mod"] > 0:
        return torch.arange(M, device=dev) % A["res_row_mod"]
    return torch.arange(M, device=dev)


def check_gemm(A, before, out):
    a, b, am, bm = A["a"], A["b"], A["a_major"], A["b_major"]
    M, N, K = gemm_rows(a, b, am, bm)
    acc = A["accumulate"]
    plan = GO.split_plan(M, N, K, acc, sms())
    return {"": gemm_ratio(a, b, am, bm, out, A["alpha"], A["bias"], A["residual"], _res_rows(A, M, a.device),
                           before.get("out") if acc else None, plan)}


def cast_check(A, before, out):
    return {"": exact(out, A["src"].contiguous().bfloat16())}


# --------------------------------------------------------------------------- LayerNorm

def check_ln_fwd(A, before, res):
    out, stats, out2, stats2 = res
    x, g, r, g2, eps = A["x"], A["g"], A["res"], A["g2"], A["eps"]
    w = Worst()
    for r0, r1 in _chunks(x.shape[0]):
        mean, rstd = BO.ln_stats64(x[r0:r1], eps)
        if stats is not None:
            w.add("mean", BO.gate_ratio(stats[r0:r1, 0], mean, BO.STAT_REL * (mean.abs() + 1 / rstd)))
            w.add("rstd", BO.gate_ratio(stats[r0:r1, 1], rstd, BO.STAT_REL * rstd))
        ref = (x[r0:r1].double() - mean[:, None]) * rstd[:, None] * g.double()
        if r is not None:
            ref = ref + r[r0:r1].double()
        w.add("out", BO.gate_ratio(out[r0:r1], ref, BO.elem_gate(ref)))
        if g2 is not None:
            mean2, rstd2 = BO.ln_stats64(out[r0:r1], eps)          # the second norm reads bf16 out
            w.add("mean2", BO.gate_ratio(stats2[r0:r1, 0], mean2, BO.STAT_REL * (mean2.abs() + 1 / rstd2)))
            w.add("rstd2", BO.gate_ratio(stats2[r0:r1, 1], rstd2, BO.STAT_REL * rstd2))
            ref2 = (out[r0:r1].double() - mean2[:, None]) * rstd2[:, None] * g2.double()
            w.add("out2", BO.gate_ratio(out2[r0:r1], ref2, BO.elem_gate(ref2)))
    return w


def check_ln_bwd(A, before, res):
    dy, x, stats, g, add, dg = A["dy"], A["x"], A["stats"], A["g"], A["add"], A["dg"]
    dx, xn = res if A["want_xn"] else (res, None)
    rows = x.shape[0]
    w = Worst()
    dg_sum = dg_abs = 0.0
    for r0, r1 in _chunks(rows):
        st = stats[r0:r1]
        dx_ref, dg_c, _, _ = BO.ln_bwd64(dy[r0:r1], x[r0:r1], st[:, 0], st[:, 1], g)
        if add is not None:
            dx_ref = dx_ref + add[r0:r1].double()
        w.add("dx", BO.gate_ratio(dx[r0:r1], dx_ref, BO.elem_gate(dx_ref)))
        xh = (x[r0:r1].double() - st[:, 0].double()[:, None]) * st[:, 1].double()[:, None]
        if xn is not None:
            ref = xh * g.double()
            w.add("xn", BO.gate_ratio(xn[r0:r1], ref, BO.elem_gate(ref)))
        if dg is not None:
            dg_sum = dg_sum + dg_c
            dg_abs = dg_abs + (dy[r0:r1].double() * xh).abs().sum(0)
    if dg is not None:
        d0 = before["dg"].double()
        w.add("dg", BO.gate_ratio(dg, d0 + dg_sum, red_gate(d0.abs() + dg_abs, adds_ln_dg(rows))))
    return w


# --------------------------------------------------------------------------- fused feed-forward

def check_ff_weights(A, before, res):
    w1p, w2g, colvec = res
    w = Worst()
    w.add("w1p", exact(w1p, BO.ff_permute(A["w1"].contiguous().bfloat16())))
    w.add("w2g", exact(w2g, (A["w2"] * A["g4"]).bfloat16()))
    w.add("colvec", BO.gate_ratio(colvec, w2g.double().sum(1), BO.RED_REL * w2g.double().abs().sum(1)))
    return w


def check_ff_up(A, before, res):
    u, hp, rowsum = res
    x, w1 = A["x"], BO.ff_unpermute(A["w1p"]).double()
    M, d = x.shape
    D4 = 4 * d
    w = Worst()
    for r0, r1 in _chunks(M):
        u_ref = x[r0:r1].double() @ w1.t()
        if u is not None:
            ur = u_ref.view(-1, 2, D4)
            w.add("u", BO.gate_ratio(u[r0:r1].view(-1, 2, D4), ur, BO.elem_gate(ur)))
        hp_ref = u_ref[:, :D4] * BO.gelu64(u_ref[:, D4:])
        del u_ref
        w.add("hp", BO.gate_ratio(hp[r0:r1], hp_ref, BO.elem_gate(hp_ref)))
        box = hp[r0:r1].double().view(r1 - r0, -1, 64)
        box_abs = torch.stack([box.abs().sum(-1), (box * box).sum(-1)], -1)
        w.add("rowsum", BO.gate_ratio(rowsum[r0:r1], BO.ff_rowsum64(hp[r0:r1]), BO.RED_REL * box_abs))
    return w


def check_ff_down(A, before, res):
    out, acc, stats = res
    hp, w2g, colvec, r = A["hp"], A["w2g"], A["colvec"], A["res"]
    w = Worst()
    for r0, r1 in _chunks(hp.shape[0]):
        mean, rstd = BO.ln_stats64(hp[r0:r1], A["eps"])
        st = stats[r0:r1]
        w.add("mean", BO.gate_ratio(st[:, 0], mean, BO.STAT_REL * (mean.abs() + 1 / rstd)))
        w.add("rstd", BO.gate_ratio(st[:, 1], rstd, BO.STAT_REL * rstd))
        x2_ref, acc_ref, _ = BO.ff_down64(hp[r0:r1], w2g, colvec, st[:, 0], st[:, 1], r[r0:r1])
        w.add("x2", BO.gate_ratio(out[r0:r1], x2_ref, BO.elem_gate(x2_ref)))
        w.add("acc", BO.gate_ratio(acc[r0:r1], acc_ref, BO.elem_gate(acc_ref)))
    return w


def check_ff_bwd_prep(A, before, res):
    dxs, vsum, ab = res
    dx, stats, acc, colvec = A["dx"], A["stats"], A["acc"], A["colvec"]
    M, d = dx.shape
    w = Worst()
    w.add("dxs", exact(dxs, (dx.float() * stats[:, 1:2]).bfloat16()))
    v_sum = v_abs = 0.0
    for r0, r1 in _chunks(M):
        st = stats[r0:r1]
        terms = dxs[r0:r1].double() * st[:, :1].double()
        v_sum, v_abs = v_sum + terms.sum(0), v_abs + terms.abs().sum(0)
        if ab is not None:
            dxc = dx[r0:r1]
            a_ref, b_ref = BO.ff_ab64(dxc, acc[r0:r1], colvec, st[:, 0], st[:, 1], 4 * d)
            a_scale = (dxc.double().abs() @ colvec.double().abs()) / (4 * d)
            b_scale = st[:, 1].double() * ((dxc.double() * acc[r0:r1].double()).abs().sum(1) / (4 * d)
                                           + st[:, 0].double().abs() * a_scale)
            w.add("a", BO.gate_ratio(ab[r0:r1, 0], a_ref, BO.RED_REL * a_scale))
            w.add("b", BO.gate_ratio(ab[r0:r1, 1], b_ref, BO.RED_REL * b_scale))
    w.add("vsum", BO.gate_ratio(vsum, v_sum, red_gate(v_abs, adds_vsum(M))))
    return w


def check_ff_bwd(A, before, du):
    dx, w2g, u, stats, ab = A["dx"], A["w2g"], A["u"], A["stats"], A["ab"]
    D4 = 4 * dx.shape[1]
    w = Worst()
    for r0, r1 in _chunks(dx.shape[0]):
        st, abc = stats[r0:r1], ab[r0:r1]
        ref = BO.ff_bwd64(dx[r0:r1], w2g, u[r0:r1], st[:, 0], st[:, 1], abc[:, 0], abc[:, 1]).view(-1, 2, D4)
        w.add("du", BO.gate_ratio(du[r0:r1].view(-1, 2, D4), ref, BO.elem_gate(ref)))
    return w


def check_ff_w2_grad_post(A, before, raw):
    raw0, vsum, g4 = before["raw"], A["vsum"], A["g4"]
    w = Worst()
    w.add("dw2", exact(raw, g4 * (raw0 - vsum[:, None])))
    if A["dg"] is not None:
        tt = (raw0.double() - vsum.double()[:, None]) * A["w2"].double()
        d0 = before["dg"].double()
        w.add("dg4", BO.gate_ratio(A["dg"], d0 + tt.sum(0), red_gate(tt.abs().sum(0) + d0.abs(),
                                                                       adds_dg4(raw.shape[0]))))
    return w


# --------------------------------------------------------------------------- attention, rotary

def _attn_slices(A):
    B, n = A["B"], A["n"]
    per = max(1, ATTN_TOKENS // n)
    for b0 in range(0, B, per):
        b1 = min(B, b0 + per)
        mk = None if A["key_mask"] is None else A["key_mask"][b0:b1]
        yield b0, b1, slice(b0 * n, b1 * n), mk


def _attn_ref(A, b0, b1, rows, mk, bwd):
    """attn_oracle's fp64 reference of batch items [b0, b1), or with dropout dropout_oracle's, fed the
    mask of the call's seed and layer drawn on the device (dropout_oracle.attn_drop_mul_torch)."""
    qkv, n, H = A["qkv"][rows], A["n"], A["heads"]
    o, d_o = (A["o"][rows], A["d_o"][rows]) if bwd else (None, None)
    if A["dropout"] is None:
        return AO.attn_ref64(qkv, mk, b1 - b0, n, H, A["scale"], A["causal"], o=o, d_o=d_o)
    p, seed, layer = A["dropout"]
    drop = DO.attn_drop_mul_torch(int(seed.item()), b0, b1, H, n, layer, p, qkv.device)
    return DO._attn_chunk64(qkv, mk, b1 - b0, n, H, A["scale"], A["causal"], o, d_o, drop)


def check_attn_fwd(A, before, res):
    o, lse = res
    w = Worst()
    for b0, b1, rows, mk in _attn_slices(A):
        r = _attn_ref(A, b0, b1, rows, mk, False)
        w.add("o", BO.gate_ratio(o[rows], r["o"], r["g_o"]))
        w.add("lse", BO.gate_ratio(lse[b0:b1], r["lse"], r["g_lse"]))
    return w


def check_attn_bwd(A, before, dqkv):
    w = Worst()
    for b0, b1, rows, mk in _attn_slices(A):
        r = _attn_ref(A, b0, b1, rows, mk, True)
        w.add("dqkv", BO.gate_ratio(dqkv[rows], r["dqkv"], r["g_dqkv"]))
    return w


def check_rotary(A, before, qkv):
    n, ns = A["n"], A["nslices"]
    w = Worst()
    w.add("rest", exact(qkv[:, ns * 64:], before["qkv"][:, ns * 64:]))
    for r0, r1 in _chunks(qkv.shape[0], ROWS // n * n or n):
        ref = BO.rotate64(before["qkv"][r0:r1, :ns * 64], A["cos_tab"], A["sin_tab"], A["inverse"])
        w.add("qkv", BO.gate_ratio(qkv[r0:r1, :ns * 64], ref, BO.elem_gate(ref)))
    return w


# --------------------------------------------------------------------------- latents and loss

def l2norm_gates(d):
    """Relative error of inv = rsqrt(sum p^2): the fp32 sum of squares (d / 32 per lane, a 5-level
    shuffle tree) and rsqrtf (2 ulp), with 2x headroom."""
    return (d // 32 + 8) * U24


def check_l2norm_fwd(A, before, res):
    z, zrow, zcol, inv = res
    p = A["p"]
    d = p.shape[1]
    rel = l2norm_gates(d)
    w = Worst()
    hi, lo = zrow[:, :d], zrow[:, d:2 * d]
    w.add("layout", max(exact(zrow[:, 2 * d:], hi), exact(zcol[:, :2 * d], hi.repeat(1, 2)), exact(zcol[:, 2 * d:], lo)))
    for r0, r1 in _chunks(p.shape[0]):
        p64 = p[r0:r1].double()
        nrm = p64.norm(dim=1)
        z_ref = p64 / nrm[:, None]
        w.add("inv", BO.gate_ratio(inv[r0:r1], 1.0 / nrm, rel / nrm))
        zg = (rel + U24) * z_ref.abs() + 2.0 ** -40
        w.add("z", BO.gate_ratio(z[r0:r1], z_ref, zg))
        # split bf16: hi + lo keeps 16 bits of z
        w.add("hi_lo", BO.gate_ratio(hi[r0:r1].double() + lo[r0:r1].double(), z_ref, zg + 2.0 ** -16 * z_ref.abs()))
    return w


def check_l2norm_bwd(A, before, dp):
    dz, z, inv = A["dz"], A["z"], A["inv"]
    d = z.shape[1]
    w = Worst()
    for r0, r1 in _chunks(z.shape[0]):
        z64, dz64, i64 = z[r0:r1].double(), dz[r0:r1].double(), inv[r0:r1].double()[:, None]
        s = (z64 * dz64).sum(1, keepdim=True)
        ref = i64 * (dz64 - z64 * s)
        sabs = (z64 * dz64).abs().sum(1, keepdim=True)
        gate = (BO.elem_gate(ref) + i64 * z64.abs() * l2norm_gates(d) * sabs
                + 2.0 ** -23 * i64 * (dz64.abs() + z64.abs() * s.abs()))
        w.add("dp", BO.gate_ratio(dp[r0:r1], ref, gate))
    return w


def _logits(a, b, temp, r0, r1):
    return temp * (a[r0:r1].double() @ b.double().t())


NCE_ROWS = 2048


def _loss_sum_ratio(loss, before, scale, terms_sum, terms_abs, term_gates, n_add):
    """A fused loss sum loss_accum += scale * sum(terms): the terms' own gates scaled, plus n_add fp32
    additions of the sum of |terms| and of the prefill."""
    l0 = before["loss_accum"].double().item()
    gate = abs(scale) * term_gates + n_add * U24 * (abs(l0) + abs(scale) * terms_abs)
    return abs(loss.double().item() - (l0 + scale * terms_sum)) / gate


def check_nce_fwd(A, before, res):
    lse, pos = res
    a, b, off, dcl = A["a"], A["b"], A["diag_offset"], A["dcl"]
    temp = A["temp_exp"].double().item()
    w = Worst()
    t_sum = t_abs = t_gate = 0.0
    for r0, r1 in _chunks(a.shape[0], NCE_ROWS):
        ref_lse, ref_pos = NO.ref_rows(_logits(a, b, temp, r0, r1), off + r0, dcl)
        g_lse, g_pos = NO.lse_gate(temp, ref_lse), torch.full_like(ref_pos, temp * NO.LOGIT_GATE)
        w.add("lse", BO.gate_ratio(lse[r0:r1], ref_lse, g_lse))
        w.add("pos", BO.gate_ratio(pos[r0:r1], ref_pos, g_pos))
        t = ref_lse - ref_pos
        t_sum, t_abs, t_gate = t_sum + t.sum().item(), t_abs + t.abs().sum().item(), t_gate + (g_lse + g_pos).sum().item()
    if A["loss_accum"] is not None:
        w.add("loss", _loss_sum_ratio(A["loss_accum"], before, A["loss_scale"], t_sum, t_abs, t_gate, a.shape[0]))
    return w


def check_nce_bwd(A, before, g):
    a, b, off, dcl = A["a"], A["b"], A["diag_offset"], A["dcl"]
    temp = A["temp_exp"].double().item()
    gs = A["gscale"].double().item()
    wts = (A["w_row"], A["w_col"], A["w_diag"])
    lse_row, lse_col = A["lse_row"], A["lse_col"]
    w = Worst()
    sum_gs = abs_gs = abs_g = 0.0
    R, C = a.shape[0], b.shape[0]
    for r0, r1 in _chunks(R, NCE_ROWS):
        err, s1, s2, s3 = NO.check_bwd_rows(g[r0:r1], _logits(a, b, temp, r0, r1), off + r0, dcl,
                                            None if lse_row is None else lse_row[r0:r1], lse_col, wts, gs, temp)
        w.add("g", err)
        sum_gs, abs_gs, abs_g = sum_gs + s1, abs_gs + s2, abs_g + s3
    if A["dtemp"] is not None:
        d0 = before["dtemp"].double().item()
        gate = NO.dtemp_gate(temp, abs_gs, abs_g, R, C) + 2.0 ** -23 * abs(d0)
        w.add("dtemp", abs(A["dtemp"].double().item() - (d0 + sum_gs)) / gate)
    return w


# --------------------------------------------------------------------------- embeddings

def check_text_embed_fwd(A, before, out):
    ids, tok, pos, cls = A["ids"], A["tok"], A["pos"], A["cls"]
    B, n = ids.shape
    w = Worst()
    w.add("cls", exact(out[:, 0], cls.bfloat16().expand(B, -1)))
    for b0, b1 in _chunks(B, max(1, ROWS // n)):
        w.add("tok", exact(out[b0:b1, 1:], (tok[ids[b0:b1]] + pos[:n]).bfloat16()))
    return w


def check_text_embed_bwd(A, before, res):
    dtok, dpos, dcls = res
    ids, dx, vocab, pos_rows = A["ids"], A["dx"], A["vocab"], A["pos_rows"]
    B, n = ids.shape
    d = dx.shape[-1]
    (rtok, atok), (rpos, apos), (rcls, acls) = GO.text_embed_bwd64(ids, dx, vocab, pos_rows)
    w = Worst()
    w.add("dtok", BO.gate_ratio(dtok, rtok, red_gate(atok, adds_scatter(ids.reshape(-1), vocab))))
    n_add = adds_text_colsum(B, n, d)
    w.add("dpos", BO.gate_ratio(dpos, rpos, red_gate(apos, n_add)))
    w.add("dcls", BO.gate_ratio(dcls, rcls, red_gate(acls, n_add)))
    return w


def check_patchify_gather(A, before, out):
    img, p, keep, ld = A["img"], A["patch"], A["keep"], A["ld"]
    B = img.shape[0]
    w = Worst()
    for b0, b1 in _chunks(B, 256):
        ref = GO.patchify64(img[b0:b1].contiguous(), p)
        if keep is not None:
            ref = torch.gather(ref, 1, keep[b0:b1, :, None].expand(-1, -1, ref.shape[2]))
        k, pd = ref.shape[1], ref.shape[2]
        got = out[b0 * k:b1 * k]
        w.add("rows", exact(got[:, :pd], ref.reshape(-1, pd).bfloat16()))
        if ld is not None and ld > pd:
            w.add("pad", exact(got[:, pd:], torch.zeros_like(got[:, pd:])))
    return w


def check_scatter_add_rows(A, before, dst):
    src, idx, period = A["src"], A["idx"], A["period"]
    rows = idx.long() if idx is not None else torch.arange(src.shape[0], device=src.device) % period
    d0 = before["dst"].double()
    s = src.double()
    ref = d0.index_add(0, rows, s)
    ab = d0.abs().index_add(0, rows, s.abs())
    return {"dst": BO.gate_ratio(dst, ref, red_gate(ab, adds_scatter(rows, dst.shape[0])))}


def check_colsum_rows(A, before, dst):
    src = A["src"]
    d0 = before["dst"].double()
    s_sum = s_abs = 0.0
    for r0, r1 in _chunks(src.shape[0]):
        s = src[r0:r1].double()
        s_sum, s_abs = s_sum + s.sum(0), s_abs + s.abs().sum(0)
    return {"dst": BO.gate_ratio(dst, d0 + s_sum, red_gate(d0.abs() + s_abs, adds_colsum(src.shape[0])))}


# --------------------------------------------------------------------------- optimizer

def check_adamw(A, before, _):
    w = Worst()
    hp = [A[k] for k in ("lr", "beta1", "beta2", "eps", "weight_decay", "step", "grad_scale")]
    for i0, i1 in _chunks(A["p"].numel(), FLAT_CHUNK):
        rp, rm, rv, gp, gm, gv = GO.adamw64(before["p"][i0:i1], A["g"][i0:i1], before["m"][i0:i1],
                                            before["v"][i0:i1], *hp)
        w.add("p", BO.gate_ratio(A["p"][i0:i1], rp, gp))
        w.add("m", BO.gate_ratio(A["m"][i0:i1], rm, gm))
        w.add("v", BO.gate_ratio(A["v"][i0:i1], rv, gv))
    return w


# --------------------------------------------------------------------------- FILIP
# Gates of test_gpu_filip.py: segment maxima within 2^-16 temp of fp64 (the split-bf16 product), the
# fp64 similarity at the returned index within the same of the maximum (near-ties may pick either);
# lse 1e-6 |ref| + 4e-6 and g gscale (2e-5 p + 2e-6); the weighted token sums of filip_reduce at their
# fp32 chain, one addition per token.

SEGMAX_GATE = 2.0 ** -16


def check_filip_segmax16(A, before, res):
    seg_max, seg_arg = res
    a, b, seg_len = A["a"], A["b"], A["seg_len"]
    temp = A["temp_exp"].double().item()
    col_mul, col_add = A["col_mul"], A["col_add"]
    R, C = a.shape[0], b.shape[0]
    nseg = C // seg_len
    gate = SEGMAX_GATE * temp
    w = Worst()
    for r0, r1 in _chunks(R, max(1, (1 << 24) // C)):
        s = _logits(a, b, temp, r0, r1)
        if col_mul is not None:
            s = s * col_mul.double() + col_add.double()
        s = s.view(r1 - r0, nseg, seg_len)
        ref = s.amax(-1)
        if seg_max is not None:
            w.add("max", (seg_max[r0:r1].double() - ref).abs().max().item() / gate)
        if seg_arg is not None:
            arg = (seg_arg[r0:r1].to(torch.int32) & 0xFFFF).long()
            w.add("arg_range", 0.0 if bool((arg < seg_len).all()) else EXACT_FAIL)
            at = s.gather(-1, arg.clamp_max(seg_len - 1).unsqueeze(-1)).squeeze(-1)
            w.add("arg", (ref - at).abs().max().item() / gate)
    return w


def check_filip_reduce(A, before, out):
    m, wts, samples, length, nseg = A["seg_max"], A["weights"], A["samples"], A["length"], A["nseg"]
    valid = (wts != 0)[:, None]
    mv = torch.where(valid, m, torch.zeros_like(m)).double()          # zero-weight rows are skipped
    terms = (wts.double()[:, None] * mv).view(samples, length, nseg)
    ref, scale = terms.sum(1), terms.abs().sum(1)
    if A["transpose"]:
        ref, scale = ref.t(), scale.t()
    return {"out": BO.gate_ratio(out, ref, red_gate(scale, length + 1))}


def _filip_rows(s, off, dcl, row_valid):
    R = s.shape[0]
    rows = torch.arange(R, device=s.device)
    s64 = s.double()
    lse_in = s64.clone()
    if dcl:
        lse_in[rows, rows + off] = -math.inf
    valid = torch.ones(R, dtype=torch.bool, device=s.device) if row_valid is None else row_valid
    return rows, s64, lse_in, valid


def check_filip_nce_fwd(A, before, lse):
    s, off, dcl, loss, scale = A["s"], A["diag_off"], A["dcl"], A["loss_accum"], A["loss_scale"]
    rows, s64, lse_in, valid = _filip_rows(s, off, dcl, A["row_valid"])
    ref = torch.logsumexp(lse_in, dim=1)
    gate = 1e-6 * ref.abs() + 4e-6
    w = Worst()
    w.add("lse", ((lse.double() - ref).abs() / gate)[valid].max().item() if bool(valid.any()) else 0.0)
    w.add("lse_invalid", exact(lse[~valid], torch.zeros_like(lse[~valid])))
    if loss is not None:
        terms = scale * (ref - s64[rows, rows + off])[valid]
        l0 = before["loss_accum"].double().item()
        lg = abs(scale) * gate[valid].sum().item() + s.shape[0] * U24 * (abs(l0) + terms.abs().sum().item())
        w.add("loss", abs(loss.double().item() - (l0 + terms.sum().item())) / lg)
    return w


def check_filip_nce_bwd(A, before, g):
    s, off, dcl = A["s"], A["diag_off"], A["dcl"]
    gs = A["gscale"].double().item()
    rows, s64, lse_in, valid = _filip_rows(s, off, dcl, A["row_valid"])
    ref_lse = torch.logsumexp(lse_in, dim=1)
    p = torch.exp(lse_in - ref_lse[:, None])
    ref = gs * p
    ref[rows, rows + off] -= gs
    gate = gs * (2e-5 * p + 2e-6)
    w = Worst()
    w.add("g", ((g.double() - ref).abs() / gate)[valid].max().item() if bool(valid.any()) else 0.0)
    w.add("g_invalid", exact(g[~valid], torch.zeros_like(g[~valid])))
    return w


def check_filip_expand16(A, before, g):
    seg_arg, wmat, rowscale, alpha = A["seg_arg"], A["wmat"], A["rowscale"], A["temp_exp"]
    row0, rps, seg_len, nseg = A["row0"], A["rows_per_sample"], A["seg_len"], A["nseg"]
    rows = seg_arg.shape[0]
    r = torch.arange(row0, row0 + rows, device=g.device)
    wv = wmat[r // rps] * rowscale[r][:, None]
    want = torch.zeros((rows, nseg * seg_len), device=g.device, dtype=torch.bfloat16)
    cols = torch.arange(nseg, device=g.device)[None, :] * seg_len + (seg_arg.to(torch.int32) & 0xFFFF).long()
    want.scatter_(1, cols, (wv * alpha).to(torch.bfloat16))
    return {"g": exact(g, want)}


def block_columns(n, b, B, col_run, j, device=None):
    """Columns of image view j's global samples k = 0 .. B-1 in a view-block matrix [m b, n B]:
    view-major (col_run = B) is n runs of all B samples; rank-major (col_run = b) is, per rank of b
    samples, that rank's n views in turn."""
    idx = torch.arange(n * B, device=device)
    if col_run == B:
        return idx.view(n, B)[j]
    assert col_run == b and B % b == 0, (col_run, b, B)
    return idx.view(B // b, n, b)[:, j, :].reshape(-1)


def _blocks_ref(A):
    """fp64 per (row, block): the lse over the block's columns (the positive left out under DCL, an
    empty DCL denominator ln(1e-20)), the positive's similarity, the block weight of the row, and
    p = exp(s - lse) over the block's columns.  -> (lse [R, n], pos [R, n], bw [R, n], [(cols, p)])."""
    s, m, n, col_run, off, dcl = A["s"], A["m"], A["n"], A["col_run"], A["diag_off"], A["dcl"]
    R, Ctot = s.shape
    b, B = R // m, Ctot // n
    rows = torch.arange(R, device=s.device)
    x = rows % b
    bw_all = A["block_w"].double().view(m, n)[rows // b]
    lse, pos, parts = [], [], []
    for j in range(n):
        cols = block_columns(n, b, B, col_run, j, s.device)
        sj = s[:, cols].double()
        pos.append(sj[rows, x + off])
        if dcl:
            sj[rows, x + off] = -math.inf
        lj = torch.logsumexp(sj, dim=1)
        if dcl:
            lj = torch.where(torch.isinf(lj) & (lj < 0), NO.LN_1E20, lj)
        lse.append(lj)
        parts.append((cols, torch.exp(sj - lj[:, None])))
    return torch.stack(lse, 1), torch.stack(pos, 1), bw_all, parts


def _row_valid_of(A, R, dev):
    rv = A["row_valid"]
    return torch.ones(R, dtype=torch.bool, device=dev) if rv is None else rv


def check_filip_nce_blocks_fwd(A, before, lse):
    s, loss = A["s"], A["loss_accum"]
    valid = _row_valid_of(A, s.shape[0], s.device)
    ref, pos, bw, _ = _blocks_ref(A)
    gate = 1e-6 * ref.abs() + 4e-6
    w = Worst()
    w.add("lse", ((lse.double() - ref).abs() / gate)[valid].max().item() if bool(valid.any()) else 0.0)
    if not bool(valid.all()):                 # rows without a valid token: lse 0 exactly
        w.add("lse_invalid", exact(lse[~valid], torch.zeros_like(lse[~valid])))
    if loss is not None:
        terms = (bw * (ref - pos))[valid]
        w.add("loss", _loss_sum_ratio(loss, before, 1.0, terms.sum().item(), terms.abs().sum().item(),
                                      (bw * gate)[valid].sum().item(), terms.numel()))
    return w


def check_filip_nce_blocks_bwd(A, before, g):
    s, off = A["s"], A["diag_off"]
    R = s.shape[0]
    b = R // A["m"]
    gs = A["gscale"].double().item()
    valid = _row_valid_of(A, R, s.device)
    _, _, bw, parts = _blocks_ref(A)
    rows = torch.arange(R, device=s.device)
    w = Worst()
    for j, (cols, p) in enumerate(parts):
        scale = gs * bw[:, j:j + 1]
        ref = scale * p
        ref[rows, rows % b + off] -= scale[:, 0]
        gate = scale.abs() * (2e-5 * p + 2e-6)
        err = ((g[:, cols].double() - ref).abs() / gate)[valid]
        w.add("g", err.max().item() if err.numel() else 0.0)
    if not bool(valid.all()):                 # rows without a valid token: g 0 exactly
        w.add("g_invalid", exact(g[~valid], torch.zeros_like(g[~valid])))
    return w


# --------------------------------------------------------------------------- sigmoid loss
# Gates of sigmoid_oracle (test_gpu_sigmoid_loss.py's): row losses ROW_REL relative, g G_REL relative
# where |l| < G_LIVE and exactly 0 where |l| > G_SATURATED, d temperature / d logit_bias SUM_REL of the
# sum of their terms' magnitudes.  The logits come from the bf16 operands the call received, so the
# split hi | lo product is the kernel's.

def _sig_rows(A, r0, r1):
    temp, bias = A["temp_exp"].double().item(), A["logit_bias"].double().item()
    l = _logits(A["a"], A["b"], temp, r0, r1) + bias
    z = SG.labels(r1 - r0, l.shape[1], A["diag_offset"] + r0, like=l)
    return l, z, temp, bias


def check_sigmoid_fwd(A, before, rowloss):
    w = Worst()
    total = 0.0
    for r0, r1 in _chunks(A["a"].shape[0], NCE_ROWS):
        l, z, _, _ = _sig_rows(A, r0, r1)
        ref = SG.softplus(-z * l).sum(1)
        w.add("rows", BO.gate_ratio(rowloss[r0:r1], ref, SG.ROW_REL * ref + 1e-30))
        total += ref.sum().item()
    if A["loss_accum"] is not None:
        l0, sc = before["loss_accum"].double().item(), A["loss_scale"]
        gate = SG.LOSS_REL * abs(sc) * total + 2.0 ** -23 * abs(l0) + 1e-30
        w.add("loss", abs(A["loss_accum"].double().item() - (l0 + sc * total)) / gate)
    return w


def check_sigmoid_bwd(A, before, g):
    gs = A["gscale"].double().item()
    C = A["b"].shape[0]
    w = Worst()
    w.add("pad", exact(g[:, C:], torch.zeros_like(g[:, C:])))
    dt = dt_abs = db = db_abs = 0.0
    for r0, r1 in _chunks(A["a"].shape[0], NCE_ROWS):
        l, z, temp, bias = _sig_rows(A, r0, r1)
        rg = gs * -z * torch.sigmoid(-z * l)                  # sigmoid(l) - [positive], no cancellation
        want = temp * rg
        gk = g[r0:r1, :C].double()
        live = l.abs() < SG.G_LIVE
        rel = (gk - want).abs()[live] / want.abs()[live]
        w.add("g", rel.max().item() / SG.G_REL if rel.numel() else 0.0)
        w.add("g_saturated", 0.0 if not bool(gk[l.abs() > SG.G_SATURATED].ne(0).any()) else EXACT_FAIL)
        t = rg * (l - bias)
        dt, dt_abs = dt + t.sum().item(), dt_abs + t.abs().sum().item()
        db, db_abs = db + rg.sum().item(), db_abs + rg.abs().sum().item()
    for name, val, mag in (("dtemp", dt, dt_abs), ("dbias", db, db_abs)):
        if A[name] is not None:
            d0 = before[name].double().item()
            gate = SG.SUM_REL * (mag + abs(d0)) + 1e-30
            w.add(name, abs(A[name].double().item() - (d0 + val)) / gate)
    return w


# --------------------------------------------------------------------------- vocabulary cross-entropy
# Per-element gates derived from what the kernels compute.  A logit l = x w^T + bias is an fp32
# accumulation at K = d: its error is within gemm_oracle.GAMMA of sum |x| |w| (the GEMM gate's
# accumulation term) plus one rounding of the bias add.  lse inherits the softmax-weighted logit error
# plus the fp32 log-sum-exp (nce_oracle.lse_gate's 2^-20 (1 + |lse|)); the target logit its own logit
# error.  g = bf16(gscale (exp(l - lse) - onehot)) with the call's lse: one bf16 rounding, plus
# gscale p times the logit's error, the fp32 rounding of l - lse and the exp approximation.

VCE_ROWS = 1024


def _vce_rows(A, r0, r1):
    x, wt, bias = A["x"][r0:r1].double(), A["w"].double(), A["bias"]
    l = x @ wt.t()
    e_l = GO.GAMMA * (x.abs() @ wt.abs().t())
    if bias is not None:
        l += bias.double()
    e_l += U24 * l.abs()
    return l, e_l


def check_vocab_ce_fwd(A, before, res):
    lse, pos = res
    labels = A["labels"]
    w = Worst()
    t_sum = t_abs = t_gate = 0.0
    for r0, r1 in _chunks(A["x"].shape[0], VCE_ROWS):
        l, e_l = _vce_rows(A, r0, r1)
        ref = torch.logsumexp(l, dim=1)
        g_lse = (torch.exp(l - ref[:, None]) * e_l).sum(1) + 2.0 ** -20 * (1.0 + ref.abs())
        lab = labels[r0:r1, None]
        ref_pos, g_pos = l.gather(1, lab)[:, 0], e_l.gather(1, lab)[:, 0]
        w.add("lse", BO.gate_ratio(lse[r0:r1], ref, g_lse))
        w.add("target", BO.gate_ratio(pos[r0:r1], ref_pos, g_pos))
        t = ref - ref_pos
        t_sum, t_abs, t_gate = t_sum + t.sum().item(), t_abs + t.abs().sum().item(), t_gate + (g_lse + g_pos).sum().item()
    if A["loss_accum"] is not None:
        w.add("loss", _loss_sum_ratio(A["loss_accum"], before, A["loss_scale"], t_sum, t_abs, t_gate,
                                      A["x"].shape[0]))
    return w


def check_vocab_ce_bwd(A, before, g):
    gs = A["gscale"].double().item()
    V = A["w"].shape[0]
    labels, lse_k = A["labels"], A["lse"]
    w = Worst()
    w.add("pad", exact(g[:, V:], torch.zeros_like(g[:, V:])))
    for r0, r1 in _chunks(A["x"].shape[0], VCE_ROWS):
        l, e_l = _vce_rows(A, r0, r1)
        lk = lse_k[r0:r1].double()[:, None]
        p = torch.exp(l - lk)
        ref = gs * p
        ref.scatter_add_(1, labels[r0:r1, None], torch.full((r1 - r0, 1), -gs, dtype=ref.dtype, device=ref.device))
        gate = (NO.BF16_REL * ref.abs() + gs * p * (e_l + 2.0 ** -23 * (l.abs() + lk.abs()) + 2.0 ** -22)
                + gs * 2.0 ** -120)
        w.add("g", BO.gate_ratio(g[r0:r1, :V], ref, gate))
    return w


# --------------------------------------------------------------------------- similarity regularisation
# Gates of simreg_oracle (test_gpu_simreg.py's) against E = a b^T of the call's bf16 operands, the
# diagonal column of each row zeroed.  E's own error, simreg_oracle.E_ABS, was measured on latents of
# random directions, where the partial sums of E's K = 6 D chain stay near |<t_r, t_c>| ~ D^-1/2.  A
# training step's latents are far from orthogonal (a freshly initialised tower maps every input near
# one direction), so the chain's running sums reach |<t_r, t_c>| ~ 1 before the -V V^T half brings
# them back to E: its accumulation error is then bounded by the GEMM's own per-element chain bound
# (gemm_oracle.chain_bound of the running sums), and E's error term is the larger of the two.

def _simreg_rows(A, r0, r1):
    """fp64 E of rows [r0, r1) with the diagonal zeroed, and the bound on the kernel's error of E."""
    e, S, P = GO.chain_sums64(A["a"][r0:r1], A["b"])
    e_err = torch.clamp(GO.chain_bound(S, P), min=SR.E_ABS)
    del S, P
    r = torch.arange(r1 - r0, device=e.device)
    e[r, r + r0 + A["diag_offset"]] = 0.0
    return e, e_err


def check_simreg_pack(A, before, out):
    v = -A["v"] if A["negate_v"] else A["v"]
    return {"": exact(out, torch.cat([A["t"], v], 1))}


def check_simreg_fwd(A, before, rowsum):
    w = Worst()
    total = 0.0
    for r0, r1 in _chunks(A["a"].shape[0], NCE_ROWS):
        e, e_err = _simreg_rows(A, r0, r1)
        ref = (e * e).sum(1)
        w.add("rowsum", BO.gate_ratio(rowsum[r0:r1], ref, SR.ROWSUM_REL * ref + 2 * (e_err * e.abs()).sum(1)))
        total += ref.sum().item()
    if A["loss_accum"] is not None:
        l0, sc = before["loss_accum"].double().item(), A["loss_scale"]
        gate = SR.LOSS_REL * abs(sc) * total + 2.0 ** -23 * abs(l0) + 1e-30
        w.add("loss", abs(A["loss_accum"].double().item() - (l0 + sc * total)) / gate)
    return w


def check_simreg_bwd(A, before, g):
    gs = A["gscale"].double().item()
    C, off = A["b"].shape[0], A["diag_offset"]
    R = A["a"].shape[0]
    r = torch.arange(R, device=g.device)
    w = Worst()
    w.add("pad", exact(g[:, C:], torch.zeros_like(g[:, C:])))
    w.add("diag", exact(g[r, r + off], torch.zeros_like(g[r, r + off])))
    for r0, r1 in _chunks(R, NCE_ROWS):
        e, e_err = _simreg_rows(A, r0, r1)
        ref = gs * e
        w.add("g", BO.gate_ratio(g[r0:r1, :C], ref, SR.G_REL * ref.abs() + abs(gs) * e_err))
    return w


# --------------------------------------------------------------------------- augmentation

AUG_IMAGES = 256          # images per fp64 augmentation reference chunk
AUG_ARGS = ("ops", "factor", "one_minus", "grayscale", "flip", "blur_kernel", "normalize", "crop", "out_size")


def check_augment(A, before, out):
    """augment_oracle.augment64 of the call's own arguments, at augment_oracle.GATE of max(1, max |ref|)."""
    x = A["x"]
    kw = {k: A[k] for k in AUG_ARGS}
    err = top = 0.0
    for b0, b1 in _chunks(x.shape[0], AUG_IMAGES):
        ref = AU.augment64(x[b0:b1], **kw)
        err = max(err, (out[b0:b1].double() - ref).abs().max().item())
        top = max(top, ref.abs().max().item())
    return {"": err / (AU.GATE * max(1.0, top))}


# --------------------------------------------------------------------------- image gradients

def cast_rows_check(A, before, out):
    src, cols = A["src"], A["src"].shape[1]
    return {"": exact(out[:, :cols], src.bfloat16()), "pad": exact(out[:, cols:], torch.zeros_like(out[:, cols:]))}


def unpatchify64(rows, image_shape, p, keep):
    """The inverse of gemm_oracle.patchify64 with PatchDropout's keep: rows [B k, p p C] (only their first
    p p C columns are read) -> fp64 [B, C, H, W], every pixel of a patch not in keep[b] 0."""
    B, C, H, W = (int(v) for v in image_shape)
    gh, gw, pd = H // p, W // p, p * p * C
    r = rows[:, :pd].double().view(B, -1, pd)
    if keep is not None:
        r = torch.zeros((B, gh * gw, pd), dtype=r.dtype, device=r.device).scatter_(
            1, keep[:, :, None].expand(-1, -1, pd), r)
    img = torch.zeros((B, C, H, W), dtype=r.dtype, device=r.device)
    img[:, :, :gh * p, :gw * p] = r.view(B, gh, gw, p, p, C).permute(0, 5, 1, 3, 2, 4).reshape(B, C, gh * p, gw * p)
    return img


def check_patchify_scatter(A, before, img):
    """Each pixel comes from exactly one f32 row element (or is 0): exact."""
    src, shape, p, keep = A["src"], A["image_shape"], A["patch"], A["keep"]
    B = int(shape[0])
    k = src.shape[0] // B
    w = Worst()
    for b0, b1 in _chunks(B, 256):
        ref = unpatchify64(src[b0 * k:b1 * k], (b1 - b0,) + tuple(shape[1:]), p,
                           None if keep is None else keep[b0:b1])
        w.add("", exact(img[b0:b1].double(), ref))
    return w


# --------------------------------------------------------------------------- registry

class Check:
    """check(bound arguments after the call, {name: clone before the call}, result) -> {output: ratio};
    inplace(arguments) -> names of the buffers the call writes in place or accumulates into."""

    def __init__(self, check, inplace=()):
        self.check = check
        self._inplace = inplace

    def inplace(self, A):
        names = self._inplace(A) if callable(self._inplace) else self._inplace
        return [k for k in names if A.get(k) is not None]


CHECKS = {
    "gemm": Check(check_gemm, lambda A: ("out",) if A["accumulate"] else ()),
    "cast_bf16": Check(cast_check),
    "layernorm_fwd": Check(check_ln_fwd),
    "layernorm_bwd": Check(check_ln_bwd, ("dg",)),
    "l2norm_fwd": Check(check_l2norm_fwd),
    "l2norm_bwd": Check(check_l2norm_bwd),
    "attn_fwd": Check(check_attn_fwd),
    "attn_bwd": Check(check_attn_bwd),
    "rotary_": Check(check_rotary, ("qkv",)),
    "patchify_gather": Check(check_patchify_gather),
    "scatter_add_rows_": Check(check_scatter_add_rows, ("dst",)),
    "colsum_rows_": Check(check_colsum_rows, ("dst",)),
    "ff_weights": Check(check_ff_weights),
    "ff_up": Check(check_ff_up),
    "ff_down": Check(check_ff_down),
    "ff_bwd_prep": Check(check_ff_bwd_prep),
    "ff_bwd": Check(check_ff_bwd),
    "ff_w2_grad_post_": Check(check_ff_w2_grad_post, ("raw", "dg")),
    "adamw_step_": Check(check_adamw, ("p", "m", "v")),
    "nce_fwd": Check(check_nce_fwd, ("loss_accum",)),
    "nce_bwd": Check(check_nce_bwd, ("dtemp",)),
    "text_embed_fwd": Check(check_text_embed_fwd),
    "text_embed_bwd": Check(check_text_embed_bwd),
    "filip_segmax16": Check(check_filip_segmax16),
    "filip_reduce": Check(check_filip_reduce),
    "filip_nce_fwd": Check(check_filip_nce_fwd, ("loss_accum",)),
    "filip_nce_bwd": Check(check_filip_nce_bwd),
    "filip_expand16": Check(check_filip_expand16),
    "filip_nce_blocks_fwd": Check(check_filip_nce_blocks_fwd, ("loss_accum",)),
    "filip_nce_blocks_bwd": Check(check_filip_nce_blocks_bwd),
    "sigmoid_fwd": Check(check_sigmoid_fwd, ("loss_accum",)),
    "sigmoid_bwd": Check(check_sigmoid_bwd, ("dtemp", "dbias")),
    "vocab_ce_fwd": Check(check_vocab_ce_fwd, ("loss_accum",)),
    "vocab_ce_bwd": Check(check_vocab_ce_bwd),
    "simreg_pack": Check(check_simreg_pack),
    "simreg_fwd": Check(check_simreg_fwd, ("loss_accum",)),
    "simreg_bwd": Check(check_simreg_bwd),
    "augment": Check(check_augment),
    "cast_bf16_rows": Check(cast_rows_check),
    "patchify_scatter": Check(check_patchify_scatter),
}


# --------------------------------------------------------------------------- recorder

def _desc(v):
    """What of one argument goes into a signature."""
    if isinstance(v, torch.Tensor):
        return (tuple(v.shape), str(v.dtype).replace("torch.", ""), tuple(v.stride()))
    if isinstance(v, (tuple, list)):
        return tuple(_desc(x) for x in v)
    return v


def _meta(v):
    if isinstance(v, torch.Tensor):
        return torch.empty(v.shape, dtype=v.dtype, device="meta")
    return v


def _sig_text(A) -> str:
    parts = []
    for k, v in A.items():
        if v is None or v is False:
            continue
        if isinstance(v, torch.Tensor):
            s = "x".join(str(x) for x in v.shape)
            if v.dim() == 2 and v.stride(0) != v.shape[1]:
                s += f"/ld{v.stride(0)}"
            parts.append(f"{k}={s}:{str(v.dtype).replace('torch.', '')}")
        elif isinstance(v, (tuple, list)):
            parts.append(f"{k}=set")
        elif isinstance(v, float):
            parts.append(f"{k}={v:.4g}")
        else:
            parts.append(f"{k}={v}")
    return ",".join(parts).replace(" ", "")


class Recorder:
    """Spies on every public wrapper of the kernels module K (see the module docstring).

    results: [(label, ratio)] of every checked output; calls: Counter of wrapper calls; unchecked:
    Counter of calls to wrappers with no check; signatures: the checked signatures."""

    def __init__(self, K, verbose=True):
        self.K, self.verbose = K, verbose
        self.results, self.calls, self.unchecked = [], Counter(), Counter()
        self.signatures = {}
        self.arguments = {}          # signature -> its arguments, tensors as shape-only meta tensors

    def install(self, monkeypatch):
        for name in public_wrappers(self.K):
            if name not in HOST_HELPERS:
                monkeypatch.setattr(self.K, name, self._spy(name, getattr(self.K, name)))
        return self

    def _spy(self, name, real):
        sig = inspect.signature(real)
        check = CHECKS.get(name)

        def spy(*args, **kw):
            self.calls[name] += 1
            if check is None:
                self.unchecked[name] += 1
                return real(*args, **kw)
            ba = sig.bind(*args, **kw)
            ba.apply_defaults()
            A = dict(ba.arguments)
            key = (name, _desc(tuple(A.values())))
            if key in self.signatures:
                return real(*args, **kw)
            before = {k: A[k].clone() for k in check.inplace(A)}
            out = real(*args, **kw)
            torch.cuda.synchronize()
            ratios = check.check(A, before, out)
            del before
            label = f"{name}[{_sig_text(A)}]"
            self.signatures[key] = label
            self.arguments[key] = {k: _meta(v) for k, v in A.items()}
            for k, r in ratios.items():
                self.results.append((label + k, r))
                if self.verbose:
                    print(f"GATE {label}{k} {r:.4f}", flush=True)
            torch.cuda.empty_cache()
            return out

        return spy

    def failures(self):
        return [(lab, r) for lab, r in self.results if not r <= 1.0]

    def worst(self, family: str) -> float:
        rs = [r for lab, r in self.results if lab.startswith(family + "[")]
        return max(rs) if rs else float("nan")
