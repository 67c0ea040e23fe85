"""The generic wgmma GEMM (xclip_gemm_bf16, EPI_STORE) against fp64 on the exact bf16 operands, with the
per-element gates of gemm_oracle (GAMMA * |alpha| * sum_k |a b| + epilogue / split-K additions + bf16
rounding).  Worst gate ratios on an H100 80GB HBM3 (700 W power limit): f32 0.034 (shapes) and 0.30
(epilogues), accumulated f32 0.42, split-K 0.19, bf16 0.996 (the bf16 rounding bound, see gemm_oracle);
the file runs in about 25 s there.

- every call class (tile width x operand majors x output kind x bias x residual mode x alpha != 1 x
  partial last N tile x K tail);
- N at 256-wide tiles with a partial last tile (1152, 1920, 2688: the QKV projections of widths 384,
  640, 896), N = 1032 (one 8-column last tile), N at 128-wide tiles, the dgrad shapes that run 256-wide
  tiles, and K from below one k-block to 2304;
- ragged M (1 row, M % 128 = 1 and 127) and tile counts around one and two waves of SMs;
- split-K into a random non-zero prefill with alpha = 1 and -1: short last splits, the branch where
  the wave bound hi falls below lo, bias and residual with splits;
- every output lives in a buffer with ldc > N and rows past M filled with NaN, which must come back bit
  for bit;
- an inventory of every GEMM call of a depth-1 CLIP step over six configurations, whose classes must
  all occur above.
"""
import itertools

import pytest
import torch

import block_oracle as BO
import gemm_oracle as GO

pytestmark = pytest.mark.gpu

MAJORS = [(0, 0), (0, 1), (1, 0), (1, 1)]
OUTS = ["bf16", "f32", "f32acc"]
N_CASES = [1152, 1920, 2688, 1032, 1272, 136, 384, 896]    # 1272: a partial 256-wide tile of 248 columns
K_CASES = [8, 40, 64, 72, 200, 1152, 2304]
DGRAD_SHAPES = [(768, 2304), (512, 1536)]            # (N, K): cfg3 QKV dgrad, text QKV dgrad
# (block_n, partial last N tile) -> N of the class matrix; K tail -> K
CLASS_N = {(128, False): 384, (128, True): 136, (256, False): 1536, (256, True): 1152}
CLASS_K = {False: 128, True: 72}
CLASS_M = 136                                         # two row tiles, the last one with 8 rows
RES_MODES = [None, "row", "mod", "idx"]


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def run_case(dev, M, N, K, a_major=0, b_major=0, out="f32", alpha=1.0, bias=False, res=None, seed=0):
    """One GEMM into a NaN-framed output buffer -> (gate ratio, split plan).  Asserts the frame (columns
    N..ldc, rows past M) is bit-identical afterwards."""
    from x_clip_b200 import kernels
    a, b = GO.operands(M, N, K, a_major, b_major, seed)
    bias_t, res_t, rows = GO.epilogue_inputs(M, N, K, res, seed)
    bias_t = bias_t if bias else None
    acc = out == "f32acc"
    pre = GO.prefill(M, N, seed) if acc else None
    dt = torch.bfloat16 if out == "bf16" else torch.float32
    ldc = N + 24
    buf = torch.full((M + 3, ldc), float("nan"), dtype=dt, device=dev)
    c = buf[:M, :N]
    if pre is not None:
        c.copy_(pre)
    frame = torch.ones(M + 3, ldc, dtype=torch.bool, device=dev)
    frame[:M, :N] = False
    ibits = torch.int16 if dt == torch.bfloat16 else torch.int32
    before = buf.view(ibits)[frame].clone()
    a, b = a.to(dev), b.to(dev)
    kw = {}
    if res_t is not None:
        rbuf = torch.zeros(res_t.shape[0], N + 8, dtype=torch.bfloat16, device=dev)   # ldr > N
        rbuf[:, :N] = res_t.to(dev)
        kw["residual"] = rbuf[:, :N]
        if res == "mod":
            kw["res_row_mod"] = res_t.shape[0]
        elif res == "idx":
            kw["res_row_idx"] = rows.to(dev, torch.int32)
    kernels.gemm(a, b, a_major=a_major, b_major=b_major, out=c, alpha=alpha,
                 bias=None if bias_t is None else bias_t.to(dev), accumulate=acc, **kw)
    torch.cuda.synchronize()
    assert torch.equal(buf.view(ibits)[frame], before), "GEMM wrote outside its output"
    plan = GO.split_plan(M, N, K, acc, _sms())
    r = res_t.to(dev) if res_t is not None else None
    rr = rows.to(dev) if rows is not None else None
    p = pre.to(dev) if pre is not None else None
    bb = bias_t.to(dev) if bias_t is not None else None
    ratio = 0.0
    for r0 in range(0, M, 4096):                      # fp64 reference in row chunks
        r1 = min(M, r0 + 4096)
        ac = a[r0:r1] if a_major == 0 else a[:, r0:r1]
        sl = dict(alpha=alpha, bias=bb, residual=r, res_rows=None if rr is None else rr[r0:r1],
                  prefill=None if p is None else p[r0:r1])
        ref = GO.gemm64(ac, b, a_major, b_major, **sl)
        gate = GO.gemm_gate(ac, b, a_major, b_major, **sl, bf16_out=out == "bf16", splits=plan["splits"], ref=ref)
        ratio = max(ratio, BO.gate_ratio(c[r0:r1], ref, gate))
    return ratio, plan


class Worst:
    """Largest gate ratio over the GEMMs of one test; prints `GATE name ratio` and asserts <= 1."""

    def __init__(self, name):
        self.name, self.ratio, self.case = name, 0.0, None

    def add(self, ratio, case):
        if ratio >= self.ratio:
            self.ratio, self.case = ratio, case

    def check(self):
        print(f"GATE {self.name} {self.ratio:.4f}")
        assert self.ratio <= 1.0, f"{self.name}: error is {self.ratio:.3f} x its gate at {self.case}"


def class_matrix():
    """(N, K, alpha, bias, res) of every combination of tile width, partial last N tile, K tail, bias,
    residual mode and alpha != 1 (alternately 0.5 and -1)."""
    cases = []
    for i, ((bn, part), ktail, bias, res, alt) in enumerate(itertools.product(
            CLASS_N, (False, True), (False, True), RES_MODES, (False, True))):
        N, K = CLASS_N[(bn, part)], CLASS_K[ktail]
        assert GO.block_n(N, K) == bn and (N % bn != 0) == part and (K % 64 != 0) == ktail
        alpha = (0.5 if i % 4 < 2 else -1.0) if alt else 1.0
        cases.append((N, K, alpha, bias, res))
    return cases


@pytest.mark.parametrize("out", OUTS)
@pytest.mark.parametrize("a_major,b_major", MAJORS)
def test_gemm_every_class(cuda_device, a_major, b_major, out):
    """Both tile widths, full and partial last N tile, with and without K tail, bias, the three residual
    modes (row, row % 97, gathered rows with repeats) and alpha in {1, 0.5, -1}."""
    w = Worst(f"gemm_class_{a_major}{b_major}_{out}")
    for j, (N, K, alpha, bias, res) in enumerate(class_matrix()):
        ratio, _ = run_case(cuda_device, CLASS_M, N, K, a_major, b_major, out, alpha, bias, res, seed=j)
        w.add(ratio, (N, K, alpha, bias, res))
    w.check()


@pytest.mark.parametrize("out", OUTS)
@pytest.mark.parametrize("a_major,b_major", MAJORS)
def test_gemm_n_k_shapes(cuda_device, a_major, b_major, out):
    """Every N case x every K case, and the dgrad shapes on 256-wide tiles.  M % 128 = 127 (K-major A)
    or 120 (MN-major A, whose rows must be a multiple of 8)."""
    M = 255 if a_major == 0 else 248
    w = Worst(f"gemm_nk_{a_major}{b_major}_{out}")
    shapes = [(N, K) for N in N_CASES for K in K_CASES] + DGRAD_SHAPES
    assert {GO.block_n(N, K) for N, K in DGRAD_SHAPES} == {256}
    for j, (N, K) in enumerate(shapes):
        ratio, _ = run_case(cuda_device, M, N, K, a_major, b_major, out, seed=100 + j)
        w.add(ratio, (M, N, K))
    w.check()


def _wave_rows(tiles, n_tiles):
    return -(-tiles // n_tiles) * 128 - 40


@pytest.mark.parametrize("N", [384, 1152])
@pytest.mark.parametrize("a_major,b_major", MAJORS)
def test_gemm_ragged_m_and_waves(cuda_device, N, a_major, b_major):
    """M = 1 / 129 / 255 (8 / 136 / 248 for MN-major A) and tile counts sms - 1 .. 2 sms + 1, into
    bf16, f32 and accumulated f32 (tiles >= SMs: no split)."""
    K = 200
    s = _sms()
    nt = -(-N // GO.block_n(N, K))
    ms = [1, 129, 255] if a_major == 0 else [8, 136, 248]
    ms += [_wave_rows(t, nt) for t in (s - 1, s, s + 1, 2 * s - 1, 2 * s, 2 * s + 1)]
    w = Worst(f"gemm_waves_{N}_{a_major}{b_major}")
    for j, M in enumerate(ms):
        for out in OUTS:
            ratio, plan = run_case(cuda_device, M, N, K, a_major, b_major, out, seed=200 + j)
            assert plan["splits"] == 1
            w.add(ratio, (M, out))
    w.check()


# name: (M, N, K, a_major, b_major, alpha, bias, res, expected property of the split plan)
SPLIT_CASES = {
    "short_last_256": (768, 768, 9000, 1, 1, 1.0, False, None, "short"),
    "short_last_128_alpha_neg": (1024, 640, 5000, 0, 1, -1.0, False, None, "short"),
    "hi_lt_lo_short_alpha_neg": (512, 512, 4160, 1, 1, -1.0, False, None, "hi<lo short"),
    "hi_lt_lo_partial_256": (256, 1152, 3000, 0, 1, -1.0, False, None, "hi<lo short"),
    "hi_lt_lo_even": (1024, 512, 8192, 1, 1, 1.0, False, None, "hi<lo"),
    "bias_res_mod": (768, 768, 9000, 0, 0, 0.5, True, "mod", "short"),
    "bias_res_idx_partial_256": (256, 1152, 3000, 1, 1, -1.0, True, "idx", "hi<lo short"),
}


@pytest.mark.parametrize("name", list(SPLIT_CASES))
def test_gemm_splitk_into_prefill(cuda_device, name):
    M, N, K, am, bm, alpha, bias, res, prop = SPLIT_CASES[name]
    plan = GO.split_plan(M, N, K, True, _sms())
    rng = GO.split_ranges(plan)
    assert plan["splits"] > 1, plan
    if "short" in prop:
        assert rng[-1][1] - rng[-1][0] < plan["kb_per"], plan
    if "hi<lo" in prop:
        assert plan["hi"] < plan["lo"], plan
    ratio, _ = run_case(cuda_device, M, N, K, am, bm, "f32acc", alpha, bias, res, seed=300)
    w = Worst(f"gemm_splitk_{name}")
    w.add(ratio, plan)
    w.check()


# --------------------------------------------------------------------------- inventory

def matrix_classes():
    """Every call class the tests above run."""
    out = set()
    for am, bm in MAJORS:
        for o in OUTS:
            for N, K, alpha, bias, res in class_matrix():
                out.add(GO.call_class(CLASS_M, N, K, am, bm, o, bias, res or "none", alpha))
            for N, K in [(N, K) for N in N_CASES for K in K_CASES] + DGRAD_SHAPES:
                out.add(GO.call_class(255, N, K, am, bm, o, False, "none", 1.0))
    for M, N, K, am, bm, alpha, bias, res, _ in SPLIT_CASES.values():
        out.add(GO.call_class(M, N, K, am, bm, "f32acc", bias, res or "none", alpha))
    return out


def _inventory_configs():
    import bench
    base = dict(text_enc_depth=1, visual_enc_depth=1)
    return {
        "cfg2": (dict(bench.README_CFG, **base), {}, 0.0),
        "cfg3_patch_dropout": (dict(bench.VITB16_CFG, **base), {}, 0.5),
        "vit_s16": (dict(bench.VITB16_CFG, **base, dim_text=384, dim_image=384, dim_latent=384, text_heads=6,
                         visual_heads=6), {}, 0.0),
        "b16plus_simreg_extra": (dict(bench.VITB16_CFG, **base, dim_text=640, dim_image=896, dim_latent=640,
                                      text_heads=10, visual_heads=14, visual_image_size=240),
                                 dict(extra_latent_projection=True, sim_reg_loss_weight=0.1), 0.0),
        "w128": (dict(bench.README_CFG, **base, dim_text=128, dim_image=128, dim_latent=128, text_heads=2,
                      visual_heads=2), {}, 0.0),
        "cfg4_filip": (dict(bench.README_CFG, **base), dict(use_all_token_embeds=True), 0.0),
    }


def test_gemm_call_inventory(cuda_device, monkeypatch):
    """Every kernels.gemm call of one forward + backward of a depth-1 CLIP, reduced to its class, occurs
    in the matrix above.  A call site with a new class fails here until the matrix covers it."""
    import x_clip_b200
    from x_clip_b200 import kernels
    real = kernels.gemm
    calls = []

    def spy(a, b, *, a_major=0, b_major=0, out=None, out_dtype=torch.bfloat16, alpha=1.0, bias=None,
            residual=None, res_row_mod=0, res_row_idx=None, accumulate=False):
        M, K = a.shape if a_major == 0 else a.shape[::-1]
        N = b.shape[0] if b_major == 0 else b.shape[1]
        dt = out.dtype if out is not None else (torch.float32 if accumulate else out_dtype)
        kind = "f32acc" if accumulate else ("bf16" if dt == torch.bfloat16 else "f32")
        calls.append((tag, (M, N, K), GO.call_class(M, N, K, a_major, b_major, kind, bias is not None,
                                                     GO.res_mode_of(residual, res_row_mod, res_row_idx), alpha)))
        return real(a, b, a_major=a_major, b_major=b_major, out=out, out_dtype=out_dtype, alpha=alpha, bias=bias,
                    residual=residual, res_row_mod=res_row_mod, res_row_idx=res_row_idx, accumulate=accumulate)

    monkeypatch.setattr(kernels, "gemm", spy)
    for tag, (cfg, loss_kw, drop) in _inventory_configs().items():
        torch.manual_seed(0)
        clip = x_clip_b200.CLIP(**cfg, **loss_kw, visual_patch_dropout=drop).to(cuda_device)
        clip.train()
        B = 4
        text = torch.randint(1, cfg["num_text_tokens"], (B, cfg["text_seq_len"]), device=cuda_device)
        text[:, -5:] = 0
        image = torch.randn(B, 3, cfg["visual_image_size"], cfg["visual_image_size"], device=cuda_device)
        loss = clip(text, image, return_loss=True)
        loss.backward()
        torch.cuda.synchronize()
        del clip, loss
    seen = {}
    for tag, shape, cls in calls:
        seen.setdefault(cls, []).append((tag, shape))
    print(f"GEMM call classes {GO.CLASS_FIELDS}:")
    for cls in sorted(seen, key=str):
        print("CLASS", cls, sorted({t for t, _ in seen[cls]}), sorted(set(s for _, s in seen[cls]))[:4])
    covered = matrix_classes()
    missing = {cls: seen[cls][:3] for cls in seen if cls not in covered}
    assert not missing, f"GEMM call classes with no fp64 case: {missing}"
    # the QKV projections of widths 384 / 640 / 896 run 256-wide tiles with a partial last tile
    for tag, d in (("vit_s16", 384), ("b16plus_simreg_extra", 640), ("b16plus_simreg_extra", 896)):
        qkv = [cls for t, (M, N, K), cls in calls if t == tag and N == 3 * d and K == d]
        assert qkv and all(c[0] == 256 and c[7] for c in qkv), (tag, d, qkv)
