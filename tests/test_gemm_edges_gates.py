"""CPU checks of the references and gates of test_gpu_gemm_fp64.py, test_gpu_embed_fp64.py and
test_gpu_adamw_fp64.py (no GPU).

- The fp64 helpers of gemm_oracle agree with torch in fp32 on small shapes, and the tile and split-K
  mirrors give the choices csrc/gemm.cu documents.
- On the inputs those tests build from the same seeds, each gate is at most a quarter of the effect of
  the defect it exists to catch (`bite` >= 4, as in test_block_gates.py): the defect still fails the
  GPU test after the kernel's own rounding error (at most 1 gate) is subtracted.
"""
import pytest
import torch

import block_oracle as BO
import gemm_oracle as GO
import test_gpu_adamw_fp64 as TA
import test_gpu_embed_fp64 as TE
import test_gpu_gemm_fp64 as TG

BITE = 4.0
SMS = 132                 # H100 SXM


# --------------------------------------------------------------------------- helpers

@pytest.mark.parametrize("a_major,b_major", TG.MAJORS)
def test_gemm64_matches_torch_fp32(a_major, b_major):
    M, N, K = 40, 24, 72
    a, b = GO.operands(M, N, K, a_major, b_major, seed=5)
    bias, res, rows = GO.epilogue_inputs(M, N, K, "idx", seed=5)
    pre = GO.prefill(M, N, seed=5)
    A = a.float() if a_major == 0 else a.float().t()
    B = b.float() if b_major == 0 else b.float().t()
    want = -0.5 * (A @ B.t()) + bias + res.float()[rows] + pre
    got = GO.gemm64(a, b, a_major, b_major, -0.5, bias, res, rows, pre)
    assert (got - want.double()).abs().max() <= 1e-5 * want.abs().max()
    S = GO.abs_sum64(a, b, a_major, b_major)
    assert torch.allclose(S, (A.abs() @ B.abs().t()).double(), rtol=1e-5)
    blocks = GO.gemm64(a, b, a_major, b_major, k_blocks=[(0, 1), (1, 2)])
    assert torch.allclose(blocks, GO.gemm64(a, b, a_major, b_major), rtol=1e-12, atol=1e-12)


def test_tile_and_split_mirrors():
    # production shapes (N, K) -> tile width
    assert [GO.block_n(N, K) for N, K in [(1152, 384), (1920, 640), (2688, 896), (768, 768), (512, 512),
                                          (768, 2304), (512, 1536), (136, 72), (1032, 8)]] == \
        [256, 256, 256, 128, 128, 256, 256, 128, 256]
    # 64 output tiles on 132 SMs: 6 splits fill 2.91 waves to 97 %, better than 5 (2.42 waves, 81 %)
    p = GO.split_plan(1024, 2048, 64 * 1000, True, SMS)
    assert p["tiles"] == 64 and p["splits"] == 6 and (p["lo"], p["hi"]) == (5, 16)
    assert GO.split_plan(1024, 2048, 64 * 1000, False, SMS)["splits"] == 1
    for M, N, K, *_ in TG.SPLIT_CASES.values():
        p = GO.split_plan(M, N, K, True, SMS)
        r = GO.split_ranges(p)
        assert r[0][0] == 0 and r[-1][1] == p["num_kb"] and all(x[1] == y[0] for x, y in zip(r, r[1:]))


def test_text_embed_bwd64_matches_torch_autograd():
    ids, dx = GO.text_embed_case(5, 7, 16, 11)
    tok = torch.zeros(11, 16, requires_grad=True)
    pos = torch.zeros(9, 16, requires_grad=True)
    cls = torch.zeros(16, requires_grad=True)
    out = torch.cat([cls.expand(5, 1, 16), tok[ids] + pos[:7]], 1)
    out.backward(dx.float())
    (dtok, _), (dpos, _), (dcls, _) = GO.text_embed_bwd64(ids, dx, 11, 9)
    for got, want in ((dtok, tok.grad), (dpos, pos.grad), (dcls, cls.grad)):
        assert torch.allclose(got, want.double(), atol=1e-5)


def test_adamw64_matches_torch_adamw():
    for step in (1, 2, 5):
        p, g, m, v = GO.adamw_state(1003, 0, step)
        t = torch.nn.Parameter(p.clone())
        opt = torch.optim.AdamW([t], lr=1e-3, betas=(0.9, 0.95), eps=1e-8, weight_decay=0.05)
        if step > 1:
            opt.state[t] = dict(step=torch.tensor(float(step - 1)), exp_avg=m.clone(), exp_avg_sq=v.clone())
        t.grad = g * 2.0 ** -10
        opt.step()
        rp, rm, rv, *_ = GO.adamw64(p, g, m, v, 1e-3, 0.9, 0.95, 1e-8, 0.05, step, 2.0 ** -10)
        assert torch.allclose(rp, t.detach().double(), rtol=1e-6, atol=1e-7)
        assert torch.allclose(rm, opt.state[t]["exp_avg"].double(), rtol=1e-5, atol=1e-12)
        assert torch.allclose(rv, opt.state[t]["exp_avg_sq"].double(), rtol=1e-5, atol=1e-20)


# --------------------------------------------------------------------------- GEMM defects

def _nk_case(N, K, a_major=0, b_major=0):
    """Inputs of test_gemm_n_k_shapes for (N, K): same M and seed."""
    shapes = [(n, k) for n in TG.N_CASES for k in TG.K_CASES] + TG.DGRAD_SHAPES
    j = shapes.index((N, K))
    M = 255 if a_major == 0 else 248
    return GO.operands(M, N, K, a_major, b_major, 100 + j)


@pytest.mark.parametrize("K", [40, 72, 200])
@pytest.mark.parametrize("N,a_major,b_major", [(136, 0, 0), (1152, 0, 1), (384, 1, 1)])
def test_gemm_dropped_k_tail_bites(N, K, a_major, b_major):
    a, b = _nk_case(N, K, a_major, b_major)
    nkb = -(-K // 64)
    ref = GO.gemm64(a, b, a_major, b_major)
    effect = GO.gemm64(a, b, a_major, b_major, k_blocks=[(nkb - 1, nkb)])
    for bf16 in (False, True):
        assert BO.bite(effect, GO.gemm_gate(a, b, a_major, b_major, bf16_out=bf16, ref=ref)) >= BITE


# unsplit weight-gradient chains of the training step: cfg3's feed-forward up-projection (768 x 98 rows
# per micro-batch, 1176 k-blocks) and dcl_extra's (1024 x 98 rows, 1568 k-blocks)
CHAIN_KS = [75264, 100352]
# What a dropped k-block of a chain of one sign spans under a bound that holds the tensor cores' error:
# every MMA of such a chain truncates its 16 products in one direction, up to 4 ulp (measured 3.995 on
# an H100), so over 1568 k-blocks the accumulation may legitimately lose about one k-block's worth.
SAME_SIGN_BITE = {75264: 1.2, 100352: 0.85}


@pytest.mark.parametrize("K", CHAIN_KS)
def test_gemm_long_chain_k_block_defects_bite(K):
    """Where the accumulation term is the chain bound (gemm_oracle.chain_bound), a dropped or doubled
    k-block at the start, middle or end of one long chain still spans BITE gates, on operands of both
    signs as the GPU tests build them.  With operands of one sign the running sum grows with the chain,
    and so does the error of the tensor cores' accumulation, all in one direction: there a k-block
    spans about 1.7 and 0.9 gates at these K (SAME_SIGN_BITE), and no bound that holds the hardware's
    error can give it four."""
    a, b = GO.operands(64, 64, K, 1, 1, seed=K)
    plan = GO.split_plan(6144, 768, K, True, SMS)
    assert plan["splits"] == 1 and plan["kb_per"] == K // 64
    nkb = K // 64
    for sign_free in (True, False):
        x, y = (a, b) if sign_free else (a.abs(), b.abs())
        _, S, P = GO.chain_sums64(x, y, 1, 1)
        gate = GO.gemm_gate(x, y, 1, 1, S=S, P=P)
        assert bool((gate > GO.GAMMA * S).any())              # the chain bound is the active term
        for kb in (0, nkb // 2, nkb - 1):
            effect = GO.gemm64(x, y, 1, 1, k_blocks=[(kb, kb + 1)])
            assert BO.bite(effect, gate) >= (BITE if sign_free else SAME_SIGN_BITE[K]), (K, kb, sign_free)


def test_chain_sums64_restarts_at_every_split():
    """P of chain_sums64 sums |running partial sum| per split: a two-split chain equals the sum of the
    two one-split chains of its halves, and the full sum and S do not depend on the splits."""
    a, b = GO.operands(8, 8, 640, 0, 0, seed=3)
    full, S, P = GO.chain_sums64(a, b, 0, 0, ranges=[(0, 4), (4, 10)], k_chunk=128)
    _, _, P0 = GO.chain_sums64(a[:, :256], b[:, :256], 0, 0)
    _, _, P1 = GO.chain_sums64(a[:, 256:], b[:, 256:], 0, 0)
    assert torch.allclose(P, P0 + P1, rtol=1e-12)
    assert torch.allclose(full, GO.gemm64(a, b), rtol=1e-12, atol=1e-12)
    assert torch.allclose(S, GO.abs_sum64(a, b), rtol=1e-12)


def _split_case(name):
    M, N, K, am, bm, alpha, bias, res, _ = TG.SPLIT_CASES[name]
    a, b = GO.operands(M, N, K, am, bm, 300)
    bias_t, res_t, rows = GO.epilogue_inputs(M, N, K, res, 300)
    plan = GO.split_plan(M, N, K, True, SMS)
    kw = dict(alpha=alpha, bias=bias_t if bias else None, residual=res_t, res_rows=rows, prefill=GO.prefill(M, N, 300))
    return a, b, am, bm, plan, kw


@pytest.mark.parametrize("name", ["hi_lt_lo_partial_256", "short_last_128_alpha_neg"])
def test_gemm_doubled_k_block_bites(name):
    """A split boundary off by one: the first k-block of split 1 counted by split 0 as well."""
    a, b, am, bm, plan, kw = _split_case(name)
    kb = plan["kb_per"]
    effect = GO.gemm64(a, b, am, bm, alpha=kw["alpha"], k_blocks=[(kb, kb + 1)])
    assert BO.bite(effect, GO.gemm_gate(a, b, am, bm, splits=plan["splits"], **kw)) >= BITE


def test_gemm_epilogue_in_every_split_bites():
    a, b, am, bm, plan, kw = _split_case("bias_res_idx_partial_256")
    gate = GO.gemm_gate(a, b, am, bm, splits=plan["splits"], **kw)
    extra = plan["splits"] - 1
    assert extra >= 1
    assert BO.bite(extra * kw["bias"].double().expand_as(gate), gate) >= BITE
    assert BO.bite(extra * kw["residual"].double()[kw["res_rows"]], gate) >= BITE


def _class_case(N, K, alpha, bias, res, a_major=0, b_major=0):
    """Inputs of test_gemm_every_class for one entry of class_matrix()."""
    j = TG.class_matrix().index((N, K, alpha, bias, res))
    a, b = GO.operands(TG.CLASS_M, N, K, a_major, b_major, j)
    bias_t, res_t, rows = GO.epilogue_inputs(TG.CLASS_M, N, K, res, j)
    return a, b, bias_t if bias else None, res_t, rows, j


@pytest.mark.parametrize("N,K", [(384, 72), (1152, 128)])
@pytest.mark.parametrize("out", ["bf16", "f32", "f32acc"])
def test_gemm_residual_and_alpha_defects_bite(N, K, out):
    pre = None
    for alpha, bias, res in [(1.0, False, "mod"), (1.0, True, "idx"), (-1.0, True, None), (0.5, True, None)]:
        if (N, K, alpha, bias, res) not in TG.class_matrix():
            continue
        a, b, bias_t, res_t, rows, j = _class_case(N, K, alpha, bias, res)
        if out == "f32acc":
            pre = GO.prefill(TG.CLASS_M, N, j)
        kw = dict(alpha=alpha, bias=bias_t, residual=res_t, res_rows=rows, prefill=pre)
        ref = GO.gemm64(a, b, **kw)
        gate = GO.gemm_gate(a, b, **kw, bf16_out=out == "bf16", ref=ref)
        if res == "mod":            # row % mod off by one
            off = res_t.double()[(rows + 1) % res_t.shape[0]] - res_t.double()[rows]
            assert BO.bite(off, gate) >= BITE
        if res == "idx":            # res_row_idx ignored: row r reads residual row r (rows < R only)
            R = res_t.shape[0]
            eff = res_t.double()[:R] - res_t.double()[rows[:R]]
            assert BO.bite(eff, gate[:R]) >= BITE
        if alpha != 1.0:            # alpha applied to the bias
            assert BO.bite(((alpha - 1) * bias_t.double()).expand_as(gate), gate) >= BITE
        if pre is not None:         # prefill overwritten instead of accumulated
            assert BO.bite(pre.double(), gate) >= BITE


@pytest.mark.parametrize("N", [1272, 1152])
@pytest.mark.parametrize("out", ["bf16", "f32"])
def test_gemm_zeroed_half_tile_bites(N, out):
    """A half of the partial last 256-wide tile left at zero: the second half (columns 1152..1271 of
    N = 1272) or the only valid half (columns 1024..1151 of N = 1152)."""
    a, b = _nk_case(N, 200)
    ref = GO.gemm64(a, b)
    gate = GO.gemm_gate(a, b, bf16_out=out == "bf16", ref=ref)
    c0 = 1152 if N == 1272 else 1024
    assert BO.bite(ref[:, c0:N], gate[:, c0:N]) >= BITE


# --------------------------------------------------------------------------- embedding defects

def test_text_embed_lost_duplicate_red_add_bites():
    B, n, d, vocab = 16, 77, 512, 3
    ids, dx = GO.text_embed_case(B, n, d, vocab)
    (dtok, atok), _, _ = GO.text_embed_bwd64(ids, dx, vocab, n + 5)
    # one occurrence of each id lost
    for v in range(vocab):
        b, t = (ids == v).nonzero()[-1].tolist()
        assert BO.bite(dx[b, 1 + t].double(), GO.red_gate(atok[v])) >= BITE


@pytest.mark.parametrize("name", list(TE.BSPLIT_CASES))
def test_text_embed_column_sum_defects_bite(name):
    B, n, d = TE.BSPLIT_CASES[name]
    ids, dx = GO.text_embed_case(B, n, d, 100)
    _, (dpos, apos), (dcls, acls) = GO.text_embed_bwd64(ids, dx, 100, n + 5)
    x = dx.double()
    # dcls summed over B - 1 samples
    assert BO.bite(x[B - 1, 0], GO.red_gate(acls)) >= BITE
    # one batch slice of dpos counted twice (bsplit stride off by one)
    bs = GO.text_embed_bsplit(B, n, d, SMS)
    assert BO.bite(x[0::bs, 1:].sum(0), GO.red_gate(apos[:n])) >= BITE


def test_patch_embed_scatter_and_colsum_defects_bite():
    """A lost duplicate row in d pos, and one row slice of d bias counted twice."""
    B, S, p, C, k, d = TE.PATCH_CASES[1]
    n = (S // p) ** 2
    t = GO.patch_embed_case(B, n, k, p * p * C, d)
    rows = t["keep"].reshape(-1)
    dy = t["dy"].double()
    apos = torch.zeros(n, d, dtype=torch.float64).index_add_(0, rows, dy.abs())
    dup = (rows == rows[0]).nonzero().squeeze(1)
    assert dup.numel() > 1
    assert BO.bite(dy[dup[-1]], GO.red_gate(apos[rows[0]])) >= BITE
    assert BO.bite(dy[0::256].sum(0), GO.red_gate(dy.abs().sum(0))) >= BITE


# --------------------------------------------------------------------------- AdamW defects

ADAM_DEFECTS = ["no_bc1", "bc1_step_minus_1", "eps_in_sqrt", "decay_after", "scale_m_only", "scale_v_only"]
# a defect is visible only where the knob it misuses is on: weight decay, grad_scale != 1
ADAM_DEFECT_CASES = [(d, i) for d in ADAM_DEFECTS for i, (_, wd, gs, _) in enumerate(TA.LARGE_CASES)
                     if not (d == "decay_after" and wd == 0) and not (d.startswith("scale") and gs == 1)]


@pytest.mark.parametrize("defect,case", ADAM_DEFECT_CASES)
def test_adamw_defects_bite(defect, case):
    """On the large states test_adamw_c_abi builds at step 2 (n just past the grid cap), each defect
    moves p by at least 4 of its gates."""
    betas, wd, gs, near = TA.LARGE_CASES[case]
    p, g, m, v = GO.adamw_state(TA.grid_cap_elems(SMS) + 3, case, 2, near)
    args = (1e-3, betas[0], betas[1], 1e-8, wd, 2, gs)
    rp, rm, rv, gp, gm, gv = GO.adamw64(p, g, m, v, *args)
    dp, dm, dv, *_ = GO.adamw64(p, g, m, v, *args, defect=defect)
    assert BO.bite(dp - rp, gp) >= BITE
