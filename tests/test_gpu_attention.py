"""Fused attention forward / backward against the fp64 reference of attn_oracle.py (x_clip.py:217-244),
computed from the bf16 q, k, v the kernels read, with per-element gates (derivation in attn_oracle).
Inputs come from attn_oracle's recipes: flat, peaked and late-maximum scores, block-masked keys and
rows with no visible key, with dO along o so that the - delta term of dS is large."""
import pytest
import torch

import attn_oracle as AO
import block_oracle as BO

pytestmark = pytest.mark.gpu

ATTN_STREAM = 5     # XCLIP_TUNE_ATTN_STREAM (include/xclip_b200.h)
SCALE = 64 ** -0.5

CASES = [(2, 33, 4, False), (3, 65, 8, False), (2, 128, 2, True), (2, 17, 4, True),
         (2, 197, 12, False), (2, 257, 8, True), (1, 320, 2, True), (5, 78, 8, True),
         # n = 64k+1: a last 64-row block with one row; 24*8 (b,h) items: many CTAs per SM
         (2, 129, 4, True), (3, 129, 2, False), (24, 257, 8, True), (20, 257, 8, False),
         # short sequences (attention_small.cu): ViT-B/16 with patch dropout (98), CLIP text (78),
         # README image tower (32); several items per CTA; every 16-key tail width
         (130, 98, 12, False), (90, 78, 8, True), (300, 32, 8, False), (3, 64, 4, True), (2, 112, 3, True),
         (2, 1, 2, False), (3, 16, 2, True), (2, 100, 4, True), (4, 128, 12, False), (2, 48, 2, False),
         (2, 81, 5, True),
         # batch x heads beyond 65535 CTAs in one grid dimension
         (16640, 16, 4, True)]
CAUSAL_CASES = [(3, 78, 8, True), (2, 33, 4, False), (2, 128, 2, True), (40, 64, 8, False)]
# tail widths, the causal cap of 128, the resident / streaming switch at 320 / 321
SEQ_LENS = [1, 2, 15, 16, 17, 63, 64, 65, 127, 128, 320, 321, 577, 1025]
# recipe shapes: 4 full blocks + a one-key tail; resident (and forced streaming) / streaming
RECIPE_N = {"resident": 257, "forced": 257, "streaming": 577}


def _mk(B, n, H, masked, dev, seed=0):
    g = torch.Generator().manual_seed(seed)
    qkv = torch.randn(B * n, 3 * H * 64, generator=g).to(dev).bfloat16()
    mask = None
    if masked:
        mask = (torch.rand(B, n, generator=g) > 0.3).to(dev)
        mask[:, 0] = True     # the CLS key is always attendable (x_clip.py:335)
    return qkv, mask


def fwd_bwd(case, B, n, H, scale=SCALE, causal=False, bwd=True):
    from x_clip_b200 import kernels as K
    o, lse = K.attn_fwd(case["qkv"], case["mask"], B, n, H, scale, causal=causal)
    dqkv = K.attn_bwd(case["qkv"], case["mask"], o, case["d_o"], lse, B, n, H, scale, causal=causal) if bwd else None
    torch.cuda.synchronize()
    return o, lse, dqkv


def check_attn(tag, case, B, n, H, o, lse, dqkv=None, scale=SCALE, causal=False):
    """o, lse (and dq, dk, dv) per element against the fp64 reference; prints GATE lines."""
    ref = AO.attn_ref64(case["qkv"], case["mask"], B, n, H, scale, causal,
                        o=o if dqkv is not None else None, d_o=case["d_o"] if dqkv is not None else None)
    BO.check(f"attn o {tag}", o, ref["o"], ref["g_o"])
    BO.check(f"attn lse {tag}", lse, ref["lse"], ref["g_lse"])
    if dqkv is None:
        return
    inner = H * 64
    for name, sl in (("dq", slice(0, inner)), ("dk", slice(inner, 2 * inner)), ("dv", slice(2 * inner, 3 * inner))):
        BO.check(f"attn {name} {tag}", dqkv[:, sl], ref["dqkv"][:, sl], ref["g_dqkv"][:, sl])


def run_mode(mode, fn):
    """fn() with the streaming kernels forced at n <= 320 when mode == "forced"."""
    if mode != "forced":
        return fn()
    from x_clip_b200 import _lib
    lib = _lib.load()
    prev = lib.xclip_tune_set(ATTN_STREAM, 1)
    assert prev == 0
    try:
        return fn()
    finally:
        lib.xclip_tune_set(ATTN_STREAM, prev)


@pytest.mark.parametrize("B,n,H,masked", CASES)
def test_attn_fwd(cuda_device, B, n, H, masked):
    case = AO.attn_case("peaked", B, n, H, masked=masked, device=cuda_device)
    o, lse, _ = fwd_bwd(case, B, n, H, bwd=False)
    check_attn(f"peaked B{B} n{n} H{H}", case, B, n, H, o, lse)


@pytest.mark.parametrize("B,n,H,masked", CASES)
def test_attn_bwd(cuda_device, B, n, H, masked):
    case = AO.attn_case("flat", B, n, H, masked=masked, seed=1, device=cuda_device)
    check_attn(f"flat B{B} n{n} H{H}", case, B, n, H, *fwd_bwd(case, B, n, H))


@pytest.mark.parametrize("B,n,H,masked", CAUSAL_CASES)
def test_attn_causal_fwd_bwd(cuda_device, B, n, H, masked):
    """Causal mask of the text tower (x_clip.py:233-236, text_causal_mask=True), n <= 128."""
    case = AO.attn_case("flat", B, n, H, causal=True, masked=masked, seed=2, device=cuda_device)
    check_attn(f"causal B{B} n{n} H{H}", case, B, n, H, *fwd_bwd(case, B, n, H, causal=True), causal=True)


@pytest.mark.parametrize("H", [1, 12, 16])
@pytest.mark.parametrize("n", SEQ_LENS)
def test_attn_seq_lengths(cuda_device, n, H):
    """Peaked, key-masked scores at every tail width and both schedules; causal at H = 12."""
    causal = H == 12
    case = AO.attn_case("peaked", 2, n, H, causal=causal, seed=3, device=cuda_device)
    check_attn(f"n{n} H{H}", case, 2, n, H, *fwd_bwd(case, 2, n, H, causal=causal), causal=causal)


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("mode", ["resident", "streaming", "forced"])
@pytest.mark.parametrize("recipe", AO.RECIPES)
def test_attn_recipes(cuda_device, recipe, mode, causal):
    """Every input recipe on the resident kernels, the streaming kernels, and the streaming kernels
    forced at n <= 320.  no_visible fails on a backward that lets gradient through masked scores."""
    B, n, H = 3, RECIPE_N[mode], 2
    case = AO.attn_case(recipe, B, n, H, causal=causal, seed=4, device=cuda_device)
    out = run_mode(mode, lambda: fwd_bwd(case, B, n, H, causal=causal))
    check_attn(f"{recipe} {mode}", case, B, n, H, *out, causal=causal)


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("n", [1, 5, 65])
def test_attn_rows_without_visible_key(cuda_device, n, causal):
    """Item 0: keys 0 and 1 masked (causal rows 0 and 1 see no key); item 1: every key masked.  The
    reference's softmax is uniform over the n keys and masked_fill passes no gradient to the scores:
    such a row has dq = 0, adds nothing to dk and dO / n to every dv."""
    B, H = 2, 3
    mask = torch.ones(B, n, dtype=torch.bool)
    mask[0, :2] = False
    mask[1] = False
    case = AO.attn_case("flat", B, n, H, causal=causal, seed=5, device=cuda_device, mask=mask)
    for mode in ("resident", "forced"):
        o, lse, dqkv = run_mode(mode, lambda: fwd_bwd(case, B, n, H, causal=causal))
        check_attn(f"no visible key n{n} {mode}", case, B, n, H, o, lse, dqkv, causal=causal)
        assert (lse[1] == -AO.FLT_MAX).all()
        assert (dqkv[n:, :H * 64] == 0).all(), "a row without a visible key has dq = 0"


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("n", [97, 400])
def test_attn_scale(cuda_device, n, causal):
    """A scale other than 1/8, not a power of two (scale log2(e) rounds in fp32)."""
    B, H, scale = 2, 4, 0.3
    case = AO.attn_case("flat", B, n, H, causal=causal, scale=scale, seed=6, device=cuda_device)
    out = fwd_bwd(case, B, n, H, scale=scale, causal=causal)
    check_attn(f"scale {scale} n{n}", case, B, n, H, *out, scale=scale, causal=causal)


@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("n", [129, 385])
def test_attn_strides(cuda_device, n, causal):
    """ld_qkv, ldo, lddo and ld_dqkv above their minimum: the results equal the contiguous run bit for
    bit, and the columns beyond each operand keep their sentinel bits."""
    from x_clip_b200 import _lib
    B, H = 2, 3
    inner = H * 64
    case = AO.attn_case("no_visible", B, n, H, causal=causal, seed=7, device=cuda_device)
    o_ref, lse_ref, dqkv_ref = fwd_bwd(case, B, n, H, causal=causal)
    sentinel = -777.0

    def padded(t, extra):
        buf = torch.full((t.shape[0], t.shape[1] + extra), sentinel, device=cuda_device, dtype=torch.bfloat16)
        if t.numel():
            buf[:, :t.shape[1]] = t
        return buf

    qkv = padded(case["qkv"], 24)
    d_o = padded(case["d_o"], 16)
    o = padded(torch.empty(B * n, 0, device=cuda_device), inner + 8)
    dqkv = padded(torch.empty(B * n, 0, device=cuda_device), 3 * inner + 40)
    ins = (qkv.clone(), d_o.clone())
    lse = torch.empty(B, H, n, device=cuda_device)
    delta = torch.empty(B, H, n, device=cuda_device)
    stream = torch.cuda.current_stream().cuda_stream
    mask = case["mask"].data_ptr()
    _lib.call("xclip_attn_fwd", qkv.data_ptr(), qkv.stride(0), mask, o.data_ptr(), o.stride(0), lse.data_ptr(),
              B, n, H, SCALE, int(causal), stream)
    _lib.call("xclip_attn_bwd", qkv.data_ptr(), qkv.stride(0), mask, o.data_ptr(), o.stride(0), d_o.data_ptr(),
              d_o.stride(0), lse.data_ptr(), delta.data_ptr(), dqkv.data_ptr(), dqkv.stride(0), None, B, n, H,
              SCALE, int(causal), stream)
    torch.cuda.synchronize()
    assert qkv.stride(0) % 8 == 0 and o.stride(0) == inner + 8 and dqkv.stride(0) == 3 * inner + 40
    assert torch.equal(o[:, :inner], o_ref) and torch.equal(lse, lse_ref)
    assert torch.equal(dqkv[:, :3 * inner], dqkv_ref)
    assert (o[:, inner:] == sentinel).all() and (dqkv[:, 3 * inner:] == sentinel).all()
    assert torch.equal(qkv, ins[0]) and torch.equal(d_o, ins[1])


def test_attn_refuses_bad_arguments(cuda_device):
    """Bad leading dimensions, misaligned operands, scale <= 0 and n = 0 return XCLIP_ERR_INVALID
    without launching anything."""
    from x_clip_b200 import _lib
    lib = _lib.load()
    B, n, H = 2, 33, 2
    inner = H * 64
    dev = cuda_device
    qkv = torch.zeros(B * n + 1, 3 * inner + 16, device=dev, dtype=torch.bfloat16)
    o = torch.zeros(B * n + 1, inner + 16, device=dev, dtype=torch.bfloat16)
    d_o = torch.zeros_like(o)
    dqkv = torch.zeros_like(qkv)
    lse = torch.zeros(B, H, n, device=dev)
    delta = torch.zeros_like(lse)
    stream = torch.cuda.current_stream().cuda_stream
    fwd = dict(qkv=qkv.data_ptr(), ld=3 * inner, o=o.data_ptr(), ldo=inner, n=n, scale=SCALE)
    bwd = dict(fwd, d_o=d_o.data_ptr(), lddo=inner, dqkv=dqkv.data_ptr(), ldd=3 * inner)

    def call_fwd(a):
        return lib.xclip_attn_fwd(a["qkv"], a["ld"], None, a["o"], a["ldo"], lse.data_ptr(), B, a["n"], H,
                                  a["scale"], 0, stream)

    def call_bwd(a):
        return lib.xclip_attn_bwd(a["qkv"], a["ld"], None, a["o"], a["ldo"], a["d_o"], a["lddo"], lse.data_ptr(),
                                  delta.data_ptr(), a["dqkv"], a["ldd"], None, B, a["n"], H, a["scale"], 0, stream)

    bad = [dict(ld=3 * inner + 4), dict(ld=3 * inner - 8), dict(qkv=qkv.data_ptr() + 2), dict(o=o.data_ptr() + 2),
           dict(ldo=inner + 4), dict(ldo=inner - 8), dict(scale=0.0), dict(scale=-SCALE), dict(n=0)]
    bad_bwd = [dict(d_o=d_o.data_ptr() + 2), dict(dqkv=dqkv.data_ptr() + 2), dict(lddo=inner + 4),
               dict(ldd=3 * inner + 4), dict(ldd=3 * inner - 8)]
    for call, good, cases in ((call_fwd, fwd, bad), (call_bwd, bwd, bad + bad_bwd)):
        for change in cases:
            n0 = lib.xclip_launch_count()
            assert call(dict(good, **change)) == 1, change        # XCLIP_ERR_INVALID
            assert lib.xclip_launch_count() == n0, f"{change}: a refused call launched a kernel"
        n0 = lib.xclip_launch_count()
        assert call(good) == 0
        assert lib.xclip_launch_count() > n0
    torch.cuda.synchronize()


def test_attn_bwd_checks_key_mask(cuda_device):
    from x_clip_b200 import _lib
    from x_clip_b200 import kernels as K
    B, n, H = 2, 17, 2
    case = AO.attn_case("flat", B, n, H, device=cuda_device)
    o, lse = K.attn_fwd(case["qkv"], case["mask"], B, n, H, SCALE)
    for bad in (case["mask"].to(torch.uint8), case["mask"][:, :-1], case["mask"].t().contiguous().t()):
        with pytest.raises(_lib.XClipB200Error, match="key_mask"):
            K.attn_bwd(case["qkv"], bad, o, case["d_o"], lse, B, n, H, SCALE)
