"""The workloads bench.py times, checked kernel call by kernel call against fp64 (bench_call_oracle), and
the micro-batched step's retention plan at the benchmark's own depth, batch and micro-batch.

- cfg3 nce: ViT-B/16 (patch dropout 0.5) + 77-token text tower, 4096 pairs in micro-batches of 768
  (five chunks of 768 and a ragged one of 256: vision GEMMs at M = 768 x 98 = 75 264 and 256 x 98 =
  25 088 - 98 kept patches, no class token - weight gradients with K = 75 264, attention at (768, 98,
  12) and (768, 78, 8) with pad masks), depth 2:
  every layer issues the same calls, so more depth only repeats signatures;
- cfg3 dcl_extra at bench's 8192 pairs in micro-batches of 1024, depth 2;
- cfg2: the README model at 1024 pairs, single pass, text n = 257;
- cfg4: FILIP on the README model at 256 pairs, single pass;
- one AdamW step over the parameters of the full-depth cfg3 model;
- the retention plan of cfg3 at depth 12: "auto", three compact chunks, one full chunk, each against
  the step that re-encodes every chunk.
The first call of every kernel signature is checked; a call of a wrapper with no fp64 check fails the
workload and is named.  A self-test feeds the GEMM check two wrong outputs and requires that it
rejects both.

Measured on an H100 80GB HBM3 (700 W power limit), each test with its fp64 references: run time and
peak allocated memory cfg3 nce 15 s / 44.6 GiB, cfg3 dcl_extra 7 s / 39.7 GiB, cfg2 7 s / 39.0 GiB,
cfg4 FILIP 5 s / 13.2 GiB, AdamW (191 666 433 parameters) 3 s / 8.4 GiB, retention plans 8 s / 64.8 GiB,
self-test 2 s / 4.4 GiB; the file runs in about 65 s.  NEED_GIB holds each peak plus about 10 %: a
test skips, naming both numbers, when less is free on the shared device.  Worst gate ratios over the
four step workloads: gemm 0.986, ff_up / ff_down / ff_bwd 0.992, layernorm_fwd / _bwd 0.992, attn_fwd
0.558, attn_bwd 0.981, l2norm_fwd 0.463, l2norm_bwd 0.991, nce_fwd 0.036, nce_bwd 0.493,
text_embed_bwd 0.326, colsum_rows_ 0.005, scatter_add_rows_ 0.003, ff_bwd_prep 0.004, ff_w2_grad_post_
0.013, filip_segmax16 0.052, filip_reduce 0.217, filip_nce_fwd 0.054, filip_nce_bwd 0.015; bit-exact
calls (casts, embedding forward, patch gather, expand16) exact.  The ratios near 1 are bf16 outputs at
the rounding bound.  AdamW p 0.554.  Retention plans: every gradient within 0.0004 of its 2e-3 gate;
"auto" kept four compact chunks of six.

The GEMM gate's accumulation term is the larger of GAMMA S and gemm_oracle.chain_bound, four ulp per
MMA of each element's running partial sum along its split's k-block chain.  With GAMMA alone, the
latent data gradient g @ hi at K = 8192 (dcl_extra) erred by 4.1 x its gate and a weight gradient of
1568 k-blocks in one chain by 1.8 x; under the chain bound the latent gradient uses 0.43 of it.  The
self-test's unsplit weight gradient of 1176 k-blocks uses 0.095 of its gate, and the same call with
its first or last k-block dropped 63 and 62 gates.
"""
import gc
import math
import time

import pytest
import torch

import bench_call_oracle as BC
import gemm_oracle as GO

pytestmark = pytest.mark.gpu

# free device memory (GiB) each test needs: its measured peak plus 10 %
NEED_GIB = {"cfg3_nce": 49, "cfg3_dcl_extra": 44, "cfg2": 43, "cfg4_filip": 15, "adamw": 10, "retention": 71,
            "self_test": 5}


def _need(what):
    gc.collect()
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < NEED_GIB[what] * 2 ** 30:
        pytest.skip(f"{what} needs {NEED_GIB[what]} GiB of free device memory, {free / 2 ** 30:.1f} GiB free")


def _start():
    gc.collect()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    return time.time()


def _report(what, t0):
    torch.cuda.synchronize()
    print(f"RUN {what}: {time.time() - t0:.1f} s, peak allocated {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB",
          flush=True)


def _data(cfg, batch, dev):
    gd = torch.Generator(device=dev).manual_seed(1)
    S, V, I = cfg["text_seq_len"], cfg["num_text_tokens"], cfg["visual_image_size"]
    text = torch.randint(0, V, (batch, S), generator=gd, device=dev)
    image = torch.randn(batch, 3, I, I, generator=gd, device=dev)
    return text, image


def _step(dev, monkeypatch, what, cfg, loss_kw, batch, microbatch, drop=0.5):
    import x_clip_b200
    from x_clip_b200 import kernels
    _need(what)
    t0 = _start()
    rec = BC.Recorder(kernels).install(monkeypatch)
    torch.manual_seed(0)
    clip = x_clip_b200.CLIP(**cfg, **loss_kw, visual_patch_dropout=drop, microbatch=microbatch or None).to(dev)
    clip.train()
    text, image = _data(cfg, batch, dev)
    loss = clip(text, image, return_loss=True)
    loss.backward()
    _report(what, t0)
    assert math.isfinite(loss.item())
    return rec, clip


def _verdict(rec, what):
    families = sorted({lab.split("[")[0] for lab, _ in rec.results})
    print(f"WORST {what}: " + " ".join(f"{f} {rec.worst(f):.3f}" for f in families))
    assert not rec.unchecked, f"{what}: kernel calls with no fp64 check: {dict(rec.unchecked)}"
    bad = rec.failures()
    assert not bad, f"{what}: {len(bad)} outputs outside their gates: {bad[:10]}"


def _seen(rec, name, **want):
    """Whether a checked call of `name` had every argument in `want`: a tuple is a tensor's shape, a
    callable a predicate on the argument."""
    for (nm, _), A in rec.arguments.items():
        if nm != name:
            continue
        if all((f(A.get(k)) if callable(f) else A.get(k) == f) for k, f in want.items()):
            return True
    return False


def _shape(*s):
    return lambda t: t is not None and tuple(t.shape) == s


def test_cfg3_nce_step(cuda_device, monkeypatch):
    import bench
    cfg = dict(bench.VITB16_CFG, text_enc_depth=2, visual_enc_depth=2)
    d = bench.DEFAULTS["cfg3"]
    rec, clip = _step(cuda_device, monkeypatch, "cfg3_nce", cfg, bench.LOSS_KW["nce"], d["batch"], d["microbatch"])
    print("plan", clip.last_step_plan)
    assert clip.last_step_plan["chunks"] == 6
    for M in (75264, 25088):                                     # 768 x 98 and 256 x 98 vision rows
        assert _seen(rec, "gemm", a=_shape(M, 768), a_major=0), M
        assert _seen(rec, "gemm", a=lambda t, M=M: t is not None and t.shape[0] == M, a_major=1, b_major=1), M
        assert _seen(rec, "ff_up", x=_shape(M, 768)) and _seen(rec, "ff_bwd", dx=_shape(M, 768)), M
        assert _seen(rec, "layernorm_fwd", x=_shape(M, 768)) and _seen(rec, "layernorm_bwd", x=_shape(M, 768)), M
    assert _seen(rec, "attn_fwd", B=768, n=98, heads=12) and _seen(rec, "attn_bwd", B=768, n=98, heads=12)
    masked = lambda m: m is not None                             # noqa: E731
    assert _seen(rec, "attn_fwd", B=768, n=78, heads=8, key_mask=masked)
    assert _seen(rec, "attn_bwd", B=768, n=78, heads=8, key_mask=masked)
    assert _seen(rec, "text_embed_bwd", vocab=49408)
    assert _seen(rec, "patchify_gather") and _seen(rec, "scatter_add_rows_") and _seen(rec, "colsum_rows_")
    assert _seen(rec, "l2norm_fwd", p=_shape(768, 512)) and _seen(rec, "l2norm_fwd", p=_shape(256, 512))
    assert _seen(rec, "nce_fwd", a=_shape(4096, 1536), b=_shape(4096, 1536))
    assert _seen(rec, "nce_bwd", a=_shape(4096, 1536), b=_shape(4096, 1536))
    _verdict(rec, "cfg3_nce")


def test_cfg3_dcl_extra_step(cuda_device, monkeypatch):
    import bench
    cfg = dict(bench.VITB16_CFG, text_enc_depth=2, visual_enc_depth=2)
    rec, clip = _step(cuda_device, monkeypatch, "cfg3_dcl_extra", cfg, bench.LOSS_KW["dcl_extra"], 8192, 1024)
    assert clip.last_step_plan["chunks"] == 8
    assert _seen(rec, "nce_bwd", dcl=True, w_col=0.0) and _seen(rec, "nce_bwd", dcl=True, w_row=0.0)
    _verdict(rec, "cfg3_dcl_extra")


def test_cfg2_step(cuda_device, monkeypatch):
    import bench
    d = bench.DEFAULTS["cfg2"]
    rec, _ = _step(cuda_device, monkeypatch, "cfg2", bench.README_CFG, bench.LOSS_KW["nce"], d["batch"],
                   d["microbatch"])
    assert _seen(rec, "attn_fwd", B=1024, n=257, heads=8) and _seen(rec, "attn_bwd", B=1024, n=257, heads=8)
    _verdict(rec, "cfg2")


def test_cfg4_filip_step(cuda_device, monkeypatch):
    import bench
    rec, _ = _step(cuda_device, monkeypatch, "cfg4_filip", bench.README_CFG, bench.LOSS_KW["filip"], 256, 0)
    for name in ("filip_segmax16", "filip_reduce", "filip_nce_fwd", "filip_nce_bwd", "filip_expand16"):
        assert _seen(rec, name), name
    _verdict(rec, "cfg4_filip")


def test_adamw_step_over_cfg3_parameters(cuda_device, monkeypatch):
    """One FusedAdamW step (step 2, so the moments are non-zero) over every parameter of the full-depth
    cfg3 model, with gradients spread over six orders of magnitude."""
    import bench
    import x_clip_b200
    from x_clip_b200 import kernels
    from x_clip_b200.optim import FusedAdamW
    _need("adamw")
    t0 = _start()
    torch.manual_seed(0)
    clip = x_clip_b200.CLIP(**bench.VITB16_CFG).to(cuda_device)
    opt = FusedAdamW(clip.parameters(), lr=1e-3, weight_decay=0.05)
    n = sum(p.numel() for p in opt.params)
    gen = torch.Generator(device=cuda_device).manual_seed(2)
    for p in opt.params:
        p.grad = torch.randn(p.shape, generator=gen, device=cuda_device) * 10.0 ** (
            -6 * torch.rand(p.shape, generator=gen, device=cuda_device))
    opt.step()
    for p in opt.params:
        p.grad = torch.randn(p.shape, generator=gen, device=cuda_device) * 1e-3
    rec = BC.Recorder(kernels).install(monkeypatch)
    opt.step()
    _report("adamw", t0)
    print(f"AdamW over {n} parameters ({opt.flat.numel()} with padding)")
    assert n > 1.4e8 and _seen(rec, "adamw_step_", step=2)
    _verdict(rec, "adamw")


# --------------------------------------------------------------------------- retention plan

def _rel(a, b):
    d = b.double().norm().item()
    return (a.double() - b.double()).norm().item() / (d if d > 0 else 1.0)


def test_retention_plans_at_full_depth(cuda_device, monkeypatch):
    """cfg3 at depth 12, 4096 pairs in chunks of 768: the "auto" plan (whatever it plans from the free
    HBM), three compact chunks (RETAIN_MODE = "compact", retain = 3) and one full chunk (retain = 1),
    each against retain = 0 (every chunk re-encoded in backward) from the same weights, data and RNG
    state: loss within 1e-5 relative, every parameter's gradient within 2e-3 relative Frobenius."""
    import bench
    import x_clip_b200
    from x_clip_b200 import engine as E
    _need("retention")
    dev = cuda_device
    t0 = _start()
    torch.manual_seed(0)
    clip = x_clip_b200.CLIP(**bench.VITB16_CFG, visual_patch_dropout=0.5, microbatch=768,
                            microbatch_retain=0).to(dev)
    clip.train()
    text, image = _data(bench.VITB16_CFG, 4096, dev)
    rng = (torch.get_rng_state(), torch.cuda.get_rng_state(dev))
    params = dict(clip.named_parameters())

    def step(retain, mode):
        monkeypatch.setattr(E, "RETAIN_MODE", mode)
        clip.microbatch_retain = retain
        for p in params.values():
            p.grad = None
        torch.set_rng_state(rng[0])
        torch.cuda.set_rng_state(rng[1], dev)
        loss = clip(text, image, return_loss=True)
        loss.backward()
        torch.cuda.synchronize()
        print(f"retain={retain} mode={mode}: plan {clip.last_step_plan}", flush=True)
        return loss.item(), dict(clip.last_step_plan)

    ref_loss, plan = step(0, None)
    assert plan["chunks"] == 6 and plan["retained_chunks"] == []
    ref = {k: p.grad.clone() for k, p in params.items() if p.grad is not None}
    for retain, mode, kept, compact in (("auto", None, None, None), (3, "compact", [0, 1, 2], [0, 1, 2]),
                                        (1, None, [0], [])):
        loss, plan = step(retain, mode)
        if kept is not None:
            assert plan["retained_chunks"] == kept and plan["compact_chunks"] == compact, plan
        assert plan["oom_fallbacks"] == 0, plan
        assert abs(loss - ref_loss) <= 1e-5 * abs(ref_loss), (retain, loss, ref_loss)
        worst = 0.0
        for k, p in params.items():
            assert (p.grad is None) == (k not in ref), k
            if p.grad is not None:
                r = _rel(p.grad, ref[k])
                worst = max(worst, r)
                assert r <= 2e-3, (retain, mode, k, r)
        print(f"GATE retention_{retain}_{mode or 'unforced'} {worst / 2e-3:.4f}")
    _report("retention", t0)


# --------------------------------------------------------------------------- the checker itself

def _gemm_check_ratio(got, a, b, **kw):
    """The ratio bench_call_oracle's GEMM check gives `got` as the result of K.gemm(a, b, **kw); an
    accumulated call is taken to start from zeros."""
    import inspect
    from x_clip_b200 import kernels as K
    ba = inspect.signature(K.gemm).bind(a, b, **kw)
    ba.apply_defaults()
    before = {"out": torch.zeros_like(got)} if kw.get("accumulate") else {}
    return BC.CHECKS["gemm"].check(dict(ba.arguments), before, got)[""]


def test_checker_rejects_wrong_gemm_outputs(cuda_device):
    """The GEMM check of bench_call_oracle accepts the kernel's output and rejects a wrong one at the
    shapes it covers:
    - the ragged chunk's QKV projection (M = 256 x 98 = 25 088, N = 2304, K = 768): the kernel's output
      with the last 64 columns of K dropped, and the output with its rows shifted by one;
    - the unsplit weight gradient of the cfg3 feed-forward up-projection (dW1 = du^T xn2: both operands
      MN-major, accumulated into a [6144, 768] fp32 output, K = 768 x 98 = 75 264, one chain of 1176
      k-blocks per tile): the kernel's output with the first and with the last 64-wide k-block of the
      chain dropped, where the accumulation gate is the chain bound, not GAMMA."""
    from x_clip_b200 import kernels as K
    _need("self_test")
    t0 = _start()
    dev = cuda_device
    M, N, K_ = 25088, 2304, 768
    a, b = GO.operands(M, N, K_, 0, 0, seed=5)
    a, b = a.to(dev), b.to(dev)
    good = K.gemm(a, b)
    short = K.gemm(a[:, :K_ - 64].contiguous(), b[:, :K_ - 64].contiguous())
    torch.cuda.synchronize()
    r = {"qkv_good": _gemm_check_ratio(good, a, b), "qkv_k_minus_64": _gemm_check_ratio(short, a, b),
         "qkv_rows_shifted": _gemm_check_ratio(good.roll(1, dims=0), a, b)}
    del a, b, good, short

    M, N, K_ = 6144, 768, 75264
    plan = GO.split_plan(M, N, K_, True, BC.sms())
    assert plan["splits"] == 1 and plan["kb_per"] == 1176, plan
    gen = torch.Generator(device=dev).manual_seed(6)

    def operand(rows):          # stored MN-major [K, rows], logical rows scaled over three decades
        t = torch.randn(K_, rows, generator=gen, device=dev)
        return (t * 10.0 ** (-3.0 * torch.rand(1, rows, generator=gen, device=dev))).bfloat16()

    du, xn2 = operand(M), operand(N)
    kw = dict(a_major=1, b_major=1, accumulate=True)
    good = K.gemm(du, xn2, **kw)
    no_last = K.gemm(du[:K_ - 64], xn2[:K_ - 64], **kw)
    no_first = K.gemm(du[64:], xn2[64:], **kw)
    torch.cuda.synchronize()
    r.update(wgrad_good=_gemm_check_ratio(good, du, xn2, **kw),
             wgrad_last_k_block_dropped=_gemm_check_ratio(no_last, du, xn2, **kw),
             wgrad_first_k_block_dropped=_gemm_check_ratio(no_first, du, xn2, **kw))
    _report("self_test", t0)
    for k, v in r.items():
        print(f"GATE selftest_gemm_{k} {v:.4f}")
    assert r["qkv_good"] <= 1.0 and r["wgrad_good"] <= 1.0, r
    assert min(v for k, v in r.items() if not k.endswith("good")) > 1.0, r
