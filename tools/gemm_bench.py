"""Time the wgmma GEMM at the shapes of the bench workloads.

    python tools/gemm_bench.py            (cfg3 micro-batch 768 and cfg2 shapes, then a K sweep)"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from x_clip_b200 import _lib, kernels as K  # noqa: E402

dev = torch.device("cuda:0")
lib = _lib.load()
# (label, M, N, K, a_major, b_major, accumulate)
T3, T3t = 768 * 98, 768 * 78
SHAPES = [
    ("vit qkv fwd", T3, 2304, 768, 0, 0, False), ("vit out fwd", T3, 768, 768, 0, 0, False),
    ("vit ff-up fwd", T3, 6144, 768, 0, 0, False), ("vit ff-down fwd", T3, 768, 3072, 0, 0, False),
    ("vit qkv dgrad", T3, 768, 2304, 0, 1, False), ("vit out dgrad", T3, 768, 768, 0, 1, False),
    ("vit ff-up dgrad", T3, 768, 6144, 0, 1, False), ("vit ff-down dgrad", T3, 3072, 768, 0, 1, False),
    ("vit qkv wgrad", 2304, 768, T3, 1, 1, True), ("vit out wgrad", 768, 768, T3, 1, 1, True),
    ("vit ff-up wgrad", 6144, 768, T3, 1, 1, True), ("vit ff-down wgrad", 768, 3072, T3, 1, 1, True),
    ("text qkv fwd", T3t, 1536, 512, 0, 0, False), ("text out fwd", T3t, 512, 512, 0, 0, False),
    ("text ff-up fwd", T3t, 4096, 512, 0, 0, False), ("text qkv dgrad", T3t, 512, 1536, 0, 1, False),
    ("text out dgrad", T3t, 512, 512, 0, 1, False), ("text qkv wgrad", 1536, 512, T3t, 1, 1, True),
    ("cfg2 text ff-up fwd", 263168, 4096, 512, 0, 0, False),
]


def timeit(fn, reps=10):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def run(label, M, N, Kd, am, bm, acc):
    g = torch.Generator().manual_seed(0)
    a = torch.randn((M, Kd) if am == 0 else (Kd, M), generator=g).to(dev).bfloat16()
    b = torch.randn((N, Kd) if bm == 0 else (Kd, N), generator=g).to(dev).bfloat16()
    out = torch.zeros(M, N, device=dev, dtype=torch.float32 if acc else torch.bfloat16)
    ms = timeit(lambda: K.gemm(a, b, a_major=am, b_major=bm, out=out, accumulate=acc))
    fl = 2.0 * M * N * Kd
    print(f"{label:22s} M={M} N={N} K={Kd}: {ms:.3f} ms {fl / ms / 1e9:7.1f} TF/s", flush=True)
    return ms


for shape in SHAPES:
    run(*shape)

# K sweep at a fixed output (cfg3 micro-batch 768 ViT tokens x d): every CTA runs the same number of
# tiles, so time = waves * (a + b * k-blocks); the intercept a is the fixed cost of a tile (prologue,
# epilogue, pipeline drain) that the k-loop does not hide.
M_SW, N_SW = 768 * 98, 768
sms = torch.cuda.get_device_properties(dev).multi_processor_count
for bn in (128, 256):
    waves = -(-(-(-M_SW // 128) * (N_SW // bn)) // sms)
    print(f"K sweep M={M_SW} N={N_SW}: {waves} tiles per CTA at BLOCK_N {bn}", flush=True)
ks = [256, 512, 768, 1536, 3072]
ts = [run("K sweep", M_SW, N_SW, k, 0, 0, False) for k in ks]
kbs = [k / 64 for k in ks]
n = len(ks)
mk, mt = sum(kbs) / n, sum(ts) / n
slope = sum((x - mk) * (y - mt) for x, y in zip(kbs, ts)) / sum((x - mk) ** 2 for x in kbs)
icpt = mt - slope * mk
print(f"K sweep fit: time = {icpt:.4f} ms + {slope * 1e3:.3f} us * k-blocks "
      f"(intercept = {100 * icpt / ts[ks.index(768)]:.1f} % of K=768)", flush=True)
