"""Time the wgmma GEMM at the shapes of the bench workloads.

    python tools/gemm_bench.py            (cfg3 micro-batch 512 and cfg2 shapes)"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from x_clip_b200 import _lib, kernels as K  # noqa: E402

dev = torch.device("cuda:0")
lib = _lib.load()
# (label, M, N, K, a_major, b_major, accumulate)
T3, T3t = 512 * 98, 512 * 78
SHAPES = [
    ("vit qkv fwd", T3, 2304, 768, 0, 0, False), ("vit out fwd", T3, 768, 768, 0, 0, False),
    ("vit ff-up fwd", T3, 6144, 768, 0, 0, False), ("vit ff-down fwd", T3, 768, 3072, 0, 0, False),
    ("vit ff-up dgrad", T3, 768, 6144, 0, 1, False), ("vit ff-down dgrad", T3, 3072, 768, 0, 1, False),
    ("vit ff-up wgrad", 6144, 768, T3, 1, 1, True), ("vit ff-down wgrad", 768, 3072, T3, 1, 1, True),
    ("text ff-up fwd", T3t, 4096, 512, 0, 0, False), ("text qkv fwd", T3t, 1536, 512, 0, 0, False),
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


for (label, M, N, Kd, am, bm, acc) in SHAPES:
    g = torch.Generator().manual_seed(0)
    a = torch.randn((M, Kd) if am == 0 else (Kd, M), generator=g).to(dev).bfloat16()
    b = torch.randn((N, Kd) if bm == 0 else (Kd, N), generator=g).to(dev).bfloat16()
    out = torch.zeros(M, N, device=dev, dtype=torch.float32 if acc else torch.bfloat16)
    ms = timeit(lambda: K.gemm(a, b, a_major=am, b_major=bm, out=out, accumulate=acc))
    fl = 2.0 * M * N * Kd
    print(f"{label:22s} M={M} N={N} K={Kd}: {ms:.3f} ms {fl / ms / 1e9:7.1f} TF/s", flush=True)
