"""Cost of the image gradient: the patchify_scatter kernel and a cfg3-shaped vision tower in three modes.

1. xclip_patchify_scatter at cfg3 chunk shapes (768 x 3 x 224 x 224, patch 16) with patch dropout 0 and
   0.5: CUDA-event time per call and GB/s = bytes the kernel must move (the kept rows read, the whole
   image gradient written, keep read) / time.
2. The ViT-B/16 image tower of cfg3 (768 wide, 12 heads, 12 layers, 224 px / 16, patch dropout 0.5) on a
   micro-batch of 768 images, forward + backward of (cls output . fixed target), in three modes:
     a. parameter gradients only (a training step's vision tower);
     b. parameter and image gradients;
     c. frozen parameters, torch.autograd.grad(objective, image) (one PGD step).
   Wall time per call (CUDA-synchronised) and, in a separate profiled pass, the time of each kernel
   family from x_clip_b200.kernels.PROF.

The card's name, power limit and SM clock limit are read in the same run and printed with the numbers.

    python tools/image_grad_bench.py [--batch 768] [--reps 50] [--steps 10] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from x_clip_b200 import kernels as K  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
    except (OSError, subprocess.TimeoutExpired, IndexError):
        q = torch.cuda.get_device_name(0) + ", power limit unknown, clock unknown"
    return q


def timeit(fn, reps):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps       # ms


def scatter_bench(batch, reps, dev):
    out = []
    C, H, W, P = 3, 224, 224, 16
    n = (H // P) * (W // P)
    pd = P * P * C
    for drop in (0.0, 0.5):
        g = torch.Generator(device=dev).manual_seed(1)
        keep = None if drop == 0 else torch.randn(batch, n, device=dev, generator=g).topk(
            max(1, int(n * (1 - drop))), dim=-1).indices
        k = n if keep is None else keep.shape[1]
        src = torch.randn(batch * k, pd, device=dev, generator=g)
        ms = timeit(lambda: K.patchify_scatter(src, (batch, C, H, W), P, keep), reps)
        nbytes = 4.0 * batch * k * pd + 4.0 * batch * n * pd + (0 if keep is None else 8.0 * batch * k)
        out.append(dict(patch_dropout=drop, kept=k, ms=ms, gbps=nbytes / ms / 1e6, bytes=nbytes))
    return out


def tower(dev):
    from x_clip_b200.clip import VisionTransformer
    torch.manual_seed(0)
    vt = VisionTransformer(768, image_size=224, patch_size=16, channels=3, depth=12, heads=12, dim_head=64,
                           patch_dropout=0.5).to(dev)
    vt.train()
    return vt


def tower_bench(batch, steps, dev):
    vt = tower(dev)
    g = torch.Generator(device=dev).manual_seed(2)
    image = torch.randn(batch, 3, 224, 224, device=dev, generator=g)
    target = torch.randn(batch, 768, device=dev, generator=g)

    def run(mode):
        vt.requires_grad_(mode != "c")
        for p in vt.parameters():
            p.grad = None
        x = image.clone().requires_grad_(mode != "a")
        obj = (vt(x)[:, 0].float() * target).sum()
        if mode == "c":
            torch.autograd.grad(obj, x)
        else:
            obj.backward()

    res = {}
    modes = ("a", "b", "c")
    for m in modes:                          # warm-up: every shape of every mode
        for _ in range(2):
            run(m)
    torch.cuda.synchronize()
    times = {m: [] for m in modes}
    for _ in range(steps):                   # interleaved, so drift of the shared host hits all modes alike
        for m in modes:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(m)
            torch.cuda.synchronize()
            times[m].append((time.perf_counter() - t0) * 1e3)
    for m in modes:
        K.PROF.start()
        run(m)
        fam = K.PROF.stop()
        ts = sorted(times[m])
        res[m] = dict(ms_median=ts[len(ts) // 2], ms_min=ts[0], ms_max=ts[-1],
                      families={k: dict(calls=v["calls"], ms=round(v["ms"], 3)) for k, v in sorted(fam.items())})
    res["b_over_a"] = res["b"]["ms_median"] / res["a"]["ms_median"]
    res["c_over_a"] = res["c"]["ms_median"] / res["a"]["ms_median"]
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--batch", type=int, default=768)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("image_grad_bench.py measures on the GPU; no CUDA device found")
    dev = torch.device("cuda:0")
    from x_clip_b200 import _lib
    _lib.call("xclip_init")
    out = dict(card=card(), batch=a.batch)
    print("card:", out["card"])
    out["scatter"] = scatter_bench(a.batch, a.reps, dev)
    for r in out["scatter"]:
        print(f"patchify_scatter drop {r['patch_dropout']}: {r['ms']:.3f} ms  {r['gbps']:.0f} GB/s")
    out["tower"] = tower_bench(a.batch, a.steps, dev)
    for m in ("a", "b", "c"):
        r = out["tower"][m]
        print(f"mode {m}: {r['ms_median']:.1f} ms (min {r['ms_min']:.1f}, max {r['ms_max']:.1f})")
        print("   ", {k: v["ms"] for k, v in r["families"].items()})
    print(f"b/a {out['tower']['b_over_a']:.4f}  c/a {out['tower']['c_over_a']:.4f}")
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
