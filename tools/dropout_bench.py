"""Cost of attention dropout (xclip_attn_dropout_fwd / _bwd) against the plain kernels.

1. Attention forward and backward at the cfg3 shapes - image tower with patch dropout 0.5 (B 512, n 99,
   H 12) and text tower (B 512, n 78, H 8) - and one streaming shape (B 32, n 577, H 12), at p = 0 (the
   plain kernels) and p = 0.1.  CUDA-event time per call.
2. A cfg3-shaped ViT-B/16 image tower (768 wide, 12 heads, 12 layers, 224 px / 16, patch dropout 0.5)
   on a micro-batch of 256 images, forward + backward, at attn_dropout 0 and 0.1.

The variants alternate inside every round and the rounds repeat (--rounds); the median and the spread
over the rounds are printed.  The card's name, power limit and SM clock limit are read in the same run.

    python tools/dropout_bench.py [--rounds 5] [--reps 50] [--json out.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

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
    fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def attn_variants(B, n, H, dev):
    g = torch.Generator(device=dev).manual_seed(0)
    qkv = torch.randn(B * n, 3 * H * 64, device=dev, generator=g).bfloat16()
    d_o = torch.randn(B * n, H * 64, device=dev, generator=g).bfloat16()
    mask = torch.rand(B, n, device=dev, generator=g) > 0.2
    mask[:, 0] = True
    seed = torch.tensor([12345], dtype=torch.int64, device=dev)
    out = {}
    for p in (0.0, 0.1):
        dr = None if p == 0 else (p, seed, 0)
        o, lse = K.attn_fwd(qkv, mask, B, n, H, 0.125, dropout=dr)
        out[f"fwd p{p}"] = lambda dr=dr: K.attn_fwd(qkv, mask, B, n, H, 0.125, dropout=dr)
        out[f"bwd p{p}"] = lambda dr=dr, o=o, lse=lse: K.attn_bwd(qkv, mask, o, d_o, lse, B, n, H, 0.125, dropout=dr)
    return out


def tower_variants(batch, dev):
    import x_clip_b200
    torch.manual_seed(0)
    vit = x_clip_b200.VisionTransformer(768, image_size=224, patch_size=16, channels=3, dim_head=64, depth=12,
                                        heads=12, patch_dropout=0.5, attn_dropout=0.1).to(dev).train()
    img = torch.randn(batch, 3, 224, 224, device=dev)

    def step(p):
        for attn, _ in vit.transformer.layers:
            attn.fn.dropout.p = p
        out = vit(img)
        out.float().square().mean().backward()
    return {f"tower p{p}": (lambda p=p: step(p)) for p in (0.0, 0.1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--tower-reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    res = dict(card=card(), shapes={})
    groups = [(f"attn B{B} n{n} H{H}", attn_variants(B, n, H, dev), a.reps)
              for B, n, H in ((512, 99, 12), (512, 78, 8), (32, 577, 12))]
    groups.append(("vit-b16 tower mb256", tower_variants(256, dev), a.tower_reps))
    for name, variants, reps in groups:
        times = {k: [] for k in variants}
        for _ in range(a.rounds):
            for k, fn in variants.items():
                times[k].append(timeit(fn, reps))
        summ = {k: dict(ms=statistics.median(v), spread=(max(v) - min(v)) / statistics.median(v))
                for k, v in times.items()}
        res["shapes"][name] = summ
        for k, v in summ.items():
            print(f"{name:24s} {k:10s} {v['ms']:9.4f} ms  (spread {100 * v['spread']:.1f} %)")
        for kind in ("fwd", "bwd", "tower"):
            if f"{kind} p0.0" in summ:
                r = summ[f"{kind} p0.1"]["ms"] / summ[f"{kind} p0.0"]["ms"]
                print(f"{name:24s} {kind} ratio p0.1 / p0: {r:.3f}")
    print("card:", res["card"])
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
