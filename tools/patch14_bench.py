"""Patch 14 on the H100: the patch-embedding front end and a ViT-L/14 CLIP training step.

1. xclip_patchify_gather(_rows) and xclip_patchify_scatter(_rows) at 224 / 14 and 336 / 14 (588 values
   per patch, rows padded to 592) against 224 / 16 (768 values), on the same number of images, with patch
   dropout 0 and 0.5.  GB/s from the shapes: the gather reads the kept patches' f32 pixels and writes
   their bf16 rows (padding included); the scatter reads the kept f32 rows and writes the whole f32 image.
2. The patch-embedding GEMM (xclip_gemm_bf16) at K = 588 run as K = 592, against K = 768: forward
   (M x 1024 tokens) and weight gradient (1024 x K, split-K over M).  TFLOP/s count the useful K
   (588 / 768), the padded columns are overhead.
3. A ViT-L/14 CLIP training step: image tower 1024 wide, 16 heads, 24 layers at 224 px / 14 (patch
   dropout 0.5: 128 of 256 patches), causal 77-token text tower 768 wide, 12 heads, 12 layers, EOS
   pooling, latent 768; batch 1024 per GPU in micro-batches of 256.  pairs/s and peak allocation.

Prints the card's name, power limit and SM clock limit, then one JSON line per measurement.

    python tools/patch14_bench.py [--images 768] [--reps 50] [--step-batch 1024] [--microbatch 256]
                                  [--steps 3] [--skip-step]
"""
import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def timeit(fn, reps):
    import torch
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def front_end(images, reps, dev):
    import torch
    from x_clip_b200 import kernels as K
    out = []
    for size, P in ((224, 16), (224, 14), (336, 14)):
        C = 3
        n = (size // P) ** 2
        pd = P * P * C
        ld = K.patch_row_stride(pd)
        img = torch.randn(images, C, size, size, device=dev)
        for drop in (0.0, 0.5):
            k = n if drop == 0 else int(n * (1 - drop))
            keep = None if drop == 0 else torch.rand(images, n, device=dev).topk(k, dim=-1).indices
            rows = images * k
            ms_g = timeit(lambda: K.patchify_gather(img, P, keep, ld=ld), reps)
            g_bytes = rows * pd * 4 + rows * ld * 2
            src = torch.randn(rows, ld, device=dev)[:, :pd]
            ms_s = timeit(lambda: K.patchify_scatter(src, img.shape, P, keep), reps)
            s_bytes = rows * pd * 4 + images * C * size * size * 4
            out.append(dict(what="patchify", image=size, patch=P, patch_dim=pd, ld=ld, images=images,
                            patch_dropout=drop, kept=k, gather_ms=round(ms_g, 4),
                            gather_gbps=round(g_bytes / ms_g / 1e6), scatter_ms=round(ms_s, 4),
                            scatter_gbps=round(s_bytes / ms_s / 1e6)))
            del src
        del img
        torch.cuda.empty_cache()
    return out


def gemm(reps, dev):
    import torch
    from x_clip_b200 import kernels as K
    M, N = 256 * 128, 1024          # a micro-batch of 256 images, 128 kept patches each
    out = []
    for kd in (588, 768):
        ld = K.patch_row_stride(kd)
        a = torch.randn(M, ld, device=dev).bfloat16()
        w = torch.randn(N, ld, device=dev).bfloat16()
        dy = torch.randn(M, N, device=dev).bfloat16()
        dw = torch.zeros(N, ld, device=dev)
        ms_f = timeit(lambda: K.gemm(a, w), reps)
        ms_w = timeit(lambda: K.gemm(dy, a, a_major=1, b_major=1, out=dw, accumulate=True), reps)
        fl = 2.0 * M * N * kd
        out.append(dict(what="patch_gemm", M=M, N=N, K=kd, K_run=ld, fwd_ms=round(ms_f, 4),
                        fwd_tflops=round(fl / ms_f / 1e9, 1), wgrad_ms=round(ms_w, 4),
                        wgrad_tflops=round(fl / ms_w / 1e9, 1)))
    return out


def step(batch, microbatch, steps, dev):
    import torch
    import x_clip_b200
    kw = dict(dim_text=768, dim_image=1024, dim_latent=768, num_text_tokens=49408, text_enc_depth=12,
              text_seq_len=77, text_heads=12, visual_enc_depth=24, visual_heads=16,
              visual_image_size=224, visual_patch_size=14, text_causal_mask=True, text_eos_id=49407)
    torch.manual_seed(0)
    clip = x_clip_b200.CLIP(**kw, microbatch=microbatch).to(dev)
    clip.train()
    text = torch.randint(3, 49407, (batch, 77), device=dev)
    text[:, -1] = 49407
    image = torch.randn(batch, 3, 224, 224, device=dev)
    clip(text, image, return_loss=True).backward()
    clip.zero_grad(set_to_none=True)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        loss = clip(text, image, return_loss=True)
        loss.backward()
        clip.zero_grad(set_to_none=True)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    sp = clip.last_step_plan
    return dict(what="vitl14_step", pairs_per_gpu=batch, microbatch=microbatch, steps=steps, step_ms=round(ms, 1),
                pairs_per_s=round(batch / (ms / 1e3), 1),
                peak_alloc_gib=round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 2),
                chunks=sp["chunks"], retained_chunks=sp["retained_chunks"], loss=round(loss.item(), 5))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=768)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--step-batch", type=int, default=1024)
    ap.add_argument("--microbatch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--skip-step", action="store_true")
    a = ap.parse_args()

    import torch
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    dev = torch.device("cuda:0")
    print(json.dumps(dict(card=card())), flush=True)
    for r in front_end(a.images, a.reps, dev) + gemm(a.reps, dev):
        print(json.dumps(r), flush=True)
    if not a.skip_step:
        print(json.dumps(step(a.step_batch, a.microbatch, a.steps, dev)), flush=True)


if __name__ == "__main__":
    main()
