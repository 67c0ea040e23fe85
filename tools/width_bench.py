"""Row-wise kernels at every model width 128 * {1..8}, and one training step of a ViT-S/16 CLIP.

1. LayerNorm forward (plain, and with residual + chained second norm), LayerNorm backward (with dg),
   l2norm forward / backward and ff_bwd_prep, each on ROWS rows of each width.  GB/s = bytes the
   kernel must move (computed from the shapes below) / CUDA-event time per call.
2. A ViT-S/16 CLIP step (image 384 wide, 6 heads, 12 layers, 224 px / 16, patch dropout 0.5; text 384
   wide, 6 heads, 12 layers, 77 tokens; latent 384): forward + backward as bench.py times it, pairs/s
   and peak allocation.

The card's name, power limit and SM clock limit are read in the same run and printed with the numbers.

    python tools/width_bench.py [--rows 262144] [--widths 128,...,1024] [--repeat 1] [--batch 1024]
                                [--microbatch 512] [--steps 5] [--skip-step] [--json out.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from x_clip_b200 import kernels as K  # noqa: E402

WIDTHS = [128 * k for k in range(1, 9)]
BF, F32 = 2, 4


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


def row_kernels(rows, reps, dev, widths=WIDTHS):
    out = []
    for d in widths:
        g = torch.Generator(device=dev).manual_seed(d)
        x = torch.randn(rows, d, device=dev, generator=g).bfloat16()
        r = torch.randn(rows, d, device=dev, generator=g).bfloat16()
        dy = torch.randn(rows, d, device=dev, generator=g).bfloat16()
        gain = 1 + 0.1 * torch.randn(d, device=dev, generator=g)
        p = torch.randn(rows, d, device=dev, generator=g)
        dz = torch.randn(rows, d, device=dev, generator=g)
        _, st, _, _ = K.layernorm_fwd(x, gain)
        z, _, _, inv = K.l2norm_fwd(p)
        acc = torch.randn(rows, d, device=dev, generator=g).bfloat16()
        colvec = torch.randn(d, device=dev, generator=g)
        dg = torch.zeros(d, device=dev)
        n = rows * d
        cases = [
            # name, call, bytes moved
            ("ln_fwd", lambda: K.layernorm_fwd(x, gain), n * (BF + BF) + rows * 2 * F32),
            ("ln_fwd_res_chain", lambda: K.layernorm_fwd(x, gain, res=r, g2=gain),
             n * 4 * BF + rows * 4 * F32),
            ("ln_bwd", lambda: K.layernorm_bwd(dy, x, st, gain, dg=dg), n * 3 * BF + rows * 2 * F32),
            ("l2norm_fwd", lambda: K.l2norm_fwd(p), n * (F32 + F32 + 6 * BF) + rows * F32),
            ("l2norm_bwd", lambda: K.l2norm_bwd(dz, z, inv), n * (2 * F32 + BF) + rows * F32),
            ("ff_bwd_prep", lambda: K.ff_bwd_prep(dy, st, acc, colvec),
             n * 3 * BF + rows * 4 * F32),
        ]
        for name, fn, nbytes in cases:
            ms = timeit(fn, reps)
            out.append(dict(kernel=name, d=d, rows=rows, us=round(ms * 1e3, 2), gbps=round(nbytes / ms / 1e6, 1)))
            print(f"{name:17s} d={d:4d} rows={rows}: {ms * 1e3:8.1f} us  {nbytes / ms / 1e6:7.0f} GB/s", flush=True)
    return out


VITS16 = dict(dim_text=384, dim_image=384, dim_latent=384, num_text_tokens=49408, text_enc_depth=12,
              text_seq_len=77, text_heads=6, visual_enc_depth=12, visual_heads=6,
              visual_image_size=224, visual_patch_size=16)


def vits_step(batch, microbatch, steps, dev):
    import x_clip_b200
    torch.manual_seed(0)
    clip = x_clip_b200.CLIP(**VITS16, visual_patch_dropout=0.5, microbatch=microbatch or None).to(dev)
    clip.train()
    text = torch.randint(1, VITS16["num_text_tokens"], (batch, VITS16["text_seq_len"]), device=dev)
    image = torch.randn(batch, 3, 224, 224, device=dev)
    params = [p for p in clip.parameters() if p.requires_grad]

    def step():
        for q in params:
            q.grad = None
        loss = clip(text, image, return_loss=True)
        loss.backward()
        return loss

    step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    ms = timeit(step, steps)
    peak = torch.cuda.max_memory_allocated(dev) / 2 ** 30
    loss = step().item()
    res = dict(batch=batch, microbatch=microbatch or None, ms_per_step=round(ms, 2),
               pairs_per_s=round(batch / (ms / 1e3), 1), peak_gib=round(peak, 2), loss=round(loss, 5))
    print(f"ViT-S/16 CLIP step, batch {batch}, micro-batch {microbatch or 'none'}: {ms:.1f} ms, "
          f"{res['pairs_per_s']} pairs/s, peak allocation {peak:.2f} GiB, loss {loss:.4f}", flush=True)
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--rows", type=int, default=262144)
    ap.add_argument("--widths", default=",".join(map(str, WIDTHS)), help="comma-separated subset of 128..1024")
    ap.add_argument("--repeat", type=int, default=1, help="sweep the widths this many times")
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--microbatch", type=int, default=512)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--skip-step", action="store_true")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("width_bench needs a CUDA device: no number is measured without one")
    dev = torch.device("cuda:0")
    c = card()
    print(f"card: {c}", flush=True)
    widths = [int(w) for w in a.widths.split(",")]
    assert all(w in WIDTHS for w in widths), widths
    out = dict(card=c, rows=[r for _ in range(a.repeat) for r in row_kernels(a.rows, a.reps, dev, widths)])
    if not a.skip_step:
        out["vits16_step"] = vits_step(a.batch, a.microbatch, a.steps, dev)
    print(f"card: {c}", flush=True)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
