#!/usr/bin/env python
"""Training step of the cfg3 model (bench.py) at 384 px: ViT-B/16 image tower with 576 image tokens per
sample, so image attention runs on the streaming kernels (n = 576 > 320).

    python tools/highres_step.py [--batch 1024] [--microbatch 256] [--steps 5] [--warmup 2]

Patch dropout 0.0 (every patch reaches attention).  Prints one JSON line: ms per step, pairs/s, peak
memory and the micro-batch plan.  A measurement tool, not the bench metric."""
import argparse
import json
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
import torch  # noqa: E402
import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--image-size", type=int, default=384)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--microbatch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cfg = dict(bench.VITB16_CFG, visual_image_size=a.image_size)
    run = bench.Runner(cfg, "nce", a.batch, a.microbatch, 0.0, dev, 0, 1)
    torch.cuda.reset_peak_memory_stats(dev)
    ms, loss = run.timed(a.steps, a.warmup)
    print(json.dumps({
        "gpu": torch.cuda.get_device_name(dev), "image_size": a.image_size,
        "image_tokens": (a.image_size // cfg["visual_patch_size"]) ** 2, "batch": a.batch,
        "microbatch": a.microbatch, "steps": a.steps, "ms_per_step": round(ms / a.steps, 2),
        "pairs_per_s": round(a.batch * a.steps / (ms / 1e3), 1), "loss": round(loss, 4),
        "peak_GB": round(torch.cuda.max_memory_allocated(dev) / 1e9, 2), "plan": run.clip.last_step_plan}),
        flush=True)
    run.close()


if __name__ == "__main__":
    main()
