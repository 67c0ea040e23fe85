"""The auxiliary losses at large batch through the micro-batched step: the README model with SimSiam
(DCL + extra latent projections + use_visual_ssl, README.md) at 1024 and 4096 pairs per GPU, and cfg3
with MLM at 4096 pairs per GPU, micro-batch 768.  Prints one JSON line per run with pairs/s, the peak
allocation, the retention plan, and the card's name and power limit read in the same run.  The SSL
views are augmented on the whole batch at once by the default augmentation (SimCLRAugmentation, on the
CUDA kernels); `--augment flip` replaces it by a horizontal flip.  `--lr` > 0 takes a fused AdamW step
after every step and prints the loss of each timed step (a training run on one fixed batch).

    python tools/aux_microbatch_bench.py [--runs readme_simsiam:1024,readme_simsiam:4096,cfg3_mlm:4096]
                                         [--microbatch 768] [--steps 3] [--warmup 1] [--lr 0]
"""
import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", default="readme_simsiam:1024,readme_simsiam:4096,cfg3_mlm:4096")
    ap.add_argument("--microbatch", type=int, default=768)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--augment", default="default", choices=["default", "flip"],
                    help="SSL views: the reference's pipeline, or a horizontal flip only")
    ap.add_argument("--lr", type=float, default=0.0, help="> 0: an AdamW step after every step")
    a = ap.parse_args()

    import torch
    import bench
    import x_clip_b200
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    dev = torch.device("cuda:0")
    gpu = card()
    models = {
        "readme_simsiam": dict(bench.README_CFG, decoupled_contrastive_learning=True, extra_latent_projection=True,
                               use_visual_ssl=True),
        "cfg3_mlm": dict(bench.VITB16_CFG, use_mlm=True),
    }
    for run in a.runs.split(","):
        name, batch = run.split(":")
        batch = int(batch)
        kw = models[name]
        torch.manual_seed(0)
        clip = x_clip_b200.CLIP(**kw, microbatch=a.microbatch).to(dev)
        clip.train()
        if a.augment == "flip" and kw.get("use_visual_ssl"):
            from torchvision import transforms as T
            clip.visual_ssl.augment1 = clip.visual_ssl.augment2 = T.RandomHorizontalFlip()
        opt = None
        if a.lr > 0:
            from x_clip_b200.optim import FusedAdamW
            opt = FusedAdamW(clip.parameters(), lr=a.lr)
        losses = []
        text = torch.randint(3, kw["num_text_tokens"], (batch, kw["text_seq_len"]), device=dev)
        image = torch.randn(batch, 3, kw["visual_image_size"], kw["visual_image_size"], device=dev)
        t0 = time.perf_counter()
        for _ in range(a.warmup):
            clip(text, image, return_loss=True).backward()
            if opt is not None:
                opt.step()
            clip.zero_grad(set_to_none=True)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.steps):
            loss = clip(text, image, return_loss=True)
            loss.backward()
            if opt is not None:
                opt.step()
                losses.append(loss.detach())
            clip.zero_grad(set_to_none=True)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / a.steps
        sp = clip.last_step_plan
        print(json.dumps(dict(model=name, pairs_per_gpu=batch, microbatch=a.microbatch, steps=a.steps,
                              step_ms=round(ms, 1), pairs_per_s=round(batch / (ms / 1e3), 1),
                              peak_alloc_gib=round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 2),
                              chunks=sp["chunks"], retained_chunks=sp["retained_chunks"], passes=sp["passes"],
                              augment=a.augment, loss=round(loss.item(), 5),
                              **(dict(lr=a.lr, losses=[round(v.item(), 5) for v in losses]) if opt else {}),
                              wall_s=round(time.perf_counter() - t0, 1), card=gpu)),
              flush=True)
        del clip, text, image, loss
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
