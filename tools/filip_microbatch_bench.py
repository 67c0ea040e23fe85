"""cfg3-shaped FILIP at 4096 pairs per GPU through the micro-batched step (micro-batch 768): pairs/s,
peak allocation, encoder chunks retained, FILIP rows saved / recomputed, under the default save plan
and with every FILIP chunk forced to be recomputed.  Prints one JSON line per plan, with the card's
name and power limit read in the same run.

    python tools/filip_microbatch_bench.py [--batch 4096] [--microbatch 768] [--steps 3] [--warmup 1]
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
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--microbatch", type=int, default=768)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--plans", default="default,recompute")
    a = ap.parse_args()

    import torch
    import bench
    from x_clip_b200 import filip
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    dev = torch.device("cuda:0")
    gpu = card()
    for plan in a.plans.split(","):
        filip.FILIP_SAVE_BYTES = {"default": None, "recompute": 0}[plan]
        run = bench.Runner(bench.VITB16_CFG, "filip", a.batch, a.microbatch, 0.5, dev, 0, 1)
        t0 = time.perf_counter()
        torch.cuda.reset_peak_memory_stats(dev)
        ms, loss = run.timed(a.steps, a.warmup)
        sp = run.clip.last_step_plan
        out = dict(plan=plan, pairs_per_gpu=a.batch, microbatch=a.microbatch, steps=a.steps,
                   step_ms=round(ms / a.steps, 1), pairs_per_s=round(a.batch * a.steps / (ms / 1e3), 1),
                   peak_alloc_gib=round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 2),
                   encoder_chunks=sp["chunks"], encoder_chunks_retained=sp["retained"],
                   filip_rows_saved=sp["filip"]["rows_saved"], filip_rows_recomputed=sp["filip"]["rows_recomputed"],
                   filip_saved_gb=round(sp["filip"]["saved_bytes"] / 1e9, 2), loss=loss,
                   wall_s=round(time.perf_counter() - t0, 1), card=gpu)
        print(json.dumps(out), flush=True)
        run.close()
        del run
        torch.cuda.empty_cache()
    filip.FILIP_SAVE_BYTES = None


if __name__ == "__main__":
    main()
