"""Cost of the pairwise sigmoid loss (CLIP(sigmoid_loss=True), xclip_sigmoid_* in csrc/nce.cu).

    python tools/sigmoid_bench.py [--skip-step] [--rounds 3]

(1) The loss kernels alone at R = 4096 rows, C = 4096 and 32768 columns (one rank block of an 8-GPU
    step), latent 512 (K = 3 x 512 split-bf16): xclip_sigmoid_fwd against xclip_nce_fwd and
    xclip_sigmoid_bwd against xclip_nce_bwd, alternated.  TFLOP/s count 2 R C K per call.
(2) bench.py's cfg3 step at 4096 pairs per GPU, micro-batch 768, with the default loss and with
    sigmoid_loss=True, alternated `--rounds` times: pairs/s and peak allocation.
Prints one JSON line per measurement, each with the card's name and power limit read in the same run."""
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


def _time(fn, reps, warmup=3):
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def kernels(R, C, D, dev, gpu, rounds):
    import torch
    from x_clip_b200 import kernels as K
    _, rows, _, _ = K.l2norm_fwd(torch.randn((R, D), device=dev))
    _, _, cols, _ = K.l2norm_fwd(torch.randn((C, D), device=dev))
    te = torch.full((1,), 10.0, device=dev)
    lb = torch.full((1,), -10.0, device=dev)
    gs = torch.full((1,), 1.0 / C, device=dev)
    lse_r, _ = K.nce_fwd(rows, cols, te, 0, False)
    lse_c = torch.zeros(C, device=dev)
    dt = torch.zeros(2, device=dev)
    calls = {
        "sigmoid_fwd": lambda: K.sigmoid_fwd(rows, cols, te, lb, 0),
        "nce_fwd": lambda: K.nce_fwd(rows, cols, te, 0, False),
        "sigmoid_bwd": lambda: K.sigmoid_bwd(rows, cols, te, lb, 0, gs, dt[0:1], dt[1:2]),
        "nce_bwd": lambda: K.nce_bwd(rows, cols, te, 0, False, lse_r, lse_c, 1.0, 1.0, 2.0, gs, dt[0:1]),
    }
    reps = max(20, int(2e12 // (2 * R * C * 3 * D)))
    ms = {k: [] for k in calls}
    for _ in range(rounds):
        for k, f in calls.items():
            ms[k].append(_time(f, reps))
    flop = 2.0 * R * C * 3 * D
    for k, v in ms.items():
        best = min(v)
        print(json.dumps(dict(kernel=k, R=R, C=C, latent=D, reps=reps, ms=[round(x, 4) for x in v],
                              tflops=round(flop / (best * 1e-3) / 1e12, 1), card=gpu)), flush=True)


def step(sigmoid, batch, microbatch, steps, warmup, dev, gpu):
    import torch
    import bench
    import x_clip_b200
    kw = dict(bench.VITB16_CFG)
    torch.manual_seed(0)
    clip = x_clip_b200.CLIP(**kw, microbatch=microbatch, sigmoid_loss=sigmoid).to(dev)
    clip.train()
    text = torch.randint(3, kw["num_text_tokens"], (batch, kw["text_seq_len"]), device=dev)
    image = torch.randn(batch, 3, kw["visual_image_size"], kw["visual_image_size"], device=dev)
    for _ in range(warmup):
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
    out = dict(model="cfg3", loss_fn="sigmoid" if sigmoid else "infonce", pairs_per_gpu=batch,
               microbatch=microbatch, steps=steps, step_ms=round(ms, 1), pairs_per_s=round(batch / (ms / 1e3), 1),
               peak_alloc_gib=round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 2),
               retained_chunks=clip.last_step_plan["retained"], loss=round(loss.item(), 5), card=gpu)
    print(json.dumps(out), flush=True)
    del clip, text, image, loss
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-step", action="store_true")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--microbatch", type=int, default=768)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    dev = torch.device("cuda:0")
    gpu = card()
    t0 = time.perf_counter()
    for C in (4096, 32768):
        kernels(4096, C, 512, dev, gpu, a.rounds)
    if not a.skip_step:
        for _ in range(a.rounds):
            for sig in (False, True):
                step(sig, a.batch, a.microbatch, a.steps, a.warmup, dev, gpu)
    print(json.dumps(dict(wall_s=round(time.perf_counter() - t0, 1), card=gpu)), flush=True)


if __name__ == "__main__":
    main()
