"""The SimCLR augmentation of SimSiam / SimCLR (SimCLRAugmentation on xclip_augment_mean / _apply) at
training batch sizes, with forced parameters so every call moves the same bytes:

    full  : full-image crop with every branch on (jitter with contrast, so the mean pass runs;
            grayscale, flip, blur) - the worst case
    crop8 : the same with a centred crop of 8 % of the image area (RandomResizedCrop's smallest)

For B in 256, 1024, 4096 at 224 and 256 px it times one view with CUDA events over many calls and
reports GB/s from the bytes the call must move (computed here: the mean pass reads the image, the
fused pass reads the crop window and writes the view), and the peak allocation above the input.  The
torchvision functional pipeline with the same parameters runs in the same process where it fits.
Prints one JSON line per measurement and the card's name and power limit.

    python tools/augment_bench.py [--batches 256,1024,4096] [--sizes 224,256] [--iters 20]
"""
import argparse
import json
import math
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="256,1024,4096")
    ap.add_argument("--sizes", default="224,256")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--torchvision-iters", type=int, default=3)
    a = ap.parse_args()

    import torch
    from x_clip_b200.aux import AugmentParams, SimCLRAugmentation
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    dev = torch.device("cuda:0")
    torch.backends.cudnn.allow_tf32 = False
    print(json.dumps(dict(card=card())), flush=True)

    def timed(fn, iters):
        fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters

    for S in (int(s) for s in a.sizes.split(",")):
        aug = SimCLRAugmentation(S, 3)
        for B in (int(b) for b in a.batches.split(",")):
            x = torch.rand(B, 3, S, S, device=dev)
            side = round(math.sqrt(0.08) * S)
            cases = {"full": (0, 0, S, S), "crop8": ((S - side) // 2, (S - side) // 2, side, side)}
            for name, crop in cases.items():
                p = AugmentParams((2, 0, 3, 1), (1.37, 0.61, 1.52, 0.13), True, True, 1.5, crop)
                h, w = crop[2], crop[3]
                # mean pass: the whole image; fused pass: the crop plus the blur halo (clipped at the
                # border), once; the view written once
                win = (min(h + 2, S) * min(w + 2, S))
                nbytes = 4 * B * 3 * (S * S + win + S * S)
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated(dev)
                torch.cuda.reset_peak_memory_stats(dev)
                ms = timed(lambda: aug.apply(x, p), a.iters)
                peak = torch.cuda.max_memory_allocated(dev) - base
                row = dict(path="kernels", B=B, size=S, case=name, crop=crop, ms=round(ms, 3),
                           gb_per_s=round(nbytes / (ms * 1e-3) / 1e9, 1), bytes=nbytes,
                           peak_above_input_gib=round(peak / 2 ** 30, 3),
                           view_gib=round(B * 3 * S * S * 4 / 2 ** 30, 3))
                print(json.dumps(row), flush=True)
                torch.cuda.reset_peak_memory_stats(dev)
                try:
                    ms = timed(lambda: aug.apply_torchvision(x, p), a.torchvision_iters)
                    tv = dict(ms=round(ms, 3),
                              peak_above_input_gib=round((torch.cuda.max_memory_allocated(dev) - base) / 2 ** 30, 3))
                except torch.cuda.OutOfMemoryError:
                    tv = dict(ms=None, oom=True)
                torch.cuda.empty_cache()
                print(json.dumps(dict(path="torchvision", B=B, size=S, case=name, **tv)), flush=True)
            del x
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
