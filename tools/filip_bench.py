"""Cost of the FILIP loss (use_all_token_embeds=True, csrc/filip.cu) at the token counts of the
project's towers.

    python tools/filip_bench.py [--skip-step] [--reps N]

(1) Segment-max passes, D = 512 (K = 3 D = 1536), local batch 256: for T text tokens against I
    image tokens, pass A is (256 T) rows x (256 I) columns in segments of I, pass B (256 I) x (256 T)
    in segments of T.  Algorithmic TFLOP/s = 2 R C 3D / time.  Also one rank's pass A at an 8-GPU
    cfg3 batch (256 x 77 rows against 2048 x 98 columns).
(2) FilipLossFn forward + backward at the same (T, I), batch 256, no encoder.
(3) The cfg3 step of bench.py with FILIP against the same step with InfoNCE (256 pairs, patch
    dropout 0.5): FILIP's share of the step.
Prints the card's name and power limit and one JSON line."""
import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))

F32, BF16 = torch.float32, torch.bfloat16


def _card(dev):
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(dev.index)], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "nvidia-smi unavailable"
    return dict(gpu=torch.cuda.get_device_name(dev), nvidia_smi=q)


def _time(fns, reps, warmup=3):
    """ms per call of each fn, the fns alternated call by call inside one window per fn"""
    for _ in range(warmup):
        for fn in fns:
            fn()
    torch.cuda.synchronize()
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(2 * reps)] for _ in fns]
    for r in range(reps):
        for j, fn in enumerate(fns):
            ev[j][2 * r].record()
            fn()
            ev[j][2 * r + 1].record()
    torch.cuda.synchronize()
    return [sum(e[2 * r].elapsed_time(e[2 * r + 1]) for r in range(reps)) / reps for e in ev]


def _split(z):
    hi = z.to(BF16)
    lo = (z - hi.float()).to(BF16)
    return torch.cat([hi, lo, hi], 1).contiguous(), torch.cat([hi, hi, lo], 1).contiguous()


def _unit(shape, dev):
    return torch.nn.functional.normalize(torch.randn(shape, device=dev), dim=-1)


def segmax_pass(R, C, seg_len, D, dev, reps):
    from x_clip_b200 import kernels as K
    a, _ = _split(_unit((R, D), dev))
    _, b = _split(_unit((C, D), dev))
    t = torch.tensor([100.0], device=dev, dtype=F32)
    (ms,) = _time([lambda: K.filip_segmax16(a, b, t, seg_len, None, None)], reps)
    fl = 2.0 * R * C * 3 * D
    return dict(R=R, C=C, seg_len=seg_len, segmax_ms=round(ms, 3), segmax_tflops=round(fl / ms / 1e9, 1))


def loss_fn(B, T, I, D, dev, reps):
    from x_clip_b200.filip import FilipLossFn
    zt, zi = _unit((B, T, D), dev), _unit((B, I, D), dev)
    lens = torch.randint(1, T + 1, (B,), device=dev)
    mask = (torch.arange(T, device=dev)[None, :] < lens[:, None]).contiguous()
    ops = (_split(zt.reshape(-1, D)), _split(zi.reshape(-1, D)))
    zt_, zi_ = zt.requires_grad_(True), zi.requires_grad_(True)
    temp = torch.tensor(4.0, device=dev, dtype=F32, requires_grad=True)

    def step():
        FilipLossFn.apply(zt_, zi_, None, None, temp, ops, mask, False, False).backward()

    (ms,) = _time([step], reps)
    fl = 2 * 2.0 * B * T * B * I * 3 * D            # the two segment-max passes
    return dict(B=B, T=T, I=I, D=D, fwd_bwd_ms=round(ms, 3), segmax_share_tflops=round(fl / ms / 1e9, 1),
                peak_gib=round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 2))


def cfg3_step(dev, loss, steps=5):
    import bench
    r = bench.Runner(bench.WORKLOADS["cfg3"][0], loss, 256, 0, 0.5, dev, 0, 1)
    torch.cuda.reset_peak_memory_stats(dev)
    ms, lv = r.timed(steps, 2)
    out = dict(loss=loss, ms_per_step=round(ms / steps, 2), pairs_per_s=round(256 * steps / (ms / 1e3), 1),
               loss_value=round(lv, 5), peak_gib=round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 2))
    r.close()
    del r
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-step", action="store_true")
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    if not torch.cuda.is_available():
        raise SystemExit("filip_bench needs a GPU")
    D, b = 512, 256
    shapes = [(256, 64), (256, 32), (48, 144), (77, 98), (77, 196), (77, 576)]
    res = dict(card=_card(dev), segmax=[], loss_fn=[])
    for T, I in shapes:
        res["segmax"].append(dict(pass_="A", **segmax_pass(b * T, b * I, I, D, dev, args.reps)))
        res["segmax"].append(dict(pass_="B", **segmax_pass(b * I, b * T, T, D, dev, args.reps)))
        torch.cuda.empty_cache()
    res["segmax"].append(dict(pass_="A, one rank of 8 (B_g 2048)",
                              **segmax_pass(b * 77, 2048 * 98, 98, D, dev, args.reps)))
    for T, I in shapes:
        torch.cuda.reset_peak_memory_stats(dev)
        res["loss_fn"].append(loss_fn(b, T, I, D, dev, max(3, args.reps // 4)))
        torch.cuda.empty_cache()
    if not args.skip_step:
        res["cfg3_step"] = [cfg3_step(dev, "nce"), cfg3_step(dev, "filip"), cfg3_step(dev, "nce"),
                            cfg3_step(dev, "filip")]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
