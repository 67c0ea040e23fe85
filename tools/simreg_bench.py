"""Cost of the similarity regularisation (sim_reg_loss_weight > 0, csrc/simreg.cu).

    python tools/simreg_bench.py [--skip-step]

(1) Kernels at D = 512, both latent pairs as in a training step: forward = 4 packs + 2 xclip_simreg_fwd;
    backward = 2 xclip_simreg_bwd + 4 latent-gradient GEMMs.  R x C = 4096 x 4096 and 4096 x 32768
    (one rank of an 8-GPU cfg3 batch).  TFLOP/s count 2 R C K per similarity GEMM (K = 6 D) and
    2 R C D per gradient GEMM.
(2) The cfg5 step of bench.py (README CLIP, DCL + extra latent projection, 8192 pairs, micro-batch
    1024) with the term off and on: step time and peak memory.
Prints one JSON line."""
import argparse
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))


def _time(fn, reps=10, warmup=3):
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


def kernels(R, C, D, dev):
    from x_clip_b200 import kernels as K
    from x_clip_b200.engine import _pad_rows
    ops = []
    for _ in range(4):                                   # t, v, t', v'
        p = torch.randn((C, D), device=dev)
        _, zrow, zcol, _ = K.l2norm_fwd(p)
        ops.append((zrow[:R].contiguous(), zcol))
    gs = torch.full((1,), 1e-6, device=dev)

    def fwd():
        out = []
        for t, v in ((0, 1), (2, 3)):
            a = K.simreg_pack(ops[t][0], ops[v][0], False)
            b = K.simreg_pack(ops[t][1], ops[v][1], True)
            out.append((a, b, K.simreg_fwd(a, b, 0)))
        return out

    packed = fwd()
    hi = [_pad_rows(o[1][:, :D], (C + 7) // 8 * 8) for o in ops]
    dz = [torch.zeros((R, D), device=dev) for _ in range(4)]

    def bwd():
        for (a, b, _), t, v in zip(packed, (0, 2), (1, 3)):
            g = K.simreg_bwd(a, b, 0, gs)
            K.gemm(g, hi[t], b_major=1, out=dz[t], accumulate=True)
            K.gemm(g, hi[v], b_major=1, out=dz[v], alpha=-1.0, accumulate=True)

    ms_f, ms_b = _time(fwd), _time(bwd)
    fl_f = 2 * 2.0 * R * C * 6 * D
    fl_b = fl_f + 4 * 2.0 * R * C * D
    return dict(R=R, C=C, D=D, fwd_ms=round(ms_f, 3), bwd_ms=round(ms_b, 3),
                fwd_tflops=round(fl_f / ms_f / 1e9, 1), bwd_tflops=round(fl_b / ms_b / 1e9, 1))


def cfg5_step(dev, weight, steps=3):
    import bench
    r = bench.Runner(bench.WORKLOADS["cfg2"][0], "dcl_extra", 8192, 1024, 0.0, dev, 0, 1)
    r.clip.sim_reg_loss_weight, r.clip.has_sim_reg_loss = weight, weight > 0
    torch.cuda.reset_peak_memory_stats(dev)
    ms, loss = r.timed(steps, 2)
    out = dict(sim_reg_loss_weight=weight, ms_per_step=round(ms / steps, 1), loss=round(loss, 5),
               peak_gib=round(torch.cuda.max_memory_allocated(dev) / 2 ** 30, 2))
    r.close()
    del r
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--skip-step", action="store_true")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    res = dict(gpu=torch.cuda.get_device_name(dev),
               kernels=[kernels(4096, 4096, 512, dev), kernels(4096, 32768, 512, dev)])
    if not args.skip_step:
        res["cfg5"] = [cfg5_step(dev, 0.0), cfg5_step(dev, 1.0), cfg5_step(dev, 0.0), cfg5_step(dev, 1.0)]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
