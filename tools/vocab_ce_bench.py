"""The MLM head's cross-entropy over the vocabulary: the fused kernel (engine.VocabCrossEntropyFn)
against the unfused head it replaces (bf16 logits from engine.LinearFn, an fp32 copy and
F.cross_entropy), forward + backward with every gradient, at the rows a cfg3-shaped batch of 4096
captions selects (77 tokens, 15 % masked: about 49 k rows) and d = 512.  Prints one JSON line per
(V, head) with the time per step, the peak allocation above the inputs and the loss, and the card's
name and power limit read in the same run.  The two heads alternate inside each timed round.

    python tools/vocab_ce_bench.py [--rows 49152] [--vocab 10000,49408] [--dim 512] [--steps 5] [--rounds 3]
"""
import argparse
import json
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
    ap.add_argument("--rows", type=int, default=49152)
    ap.add_argument("--vocab", default="10000,49408")
    ap.add_argument("--dim", type=int, default=512)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()

    import torch
    import torch.nn.functional as F
    from x_clip_b200 import engine as E
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    dev = torch.device("cuda:0")
    gpu = card()

    def fused(rows, w, b, labels):
        return E.VocabCrossEntropyFn.apply(rows, w, b, labels)

    def unfused(rows, w, b, labels):
        return F.cross_entropy(E.LinearFn.apply(rows, w, b, None).float(), labels)

    for V in (int(v) for v in a.vocab.split(",")):
        gen = torch.Generator(device=dev).manual_seed(V)
        rows = torch.randn((a.rows, a.dim), generator=gen, device=dev).to(torch.bfloat16).requires_grad_(True)
        w = (torch.randn((V, a.dim), generator=gen, device=dev) * a.dim ** -0.5).requires_grad_(True)
        b = torch.zeros(V, device=dev).requires_grad_(True)
        labels = torch.randint(0, V, (a.rows,), generator=gen, device=dev)
        heads = dict(fused=fused, unfused=unfused)
        if V % 8:
            heads.pop("unfused")                  # LinearFn's GEMM needs V % 8 == 0

        def step(fn):
            rows.grad = w.grad = b.grad = None
            loss = fn(rows, w, b, labels)
            loss.backward()
            return loss

        res = {k: dict(ms=[], peak=0, loss=None) for k in heads}
        for k, fn in heads.items():               # warm-up
            step(fn)
        torch.cuda.synchronize()
        for _ in range(a.rounds):
            for k, fn in heads.items():
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated(dev)
                torch.cuda.reset_peak_memory_stats(dev)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(a.steps):
                    loss = step(fn)
                e1.record()
                torch.cuda.synchronize()
                res[k]["ms"].append(e0.elapsed_time(e1) / a.steps)
                res[k]["peak"] = max(res[k]["peak"], torch.cuda.max_memory_allocated(dev) - base)
                res[k]["loss"] = loss.item()
        for k, r in res.items():
            print(json.dumps(dict(head=k, rows=a.rows, vocab=V, dim=a.dim, steps=a.steps, rounds=a.rounds,
                                  ms_per_step=[round(m, 2) for m in r["ms"]],
                                  peak_above_inputs_gib=round(r["peak"] / 2 ** 30, 2),
                                  loss=round(r["loss"], 6), card=gpu)), flush=True)
        del rows, w, b, labels
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
