"""Cost of FILIP with augmented views (filip.FilipLossFn with views) at cfg4's shapes: the README model
(`bench.py --workload cfg2 --loss filip`), 256 pairs, 256 text tokens, 256 px / patch 32 with patch
dropout 0.5 (32 image tokens), D = 512.

    python tools/filip_multiview_bench.py [--reps N] [--skip-step]

(1) The loss alone, forward + backward on fixed latents, at (m, n) = (1, 1), (1, 2), (2, 2) text x
    image views: the one-pass multiview loss against the same loss computed as a loop of m n
    single-view FilipLossFn calls (weighted the same way).  (1, 1) is FilipLossFn itself.
(2) The whole CLIP step at the same (m, n): the encoders see m b texts and n b images.
All variants of a section are alternated call by call in one window; each prints ms per call and peak
allocation.  Prints the card's name and power limit and one JSON line."""
import argparse
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from tools.filip_bench import _card, _split, _time, _unit  # noqa: E402

F32 = torch.float32
B, T, I, D = 256, 256, 32, 512
VIEWS = [(1, 1), (1, 2), (2, 2)]
WEIGHTS = (0.9, 0.1)


def _latents(dev, m, n):
    zt, zi = _unit((m * B, T, D), dev), _unit((n * B, I, D), dev)
    lens = torch.randint(1, T + 1, (m * B,), device=dev)
    mask = (torch.arange(T, device=dev)[None, :] < lens[:, None]).contiguous()
    return zt, zi, mask


def _one_pass(dev, m, n):
    from x_clip_b200.filip import FilipLossFn
    zt, zi, mask = _latents(dev, m, n)
    ops = (_split(zt.reshape(-1, D)), _split(zi.reshape(-1, D)))
    zt, zi = zt.requires_grad_(True), zi.requires_grad_(True)
    temp = torch.tensor(4.6, device=dev, requires_grad=True)

    def run():
        loss = FilipLossFn.apply(zt, zi, None, None, temp, ops, mask, False, False, None, (m, n), WEIGHTS)
        loss.backward()
        zt.grad = zi.grad = temp.grad = None
    return run


def _loop(dev, m, n):
    """The same loss as m n single-view FilipLossFn calls on the views' operands."""
    from x_clip_b200.filip import FilipLossFn
    zt, zi, mask = _latents(dev, m, n)
    zts = [zt[i * B:(i + 1) * B].clone().requires_grad_(True) for i in range(m)]
    zis = [zi[j * B:(j + 1) * B].clone().requires_grad_(True) for j in range(n)]
    ot = [_split(z.detach().reshape(-1, D)) for z in zts]
    oi = [_split(z.detach().reshape(-1, D)) for z in zis]
    masks = [mask[i * B:(i + 1) * B].contiguous() for i in range(m)]
    temp = torch.tensor(4.6, device=dev, requires_grad=True)
    other = WEIGHTS[1] / (m * n - 1)

    def run():
        total = 0
        for i in range(m):
            for j in range(n):
                w = WEIGHTS[0] if i == j == 0 else other
                total = total + w * FilipLossFn.apply(zts[i], zis[j], None, None, temp, (ot[i], oi[j]), masks[i],
                                                      False, False)
        total.backward()
        for z in zts + zis:
            z.grad = None
        temp.grad = None
    return run


def _step(dev, m, n):
    import x_clip_b200
    from bench import README_CFG
    clip = x_clip_b200.CLIP(**README_CFG, use_all_token_embeds=True, visual_patch_dropout=0.5).to(dev)
    clip.train()
    g = torch.Generator(device=dev).manual_seed(0)
    texts = [torch.randint(1, README_CFG["num_text_tokens"], (B, README_CFG["text_seq_len"]), device=dev, generator=g)
             for _ in range(m)]
    ims = [torch.randn(B, 3, 256, 256, device=dev, generator=g) for _ in range(n)]

    def run():
        loss = clip(texts[0], ims[0], return_loss=True, aug_text=tuple(texts[1:]) or None,
                    aug_image=tuple(ims[1:]) or None)
        loss.backward()
        clip.zero_grad(set_to_none=True)
    return run


def _measure(dev, label, makers, reps):
    fns = [mk() for mk in makers.values()]
    ms = _time(fns, reps)
    out = {}
    for (name, _), fn, t in zip(makers.items(), fns, ms):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats(dev)
        fn()
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated(dev) / 2 ** 30
        out[name] = dict(ms=round(t, 3), peak_gib=round(peak, 2))
        print(f"{label} {name}: {t:.2f} ms, peak {peak:.2f} GiB")
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--skip-step", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU; there is no CPU path"
    dev = torch.device("cuda", 0)
    card = _card(dev)
    print(f"card: {card}")
    loss_makers = {}
    for m, n in VIEWS:
        loss_makers[f"one_pass_{m}x{n}"] = (lambda m=m, n=n: _one_pass(dev, m, n))
        if m * n > 1:
            loss_makers[f"loop_{m}x{n}"] = (lambda m=m, n=n: _loop(dev, m, n))
    res = dict(card=card, shape=dict(b=B, T=T, I=I, D=D), loss=_measure(dev, "loss", loss_makers, a.reps))
    if not a.skip_step:
        step_makers = {f"step_{m}x{n}": (lambda m=m, n=n: _step(dev, m, n)) for m, n in VIEWS}
        res["step"] = _measure(dev, "step", step_makers, max(3, a.reps // 2))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
