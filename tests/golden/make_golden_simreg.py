"""Generate the similarity-regularisation fixtures (sim_reg_loss_weight > 0) with the machinery of
make_golden.py: the REFERENCE on deterministic protocol weights and inputs, cross-checked against the
oracle plus tests/simreg_oracle.py before anything is written.

The weight of every case is chosen so that w * L_sim is about twice the contrastive loss: the parity
tests then see the term.  Each file records the loss with weight w ("loss") and with weight 0
("loss_without_sim_reg").  The weight lives beside "cfg", not in it, because the oracle's ClipConfig
has no such field.

The script also asserts that the reference fails where x_clip_b200 raises Unsupported: without the
extra latent projection, with FILIP, and with augmented views (all at x_clip.py:779).

Run in the build container only (the GPU box has no /root/reference):

    python tests/golden/make_golden_simreg.py
"""
from __future__ import annotations

import json
import os
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent))
import make_golden as M  # noqa: E402

sys.path.insert(0, str(M.HERE.parent))
import simreg_oracle as SR  # noqa: E402
from oracle import clip_oracle as O  # noqa: E402

EXTRA = dict(extra_latent_projection=True)
CASES = {
    # name: (cfg overrides, batch, pad_fraction, patch_dropout)
    "tiny_simreg_extra": (dict(M.TINY, **EXTRA), 6, 0.2, 0.0),
    "tiny_simreg_dcl_extra": (dict(M.TINY, decoupled_contrastive_learning=True, **EXTRA), 6, 0.2, 0.0),
    "vitb16_shaped_simreg_extra": (dict(M.VITB16_2L, **EXTRA), 4, 0.1, 0.0),
}


def pick_weight(cfgk, batch, padf):
    """w (two significant digits) with w * L_sim ~ 2 x the contrastive loss, from the oracle."""
    cfg = O.ClipConfig(**cfgk)
    state = O.protocol_state_dict(cfg, M.WEIGHT_SEED)
    text, image = O.protocol_inputs(cfg, batch, M.INPUT_SEED, padf)
    with torch.no_grad():
        cl, parts = O.clip_forward(state, text, image, cfg, return_parts=True)
        ls = SR.sim_reg_loss(parts["text_latents"], parts["image_latents"], parts["text_latents_extra"],
                             parts["image_latents_extra"])
    w = 2.0 * cl.item() / ls.item()
    return float(f"{w:.2g}")


def run_case(x_clip, name, cfgk, batch, padf, drop, w):
    cfg = O.ClipConfig(**cfgk)
    state = O.protocol_state_dict(cfg, M.WEIGHT_SEED)
    text, image = O.protocol_inputs(cfg, batch, M.INPUT_SEED, padf)
    clip = M.build_reference(x_clip, dict(cfgk, sim_reg_loss_weight=w), drop, state)
    assert clip.has_sim_reg_loss
    torch.manual_seed(M.DROP_SEED)
    loss = clip(text, image, return_loss=True)
    loss.backward()
    grads = {k: p.grad for k, p in clip.named_parameters() if p.grad is not None}
    with torch.no_grad():
        torch.manual_seed(M.DROP_SEED)
        enc_t, enc_i = clip(text, image, return_encodings=True)
        torch.manual_seed(M.DROP_SEED)
        lat = clip(text, image, return_latents=True)
    ref0 = M.build_reference(x_clip, cfgk, drop, state)
    torch.manual_seed(M.DROP_SEED)
    loss0 = ref0(text, image, return_loss=True).item()

    p = {k: v.clone().requires_grad_(True) for k, v in state.items()}
    o_loss = SR.clip_forward(p, text, image, cfg, w)
    o_loss.backward()
    assert abs(o_loss.item() - loss.item()) <= 2e-6 * max(1.0, abs(loss.item())), (name, o_loss.item(), loss.item())
    for k, g in grads.items():
        denom = g.norm().item() + 1e-12
        assert (p[k].grad - g).norm().item() / denom < 2e-4, (name, k)
    assert loss.item() - loss0 >= abs(loss0), (name, loss.item(), loss0)   # the term is visible

    total = torch.sqrt(sum((g.double() ** 2).sum() for g in grads.values())).item()
    return dict(case=name, cfg=cfgk, sim_reg_loss_weight=w, batch=batch, pad_fraction=padf, patch_dropout=drop,
                weight_seed=M.WEIGHT_SEED, input_seed=M.INPUT_SEED, drop_seed=M.DROP_SEED,
                loss=loss.item(), loss_without_sim_reg=loss0, dtemperature=grads["temperature"].item(),
                grad_norm=total, grad_norms={k: g.double().norm().item() for k, g in grads.items()},
                enc_text=M.summ(enc_t), enc_image=M.summ(enc_i), latents=[M.summ(z) for z in lat], keep=None,
                torch_version=torch.__version__)


def sharded_case(name, cfgk, w, world=2, per_rank=3):
    import torch.multiprocessing as mp
    cfg = O.ClipConfig(**cfgk)
    state = O.protocol_state_dict(cfg, M.WEIGHT_SEED)
    text, image = O.protocol_inputs(cfg, world * per_rank, M.INPUT_SEED, 0.2)
    texts, images = list(text.chunk(world)), list(image.chunk(world))
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    ref_kw = dict(cfgk, sim_reg_loss_weight=w)
    procs = [ctx.Process(target=M._rank_worker, args=(r, world, ref_kw, state, texts, images, 29631, q))
             for r in range(world)]
    for pr in procs:
        pr.start()
    res = sorted(q.get(timeout=600) for _ in range(world))
    for pr in procs:
        pr.join()
    ranks = []
    for rank, loss, gn, dtemp, norms in res:
        p = {k: v.clone().requires_grad_(True) for k, v in state.items()}
        o_loss = SR.clip_forward_sharded(p, texts, images, cfg, rank, w)
        o_loss.backward()
        assert abs(o_loss.item() - loss) < 5e-6 * max(1.0, abs(loss)), (name, rank, o_loss.item(), loss)
        for k, v in norms.items():
            og = p[k].grad
            on = 0.0 if og is None else og.double().norm().item()
            assert abs(on - v) <= 2e-4 * max(v, 1e-6) + 1e-9, (name, rank, k, on, v)
        ranks.append(dict(rank=rank, loss=loss, grad_norm=gn, dtemperature=dtemp, grad_norms=norms))
    return dict(case=name, cfg=cfgk, sim_reg_loss_weight=w, world=world, per_rank=per_rank, pad_fraction=0.2,
                weight_seed=M.WEIGHT_SEED, input_seed=M.INPUT_SEED, ranks=ranks)


def check_reference_refuses(x_clip):
    """The three combinations x_clip_b200 refuses fail inside the reference too."""
    cfg = O.ClipConfig(**M.TINY)
    state = O.protocol_state_dict(cfg, M.WEIGHT_SEED)
    text, image = O.protocol_inputs(cfg, 4, M.INPUT_SEED, 0.2)
    t2, i2 = O.protocol_inputs(cfg, 4, M.INPUT_SEED + 17, 0.2)
    for kw, call in ((dict(M.TINY, sim_reg_loss_weight=0.1), dict()),
                     (dict(M.TINY, sim_reg_loss_weight=0.1, use_all_token_embeds=True, **EXTRA), dict()),
                     (dict(M.TINY, sim_reg_loss_weight=0.1, **EXTRA), dict(aug_text=t2, aug_image=i2))):
        clip = M.build_reference(x_clip, kw, 0.0, state)
        try:
            clip(text, image, return_loss=True, **call)
        except (RuntimeError, IndexError, ValueError) as e:
            print("reference refuses", {k: v for k, v in kw.items() if k not in M.TINY}, sorted(call),
                  type(e).__name__)
            continue
        raise AssertionError(f"the reference ran {kw} {sorted(call)}")


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    x_clip = M.import_reference()
    check_reference_refuses(x_clip)
    for name, (cfgk, batch, padf, drop) in CASES.items():
        w = pick_weight(cfgk, batch, padf)
        out = run_case(x_clip, name, cfgk, batch, padf, drop, w)
        (M.HERE / f"{name}.json").write_text(json.dumps(out))
        print(f"{name}: w={w} loss={out['loss']:.7f} (w=0: {out['loss_without_sim_reg']:.7f}) "
              f"grad_norm={out['grad_norm']:.6f} dtemp={out['dtemperature']:.7f}")
    cfgk = dict(M.TINY, **EXTRA)
    w = pick_weight(cfgk, 6, 0.2)
    out = sharded_case("sharded_simreg_extra", cfgk, w)
    (M.HERE / "sharded_simreg_extra.json").write_text(json.dumps(out))
    print("sharded_simreg_extra", w, [(r["loss"], r["grad_norm"], r["dtemperature"]) for r in out["ranks"]])


if __name__ == "__main__":
    main()
