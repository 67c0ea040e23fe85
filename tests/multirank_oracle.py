"""Per-rank fp64 reference of the data-parallel CLIP step.  TEST INFRASTRUCTURE ONLY.

With W ranks of b pairs each, ContrastiveLossFn and FilipLossFn (the CLS and FILIP losses) keep one
contract:
- every rank returns the loss of the global batch of W * b pairs;
- rank r's parameter gradients are d(global loss) through rank r's samples only - the other ranks'
  latents arrive through the all-gather as constants;
- d temperature is the full-batch value on every rank.

That is step_oracle.step_loss on the global batch with the latents of the other ranks' rows detached
(oracle.clip_forward_sharded says the same of the reference's CLS path).  It is not restated here:
`rank_reference` runs step_oracle.reference with clip_oracle.unit_rows wrapped, the normalisation that
ends every latent step_loss makes, so that its output rows outside [r*b, (r+1)*b) are detached.  Detaching
the encoder outputs instead would not do: the latent projections would still take gradient from every
rank's rows, where the GPU step projects only its own.  test_multirank_gates.py checks that the rank
gradients add up to the full one.

Used by test_gpu_multirank_fp64.py (W ranks on one H100) and test_multirank_gates.py (CPU).
"""
from __future__ import annotations

import contextlib
from typing import Sequence
from unittest import mock

import torch

import step_oracle as SO
from oracle import clip_oracle as O


def make_case(name: str, world: int, b: int, spec: dict = None, empty: Sequence[int] = ()) -> dict:
    """step_oracle.make_case of the spec `spec` (default: step_oracle.CASES[name]) at the global batch
    world * b; `empty` lists global rows whose caption is made all padding (an empty string).  Build it
    after init_process_group: CLIP reads the world size when it is constructed."""
    spec = dict(SO.CASES[name] if spec is None else spec, batch=world * b)
    key = f"mr{world}_{name}"
    with mock.patch.dict(SO.CASES, {key: spec}):
        c = SO.make_case(key)
    text = c["batches"][0][0]
    for row in empty:
        text[row] = c["cfg"].text_pad_id
    c.update(world=world, b=b)
    return c


def rows(c, rank: int) -> slice:
    """Rank `rank`'s rows of the global batch."""
    return slice(rank * c["b"], (rank + 1) * c["b"])


@contextlib.contextmanager
def _only_rank_rows(fn: str, world: int, rank: int):
    """Wrap clip_oracle.`fn` (its first arguments are [W*b, ...] tensors) so that every row of its
    inputs (unit_rows: of its output) outside rank `rank`'s block carries no gradient."""
    real = getattr(O, fn)

    def detach_others(t):
        assert t.shape[0] % world == 0, (fn, t.shape, world)
        b = t.shape[0] // world
        mine = torch.zeros(t.shape[0], dtype=torch.bool, device=t.device)
        mine[rank * b:(rank + 1) * b] = True
        return torch.where(mine.view(-1, *[1] * (t.dim() - 1)), t, t.detach())

    if fn == "unit_rows":
        def wrapped(t):
            return detach_others(real(t))
    else:
        def wrapped(*args, **kw):
            return real(*[detach_others(a) if torch.is_tensor(a) else a for a in args], **kw)
    with mock.patch.object(O, fn, wrapped):
        yield


def rank_reference(c, dev, world: int, rank: int, keep=None) -> dict:
    """What rank `rank` of `world` must compute: step_oracle.reference's dict (loss, grads, image_grads)
    of the global batch, gradients through rank `rank`'s latents only."""
    with _only_rank_rows("unit_rows", world, rank):
        return SO.reference(c, dev, keep=keep)


def full_reference(c, dev, keep=None) -> dict:
    """The single-process fp64 step on the global batch: the loss, d temperature and d image every
    rank must reproduce."""
    return SO.reference(c, dev, keep=keep)


def row_terms_dtemp(c, dev, world: int, rank: int, keep=None) -> float:
    """d loss / d temperature of rank `rank`'s rows of the similarity matrices alone (both directions):
    what a rank returns for the temperature before its all-reduce, with an extra latent pair or FILIP,
    whose backward forms each direction's row block on the rank that owns the rows.  Each row's
    log-sum-exp term reads only its own row, so detaching the other rows at the InfoNCE leaves these."""
    with _only_rank_rows("_nce_from_logits", world, rank):
        return SO.reference(c, dev, keep=keep)["grads"]["temperature"].item()
