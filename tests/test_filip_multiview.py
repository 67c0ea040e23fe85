"""FILIP with augmented views on the CPU: the fp64 restatement (tests/filip_multiview_oracle.py) against
the reference's goldens (tests/golden/filip_mv_*.json, make_golden_filip_multiview.py), the view-block
layout and positive columns in both column orders, the block weights, the multiview chunk plan and
saved-argmax arithmetic.  CLIP.forward's routing of a FILIP call with views is in test_loss_head.py."""
import json
from pathlib import Path

import pytest
import torch

import x_clip_b200
from oracle import clip_oracle as O
import filip_multiview_oracle as FMV
from golden.make_golden_filip_multiview import CASES, view_inputs
from x_clip_b200 import filip as F

GOLD = Path(__file__).parent / "golden"


def load(name):
    return json.loads((GOLD / f"{name}.json").read_text())


def oracle_case(gold, image_grad=False):
    cfg = O.ClipConfig(**gold["cfg"])
    state = O.protocol_state_dict(cfg, gold["weight_seed"])
    texts, images = view_inputs(cfg, gold["batch"], gold["pad_fraction"], gold["n_text_views"],
                                gold["n_image_views"], [tuple(e) for e in gold["empty"]])
    p = {k: v.clone().requires_grad_(True) for k, v in state.items()}
    ims = [im.clone().requires_grad_(image_grad) for im in images]
    loss = FMV.clip_forward_filip_multiview(p, texts, ims, cfg, gold["multiview_loss_weight"])
    loss.backward()
    return loss, p, ims, texts


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_reproduces_the_reference(case):
    gold = load(case)
    loss, p, ims, texts = oracle_case(gold, "images" in gold)
    assert abs(loss.item() - gold["loss"]) <= 3e-6 * max(1.0, abs(gold["loss"])), (loss.item(), gold["loss"])
    assert abs(p["temperature"].grad.item() - gold["dtemperature"]) <= 1e-5 * max(1.0, abs(gold["dtemperature"]))
    for k, n in gold["grad_norms"].items():
        assert abs(p[k].grad.double().norm().item() - n) <= 2e-4 * n + 1e-9, k
    if "images" in gold:
        for im, rec in zip(ims, gold["images"]):
            got = im.grad.double().flatten(1).norm(dim=1)
            assert torch.allclose(got, torch.tensor(rec["sample_norms"], dtype=torch.float64), rtol=2e-4)
    for v, row in gold["empty"]:                              # an entirely padded augmented caption
        assert not bool((texts[v][row] != gold["cfg"].get("text_pad_id", 0)).any())


def test_cases_cover_the_view_shapes():
    shapes = {(c[3], c[4]) for c in CASES.values()}
    assert {(1, 2), (2, 1), (2, 2)} <= shapes
    assert any(c[5] and all(v > 0 for v, _ in c[5]) for c in CASES.values())   # an empty augmented caption
    assert any(c[6] for c in CASES.values())                                    # an image gradient


def test_augmented_captions_have_their_own_pad_pattern():
    gold = load("filip_mv_t2i2")
    cfg = O.ClipConfig(**gold["cfg"])
    texts, _ = view_inputs(cfg, gold["batch"], gold["pad_fraction"], 2, 2, ())
    assert not torch.equal(texts[0] != 0, texts[1] != 0)


# --------------------------------------------------------------------------- layout

def _gathered_labels(W, n, b):
    """(rank, view, local sample) of every column of the gathered image samples: each rank stacks
    its n views (view-major within the rank), the all-gather concatenates the ranks."""
    local = [[(r, j, y) for j in range(n) for y in range(b)] for r in range(W)]
    return [lab for r in range(W) for lab in local[r]]


@pytest.mark.parametrize("W,m,n,b", [(1, 1, 2, 3), (1, 2, 2, 4), (2, 2, 1, 3), (3, 2, 3, 2), (4, 3, 3, 1)])
def test_positive_columns_in_both_orders(W, m, n, b):
    """col_run = b indexes the gathered (rank-major) columns; col_run = W b the view-major permutation
    of the same columns.  The positive of text view i's local row x on rank r in image view j's block
    is view j's copy of global sample r b + x, and the B columns of a block are view j's samples."""
    B = W * b
    rank_major = _gathered_labels(W, n, b)
    view_major = sorted(rank_major, key=lambda t: (t[1], t[0], t[2]))
    for labels, run in ((rank_major, b), (view_major, B)):
        for r in range(W):
            for i in range(m):
                for j in range(n):
                    for x in range(b):
                        c = F.positive_column(i, j, x, r, b, n, run)
                        assert labels[c] == (r, j, x)
                    cols = [(k // run) * n * run + j * run + k % run for k in range(B)]
                    assert sorted(labels[c] for c in cols) == [(q, j, y) for q in range(W) for y in range(b)]
                    # global sample order within the block
                    assert [labels[c][0] * b + labels[c][2] for c in cols] == list(range(B))
    if W == 1:
        assert all(F.positive_column(0, j, x, 0, b, n, b) == F.positive_column(0, j, x, 0, b, n, B)
                   for j in range(n) for x in range(b))


@pytest.mark.parametrize("m,n", [(1, 2), (2, 1), (2, 2), (4, 4)])
def test_block_weights(m, n):
    B, cl_w, mv_w = 6, 0.8, 0.1
    w = F.view_block_weights(m, n, cl_w, mv_w, B)
    assert len(w) == m * n
    assert w[0] == pytest.approx(cl_w / (2 * B))
    assert sum(w[1:]) == pytest.approx(mv_w / (2 * B))
    assert len(set(w[1:])) == 1


# --------------------------------------------------------------------------- plan arithmetic

@pytest.mark.parametrize("m,n", [(1, 1), (1, 2), (2, 2), (3, 2)])
def test_saved_bytes_grow_with_the_view_counts(m, n):
    b, B, T, I, D = 8, 16, 77, 98, 512
    assert F.saved_bytes(b, B, T, I, m, n) == m * n * F.saved_bytes(b, B, T, I)
    assert F.saved_bytes(b, B, T, I) == F.saved_bytes(b, B, T, I, 1, 1)
    for extra in (False, True):
        pairs = 2 if extra else 1
        assert F.step_reserve_bytes(b, B, T, I, D, extra, m, n) == (
            F.saved_bytes(b, B, T, I, m, n) + F.FILIP_CHUNK_BYTES + 24 * D * (m * b * T + n * B * I) * pairs)
        assert F.step_reserve_bytes(b, B, T, I, D, extra) == F.step_reserve_bytes(b, B, T, I, D, extra, 1, 1)


@pytest.mark.parametrize("m,n", [(1, 2), (2, 2)])
def test_multiview_passes_plan_like_the_single_view_ones(monkeypatch, m, n):
    """The multiview passes are single-view passes with m b text samples and n B image samples: chunks of
    whole samples within the chunk budget, and a full save of exactly saved_bytes(..., m, n)."""
    monkeypatch.setattr(F, "FILIP_CHUNK_BYTES", 1 << 16)
    b, W, T, I = 6, 2, 48, 144
    B = W * b
    op = lambda rows: torch.empty((rows, 8), dtype=torch.bfloat16)
    pa = F._Pass(op(m * b * T), op(n * B * I), I, None, None, T)
    pb = F._Pass(op(n * B * I), op(m * b * T), T, None, None, I)
    assert (pa.nseg, pb.nseg) == (n * B, m * b)
    for p, rps in ((pa, T), (pb, I)):
        assert p.chunks[0][0] == 0 and p.chunks[-1][1] == p.R
        assert all(r0 % rps == 0 and r1 % rps == 0 for r0, r1 in p.chunks)
        assert all(p2[0] == p1[1] for p1, p2 in zip(p.chunks, p.chunks[1:]))
        assert max((r1 - r0) // rps for r0, r1 in p.chunks) * rps * p.nseg * 12 <= max(F.FILIP_CHUNK_BYTES // 2, rps * p.nseg * 12)
        assert len(p.chunks) > 1
    kept = pa.plan(1 << 40) + pb.plan(1 << 40)
    assert kept == F.saved_bytes(b, B, T, I, m, n)
    pa2 = F._Pass(op(m * b * T), op(n * B * I), I, None, None, T)
    assert pa2.plan(0) == 0 and pa2.saved is None


# --------------------------------------------------------------------------- refusals

TINY = dict(dim_text=256, dim_image=256, dim_latent=256, num_text_tokens=128, text_enc_depth=1,
            text_seq_len=16, text_heads=4, visual_enc_depth=1, visual_heads=4, visual_image_size=64,
            visual_patch_size=16, visual_patch_dropout=0.0, use_all_token_embeds=True)


def test_filip_simreg_with_views_still_raises():
    with pytest.raises(x_clip_b200.Unsupported, match="779"):
        x_clip_b200.CLIP(**TINY, extra_latent_projection=True, sim_reg_loss_weight=0.1)
