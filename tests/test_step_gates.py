"""CPU checks of the whole-step reference and gates of test_gpu_step_fp64.py (no GPU).

- Without a defect, step_oracle's restatement run in fp32 is oracle.clip_forward (loss and every
  gradient, to 1e-5) on committed golden cases, and its loss is the reference's golden loss.
- Every gate is at most a quarter of the effect of a glue defect it exists to catch, on the inputs of
  the GPU cases: restated in the reference, the defect moves some gated quantity (the loss, d
  temperature, a parameter family's gradient, d image) by at least 4 of its gates (`bite` >= 4), so it
  still fails the GPU test after the kernels' own error (at most 1 gate) is subtracted.
"""
import json
from pathlib import Path

import pytest
import torch

import step_oracle as SO
from oracle import clip_oracle as O

GOLD = Path(__file__).parent / "golden"
BITE = 4.0


@pytest.mark.parametrize("case", ["tiny_plain", "tiny_dcl_extra", "tiny_patchdrop", "tiny_filip_dcl_extra",
                                  "tiny_rotary", "tiny_causal"])
def test_restatement_matches_oracle_fp32(case):
    gold = json.loads((GOLD / f"{case}.json").read_text())
    cfg = O.ClipConfig(**gold["cfg"])
    state = O.protocol_state_dict(cfg, gold["weight_seed"])
    text, image = O.protocol_inputs(cfg, gold["batch"], gold["input_seed"], gold["pad_fraction"])
    keep = None if gold["keep"] is None else torch.tensor(gold["keep"])
    p = {k: v.clone().requires_grad_(True) for k, v in state.items()}
    q = {k: v.clone().requires_grad_(True) for k, v in state.items()}
    ref = O.clip_forward(p, text, image, cfg, keep=keep)
    ref.backward()
    mine = SO.step_loss(q, dict(cfg=cfg, kw={}), [text], [image], keep)
    mine.backward()
    assert abs(mine.item() - ref.item()) <= 1e-5 * abs(ref.item())
    assert abs(mine.item() - gold["loss"]) <= 1e-5 * abs(gold["loss"])
    for k in p:
        if p[k].grad is None:
            assert q[k].grad is None or not q[k].grad.ne(0).any(), k
            continue
        err = (q[k].grad - p[k].grad).norm().item()
        assert err <= 1e-5 * p[k].grad.norm().item() + 1e-12, (k, err)


def test_pinned_reference_restores_the_oracle():
    with SO.pinned():
        assert O.PINNED_LN_EPS == SO.LN_EPS and not O.SOFTMAX_FP32
    assert O.PINNED_LN_EPS is None and O.SOFTMAX_FP32


def test_every_parameter_has_a_family():
    for name in SO.CASES:
        for k in SO.make_case(name)["names"]:
            assert k == "temperature" or SO.family(k) in SO.STEP_GATES, k


_REF = {}


def _ref(case):
    if case not in _REF:
        c = SO.make_case(case)
        _REF[case] = (c, SO.reference(c, "cpu"))
    return _REF[case]


def worst(case, defect):
    c, ref = _ref(case)
    bad = SO.reference(c, "cpu", defects=(defect,))
    r = SO.ratios(bad, ref, SO.GATE_SCALE.get(case, 1.0))
    k = max(r, key=r.get)
    exact = SO.structural_errors(c["names"], bad, ref)
    print(f"BITE {defect}[{case}] {r[k]:.2f} ({k}){' + ' + '; '.join(exact) if exact else ''}")
    return float("inf") if exact else r[k]


@pytest.mark.parametrize("defect,case", [
    ("pos_cls", "default"), ("pos_shift", "default"), ("eos_last", "causal"), ("pos_kept_order", "drop"),
    ("pos_kept_order", "imggrad_drop"), ("ln_eps", "cfg3"), ("filip_pad_mean", "filip_dcl_extra"),
    ("mv_weight", "multiview"), ("simreg_b2", "simreg"), ("mlm_all", "aux")])
def test_step_gates_bite(defect, case):
    assert worst(case, defect) >= BITE


def test_vision_cls_sum_is_invisible_to_the_step():
    """The vision CLS is projected and l2-normalised (to_cls_tokens has no bias), so projecting the SUM of
    the tokens instead of their mean scales the latent's pre-image and changes neither the loss nor any
    gradient: no check of the loss, the latents or the gradients can catch this defect, only a check of
    the encodings (`return_encodings=True`) themselves."""
    assert worst("default", "cls_sum") < 1e-3
