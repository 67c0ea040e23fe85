"""CPU checks of the per-rank fp64 reference (multirank_oracle.py) and of what the gates of
test_gpu_multirank_fp64.py can see (no GPU).

- The rank gradients add up to the single-process gradient of the global batch, parameter by
  parameter; the loss and d temperature are the full values on every rank, not shares of them.
- A rank that returns another rank's gradients (rows mis-sliced by a gather or a reduce-scatter), or the
  gradient of the whole batch (a backward through every rank's latents), moves at least 4 gated families
  by at least 4 of their gates each (`BITE`): it still fails after the kernels' own error, at most one
  gate, is subtracted.
- A rank that skips the all-reduce of d temperature returns d temperature of its own rows only: that
  misses the full value by at least 4 of the d-temperature gate.
"""
import pytest

import multirank_oracle as MR
import step_oracle as SO

BITE = 4.0
FAMILIES = 4          # families a rank defect must move by BITE gates

# (name, world, local batch, empty captions): small cases of test_gpu_multirank_fp64.py
CASES = {"default": ("default", 2, 3, ()), "dcl_extra": ("dcl_extra", 3, 1, ()),
         "simreg": ("simreg", 2, 3, ()), "filip": ("filip_dcl_extra", 2, 3, (4,))}
# d temperature of a rank's own rows is what its backward returns before the all-reduce with an extra
# latent pair and with FILIP; without the pair each rank forms a block of entries instead (both
# directions of its rows' columns), a different partial sum that the check below does not model
DTEMP_CASES = ["dcl_extra", "simreg", "filip"]

_REF = {}


def _refs(case):
    if case not in _REF:
        name, world, b, empty = CASES[case]
        c = MR.make_case(name, world, b, empty=empty)
        _REF[case] = (c, MR.full_reference(c, "cpu"),
                      [MR.rank_reference(c, "cpu", world, r) for r in range(world)])
    return _REF[case]


def _scale(c):
    return SO.GATE_SCALE["filip_dcl_extra"] if c["cfg"].use_all_token_embeds else 1.0


@pytest.mark.parametrize("case", list(CASES))
def test_rank_gradients_add_up_to_the_full_gradient(case):
    c, full, ranks = _refs(case)
    for r, ref in enumerate(ranks):
        assert ref["loss"] == pytest.approx(full["loss"], rel=1e-12), r
        t = ref["grads"]["temperature"].item()
        assert t == pytest.approx(full["grads"]["temperature"].item(), rel=1e-10), (r, "d temperature")
    for k in c["names"]:
        if k == "temperature":
            continue
        f = full["grads"][k]
        parts = [ref["grads"][k] for ref in ranks]
        if SO.is_zero(f):
            assert all(SO.is_zero(p) for p in parts), k
            continue
        total = sum(p for p in parts if p is not None)
        assert SO.rel_fro(total, f) <= 1e-10, (k, SO.rel_fro(total, f))


def _bitten(got, ref, scale):
    r = SO.ratios(got, ref, scale)
    return sorted(f for f, v in r.items() if f not in ("loss", "dtemp") and v >= BITE)


@pytest.mark.parametrize("case", list(CASES))
def test_rank_slicing_defects_are_caught(case):
    c, full, ranks = _refs(case)
    scale = _scale(c)
    for r, ref in enumerate(ranks):
        whole = _bitten(full, ref, scale)
        print(f"BITE whole_batch[{case}.r{r}] {len(whole)} families: {whole}")
        assert len(whole) >= FAMILIES, (r, whole)
        for r2, other in enumerate(ranks):
            if r2 == r:
                continue
            swapped = _bitten(other, ref, scale)
            print(f"BITE rank{r2}_rows[{case}.r{r}] {len(swapped)} families: {swapped}")
            assert len(swapped) >= FAMILIES, (r, r2, swapped)


@pytest.mark.parametrize("case", DTEMP_CASES)
def test_missing_dtemp_all_reduce_is_caught(case):
    c, full, _ = _refs(case)
    world = c["world"]
    want = full["grads"]["temperature"].item()
    gate = SO.DTEMP_REL * abs(want) + SO.DTEMP_ABS
    own = [MR.row_terms_dtemp(c, "cpu", world, r) for r in range(world)]
    assert sum(own) == pytest.approx(want, rel=1e-10, abs=1e-12)
    for r, v in enumerate(own):
        print(f"BITE dtemp_own_rows[{case}.r{r}] {abs(v - want) / gate:.2f}")
        assert abs(v - want) >= BITE * gate, (r, v, want)
