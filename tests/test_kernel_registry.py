"""Every public wrapper of x_clip_b200.kernels has an fp64 per-call check in bench_call_oracle.CHECKS, or is
a host helper that launches nothing.  A new wrapper fails here until it is one of the two.  Runs without
a GPU."""
import inspect

import bench_call_oracle as BC


def test_every_wrapper_is_checked_or_listed():
    """Listed: a host helper, with the reason it launches nothing."""
    from x_clip_b200 import kernels
    names = set(BC.public_wrappers(kernels))
    checked, helpers = set(BC.CHECKS), set(BC.HOST_HELPERS)
    assert not (checked & helpers), checked & helpers
    listed = checked | helpers
    assert not (names - listed), f"kernels wrappers with no fp64 check: {sorted(names - listed)}"
    assert not (listed - names), f"listed names that are not kernels wrappers: {sorted(listed - names)}"
    for name, why in BC.HOST_HELPERS.items():
        assert why.strip() and "\n" not in why, name
    assert not hasattr(BC, "NOT_REACHED")


def test_no_check_skips_a_variant():
    """A check returns its ratios for every call: none has a path that returns None."""
    for name, c in BC.CHECKS.items():
        src = inspect.getsource(c.check)
        assert "return None" not in src, name


def test_reduction_gates_grow_with_the_rows():
    """The fp32 addition chains of the row reductions at the cfg3 vision shapes (132 SMs): a chunk of
    768 x 98 = 75 264 rows and the ragged one of 256 x 98 = 25 088."""
    import unittest.mock as mock
    with mock.patch.object(BC, "sms", lambda: 132):
        assert BC.adds_ln_dg(75264) == -(-75264 // (264 * 8)) + 8 + 264 + 1
        assert BC.adds_vsum(75264) == -(-75264 // (528 * 8)) + 8 + 528 + 1
        assert BC.adds_ln_dg(1000) == 1 + 8 + 125 + 1
        assert BC.adds_colsum(75264) == 294 + 256 + 1 and BC.adds_colsum(7) == 1 + 7 + 1
        assert BC.adds_ln_dg(75264) > BC.adds_ln_dg(25088) > BC.adds_ln_dg(2112)
