"""Compile-side checks of every gemm_bf16_kernel instantiation in the built library: no local-memory
stack (register spills), the producer / consumer register split through setmaxnreg, and no CALL
(ptxas serialises the wgmma pipeline of a kernel that contains a call)."""
import re
import shutil
import subprocess
from pathlib import Path

import pytest

from x_clip_b200 import _lib


def _cuobjdump():
    for cand in ("/usr/local/cuda/bin/cuobjdump", shutil.which("cuobjdump")):
        if cand and Path(cand).exists():
            return cand
    pytest.skip("cuobjdump not found")


def _dump(flag):
    assert _lib.LIB_PATH.exists(), "libxclip_b200.so is not built"
    r = subprocess.run([_cuobjdump(), flag, str(_lib.LIB_PATH)], capture_output=True, text=True, check=True)
    return r.stdout


def _per_function(text):
    """{mangled gemm_bf16_kernel name: its lines}"""
    funcs, cur = {}, None
    for line in text.splitlines():
        m = re.search(r"Function\s*:?\s*(\S+)", line)
        if m:
            name = m.group(1).rstrip(":")
            cur = name if "gemm_bf16_kernel" in name else None
            if cur:
                funcs.setdefault(cur, [])
            continue
        if cur:
            funcs[cur].append(line)
    return funcs


@pytest.fixture(scope="module")
def res_usage():
    funcs = _per_function(_dump("-res-usage"))
    assert funcs, "no gemm_bf16_kernel in the library"
    return funcs


@pytest.fixture(scope="module")
def sass():
    funcs = _per_function(_dump("-sass"))
    assert funcs, "no gemm_bf16_kernel in the library"
    return funcs


def test_gemm_kernels_do_not_spill(res_usage):
    bad = {}
    for name, lines in res_usage.items():
        m = re.search(r"STACK:(\d+)", "\n".join(lines))
        assert m, f"no resource line for {name}"
        if int(m.group(1)) != 0:
            bad[name] = int(m.group(1))
    assert not bad, f"local-memory stack in {bad}"


def test_gemm_kernels_set_register_budgets(sass):
    missing = [n for n, lines in sass.items() if not any("USETMAXREG" in l for l in lines)]
    assert not missing, f"no setmaxnreg in {missing}"


def test_gemm_kernels_contain_no_call(sass):
    calls = [n for n, lines in sass.items() if any(re.search(r"\bCALL\b", l) for l in lines)]
    assert not calls, f"CALL in {calls}"
