"""The C-ABI library loads without a GPU and exports exactly what include/xclip_b200.h declares."""
import ctypes
import re
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


def _declared():
    text = (ROOT / "include" / "xclip_b200.h").read_text()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(xclip_[a-z0-9_]+)\s*\(", text)))


def test_header_symbols_exported_and_bound():
    from x_clip_b200 import _lib, build
    build.build()
    lib = _lib.load()
    names = _declared()
    assert len(names) >= 15
    for n in names:
        assert hasattr(lib, n), f"{n} declared in the header but not exported"
        assert n in _lib.SIGNATURES, f"{n} has no ctypes signature"
    for n in _lib.SIGNATURES:
        assert n in names, f"{n} bound in python but not declared in the header"


def test_abi_version_and_error_string_without_gpu():
    """ABI 3: the FILIP segment-max and expand entry points take the 16-bit argmax only, and the
    un-fused GEGLU + LayerNorm kernels are gone."""
    from x_clip_b200 import _lib
    lib = _lib.load()
    assert lib.xclip_abi_version() == 3
    assert isinstance(lib.xclip_last_error(), bytes)
    assert lib.xclip_nce_num_col_blocks(1024) == 4
    assert lib.xclip_nce_num_col_blocks(100) == 1


def test_no_cpu_fallback():
    """Without a CUDA device every compute entry fails loudly instead of falling back."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from x_clip_b200 import _lib, kernels
    rc = _lib.load().xclip_init()
    assert rc != 0 and _lib.load().xclip_last_error()
    with pytest.raises(_lib.XClipB200Error):
        kernels.gemm(torch.zeros(8, 8, dtype=torch.bfloat16), torch.zeros(8, 8, dtype=torch.bfloat16))


def test_product_never_imports_oracle():
    import re
    for f in (ROOT / "x_clip_b200").rglob("*.py"):
        assert not re.search(r"^\s*(from|import)\s+oracle|import_module\(.oracle", f.read_text(), re.M), f
        assert "oracle" not in f.read_text(), f   # not even mentioned: keeps the boundary obvious


def test_library_sass_is_wgmma_tma_code():
    """The shipped kernels are sm_90a code: the GEMMs run on warpgroup MMA (HGMMA = wgmma) fed by
    TMA tensor loads (UTMALDG) behind mbarrier pipelines (SYNCS), not on recompiled generic code."""
    import shutil
    import subprocess
    from x_clip_b200 import _lib
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    try:
        sass = subprocess.run([exe, "-sass", str(_lib.LIB_PATH)], capture_output=True, text=True, timeout=300).stdout
    except (FileNotFoundError, subprocess.TimeoutExpired):
        import pytest
        pytest.skip("cuobjdump not available")
    assert "sm_90a" in sass
    for op, least in (("HGMMA", 100), ("UTMALDG", 20), ("SYNCS", 100)):
        assert sass.count(op) >= least, (op, sass.count(op))
