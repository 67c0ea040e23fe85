"""Model and latent widths 128 * {1..8} on the CPU: the oracle against the reference's fixtures at the
new widths (tests/golden/make_golden_widths.py), the parameter tree at those widths, the widths that
stay refused, and no local memory in any row-wise kernel instantiation of the built library."""
import re
import shutil
import subprocess
from pathlib import Path

import pytest

import test_oracle_golden
import test_simreg
from oracle import clip_oracle as O

GOLD = Path(__file__).parent / "golden"
WIDTH_CASES = ["tiny128_h2", "vits16_shaped", "vits16_shaped_drop", "w384_h8", "b16plus_shaped_dcl_extra",
               "vits16_filip", "vits16_text_causal"]
WIDTH_SIMREG_CASES = ["vits16_simreg_extra"]
TINY = dict(num_text_tokens=128, text_enc_depth=1, text_seq_len=16, visual_enc_depth=1,
            visual_image_size=64, visual_patch_size=16)


@pytest.mark.parametrize("case", WIDTH_CASES)
def test_oracle_reproduces_width_goldens(case):
    test_oracle_golden.test_oracle_reproduces_reference(case)


@pytest.mark.parametrize("case", WIDTH_SIMREG_CASES)
def test_oracle_reproduces_width_simreg_goldens(case):
    test_simreg.test_oracle_reproduces_simreg_goldens(case)


@pytest.mark.parametrize("kw", [
    dict(dim_text=128, dim_image=128, dim_latent=128, text_heads=2, visual_heads=2),
    dict(dim_text=384, dim_image=384, dim_latent=384, text_heads=6, visual_heads=6),
    dict(dim_text=384, dim_image=384, dim_latent=384),                                   # 8 heads: inner 512
    dict(dim_text=640, dim_image=896, dim_latent=640, text_heads=10, visual_heads=14,
         decoupled_contrastive_learning=True, extra_latent_projection=True),
    dict(dim_text=1024, dim_image=128, dim_latent=896, text_heads=16, visual_heads=2),
])
def test_state_dict_matches_reference_tree_at_new_widths(kw):
    import x_clip_b200
    kw = dict(TINY, **kw)
    clip = x_clip_b200.CLIP(**kw, visual_patch_dropout=0.)
    shapes = O.param_shapes(O.ClipConfig(**kw))
    sd = clip.state_dict()
    assert set(sd.keys()) == set(shapes.keys())
    for k, v in sd.items():
        assert tuple(v.shape) == shapes[k], k


@pytest.mark.parametrize("key", ["dim_text", "dim_image", "dim_latent"])
@pytest.mark.parametrize("width", [64, 192, 320, 1152])
def test_widths_outside_128_steps_are_refused(key, width):
    import x_clip_b200
    kw = dict(TINY, dim_text=256, dim_image=256, dim_latent=256, text_heads=4, visual_heads=4)
    kw[key] = width
    with pytest.raises(x_clip_b200.Unsupported):
        x_clip_b200.CLIP(**kw)


@pytest.mark.parametrize("kw", [dict(text_dim_head=32), dict(visual_dim_head=32)])
def test_dim_head_32_is_refused_at_new_widths(kw):
    import x_clip_b200
    with pytest.raises(x_clip_b200.Unsupported):
        x_clip_b200.CLIP(**TINY, dim_text=384, dim_image=384, dim_latent=384, text_heads=12, visual_heads=12, **kw)


ROW_KERNELS = ("ln_fwd_kernel", "ln_bwd_kernel", "l2norm_fwd_kernel", "l2norm_bwd_kernel", "ff_bwd_prep_kernel")


def _row_kernel(mangled):
    """which of ROW_KERNELS a mangled name instantiates (the length prefix of the mangled name keeps a
    kernel from matching inside a longer name that ends in it)"""
    return next((k for k in ROW_KERNELS if f"xclip{len(k)}{k}I" in mangled), None)


def test_row_kernels_do_not_spill():
    """Every row-wise instantiation, the 128-column half-vector ones included (Lb1E in the mangled
    name), has no local-memory stack, and all 8 widths of each kernel are in the library."""
    from x_clip_b200 import _lib
    exe = "/usr/local/cuda/bin/cuobjdump"
    if not Path(exe).exists():
        exe = shutil.which("cuobjdump")
    if not exe:
        pytest.skip("cuobjdump not found")
    assert _lib.LIB_PATH.exists(), "libxclip_b200.so is not built"
    text = subprocess.run([exe, "-res-usage", str(_lib.LIB_PATH)], capture_output=True, text=True, check=True).stdout
    found, bad, cur = {}, {}, None
    for line in text.splitlines():
        m = re.search(r"Function\s*:?\s*(\S+)", line)
        if m:
            name = m.group(1).rstrip(":")
            cur = name if _row_kernel(name) else None
            continue
        m = re.search(r"STACK:(\d+)", line)
        if cur and m:
            found.setdefault(_row_kernel(cur), set()).add(cur)
            if int(m.group(1)) != 0:
                bad[cur] = int(m.group(1))
            cur = None
    assert not bad, f"local-memory stack in {bad}"
    for k in ROW_KERNELS:
        names = found.get(k, set())
        assert len(names) == 8, (k, sorted(names))
        assert sum("Lb1E" in n for n in names) == 4, (k, sorted(names))
