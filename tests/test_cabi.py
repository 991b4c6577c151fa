"""CPU: the C-ABI library builds for sm_90a, loads without a GPU and exports every symbol the header declares."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def built():
    import __graft_entry__ as ge
    ge.build()
    import depthmap_b200._lib as L
    return L


def _declared():
    src = open(os.path.join(ROOT, "include", "depthmap_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(dm_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol(built):
    lib = ctypes.CDLL(built.LIB_PATH)
    names = _declared()
    assert len(names) >= 9
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/depthmap_b200.h but not exported"
    assert set(built.EXPORTS) <= set(names)


def test_version_and_error_string(built):
    lib = built.load()
    assert lib.dm_version() >= 100
    assert isinstance(lib.dm_last_error(), bytes)


def test_stereo_params_struct_layout(built):
    # must mirror dm_stereo_params in the header: 5 doubles, 7 int32, 4 int64
    assert ctypes.sizeof(built.StereoParams) == 5 * 8 + 8 * 4 + 4 * 8


def test_ops_fail_loudly_without_gpu(built):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import numpy as np
    from depthmap_b200.normalmap_generation import create_normalmap
    from depthmap_b200.stereoimage_generation import create_stereoimages
    with pytest.raises(RuntimeError, match="no CUDA device"):
        create_normalmap(np.zeros((4, 4), np.uint16))
    with pytest.raises(RuntimeError, match="no CUDA device"):
        create_stereoimages(np.zeros((4, 4, 3), np.uint8), np.zeros((4, 4), np.uint16), 2.5)


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "stable-diffusion-webui-depthmap-script_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", txt, flags=re.M), f
                assert "liboracle" not in txt, f


def test_no_vimnmx_predicate_output_in_sass(built):
    """CUDA 12.9 ptxas has been seen to miscompile (on a Blackwell target; not re-examined on sm_90a) `min/max` followed by an equality test on the same operands (fused into
    VIMNMX with a predicate output of the wrong sense, DESIGN.md "Toolchain note").  The kernels are written to avoid
    the pattern; this keeps it out of the built objects."""
    import glob
    import os
    import re
    import shutil
    import subprocess
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(cuobjdump):
        import pytest
        pytest.skip("cuobjdump not available")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    objs = glob.glob(os.path.join(root, "stable-diffusion-webui-depthmap-script_b200", "_native", "obj", "*.o"))
    assert objs, "build the native library first (python stable-diffusion-webui-depthmap-script_b200/csrc/build.py)"
    pat = re.compile(r"VIMNMX.*P[0-6], P")
    for o in objs:
        sass = subprocess.run([cuobjdump, "-sass", o], capture_output=True, text=True).stdout
        assert not pat.search(sass), o
