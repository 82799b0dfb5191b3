"""CPU-side checks of the drop-in boundary: the C-ABI library builds for sm_90a, loads, exports every
symbol include/ghicp_b200.h declares, and refuses to run without a GPU (no CPU fallback)."""
import ctypes as C
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    txt = open(os.path.join(ROOT, "include", "ghicp_b200.h")).read()
    return sorted(set(re.findall(r"^(?:int|const char \*)\s*(ghicp_[a-z0-9_]+)\(", txt, flags=re.M)))


def test_header_symbols_all_exported(g):
    L = C.CDLL(g.lib_path())
    syms = declared_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(L, s), f"{s} declared in include/ghicp_b200.h but not exported"
    assert set(syms) == set(g.capi.EXPORTS)


def test_abi_version(g):
    assert g.lib().ghicp_abi_version() == 2


def test_struct_sizes_match_header(g):
    # ghicp_config: 3 int + 7 float + 2 int + double + 2 int + fpfh_matrix_free + solver + 4 reserved (natural alignment)
    assert C.sizeof(g.Config) == 88
    assert C.sizeof(g.IterStats) % 8 == 0


def test_no_gpu_means_loud_failure(g):
    if g.device_count() > 0:
        pytest.skip("a GPU is visible here")
    sc = g.synth.config1(50, 60)
    with pytest.raises(g.GhicpError) as ei:
        g.registration.from_scene(sc, g.FT_NONE, g.CT_NN)
    assert ei.value.code == -6  # GHICP_E_NODEV


def test_product_never_imports_oracle():
    """The product path must not route through the oracle (or any CPU fallback)."""
    pkg = os.path.join(ROOT, "gh-icp_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp", ".hpp")):
                txt = open(os.path.join(dirpath, f), errors="ignore").read()
                assert "import oracle" not in txt and "from oracle" not in txt, f
                assert "liboracle" not in txt and "ghicp_oracle.h" not in txt, f


def test_sass_is_sm90a(g):
    import shutil
    import subprocess
    tool = shutil.which("cuobjdump") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    out = subprocess.run([tool, "-lelf", g.lib_path()], capture_output=True, text=True).stdout
    assert "sm_90a" in out
