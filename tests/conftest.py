import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def build_emulated_library(out_dir):
    """tests/harness/emu_library.cpp -> <out_dir>/libghicp_b200.so: the whole C ABI over the emulated kernels (TEST
    INFRASTRUCTURE; see tests/test_emulated_abi.py).  GHICP_EMU_CXXFLAGS adds compiler flags (sanitizers)."""
    import subprocess
    out = os.path.join(str(out_dir), "libghicp_b200.so")   # the product's soname: ghicp_cli finds it through LD_LIBRARY_PATH
    extra = os.environ.get("GHICP_EMU_CXXFLAGS", "").split()
    r = subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-ffp-contract=off", "-DGHICP_EMU_HOST"] + extra +
                       ["-I" + os.path.join(ROOT, "tests", "harness", "cuda_emu"), "-I" + os.path.join(ROOT, "include"), "-x", "c++",
                        "-shared", "-Wl,--no-undefined", "-o", out, os.path.join(ROOT, "tests", "harness", "emu_library.cpp"), "-ldl"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return out


def swap_in_library(g, path):
    """Make the Python binding call `path` instead of libghicp_b200.so; returns the real handle (to restore)."""
    import ctypes
    real = g.capi.lib()
    emu = ctypes.CDLL(path)
    for name in g.capi.EXPORTS:
        f, e = getattr(real, name), getattr(emu, name)
        if f.argtypes is not None:
            e.argtypes = f.argtypes
        e.restype = f.restype
    g.capi._lib = emu
    return real


@pytest.fixture(scope="session")
def emu_library_path(tmp_path_factory):
    return build_emulated_library(tmp_path_factory.mktemp("emulib"))


@pytest.fixture(scope="session")
def g(request):
    """The product package, with the library built (nvcc cross-compiles here without a GPU).
    Developer switch, never set by the driver: GHICP_TEST_EMULATED_ABI=1 runs the `-m gpu` tests on a machine WITHOUT a GPU
    against the emulated library (all-double kernels; nothing about the TMA / wgmma kernels is exercised that way):
        GHICP_TEST_EMULATED_ABI=1 python -m pytest tests/test_gpu_parity.py -m gpu -q"""
    import ghicp_b200
    ghicp_b200.build_library()
    if os.environ.get("GHICP_TEST_EMULATED_ABI"):
        emu = request.getfixturevalue("emu_library_path")
        swap_in_library(ghicp_b200, emu)
        # the C++ drivers the tests start (dropin_demo, ghicp_cli) resolve libghicp_b200.so through the loader path
        os.environ["LD_LIBRARY_PATH"] = os.path.dirname(emu) + os.pathsep + os.environ.get("LD_LIBRARY_PATH", "")
    return ghicp_b200


@pytest.fixture(scope="session")
def orc():
    """The CPU oracle (test infrastructure)."""
    import oracle
    oracle.build()
    return oracle


@pytest.fixture()
def scratch_cwd(tmp_path, monkeypatch):
    """The reference's Km::output writes Corres.txt into the CWD (src/km.cpp:148)."""
    monkeypatch.chdir(tmp_path)
    return tmp_path


@pytest.fixture(scope="session")
def emu_harness_path(tmp_path_factory):
    """tests/harness/kernel_logic_harness.cpp: the product's .cu files compiled as plain C++ against the host emulation shim
    (tests/harness/cuda_emu), built once per session.  GHICP_EMU_CXXFLAGS="-fsanitize=address,undefined
    -fno-omit-frame-pointer" (with LD_PRELOAD=libasan.so) runs the emulated kernels under the sanitizers."""
    import subprocess
    out = tmp_path_factory.mktemp("emu") / "libkernel_logic_harness.so"
    src = os.path.join(ROOT, "tests", "harness", "kernel_logic_harness.cpp")
    extra = os.environ.get("GHICP_EMU_CXXFLAGS", "").split()
    r = subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-ffp-contract=off", "-DGHICP_EMU_HOST"] + extra +
                       ["-I" + os.path.join(ROOT, "tests", "harness", "cuda_emu"), "-x", "c++", "-shared", "-o", str(out), src],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return str(out)
