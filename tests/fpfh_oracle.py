"""ctypes face of tests/harness/fpfh_oracle.cpp — the canonical FPFH definition, one thread, brute-force k-NN (TEST
INFRASTRUCTURE).  Compiled on first use into the temporary directory (the source tree may be read-only)."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "harness", "fpfh_oracle.cpp")
_lib = None


def lib():
    global _lib
    if _lib is None:
        with open(SRC, "rb") as f:
            tag = hashlib.sha1(f.read()).hexdigest()[:12]
        out = os.path.join(tempfile.gettempdir(), f"ghicp_fpfh_oracle_{os.getuid()}_{tag}.so")
        if not os.path.exists(out):
            tmp = f"{out}.{os.getpid()}.tmp"
            r = subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-o", tmp, SRC],
                               capture_output=True, text=True)
            assert r.returncode == 0, r.stderr[-3000:]
            os.replace(tmp, out)
        L = C.CDLL(out)
        fp, ip = C.POINTER(C.c_float), C.POINTER(C.c_int)
        L.fpfh_oracle.restype = C.c_int
        L.fpfh_oracle.argtypes = [fp, C.c_int, ip, C.c_int, C.c_int, C.c_int, fp, fp, ip, ip, fp, ip]
        _lib = L
    return _lib


def fpfh(xyz, idx=None, k=20, all_normals=True):
    """(fpfh [len(idx) or n][33], normals [n][3], status [n], nb_idx [n][k_eff], nb_d2 [n][k_eff], computed [n]).
    Rows the histograms did not need (and all_normals = False) are NaN / -1 / 0 and flagged in `computed`
    (bit 0 k-NN, bit 1 normal)."""
    xyz = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
    n = len(xyz)
    ia = None if idx is None else np.ascontiguousarray(idx, dtype=np.int32).reshape(-1)
    m = n if ia is None else len(ia)
    ke = min(k, int(np.isfinite(xyz).all(axis=1).sum()))   # non-finite points take no part
    out = np.zeros((m, 33), np.float32)
    nrm = np.full((n, 3), np.nan, np.float32)
    st = np.full(n, -1, np.int32)
    nb = np.full((n, ke), -1, np.int32)
    d2 = np.full((n, ke), np.nan, np.float32)
    comp = np.zeros(n, np.int32)
    fp, ip = C.POINTER(C.c_float), C.POINTER(C.c_int)
    r = lib().fpfh_oracle(xyz.ctypes.data_as(fp), n, None if ia is None else ia.ctypes.data_as(ip), m, k, int(all_normals),
                          out.ctypes.data_as(fp), nrm.ctypes.data_as(fp), st.ctypes.data_as(ip), nb.ctypes.data_as(ip),
                          d2.ctypes.data_as(fp), comp.ctypes.data_as(ip))
    assert r == ke
    return out, nrm, st, nb, d2, comp
