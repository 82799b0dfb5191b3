"""ctypes face of tests/harness/fpfh_radius_oracle.cpp — the canonical FPFH over radius neighbourhoods, one thread, brute
force (TEST INFRASTRUCTURE).  Compiled on first use into the temporary directory (the source tree may be read-only)."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HARNESS = os.path.join(ROOT, "tests", "harness")
SRC = os.path.join(HARNESS, "fpfh_radius_oracle.cpp")
_lib = None


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha1()
        for f in (SRC, os.path.join(HARNESS, "fpfh_oracle.cpp")):
            with open(f, "rb") as fh:
                h.update(fh.read())
        out = os.path.join(tempfile.gettempdir(), f"ghicp_fpfh_radius_oracle_{os.getuid()}_{h.hexdigest()[:12]}.so")
        if not os.path.exists(out):
            tmp = f"{out}.{os.getpid()}.tmp"
            r = subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-o", tmp, SRC],
                               capture_output=True, text=True)
            assert r.returncode == 0, r.stderr[-3000:]
            os.replace(tmp, out)
        L = C.CDLL(out)
        fp, ip, lp = C.POINTER(C.c_float), C.POINTER(C.c_int), C.POINTER(C.c_longlong)
        L.fpfh_radius_oracle.restype = C.c_longlong
        L.fpfh_radius_oracle.argtypes = [fp, C.c_int, ip, C.c_int, C.c_float, C.c_float, C.c_int, fp, fp, ip, ip, C.c_int, lp,
                                         ip, fp, C.c_longlong]
        _lib = L
    return _lib


def fpfh(xyz, idx=None, rn=0.5, rf=1.0, all_normals=True):
    """(fpfh [len(idx) or n][33], normals [n][3], status [n], computed [n]).  Normals the histograms did not need (and
    all_normals = False) are NaN with status -1; `computed` bit 0 = N_rn list, bit 1 = normal, bit 2 = N_rf list."""
    xyz = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
    n = len(xyz)
    ia = None if idx is None else np.ascontiguousarray(idx, dtype=np.int32).reshape(-1)
    m = n if ia is None else len(ia)
    out = np.zeros((m, 33), np.float32)
    nrm = np.full((n, 3), np.nan, np.float32)
    st = np.full(n, -1, np.int32)
    comp = np.zeros(n, np.int32)
    fp, ip = C.POINTER(C.c_float), C.POINTER(C.c_int)
    r = lib().fpfh_radius_oracle(xyz.ctypes.data_as(fp), n, None if ia is None else ia.ctypes.data_as(ip), m, rn, rf,
                                 int(all_normals), out.ctypes.data_as(fp), nrm.ctypes.data_as(fp), st.ctypes.data_as(ip),
                                 comp.ctypes.data_as(ip), -1, None, None, None, 0)
    assert r >= 0
    return out, nrm, st, comp


def lists(xyz, r):
    """N_r of every point: (counts [n] int64, idx [sum] int32, d2 [sum] float32), rows concatenated in point order."""
    xyz = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
    n = len(xyz)
    fp, ip, lp = C.POINTER(C.c_float), C.POINTER(C.c_int), C.POINTER(C.c_longlong)
    counts = np.zeros(n, np.int64)
    dummy = np.zeros((1, 33), np.float32)
    total = lib().fpfh_radius_oracle(xyz.ctypes.data_as(fp), n, np.zeros(1, np.int32).ctypes.data_as(ip), 0, r, r, 0,
                                     dummy.ctypes.data_as(fp), None, None, None, 0, counts.ctypes.data_as(lp), None, None, 0)
    assert total >= 0
    idx, d2 = np.zeros(max(total, 1), np.int32), np.zeros(max(total, 1), np.float32)
    got = lib().fpfh_radius_oracle(xyz.ctypes.data_as(fp), n, np.zeros(1, np.int32).ctypes.data_as(ip), 0, r, r, 0,
                                   dummy.ctypes.data_as(fp), None, None, None, 0, counts.ctypes.data_as(lp),
                                   idx.ctypes.data_as(ip), d2.ctypes.data_as(fp), total)
    assert got == total
    return counts, idx[:total], d2[:total]
