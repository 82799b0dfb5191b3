"""ctypes face of tests/harness/sor_oracle.cpp — the canonical statistical outlier removal of DESIGN.md §3.16, on the CPU (TEST
INFRASTRUCTURE).  Compiled on first use into the temporary directory (the source tree may be read-only)."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "harness", "sor_oracle.cpp")
_lib = None
fp, dp, ip, lp = C.POINTER(C.c_float), C.POINTER(C.c_double), C.POINTER(C.c_int), C.POINTER(C.c_longlong)


def lib():
    global _lib
    if _lib is None:
        with open(SRC, "rb") as fh:
            tag = hashlib.sha1(fh.read()).hexdigest()[:12]
        out = os.path.join(tempfile.gettempdir(), f"ghicp_sor_oracle_{os.getuid()}_{tag}.so")
        if not os.path.exists(out):
            tmp = f"{out}.{os.getpid()}.tmp"
            r = subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-pthread", "-shared", "-o", tmp, SRC],
                               capture_output=True, text=True)
            assert r.returncode == 0, r.stderr[-3000:]
            os.replace(tmp, out)
        L = C.CDLL(out)
        L.sor_oracle.argtypes = [fp, C.c_longlong, C.c_int, C.c_double, C.c_int, fp, ip, lp, dp, lp]
        _lib = L
    return _lib


def sor(xyz, mean_k, std_mul, grid=False):
    """dict: kept (ascending indices), distances [n] float32 (NaN for non-finite points), mean, stddev, threshold, n_finite,
    k_eff.  grid=True searches through the oracle's own grid instead of brute force (same bits)."""
    P = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
    n = len(P)
    dist = np.zeros(n, np.float32)
    kept = np.zeros(max(n, 1), np.int32)
    nk, stats, counts = C.c_longlong(0), np.zeros(3), np.zeros(2, np.int64)
    rc = lib().sor_oracle(P.ctypes.data_as(fp), n, int(mean_k), float(std_mul), int(grid), dist.ctypes.data_as(fp),
                          kept.ctypes.data_as(ip), C.byref(nk), stats.ctypes.data_as(dp), counts.ctypes.data_as(lp))
    assert rc == 0, rc
    return dict(kept=kept[:nk.value].copy(), distances=dist, mean=float(stats[0]), stddev=float(stats[1]),
                threshold=float(stats[2]), n_finite=int(counts[0]), k_eff=int(counts[1]))


def with_std_mul(o, std_mul):
    """The oracle result `o` at another std_mul: the distances, mean and stddev do not depend on it."""
    thr = o["mean"] + float(std_mul) * o["stddev"]
    d = o["distances"].astype(np.float64)
    keep = ~np.isnan(d) & ~(d > thr)
    return dict(o, threshold=thr, kept=np.flatnonzero(keep).astype(np.int32))
