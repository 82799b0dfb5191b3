"""ctypes face of tests/harness/overlap_oracle.cpp — the canonical overlap and fitness of DESIGN.md §3.12, one thread (TEST
INFRASTRUCTURE).  Compiled on first use into the temporary directory (the source tree may be read-only)."""
import ctypes as C
import hashlib
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "harness", "overlap_oracle.cpp")
_lib = None
fp, dp, lp = C.POINTER(C.c_float), C.POINTER(C.c_double), C.POINTER(C.c_longlong)


def lib():
    global _lib
    if _lib is None:
        with open(SRC, "rb") as fh:
            tag = hashlib.sha1(fh.read()).hexdigest()[:12]
        out = os.path.join(tempfile.gettempdir(), f"ghicp_overlap_oracle_{os.getuid()}_{tag}.so")
        if not os.path.exists(out):
            tmp = f"{out}.{os.getpid()}.tmp"
            r = subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-o", tmp, SRC],
                               capture_output=True, text=True)
            assert r.returncode == 0, r.stderr[-3000:]
            os.replace(tmp, out)
        L = C.CDLL(out)
        L.overlap_oracle.argtypes = [fp, C.c_longlong, fp, C.c_longlong, dp, C.c_float, C.c_double, C.c_int, fp, lp, dp]
        _lib = L
    return _lib


def overlap(A, B, Rt=None, thre_dis=1.0, max_range=float("inf"), grid=False):
    """dict: d2 [n] float32, overlap, ratio, overlap_rmse, n_fit, fitness, and the point-order sums (overlap_sum, fit_sum).
    grid=True searches through the oracle's own grid instead of brute force (same bits)."""
    A = np.ascontiguousarray(A, dtype=np.float32).reshape(-1, 3)
    B = np.ascontiguousarray(B, dtype=np.float32).reshape(-1, 3)
    m = None if Rt is None else np.ascontiguousarray(np.asarray(Rt, np.float64).reshape(4, 4).T).reshape(16)
    d2 = np.zeros(len(A), np.float32)
    counts, sums = np.zeros(2, np.int64), np.zeros(2)
    rc = lib().overlap_oracle(A.ctypes.data_as(fp), len(A), B.ctypes.data_as(fp), len(B), None if m is None else m.ctypes.data_as(dp),
                              float(thre_dis), float(max_range), int(grid), d2.ctypes.data_as(fp), counts.ctypes.data_as(lp),
                              sums.ctypes.data_as(dp))
    assert rc == 0, rc
    n, ov, nf = len(A), int(counts[0]), int(counts[1])
    return dict(d2=d2, n=n, overlap=ov, ratio=float(np.float32((0.01 + ov) / float(n))),
                overlap_rmse=float(np.sqrt(sums[0] / ov)) if ov else float("nan"), n_fit=nf,
                fitness=float(sums[1] / nf) if nf else sys.float_info.max, overlap_sum=float(sums[0]), fit_sum=float(sums[1]))


def move(A, Rt):
    """The float32 transform of §3.12 in numpy, every operation rounded separately."""
    A = np.asarray(A, np.float32)
    if Rt is None:
        return A.copy()
    R, t = np.asarray(Rt)[:3, :3].astype(np.float32), np.asarray(Rt)[:3, 3].astype(np.float32)
    return np.stack([((R[r, 0] * A[:, 0] + R[r, 1] * A[:, 1]) + R[r, 2] * A[:, 2]) + t[r] for r in range(3)], axis=1)


def numpy_d2(A, B, Rt=None):
    """Brute force in numpy float32 with the same operation order (no limit): min over B of (dx*dx + dy*dy) + dz*dz."""
    P = move(A, Rt)
    B = np.asarray(B, np.float32)
    out = np.empty(len(P), np.float32)
    for s in range(0, len(P), 256):
        Q = P[s:s + 256]
        dx, dy, dz = (Q[:, None, k] - B[None, :, k] for k in range(3))
        out[s:s + 256] = ((dx * dx + dy * dy) + dz * dz).min(axis=1)
    return out
