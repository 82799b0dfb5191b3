"""ctypes face of tests/harness/icp_plane_oracle.cpp — the canonical point-to-plane ICP of DESIGN.md §3.14, one thread (TEST
INFRASTRUCTURE), and the deterministic sin / cos it uses.  Compiled on first use into the temporary directory (the source
tree may be read-only).  Outputs have the layout of icp_oracle.icp's."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HARNESS = os.path.join(ROOT, "tests", "harness")
CSRC = os.path.join(ROOT, "gh-icp_b200", "csrc")
SRCS = [os.path.join(HARNESS, "icp_plane_oracle.cpp"), os.path.join(HARNESS, "icp_oracle.cpp"), os.path.join(HARNESS, "sac_oracle.cpp"),
        os.path.join(HARNESS, "fpfh_oracle.cpp"), os.path.join(CSRC, "ghicp_sac.h"), os.path.join(CSRC, "ghicp_solvers_math.h")]
_lib = None
fp, ip, dp = C.POINTER(C.c_float), C.POINTER(C.c_int), C.POINTER(C.c_double)
STATES = {1: "ITERATIONS", 2: "TRANSFORM", 3: "ABS_MSE", 4: "REL_MSE", 5: "NO_CORRESPONDENCES", 7: "SINGULAR"}


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha1()
        for f in SRCS:
            with open(f, "rb") as fh:
                h.update(fh.read())
        out = os.path.join(tempfile.gettempdir(), f"ghicp_icp_plane_oracle_{os.getuid()}_{h.hexdigest()[:12]}.so")
        if not os.path.exists(out):
            tmp = f"{out}.{os.getpid()}.tmp"
            r = subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-o", tmp, SRCS[0]],
                               capture_output=True, text=True)
            assert r.returncode == 0, r.stderr[-3000:]
            os.replace(tmp, out)
        L = C.CDLL(out)
        L.icp_plane_oracle.argtypes = [fp, C.c_longlong, fp, C.c_longlong, dp, C.c_int, C.c_int, C.c_float, C.c_double, C.c_double,
                                       C.c_int, C.c_int, dp, ip, dp, dp, ip, dp, fp, ip, fp, fp]
        L.icp_det_sincos.argtypes = [dp, C.c_longlong, dp, dp]
        _lib = L
    return _lib


def icp_plane(P, Q, guess=None, max_iterations=50, reciprocal=False, trim_ratio=0.0, transformation_epsilon=1e-8,
              fitness_epsilon=1e-5, normal_k=20, grid=False, steps=False):
    """(Rt 4x4, info) as capi.cloud_icp(metric="plane", normal_k=normal_k) returns them with return_moved and trace: info holds
    iterations, state (name), converged, cor, mse, fitness, moved, cor_trace, mse_trace.  steps=True adds T [k][4][4] (each
    iteration's T_k, float32), corr [k][n_finite] (j(i) after the rejectors, -1 none) and normals [n_finite_target][3] (the
    normals the loop reads).  grid=True searches through the oracle's own grid (same bits)."""
    P = np.ascontiguousarray(P, dtype=np.float32).reshape(-1, 3)
    Q = np.ascontiguousarray(Q, dtype=np.float32).reshape(-1, 3)
    g = None if guess is None else np.ascontiguousarray(np.asarray(guess, np.float64).reshape(4, 4).T).reshape(16)
    K = int(max_iterations)
    nf = int(np.isfinite(P).all(axis=1).sum())
    Rt, info = np.zeros(16), np.zeros(4, np.int32)
    mse, fit = C.c_double(0), C.c_double(0)
    cor_tr, mse_tr, moved = np.zeros(K, np.int32), np.zeros(K), np.zeros_like(P)
    T = np.zeros((K, 16), np.float32) if steps else None
    corr = np.zeros((K, nf), np.int32) if steps else None
    N = np.zeros((int(np.isfinite(Q).all(axis=1).sum()), 3), np.float32) if steps else None
    rc = lib().icp_plane_oracle(P.ctypes.data_as(fp), len(P), Q.ctypes.data_as(fp), len(Q), None if g is None else g.ctypes.data_as(dp),
                                K, int(bool(reciprocal)), float(trim_ratio), float(transformation_epsilon), float(fitness_epsilon),
                                int(grid), int(normal_k), Rt.ctypes.data_as(dp), info.ctypes.data_as(ip), C.byref(mse), C.byref(fit),
                                cor_tr.ctypes.data_as(ip), mse_tr.ctypes.data_as(dp), None if T is None else T.ctypes.data_as(fp),
                                None if corr is None else corr.ctypes.data_as(ip), moved.ctypes.data_as(fp),
                                None if N is None else N.ctypes.data_as(fp))
    assert rc == 0, rc
    k = int(info[0])
    out = dict(iterations=k, state=STATES[int(info[1])], converged=bool(info[2]), cor=int(info[3]), mse=mse.value, fitness=fit.value,
               moved=moved, cor_trace=cor_tr[:k].copy(), mse_trace=mse_tr[:k].copy())
    if steps:
        out["T"] = T[:k].reshape(k, 4, 4)
        out["corr"] = corr[:k]
        out["normals"] = N
    return Rt.reshape(4, 4).T.copy(), out


def det_sincos(x):
    """(sin, cos) of x by ghicp_solvers_math.h's det_sincos, the deterministic pair the point-to-plane step uses."""
    x = np.ascontiguousarray(x, dtype=np.float64).reshape(-1)
    s, c = np.zeros_like(x), np.zeros_like(x)
    lib().icp_det_sincos(x.ctypes.data_as(dp), len(x), s.ctypes.data_as(dp), c.ctypes.data_as(dp))
    return s, c
