"""ctypes face of tests/harness/gicp_oracle.cpp — the canonical Generalized ICP of DESIGN.md §3.15, one thread (TEST
INFRASTRUCTURE), and the per-pair metric it shares with the kernels.  Compiled on first use into the temporary directory (the
source tree may be read-only).  Outputs have the layout of icp_oracle.icp's."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HARNESS = os.path.join(ROOT, "tests", "harness")
CSRC = os.path.join(ROOT, "gh-icp_b200", "csrc")
SRCS = [os.path.join(HARNESS, "gicp_oracle.cpp"), os.path.join(HARNESS, "icp_plane_oracle.cpp"), os.path.join(HARNESS, "icp_oracle.cpp"),
        os.path.join(HARNESS, "sac_oracle.cpp"), os.path.join(HARNESS, "fpfh_oracle.cpp"), os.path.join(CSRC, "ghicp_sac.h"),
        os.path.join(CSRC, "ghicp_solvers_math.h")]
_lib = None
fp, ip, dp = C.POINTER(C.c_float), C.POINTER(C.c_int), C.POINTER(C.c_double)
STATES = {1: "ITERATIONS", 2: "TRANSFORM", 3: "ABS_MSE", 4: "REL_MSE", 5: "NO_CORRESPONDENCES", 7: "SINGULAR"}
INNER_END = {0: None, 1: "tolerance", 2: "steps", 3: "rejected"}


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha1()
        for f in SRCS:
            with open(f, "rb") as fh:
                h.update(fh.read())
        out = os.path.join(tempfile.gettempdir(), f"ghicp_gicp_oracle_{os.getuid()}_{h.hexdigest()[:12]}.so")
        if not os.path.exists(out):
            tmp = f"{out}.{os.getpid()}.tmp"
            r = subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-o", tmp, SRCS[0]],
                               capture_output=True, text=True)
            assert r.returncode == 0, r.stderr[-3000:]
            os.replace(tmp, out)
        L = C.CDLL(out)
        L.gicp_oracle.argtypes = [fp, C.c_longlong, fp, C.c_longlong, dp, C.c_int, C.c_int, C.c_float, C.c_double, C.c_double,
                                  C.c_int, C.c_int, dp, ip, dp, dp, ip, dp, fp, ip, ip, fp, fp, fp]
        L.gicp_oracle_mahalanobis.argtypes = [dp, fp, fp, C.c_longlong, dp]
        _lib = L
    return _lib


def gicp(P, Q, guess=None, max_iterations=50, reciprocal=False, trim_ratio=0.0, transformation_epsilon=1e-8,
         rotation_epsilon=1e-6, normal_k=20, grid=False, steps=False):
    """(Rt 4x4, info) as capi.cloud_icp(metric="gicp", normal_k=normal_k) returns them with return_moved and trace: info holds
    iterations, state (name), converged, cor, mse, fitness, moved, cor_trace, mse_trace, and inner_passes / inner_end per
    iteration (the sums the inner loop evaluated, and "tolerance", "steps", "rejected" or None).  steps=True adds F [k][4][4]
    (F after each iteration, float32), corr [k][n_finite] (j(i) after the gate and the rejectors, -1 none) and normals_s /
    normals_t (the normals the loop reads).  grid=True searches through the oracle's own grid (same bits)."""
    P = np.ascontiguousarray(P, dtype=np.float32).reshape(-1, 3)
    Q = np.ascontiguousarray(Q, dtype=np.float32).reshape(-1, 3)
    g = None if guess is None else np.ascontiguousarray(np.asarray(guess, np.float64).reshape(4, 4).T).reshape(16)
    K = int(max_iterations)
    nf = int(np.isfinite(P).all(axis=1).sum())
    Rt, info = np.zeros(16), np.zeros(4, np.int32)
    mse, fit = C.c_double(0), C.c_double(0)
    cor_tr, mse_tr, moved, inner = np.zeros(K, np.int32), np.zeros(K), np.zeros_like(P), np.zeros((K, 2), np.int32)
    F = np.zeros((K, 16), np.float32) if steps else None
    corr = np.zeros((K, nf), np.int32) if steps else None
    Ns = np.zeros((nf, 3), np.float32) if steps else None
    Nt = np.zeros((int(np.isfinite(Q).all(axis=1).sum()), 3), np.float32) if steps else None
    rc = lib().gicp_oracle(P.ctypes.data_as(fp), len(P), Q.ctypes.data_as(fp), len(Q), None if g is None else g.ctypes.data_as(dp),
                           K, int(bool(reciprocal)), float(trim_ratio), float(transformation_epsilon), float(rotation_epsilon),
                           int(grid), int(normal_k), Rt.ctypes.data_as(dp), info.ctypes.data_as(ip), C.byref(mse), C.byref(fit),
                           cor_tr.ctypes.data_as(ip), mse_tr.ctypes.data_as(dp), None if F is None else F.ctypes.data_as(fp),
                           inner.ctypes.data_as(ip), None if corr is None else corr.ctypes.data_as(ip), moved.ctypes.data_as(fp),
                           None if Ns is None else Ns.ctypes.data_as(fp), None if Nt is None else Nt.ctypes.data_as(fp))
    assert rc == 0, rc
    k = int(info[0])
    out = dict(iterations=k, state=STATES[int(info[1])], converged=bool(info[2]), cor=int(info[3]), mse=mse.value, fitness=fit.value,
               moved=moved, cor_trace=cor_tr[:k].copy(), mse_trace=mse_tr[:k].copy(), inner_passes=inner[:k, 0].copy(),
               inner_end=[INNER_END[int(w)] for w in inner[:k, 1]])
    if steps:
        out["F"] = F[:k].reshape(k, 4, 4)
        out["corr"] = corr[:k]
        out["normals_s"] = Ns
        out["normals_t"] = Nt
    return Rt.reshape(4, 4).T.copy(), out


def mahalanobis(R, ns, nt):
    """gicp_mahalanobis (ghicp_solvers_math.h) per pair: R 3x3, ns / nt [n][3] float32 normals -> M [n][3][3]."""
    R = np.ascontiguousarray(np.asarray(R, np.float64).reshape(3, 3)).reshape(9)
    ns = np.ascontiguousarray(ns, dtype=np.float32).reshape(-1, 3)
    nt = np.ascontiguousarray(nt, dtype=np.float32).reshape(-1, 3)
    M6 = np.zeros((len(ns), 6))
    lib().gicp_oracle_mahalanobis(R.ctypes.data_as(dp), ns.ctypes.data_as(fp), nt.ctypes.data_as(fp), len(ns), M6.ctypes.data_as(dp))
    M = np.empty((len(ns), 3, 3))
    for e, (a, b) in enumerate(((0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2))):
        M[:, a, b] = M6[:, e]
        M[:, b, a] = M6[:, e]
    return M
