"""ctypes face of tests/harness/sac_oracle.cpp — the canonical SAC-IA definition, one thread (TEST INFRASTRUCTURE), and of the
emulated kernels (tests/harness/sac_emu_harness.cpp).  Compiled on first use into the temporary directory (the source tree may
be read-only)."""
import ctypes as C
import hashlib
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "harness", "sac_oracle.cpp")
SAC_H = os.path.join(ROOT, "gh-icp_b200", "csrc", "ghicp_sac.h")
_lib = None
fp, ip, dp = C.POINTER(C.c_float), C.POINTER(C.c_int), C.POINTER(C.c_double)
u64p = C.POINTER(C.c_ulonglong)


def lib():
    global _lib
    if _lib is None:
        h = hashlib.sha1()
        for f in (SRC, SAC_H):
            with open(f, "rb") as fh:
                h.update(fh.read())
        out = os.path.join(tempfile.gettempdir(), f"ghicp_sac_oracle_{os.getuid()}_{h.hexdigest()[:12]}.so")
        if not os.path.exists(out):
            tmp = f"{out}.{os.getpid()}.tmp"
            r = subprocess.run(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-shared", "-o", tmp, SRC],
                               capture_output=True, text=True)
            assert r.returncode == 0, r.stderr[-3000:]
            os.replace(tmp, out)
        L = C.CDLL(out)
        L.sac_oracle.argtypes = [fp, fp, C.c_int, fp, fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_ulonglong,
                                 ip, ip, ip, fp, u64p, dp, dp, ip]
        L.sac_oracle_feat_knn.argtypes = [fp, ip, C.c_int, fp, C.c_int, C.c_int, ip]
        L.sac_oracle_nearest.argtypes = [fp, C.c_int, fp, C.c_int, fp, C.c_float, fp]
        L.sac_oracle_umeyama.argtypes = [fp, fp, fp, fp, fp]
        _lib = L
    return _lib


def _f32(a, cols):
    return np.ascontiguousarray(a, dtype=np.float32).reshape(-1, cols)


def _call(fn, P, Fs, Q, Ft, iterations=1000, samples=3, k=6, min_sample_distance=0.0, threshold=100.0, seed=0):
    P, Fs, Q, Ft = _f32(P, 3), _f32(Fs, 33), _f32(Q, 3), _f32(Ft, 33)
    H = iterations
    out = dict(samples=np.zeros((H, samples), np.int32), valid=np.zeros(H, np.int32), corr=np.zeros((H, samples), np.int32),
               rt=np.zeros((H, 12), np.float32), err=np.zeros(H, np.uint64))
    Rt, dres, ires = np.zeros(16), np.zeros(3), np.zeros(3, np.int32)
    rc = fn(P.ctypes.data_as(fp), Fs.ctypes.data_as(fp), len(P), Q.ctypes.data_as(fp), Ft.ctypes.data_as(fp), len(Q), H, samples, k,
            min_sample_distance, threshold, seed, out["samples"].ctypes.data_as(ip), out["valid"].ctypes.data_as(ip),
            out["corr"].ctypes.data_as(ip), out["rt"].ctypes.data_as(fp), out["err"].ctypes.data_as(u64p), Rt.ctypes.data_as(dp),
            dres.ctypes.data_as(dp), ires.ctypes.data_as(ip))
    assert rc == 0, rc
    out.update(Rt=Rt.reshape(4, 4).T.copy(), error=float(dres[0]), fitness=float(dres[1]), inliers=int(ires[0]),
               best=int(ires[1]), invalid=int(ires[2]), cell=float(dres[2]))
    return out


def sac(P, Fs, Q, Ft, **kw):
    """The oracle: dict of per-hypothesis samples / valid / corr / rt [H][12] (R row-major, t) / err (units of 2^-32) and the
    result Rt (4x4), error, fitness, inliers, best (h*), invalid."""
    return _call(lib().sac_oracle, P, Fs, Q, Ft, **kw)


def feat_knn(Fs, idx, Ft, k):
    Fs, Ft = _f32(Fs, 33), _f32(Ft, 33)
    idx = np.ascontiguousarray(idx, np.int32)
    ke = min(k, len(Ft))
    out = np.zeros((len(idx), ke), np.int32)
    assert lib().sac_oracle_feat_knn(Fs.ctypes.data_as(fp), idx.ctypes.data_as(ip), len(idx), Ft.ctypes.data_as(fp), len(Ft), k,
                                     out.ctypes.data_as(ip)) == ke
    return out


def nearest(P, Q, rt12, threshold):
    P, Q = _f32(P, 3), _f32(Q, 3)
    rt12 = np.ascontiguousarray(rt12, np.float32)
    out = np.zeros(len(P), np.float32)
    lib().sac_oracle_nearest(P.ctypes.data_as(fp), len(P), Q.ctypes.data_as(fp), len(Q), rt12.ctypes.data_as(fp), threshold,
                             out.ctypes.data_as(fp))
    return out


def umeyama(mu_s, mu_d, sigma):
    """The oracle's float32 Umeyama on float32 moments (sigma row-major 3x3): (R 3x3, t) as float32."""
    mu_s, mu_d = np.ascontiguousarray(mu_s, np.float32), np.ascontiguousarray(mu_d, np.float32)
    sigma = np.ascontiguousarray(sigma, np.float32).reshape(9)
    R, t = np.zeros(9, np.float32), np.zeros(3, np.float32)
    lib().sac_oracle_umeyama(mu_s.ctypes.data_as(fp), mu_d.ctypes.data_as(fp), sigma.ctypes.data_as(fp), R.ctypes.data_as(fp),
                             t.ctypes.data_as(fp))
    return R.reshape(3, 3), t


def build_emu_harness(out_dir):
    out = os.path.join(str(out_dir), "libsac_emu_harness.so")
    src = os.path.join(ROOT, "tests", "harness", "sac_emu_harness.cpp")
    extra = os.environ.get("GHICP_EMU_CXXFLAGS", "").split()
    r = subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-ffp-contract=off", "-DGHICP_EMU_HOST"] + extra +
                       ["-I" + os.path.join(ROOT, "tests", "harness", "cuda_emu"), "-x", "c++", "-shared", "-o", out, src],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return out


def emu(path, P, Fs, Q, Ft, **kw):
    """The product's kernels on the CPU emulation shim, same dict as sac() (+ the scoring grid's cell edge)."""
    L = C.CDLL(path)
    L.emu_sac.argtypes = [fp, fp, C.c_int, fp, fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_ulonglong,
                          ip, ip, ip, fp, u64p, dp, dp, ip]
    return _call(L.emu_sac, P, Fs, Q, Ft, **kw)
