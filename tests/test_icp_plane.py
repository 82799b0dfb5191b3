"""CPU checks of point-to-plane ICP on the dense clouds (DESIGN.md §3.14).

  * the oracle (tests/harness/icp_plane_oracle.cpp) against an independent numpy restatement: the same kept pairs
    every iteration, target normals equal to numpy's k-NN covariance eigenvectors up to sign, and each step within 1e-6 rad /
    1e-6 m of a float64 solve of PCL's normal equations at the origin on the same pairs; at UTM offsets its centred equations
    hold where PCL's float32 raw-coordinate ones do not; convergence to the truth on a scene of three planes;
  * the product's kernels (ghicp_icp.cu) through the C ABI of the emulated library (tests/harness/emu_library.cpp) against
    the oracle, bit for bit, over the cases of tests/test_icp.py, the four option combinations and k = 3, 20, 32, also under a
    random fiber schedule;
  * the oracle's normals against ghicp_fpfh_extract's, each convergence state (SINGULAR included), argument errors, injected
    allocation failures, Prep.icp and its normal cache, pipeline.ptplicp_reg, register_clouds(refine={"metric": "plane"}),
    the deterministic sin / cos against the C library's, and the `-m gpu` test functions of tests/test_zz9_icp_plane_gpu.py
    on small clouds."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import icp_oracle as io
import icp_plane_oracle as po
from test_icp import OPTIONS, cases, clouds, ge, move32, nn, pose, rot_angle, same  # noqa: F401  (ge: fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
UTM = np.float32([500000.0, 4400000.0, 50.0])


def knn_normals(Q, k):
    """numpy k-NN normals: the k_eff nearest (d2, index) targets, float64 covariance, the smallest eigh vector (sign free)."""
    ke = min(k, len(Q))
    N = np.empty((len(Q), 3))
    for j in range(len(Q)):
        d = Q - Q[j]
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        nb = np.lexsort((np.arange(len(Q)), d2))[:ke]
        X = Q[nb].astype(np.float64)
        _, V = np.linalg.eigh(np.cov(X.T))
        N[j] = V[:, 0]
    return N


def rt_of(x):
    """PCL's constructTransformationMatrix(alpha, beta, gamma, tx, ty, tz) in float64."""
    a, b, c = x[:3]
    sa, ca, sb, cb, sg, cg = math.sin(a), math.cos(a), math.sin(b), math.cos(b), math.sin(c), math.cos(c)
    T = np.eye(4)
    T[:3, :3] = [[cg * cb, -sg * ca + cg * sb * sa, sg * sa + cg * sb * ca],
                 [sg * cb, cg * ca + sg * sb * sa, -cg * sa + sg * sb * ca],
                 [-sb, cb * sa, cb * ca]]
    T[:3, 3] = x[3:]
    return T


def pcl_solve(S, Qc, Nc, dtype=np.float64):
    """PCL's TransformationEstimationPointToPlaneLLS on the pairs (S_i, Qc_i, Nc_i): rows [s x n, n], rhs n.(q - s), the
    rows and rhs formed in `dtype` (float32 as PCL does, or float64), the normal equations summed and solved in float64."""
    S, Qc, Nc = (np.asarray(a, dtype) for a in (S, Qc, Nc))
    r = np.concatenate([np.cross(S, Nc), Nc], axis=1).astype(np.float64)
    b = (((Nc[:, 0] * Qc[:, 0] + Nc[:, 1] * Qc[:, 1]) + Nc[:, 2] * Qc[:, 2]) -
         ((Nc[:, 0] * S[:, 0] + Nc[:, 1] * S[:, 1]) + Nc[:, 2] * S[:, 2])).astype(np.float64)
    return rt_of(np.linalg.solve(r.T @ r, r.T @ b))


def reject(W, Q, kw):
    """One iteration's kept pairs, restated: brute-force nearest targets, reciprocity, trimming (as tests/test_icp.py)."""
    j, d = nn(W.astype(np.float32), Q)
    corr = j.copy()
    if kw.get("reciprocal"):
        for i in range(len(W)):
            ii, _ = nn(Q[corr[i]][None, :], W)
            if ii[0] != i:
                corr[i] = -1
    if kw.get("trim_ratio"):
        kept = np.flatnonzero(corr >= 0)
        order = kept[np.lexsort((kept, d[kept]))]
        keep = int(math.floor(np.float32(kw["trim_ratio"]) * np.float32(len(kept))))
        corr[order[keep:]] = -1
    return corr


# ---- the oracle against an independent restatement -------------------------------------------------------------------------
@pytest.mark.parametrize("opt", range(4))
def test_oracle_equals_numpy_restatement(opt):
    kw = OPTIONS[opt]
    P, Q = clouds(400, 600, 21 + opt)
    _, o = po.icp_plane(P, Q, max_iterations=5, normal_k=12, steps=True, **kw)
    N = o["normals"]
    ref = knn_normals(Q, 12)
    assert np.all(np.abs(np.abs(np.sum(N * ref, axis=1)) - 1.0) < 1e-4)
    W = P.copy()
    for k in range(o["iterations"]):
        corr = reject(W, Q, kw)
        assert np.array_equal(corr, o["corr"][k]), (k, int((corr != o["corr"][k]).sum()))
        m = corr >= 0
        assert int(m.sum()) == o["cor_trace"][k]
        T = o["T"][k].astype(np.float64)
        R = pcl_solve(W[m], Q[corr[m]], N[corr[m]])
        assert rot_angle(R[:3, :3], T[:3, :3]) <= 1e-6 and np.abs(R[:3, 3] - T[:3, 3]).max() <= 1e-6
        W = move32(W, o["T"][k])


def test_oracle_utm_centred_normal_equations_hold_where_raw_ones_fail():
    """At UTM-scale coordinates PCL's rows, formed in float32 from the raw coordinates, mix entries of ~1e13 with entries of
    ~1 and lose the rotation; the oracle's centred step stays within 1e-5 rad of a float64 solve on the same pairs."""
    P, Q = clouds(500, 700, 5, deg=2.0)
    P, Q = P + UTM, Q + UTM
    _, o = po.icp_plane(P, Q, max_iterations=1, normal_k=12, steps=True)
    m = o["corr"][0] >= 0
    S, Qc, Nc = P[m], Q[o["corr"][0][m]], o["normals"][o["corr"][0][m]]
    # the float64 solve in coordinates centred on the target's first point (the same least-squares problem, well posed)
    c = Q[0].astype(np.float64)
    R = pcl_solve(S.astype(np.float64) - c, Qc.astype(np.float64) - c, Nc)
    assert rot_angle(R[:3, :3], o["T"][0][:3, :3].astype(np.float64)) < 1e-5
    R32 = pcl_solve(S, Qc, Nc, np.float32)
    assert rot_angle(R[:3, :3], R32[:3, :3]) > 1e-4


def three_planes(n, seed, jitter=0.0):
    """Three separate non-parallel patches (ground, two walls), 2 m apart so that no k-NN neighbourhood mixes two of them."""
    rng = np.random.default_rng(seed)
    a, b = rng.random((2, n)) * 8.0
    g = np.stack([a, b, np.zeros(n)], 1)
    w1 = np.stack([np.full(n, 10.0), a, 2.0 + 0.5 * b], 1)
    w2 = np.stack([a, np.full(n, 10.0), 2.0 + 0.5 * b], 1)
    return np.concatenate([g, w1, w2]).astype(np.float32)


def test_oracle_converges_to_the_truth_on_three_planes():
    Q = three_planes(700, 1)
    G = pose(3.0, [0.2, -0.1, 0.15])
    X = three_planes(400, 2)[::1].astype(np.float64)
    P = ((X - G[:3, 3]) @ G[:3, :3]).astype(np.float32)
    Rt, o = po.icp_plane(P, Q, max_iterations=50, normal_k=20)
    assert o["converged"], o["state"]
    assert rot_angle(Rt[:3, :3], G[:3, :3]) <= 1e-4 and np.abs(Rt[:3, 3] - G[:3, 3]).max() <= 1e-3
    print(dict(iterations=o["iterations"], state=o["state"], rot=rot_angle(Rt[:3, :3], G[:3, :3]),
               t=float(np.abs(Rt[:3, 3] - G[:3, 3]).max()), point_to_point=io.icp(P, Q, max_iterations=50)[1]["iterations"]))


def test_deterministic_sincos_within_two_ulp_of_the_c_library():
    """det_sincos (ghicp_solvers_math.h) against numpy's sin / cos (the C library's) over |x| <= 2^20, its documented range;
    NaN beyond it."""
    rng = np.random.default_rng(0)
    x = np.concatenate([[0.0, -0.0, 5e-324, -5e-324, 2.2250738585072014e-308, 1e-300, 1e-20, 1e-9, np.pi, -np.pi, np.pi / 2,
                         -np.pi / 2, np.pi / 4, 3 * np.pi / 4, 2.0 ** 20, -(2.0 ** 20)],
                        rng.uniform(-1e-3, 1e-3, 20000), rng.uniform(-4.0, 4.0, 50000), rng.uniform(-2.0 ** 20, 2.0 ** 20, 50000),
                        np.pi / 2 * np.arange(1, 600000, 97), np.sign(rng.uniform(-1, 1, 50000)) * 10.0 ** rng.uniform(-300, 6, 50000)])
    x = x[np.abs(x) <= 2.0 ** 20]
    s, c = po.det_sincos(x)
    for got, want in ((s, np.sin(x)), (c, np.cos(x))):
        ulps = np.abs(got - want) / np.spacing(np.abs(want))
        assert ulps.max() <= 2.0, (x[ulps.argmax()], ulps.max())
    assert np.array_equal(s[:2], x[:2]) and np.array_equal(np.signbit(s[:2]), np.signbit(x[:2])) and np.all(c[:4] == 1.0)
    s, c = po.det_sincos([2.0 ** 20 + 1.0, np.inf, np.nan])
    assert np.all(np.isnan(s)) and np.all(np.isnan(c))


# ---- the emulated kernels through the C ABI --------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [3, 20, 32])
@pytest.mark.parametrize("opt", range(4))
@pytest.mark.parametrize("name", ["random", "outside", "far", "utm", "ties", "nan"])
def test_emulated_abi_equals_the_oracle(ge, name, opt, k):
    _, P, Q, G = next(c for c in cases() if c[0] == name)
    kw = dict(OPTIONS[opt], max_iterations=6)
    got = ge.cloud_icp(P, Q, G, return_moved=True, trace=True, metric="plane", normal_k=k, **kw)
    want = po.icp_plane(P, Q, G, normal_k=k, **kw)
    same(got, want)
    assert got[1]["cells_visited"] > 0


def test_emulated_abi_under_a_random_schedule(g, emu_library_path, tmp_path):
    """GHICP_EMU_SCHED: fibers visited in a fresh random order at every sweep (read once per process: a child process)."""
    _, P, Q, _ = next(cases())
    np.savez(tmp_path / "in.npz", P=P, Q=Q)
    code = ("import sys, numpy as np; sys.path.insert(0, %r); sys.path.insert(0, %r); import ghicp_b200 as g;"
            "from conftest import swap_in_library; swap_in_library(g, %r); a = np.load(%r);"
            "Rt, i = g.cloud_icp(a['P'], a['Q'], None, max_iterations=6, reciprocal=True, trim_ratio=0.8, trace=True,"
            " metric='plane', normal_k=20);"
            "np.savez(%r, Rt=Rt, mse=i['mse_trace'], cor=i['cor_trace'], f=np.array([i['fitness']]))"
            % (ROOT, os.path.join(ROOT, "tests"), emu_library_path, str(tmp_path / "in.npz"), str(tmp_path / "out.npz")))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, GHICP_EMU_SCHED="11"))
    assert r.returncode == 0, r.stderr[-3000:]
    got = np.load(tmp_path / "out.npz")
    wRt, w = po.icp_plane(P, Q, None, max_iterations=6, reciprocal=True, trim_ratio=0.8, normal_k=20)
    assert np.array_equal(got["Rt"], wRt) and np.array_equal(got["mse"], w["mse_trace"]) and np.array_equal(got["cor"], w["cor_trace"])
    assert got["f"][0] == w["fitness"]


@pytest.mark.parametrize("k", [3, 20, 32])
def test_oracle_normals_equal_fpfh_extract(ge, k):
    """The loop's normals are the §3.10 k-NN normals: the oracle's equal ghicp_fpfh_extract's for the same k (the ABI does not
    output the loop's own; its bit-exact Rt against the oracle covers them)."""
    _, _, Q, _ = next(cases())
    _, o = po.icp_plane(Q[:50], Q, max_iterations=1, normal_k=k, steps=True)
    _, N, status = ge.fpfh_extract(Q, idx=np.zeros(1, np.int32), k=k)
    assert np.array_equal(o["normals"], N) and not status.any()
    for nt in (1, 2):   # fewer than 3 neighbours: CheckNormals' substitute
        _, o = po.icp_plane(Q[:10], Q[:nt], max_iterations=1, normal_k=k, steps=True)
        assert np.array_equal(o["normals"], np.full((nt, 3), 0.577, np.float32))


def test_convergence_states(ge):
    g = ge
    P, Q = clouds(400, 600, 13)
    pl = dict(metric="plane", normal_k=20)
    Rt, i = g.cloud_icp(P, Q, max_iterations=1, trace=True, **pl)
    assert i["state"] == "ITERATIONS" and i["iterations"] == 1 and i["converged"] and i["warnings"] == 0
    Rt, i = g.cloud_icp(Q, Q, max_iterations=20, **pl)                 # identical clouds: the step is exactly the identity
    assert i["state"] == "TRANSFORM" and i["iterations"] == 1 and i["mse"] == 0.0 and np.array_equal(Rt, np.eye(4))
    kw = dict(max_iterations=60, fitness_epsilon=1e-2, transformation_epsilon=0.0)
    Rt, i = g.cloud_icp(P, Q, **kw, **pl)
    assert i["state"] == "REL_MSE" and 1 < i["iterations"] < 60
    same(g.cloud_icp(P, Q, return_moved=True, trace=True, **kw, **pl), po.icp_plane(P, Q, **kw))
    G = pose(5.0, [1.0, 2.0, 0.5])
    Rt, i = g.cloud_icp(P[:2], Q, G, max_iterations=5, trace=True, **pl)  # two source points: fewer than 3 pairs
    assert i["state"] == "NO_CORRESPONDENCES" and not i["converged"] and i["warnings"] == g.capi.GHICP_W_FEW_PAIRS
    # a single plane: every normal parallel, the 6 x 6 system has rank 3 -> SINGULAR at once, F is the guess
    rng = np.random.default_rng(4)
    Qp = np.concatenate([rng.random((500, 2)) * 10.0, np.zeros((500, 1))], 1).astype(np.float32)
    Pp = np.concatenate([rng.random((300, 2)) * 9.0, np.zeros((300, 1))], 1).astype(np.float32)
    Rt, i = g.cloud_icp(Pp, Qp, G, max_iterations=5, trace=True, **pl)
    assert i["state"] == "SINGULAR" and not i["converged"] and i["warnings"] == g.capi.GHICP_W_SINGULAR
    assert np.array_equal(Rt, G.astype(np.float32).astype(np.float64)) and i["iterations"] == 1 and i["cor"] == 300
    w = po.icp_plane(Pp, Qp, G, max_iterations=5)
    assert w[1]["state"] == "SINGULAR" and np.array_equal(w[0], Rt) and w[1]["fitness"] == i["fitness"]
    Rt, i = g.cloud_icp(P, Q[:2], max_iterations=5, **pl)               # two targets: substitute normals, all parallel
    assert i["state"] == "SINGULAR" and i["warnings"] == g.capi.GHICP_W_SINGULAR


def test_argument_errors_write_nothing_and_metric_0_ignores_normal_k(ge):
    g = ge
    P, Q = clouds(60, 80, 14)
    L = g.capi.lib()
    fpp = C.POINTER(C.c_float)
    p, q = P.ctypes.data_as(fpp), Q.ctypes.data_as(fpp)
    good = dict(max_iterations=5, reciprocal=0, trim_ratio=0.0, transformation_epsilon=1e-8, fitness_epsilon=1e-5)
    moved = np.full((60, 3), 7.0, np.float32)
    cor = np.full(5, 7, np.int32)
    mse = np.full(5, 7.0)
    for bad in (dict(metric=2), dict(metric=-1), dict(metric=1, normal_k=2), dict(metric=1, normal_k=33), dict(metric=1, normal_k=0)):
        out = g.capi.IcpResult()
        out.iterations = 12345
        rc = L.ghicp_cloud_icp(0, p, 60, q, 80, None, C.byref(g.capi.IcpParams(**good, **bad)), C.byref(out),
                               moved.ctypes.data_as(fpp), cor.ctypes.data_as(C.POINTER(C.c_int)),
                               mse.ctypes.data_as(C.POINTER(C.c_double)))
        assert rc == -1, (bad, rc)
        assert out.iterations == 12345 and np.all(moved == 7.0) and np.all(cor == 7) and np.all(mse == 7.0)
        assert "metric" in L.ghicp_last_error(None).decode()
    with pytest.raises(g.GhicpError):
        g.cloud_icp(P, Q, metric="planar")
    want = g.cloud_icp(P, Q, max_iterations=5, return_moved=True, trace=True)
    for k in (0, -4, 3, 20, 99):
        got = g.cloud_icp(P, Q, max_iterations=5, return_moved=True, trace=True, metric="point", normal_k=k)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1]["moved"], want[1]["moved"])
        assert np.array_equal(got[1]["mse_trace"], want[1]["mse_trace"]) and got[1]["fitness"] == want[1]["fitness"]


def test_allocation_failure_returns_nomem_and_leaks_nothing(ge):
    g = ge
    L = g.capi.lib()
    L.ghicp_emu_live_allocations.restype = C.c_longlong
    L.ghicp_emu_fail_allocation.argtypes = [C.c_longlong]
    P, Q = clouds(200, 300, 15)
    fpp = C.POINTER(C.c_float)
    base = L.ghicp_emu_live_allocations()
    failed = 0
    for k in range(0, 2000):
        moved = np.full((200, 3), 7.0, np.float32)
        out = g.capi.IcpResult()
        out.iterations = 12345
        L.ghicp_emu_fail_allocation(k)
        rc = L.ghicp_cloud_icp(0, P.ctypes.data_as(fpp), 200, Q.ctypes.data_as(fpp), 300, None,
                               C.byref(g.capi.IcpParams(3, 1, 0.8, 1e-8, 1e-5, 1, 20)), C.byref(out), moved.ctypes.data_as(fpp),
                               None, None)
        L.ghicp_emu_fail_allocation(-1)
        assert L.ghicp_emu_live_allocations() == base, k
        if rc == 0:
            break
        failed += 1
        assert rc == -2, (k, rc)
        assert out.iterations == 12345 and np.all(moved == 7.0)
        assert "cloud_icp" in L.ghicp_last_error(None).decode()
    assert failed >= 14 and rc == 0


def test_prep_icp_equals_the_stand_alone_call_and_caches_the_normals(ge):
    g = ge
    T, S, R, t = g.synth.scan_pair(6000, seed=4)
    pt, ps = g.Prep(T, 0.3, 1.0, 1.5), g.Prep(S, 0.3, 1.0, 1.5)
    try:
        G = np.eye(4); G[:3, :3], G[:3, 3] = R, t
        G0 = pose(2.0, [0.3, -0.2, 0.1]) @ G
        pl = dict(metric="plane", normal_k=20)
        # (the emulator's events time nothing: tests/test_zz9_icp_plane_gpu.py checks the build times of the cache)
        a = ps.icp(pt, G0, max_iterations=6, reciprocal=True, trim_ratio=0.7, **pl)
        b = ps.icp(pt, G0, max_iterations=6, reciprocal=True, trim_ratio=0.7, **pl)
        assert b[1]["stage_ms"]["grid"] == 0.0                          # grid and normals cached
        w = g.cloud_icp(ps.down(), pt.down(), G0, max_iterations=6, reciprocal=True, trim_ratio=0.7, **pl)
        for x in (a, b):
            assert np.array_equal(x[0], w[0]) and x[1]["fitness"] == w[1]["fitness"] and x[1]["cor"] == w[1]["cor"]
            assert x[1]["iterations"] == w[1]["iterations"] and x[1]["cells_visited"] == w[1]["cells_visited"]
        assert np.array_equal(a[0], po.icp_plane(ps.down(), pt.down(), G0, max_iterations=6, reciprocal=True, trim_ratio=0.7)[0])
        c = ps.icp(pt, G0, max_iterations=6, metric="plane", normal_k=8)   # another k: the normals are replaced
        assert np.array_equal(c[0], g.cloud_icp(ps.down(), pt.down(), G0, max_iterations=6, metric="plane", normal_k=8)[0])
        assert ps.icp(pt, G0, max_iterations=2, metric="plane", normal_k=8)[1]["stage_ms"]["grid"] == 0.0
        assert ps.icp(pt, G0, max_iterations=2)[1]["stage_ms"]["grid"] == 0.0          # point-to-point: the grid alone
        d = ps.icp(pt, G0, max_iterations=6, reciprocal=True, trim_ratio=0.7, **pl)    # back to k = 20
        assert np.array_equal(d[0], a[0])
    finally:
        pt.close(); ps.close()


def test_pipeline_ptplicp_reg(ge):
    g = ge
    P, Q = clouds(400, 600, 16)
    assert g.ptplicp_reg(P, Q + np.float32(100.0), 10, False, True, 0.1, 20, 0.3) is None      # no overlap at all
    Rt, info = g.ptplicp_reg(P, Q, 10, True, True, 0.1, 12, 0.0)
    rho = g.cal_overlap(P, Q, 0.1)
    assert info["overlap_ratio"] == rho
    want = po.icp_plane(P, Q, None, max_iterations=10, reciprocal=True, trim_ratio=min(rho, 1.0), normal_k=12)
    assert np.array_equal(Rt, want[0]) and np.array_equal(info["moved"], want[1]["moved"])
    Rt2, _ = g.ptplicp_reg(P, Q, 10, False, False, 0.1, 20)
    assert np.array_equal(Rt2, po.icp_plane(P, Q, None, max_iterations=10, normal_k=20)[0])


def test_register_clouds_refine_point_to_plane(ge):
    g = ge
    T, S, _, _ = g.synth.scan_pair(6000, seed=4)
    kw = dict(corr_type=g.CT_NNR, feature_type=g.FT_FPFH, max_iter=20)
    Rt0, base = g.register_clouds(T, S, 0.3, 1.0, 1.5, **kw)
    ref = dict(max_iter=8, reciprocal=True, trimmed_thre_dis=0.3)
    Rt_p, ip = g.register_clouds(T, S, 0.3, 1.0, 1.5, refine=ref, **kw)
    Rt_q, iq = g.register_clouds(T, S, 0.3, 1.0, 1.5, refine=dict(ref, metric="point"), **kw)
    assert np.array_equal(Rt_p, Rt_q) and ip["icp"]["fitness"] == iq["icp"]["fitness"]
    Rt, info = g.register_clouds(T, S, 0.3, 1.0, 1.5, refine=dict(ref, metric="plane", covariance_k=12), **kw)
    D_s, D_t = S[g.voxel_downsample(S, 0.3)], T[g.voxel_downsample(T, 0.3)]
    assert np.array_equal(info["icp"]["Rt_before"], Rt0)
    rho = g.cloud_overlap(D_s, D_t, Rt0, thre_dis=0.3, fitness=False)["ratio"]
    want = po.icp_plane(D_s, D_t, Rt0, max_iterations=8, reciprocal=True, trim_ratio=min(rho, 1.0), normal_k=12)
    assert np.array_equal(Rt, want[0])
    for bad in (dict(ref, metric="planar"), dict(ref, metric="plane", covariance_k=2)):
        with pytest.raises(g.GhicpError):
            g.register_clouds(T, S, 0.3, 1.0, 1.5, refine=bad, **kw)


@pytest.mark.parametrize("name,kw", [("test_equals_oracle", dict(n_points=3000)),
                                     ("test_million_points_equal_oracle_grid", dict(n_points=4000)),
                                     ("test_two_calls_are_identical", dict(n_points=3000)),
                                     ("test_cxx_ptplicp_reg_matches_python", dict(n_points=2000))])
def test_gpu_test_functions_on_the_emulated_library(ge, name, kw, tmp_path, emu_library_path, monkeypatch):
    import test_zz9_icp_plane_gpu as t
    fn = getattr(t, name)
    if name == "test_cxx_ptplicp_reg_matches_python":
        monkeypatch.setenv("LD_LIBRARY_PATH", os.path.dirname(emu_library_path) + os.pathsep + os.environ.get("LD_LIBRARY_PATH", ""))
        fn(ge, tmp_path, **kw)
    else:
        fn(ge, **kw)
