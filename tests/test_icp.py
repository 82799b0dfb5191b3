"""CPU checks of point-to-point ICP on the dense clouds (DESIGN.md §3.13).

  * the oracle (tests/harness/icp_oracle.cpp, one thread) against an independent numpy / float64 restatement: the same
    correspondences every iteration (brute-force float32 knn_d2, (d2, index) ties, reciprocity, trimming) and transforms within
    1e-5 rad / 1e-5 m of a float64 Kabsch on the same pairs; its grid mode against its brute force;
  * the product's kernels (ghicp_icp.cu) through the C ABI of the emulated library (tests/harness/emu_library.cpp) against
    the oracle, bit for bit, with all four option combinations: random clouds, a source partly outside the target's box, far
    outliers, UTM-offset coordinates, planted distance ties across cell boundaries, NaN points, a random fiber schedule;
  * each convergence state on purpose, argument errors, an injected allocation failure, Prep.icp, pipeline.icp_reg,
    register_clouds(refine=...), and the `-m gpu` test functions of tests/test_zz8_icp_gpu.py on small clouds."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import icp_oracle as io

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPTIONS = [dict(), dict(reciprocal=True), dict(trim_ratio=0.8), dict(reciprocal=True, trim_ratio=0.7)]


def rot(ax, ay, az):
    import ghicp_b200
    return np.asarray(ghicp_b200.synth.rot_xyz_deg(ax, ay, az))


def pose(deg, t):
    Rt = np.eye(4)
    Rt[:3, :3] = rot(0.3 * deg, -0.2 * deg, deg)
    Rt[:3, 3] = t
    return Rt


def clouds(n_s, n_t, seed, extent=10.0, deg=3.0, t=(0.2, -0.1, 0.05)):
    """Q random in a box; P = a noisy subset of Q moved by the inverse of pose(deg, t), so ICP should find pose(deg, t)."""
    rng = np.random.default_rng(seed)
    Q = (rng.random((n_t, 3)) * extent).astype(np.float32)
    G = pose(deg, t)
    X = Q[rng.choice(n_t, n_s, replace=False)].astype(np.float64) + rng.normal(0, 0.01 * extent / 10, (n_s, 3))
    P = ((X - G[:3, 3]) @ G[:3, :3]).astype(np.float32)
    return P, Q


def move32(A, T):
    """The float32 move of §3.13 in numpy, every operation rounded separately: ((T00 x + T01 y) + T02 z) + T03."""
    A = np.asarray(A, np.float32)
    T = np.asarray(T, np.float32)
    return np.stack([((T[r, 0] * A[:, 0] + T[r, 1] * A[:, 1]) + T[r, 2] * A[:, 2]) + T[r, 3] for r in range(3)], axis=1)


def nn(A, B):
    """(index, d2) of the nearest B point of every A point: float32 (dx*dx + dy*dy) + dz*dz, ties to the smallest index."""
    idx, d2 = np.empty(len(A), np.int64), np.empty(len(A), np.float32)
    for s in range(0, len(A), 256):
        Q = A[s:s + 256]
        dx, dy, dz = (Q[:, None, k] - B[None, :, k] for k in range(3))
        D = (dx * dx + dy * dy) + dz * dz
        idx[s:s + 256] = D.argmin(axis=1)           # the first minimum: the smallest index
        d2[s:s + 256] = D.min(axis=1)
    return idx, d2


def kabsch(S, T):
    ms, mt = S.mean(axis=0), T.mean(axis=0)
    H = (T - mt).T @ (S - ms)
    U, _, Vt = np.linalg.svd(H)
    D = np.diag([1.0, 1.0, np.sign(np.linalg.det(U @ Vt))])
    R = U @ D @ Vt
    return R, mt - R @ ms


def rot_angle(Ra, Rb):
    """Angle of Ra^T Rb in rad from its skew part (well conditioned near 0, unlike acos of the trace)."""
    M = Ra.T @ Rb
    v = 0.5 * np.array([M[2, 1] - M[1, 2], M[0, 2] - M[2, 0], M[1, 0] - M[0, 1]])
    return math.asin(min(1.0, float(np.linalg.norm(v))))


# ---- the oracle against an independent restatement -------------------------------------------------------------------------
@pytest.mark.parametrize("opt", range(4))
@pytest.mark.parametrize("case", ["random", "utm"])
def test_oracle_equals_numpy_restatement(case, opt):
    kw = OPTIONS[opt]
    P, Q = clouds(500, 700, 1 + opt)
    if case == "utm":
        U = np.float32([500000.0, 4400000.0, 50.0])
        P, Q = P + U, Q + U
    _, o = io.icp(P, Q, max_iterations=6, steps=True, **kw)
    W = P.copy()
    for k in range(o["iterations"]):
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
        assert np.array_equal(corr, o["corr"][k]), (k, int((corr != o["corr"][k]).sum()))
        m = corr >= 0
        assert int(m.sum()) == o["cor_trace"][k]
        R, t = kabsch(W[m].astype(np.float64), Q[corr[m]].astype(np.float64))
        T = o["T"][k].astype(np.float64)
        assert rot_angle(R, T[:3, :3]) < 1e-5
        if case == "random":   # at UTM offsets the float32 means of the definition round the translation by up to ~0.5 m
            assert np.abs(t - T[:3, 3]).max() < 1e-5
        W = move32(W, o["T"][k])


def test_oracle_utm_two_pass_moments_hold_where_one_pass_fails():
    """At UTM-scale coordinates the one-pass raw moments (sum s q^T / n - mu_q mu_s^T) lose the covariance: the oracle's
    two-pass transform stays within 1e-5 rad of a float64 Kabsch on the same pairs, the one-pass one does not."""
    P, Q = clouds(500, 700, 5, deg=2.0)
    U = np.float32([500000.0, 4400000.0, 50.0])
    P, Q = P + U, Q + U
    _, o = io.icp(P, Q, max_iterations=1, steps=True)
    m = o["corr"][0] >= 0
    S, T = P[m].astype(np.float64), Q[o["corr"][0][m]].astype(np.float64)
    R, _ = kabsch(S, T)
    assert rot_angle(R, o["T"][0][:3, :3].astype(np.float64)) < 1e-5
    n = len(S)
    raw = (T.T @ S) / n - np.outer(T.mean(axis=0), S.mean(axis=0))     # one pass, in double
    U_, _, Vt = np.linalg.svd(raw.astype(np.float32).astype(np.float64))
    R1 = U_ @ np.diag([1.0, 1.0, np.sign(np.linalg.det(U_ @ Vt))]) @ Vt
    assert rot_angle(R, R1) > 1e-4


@pytest.mark.parametrize("opt", range(4))
def test_oracle_grid_mode_equals_brute_force(opt):
    P, Q = clouds(1500, 2000, 7)
    P[::60] += np.float32([40.0, 0.0, 0.0])
    a = io.icp(P, Q, max_iterations=5, **OPTIONS[opt])
    b = io.icp(P, Q, max_iterations=5, grid=True, **OPTIONS[opt])
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1]["mse_trace"], b[1]["mse_trace"])
    assert a[1]["fitness"] == b[1]["fitness"] and np.array_equal(a[1]["moved"], b[1]["moved"])


# ---- the emulated kernels through the C ABI --------------------------------------------------------------------------------
@pytest.fixture()
def ge(g, emu_library_path):
    from conftest import swap_in_library
    real = swap_in_library(g, emu_library_path)
    try:
        yield g
    finally:
        g.capi._lib = real


def same(got, want):
    """capi.cloud_icp(return_moved=True, trace=True) against icp_oracle.icp: every output bit for bit."""
    Rt, info = got
    wRt, w = want
    assert np.array_equal(Rt, wRt), (Rt, wRt)
    for k in ("iterations", "state", "converged", "cor"):
        assert info[k] == w[k], (k, info[k], w[k])
    assert np.array_equal(info["cor_trace"], w["cor_trace"])
    assert np.array_equal(info["mse_trace"], w["mse_trace"], equal_nan=True)
    assert np.float64(info["mse"]).tobytes() == np.float64(w["mse"]).tobytes()
    assert np.float64(info["fitness"]).tobytes() == np.float64(w["fitness"]).tobytes()
    assert np.array_equal(info["moved"], w["moved"], equal_nan=True)


def cases():
    P, Q = clouds(500, 700, 11)
    yield "random", P, Q, None
    yield "outside", P + np.float32([6.0, 0.0, 0.0]), Q, pose(0.0, [-5.8, 0.0, 0.0])
    F = P.copy(); F[::25] += np.float32([3000.0, -2000.0, 500.0])
    yield "far", F, Q, None
    U = np.float32([500000.0, 4400000.0, 50.0])
    yield "utm", P + U, Q + U, None
    # ties: target points on a lattice of 0.5 m, source points exactly half-way between two lattice points along x (equal
    # float32 d2 to both, across a cell boundary of any grid)
    g = np.arange(0.0, 5.0, 0.5, dtype=np.float32)
    Qt = np.stack(np.meshgrid(g, g, g, indexing="ij"), axis=-1).reshape(-1, 3).astype(np.float32)
    rng = np.random.default_rng(3)
    Pt = Qt[rng.choice(len(Qt), 300, replace=False)].copy()
    Pt[::2, 0] += np.float32(0.25)
    yield "ties", Pt, Qt, None
    N, M = P.copy(), Q.copy()
    N[::30, 1] = np.nan
    N[7::30, 2] = np.inf
    M[::40, 0] = np.nan
    yield "nan", N, M, None


@pytest.mark.parametrize("opt", range(4))
@pytest.mark.parametrize("name", ["random", "outside", "far", "utm", "ties", "nan"])
def test_emulated_abi_equals_the_oracle(ge, name, opt):
    _, P, Q, G = next(c for c in cases() if c[0] == name)
    kw = dict(OPTIONS[opt], max_iterations=8)
    got = ge.cloud_icp(P, Q, G, return_moved=True, trace=True, **kw)
    want = io.icp(P, Q, G, **kw)
    same(got, want)
    assert got[1]["cells_visited"] > 0 and got[1]["candidates"] >= got[1]["cells_visited"] // 64


def test_emulated_abi_under_a_random_schedule(g, emu_library_path, tmp_path):
    """GHICP_EMU_SCHED: fibers visited in a fresh random order at every sweep (read once per process: a child process)."""
    _, P, Q, _ = next(cases())
    np.savez(tmp_path / "in.npz", P=P, Q=Q)
    code = ("import sys, numpy as np; sys.path.insert(0, %r); sys.path.insert(0, %r); import ghicp_b200 as g;"
            "from conftest import swap_in_library; swap_in_library(g, %r); a = np.load(%r);"
            "Rt, i = g.cloud_icp(a['P'], a['Q'], None, max_iterations=6, reciprocal=True, trim_ratio=0.8, trace=True);"
            "np.savez(%r, Rt=Rt, mse=i['mse_trace'], cor=i['cor_trace'], f=np.array([i['fitness']]))"
            % (ROOT, os.path.join(ROOT, "tests"), emu_library_path, str(tmp_path / "in.npz"), str(tmp_path / "out.npz")))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, GHICP_EMU_SCHED="11"))
    assert r.returncode == 0, r.stderr[-3000:]
    got = np.load(tmp_path / "out.npz")
    wRt, w = io.icp(P, Q, None, max_iterations=6, reciprocal=True, trim_ratio=0.8)
    assert np.array_equal(got["Rt"], wRt) and np.array_equal(got["mse"], w["mse_trace"]) and np.array_equal(got["cor"], w["cor_trace"])
    assert got["f"][0] == w["fitness"]


def test_convergence_states(ge):
    g = ge
    P, Q = clouds(400, 600, 13)
    Rt, i = g.cloud_icp(P, Q, max_iterations=1, trace=True)
    assert i["state"] == "ITERATIONS" and i["iterations"] == 1 and i["converged"] and len(i["mse_trace"]) == 1
    Rt, i = g.cloud_icp(Q, Q, max_iterations=20)                           # identical clouds: T_1 is the identity
    assert i["state"] == "TRANSFORM" and i["iterations"] == 1 and i["mse"] == 0.0
    Rt, i = g.cloud_icp(P, Q, max_iterations=60, fitness_epsilon=1e-2, transformation_epsilon=0.0)
    assert i["state"] == "REL_MSE" and 1 < i["iterations"] < 60
    same(g.cloud_icp(P, Q, max_iterations=60, fitness_epsilon=1e-2, transformation_epsilon=0.0, return_moved=True, trace=True),
         io.icp(P, Q, max_iterations=60, fitness_epsilon=1e-2, transformation_epsilon=0.0))
    G = pose(5.0, [1.0, 2.0, 0.5])
    Rt, i = g.cloud_icp(P[:2], Q, G, max_iterations=5, trace=True)       # two source points: fewer than 3 pairs
    assert i["state"] == "NO_CORRESPONDENCES" and not i["converged"] and i["warnings"] == g.capi.GHICP_W_FEW_PAIRS
    assert np.array_equal(Rt, G.astype(np.float32).astype(np.float64)) and i["cor"] == 2
    # reciprocal on two clusters of 3 target points each with 12 source points around one of them: only 3 can be reciprocal,
    # then the trimmed rejector keeps floor(0.5 * 3) = 1
    Qs = np.float32([[0, 0, 0], [1, 0, 0], [0, 1, 0], [10, 0, 0], [11, 0, 0], [10, 1, 0]])
    Ps = np.concatenate([Qs[:3] + np.float32([0.01, 0.02, 0.0]) * (k + 1) for k in range(4)])
    Rt, i = g.cloud_icp(Ps, Qs, max_iterations=5, reciprocal=True, trim_ratio=0.5)
    assert i["state"] == "NO_CORRESPONDENCES" and i["cor"] == 1 and np.array_equal(Rt, np.eye(4))
    assert io.icp(Ps, Qs, max_iterations=5, reciprocal=True, trim_ratio=0.5)[1]["state"] == "NO_CORRESPONDENCES"


def test_argument_errors_write_nothing(ge):
    g = ge
    P, Q = clouds(60, 80, 14)
    L = g.capi.lib()
    fpp = C.POINTER(C.c_float)
    p, q = P.ctypes.data_as(fpp), Q.ctypes.data_as(fpp)
    good = dict(max_iterations=5, reciprocal=0, trim_ratio=0.0, transformation_epsilon=1e-8, fitness_epsilon=1e-5)
    nan = float("nan")
    bad_params = [dict(max_iterations=0), dict(trim_ratio=-0.1), dict(trim_ratio=1.5), dict(trim_ratio=nan),
                  dict(transformation_epsilon=-1.0), dict(fitness_epsilon=nan), dict(transformation_epsilon=nan)]
    moved = np.full((60, 3), 7.0, np.float32)
    cor = np.full(5, 7, np.int32)
    mse = np.full(5, 7.0)
    calls = [(p, 0, q, 80, None, good), (p, 60, q, -1, None, good), (None, 60, q, 80, None, good), (p, 60, None, 80, None, good),
             (p, 60, q, 80, np.full(16, np.nan), good), (p, 60, q, 80, np.where(np.eye(4) > 0, np.inf, 0.0).reshape(16), good)]
    calls += [(p, 60, q, 80, None, dict(good, **b)) for b in bad_params]
    for ps, ns, qs, nt, G, prm in calls:
        out = g.capi.IcpResult()
        out.iterations = 12345
        gp = None if G is None else np.ascontiguousarray(G, np.float64)
        rc = L.ghicp_cloud_icp(0, ps, ns, qs, nt, None if gp is None else gp.ctypes.data_as(C.POINTER(C.c_double)),
                               C.byref(g.capi.IcpParams(**prm)), C.byref(out), moved.ctypes.data_as(fpp),
                               cor.ctypes.data_as(C.POINTER(C.c_int)), mse.ctypes.data_as(C.POINTER(C.c_double)))
        assert rc == -1, (prm, rc)
        assert out.iterations == 12345 and np.all(moved == 7.0) and np.all(cor == 7) and np.all(mse == 7.0)
    assert L.ghicp_cloud_icp(0, p, 60, q, 80, None, None, C.byref(g.capi.IcpResult()), None, None, None) == -1
    for bad in (np.full((10, 3), np.nan, np.float32),):
        with pytest.raises(g.GhicpError) as e:
            g.cloud_icp(bad, Q)                                           # no finite source point
        assert e.value.code == -1
        with pytest.raises(g.GhicpError) as e:
            g.cloud_icp(P, bad)                                           # no finite target point
        assert e.value.code == -1


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
                               C.byref(g.capi.IcpParams(3, 1, 0.8, 1e-8, 1e-5)), C.byref(out), moved.ctypes.data_as(fpp), None, None)
        L.ghicp_emu_fail_allocation(-1)
        assert L.ghicp_emu_live_allocations() == base, k
        if rc == 0:
            break
        failed += 1
        assert rc == -2, (k, rc)
        assert out.iterations == 12345 and np.all(moved == 7.0)
        assert "cloud_icp" in L.ghicp_last_error(None).decode()
    assert failed >= 10 and rc == 0


def test_prep_icp_equals_the_stand_alone_call(ge):
    g = ge
    T, S, R, t = g.synth.scan_pair(6000, seed=4)
    pt, ps = g.Prep(T, 0.3, 1.0, 1.5), g.Prep(S, 0.3, 1.0, 1.5)
    try:
        G = np.eye(4); G[:3, :3], G[:3, 3] = R, t
        G0 = pose(2.0, [0.3, -0.2, 0.1]) @ G
        for kw in OPTIONS:
            a = ps.icp(pt, G0, max_iterations=6, **kw)
            b = ps.icp(pt, G0, max_iterations=6, **kw)
            w = g.cloud_icp(ps.down(), pt.down(), G0, max_iterations=6, **kw)
            assert b[1]["stage_ms"]["grid"] == 0.0
            for x in (a, b):
                assert np.array_equal(x[0], w[0]) and x[1]["fitness"] == w[1]["fitness"] and x[1]["cor"] == w[1]["cor"]
                assert x[1]["iterations"] == w[1]["iterations"] and x[1]["cells_visited"] == w[1]["cells_visited"]
        assert np.array_equal(a[0], io.icp(ps.down(), pt.down(), G0, max_iterations=6, **OPTIONS[-1])[0])
    finally:
        pt.close(); ps.close()
    pt, ps = g.Prep(T, 0.3, 1.0, 1.5), g.Prep(S, 0.3, 1.0, 1.5)
    try:
        ps.overlap(pt, G, thre_dis=0.3)                                   # overlap builds the grid; ICP reuses it
        assert ps.icp(pt, G, max_iterations=2)[1]["stage_ms"]["grid"] == 0.0
    finally:
        pt.close(); ps.close()


def test_pipeline_icp_reg(ge):
    g = ge
    P, Q = clouds(400, 600, 16)
    assert g.icp_reg(P, Q + np.float32(100.0), 10, False, True, 0.1, 0.3) is None        # no overlap at all
    Rt, info = g.icp_reg(P, Q, 10, True, True, 0.1, 0.0)
    rho = g.cal_overlap(P, Q, 0.1)
    assert info["overlap_ratio"] == rho
    want = io.icp(P, Q, None, max_iterations=10, reciprocal=True, trim_ratio=min(rho, 1.0))
    assert np.array_equal(Rt, want[0]) and np.array_equal(info["moved"], want[1]["moved"])
    Rt2, _ = g.icp_reg(P, Q, 10, False, False, 0.1)
    assert np.array_equal(Rt2, io.icp(P, Q, None, max_iterations=10)[0])


def test_register_clouds_refine(ge):
    g = ge
    T, S, _, _ = g.synth.scan_pair(6000, seed=4)
    kw = dict(corr_type=g.CT_NNR, feature_type=g.FT_FPFH, max_iter=20)
    Rt0, base = g.register_clouds(T, S, 0.3, 1.0, 1.5, **kw)
    Rt1, same_info = g.register_clouds(T, S, 0.3, 1.0, 1.5, refine=None, **kw)
    for i in (base, same_info):
        i.pop("stage_ms"); i.pop("fpfh_ms", None)
    assert np.array_equal(Rt0, Rt1) and base == same_info and "icp" not in base
    Rt, info = g.register_clouds(T, S, 0.3, 1.0, 1.5, refine=dict(max_iter=8, reciprocal=True, trimmed_thre_dis=0.3),
                                 evaluate=dict(thre_dis=0.3), **kw)
    D_s, D_t = S[g.voxel_downsample(S, 0.3)], T[g.voxel_downsample(T, 0.3)]
    assert np.array_equal(info["icp"]["Rt_before"], Rt0)
    rho = g.cloud_overlap(D_s, D_t, Rt0, thre_dis=0.3, fitness=False)["ratio"]
    assert info["icp"]["trim_ratio"] == rho
    want = io.icp(D_s, D_t, Rt0, max_iterations=8, reciprocal=True, trim_ratio=min(rho, 1.0))
    assert np.array_equal(Rt, want[0])
    assert info["evaluation"]["fitness"] == g.cloud_overlap(D_s, D_t, Rt, thre_dis=0.3)["fitness"]
    with pytest.raises(g.GhicpError):
        g.register_clouds(T, S, 0.3, 1.0, 1.5, refine=dict(reciprocal=True), **kw)


@pytest.mark.parametrize("name,kw", [("test_equals_oracle", dict(n_points=3000)),
                                     ("test_million_points_equal_oracle_grid", dict(n_points=4000)),
                                     ("test_two_calls_are_identical", dict(n_points=3000)),
                                     ("test_cxx_icp_reg_matches_python", dict(n_points=2000))])
def test_gpu_test_functions_on_the_emulated_library(ge, name, kw, tmp_path, emu_library_path, monkeypatch):
    import test_zz8_icp_gpu as t
    fn = getattr(t, name)
    if name == "test_cxx_icp_reg_matches_python":
        monkeypatch.setenv("LD_LIBRARY_PATH", os.path.dirname(emu_library_path) + os.pathsep + os.environ.get("LD_LIBRARY_PATH", ""))
        fn(ge, tmp_path, **kw)
    else:
        fn(ge, **kw)
