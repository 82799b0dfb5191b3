"""CPU checks of Generalized ICP on the dense clouds (DESIGN.md §3.15).

  * the oracle (tests/harness/gicp_oracle.cpp) against independent restatements: its covariances against numpy's
    U diag(1, 1, 0.001) U^T of each k-NN neighbourhood, its metric against numpy's inverse, each inner loop's end against
    scipy's minimiser of PCL's objective for the same pairs and metric, and its outer stop against a numpy restatement of
    PCL's transformation delta; convergence to the truth on a scene of three planes;
  * the product's kernels (ghicp_icp.cu, metric 2) through the C ABI of the emulated library (tests/harness/emu_library.cpp)
    against the oracle, bit for bit, over the cases of tests/test_icp.py plus one beyond the 1e6 m gate, the four option
    combinations and k = 3, 20, 32, also under a random fiber schedule;
  * each convergence state (SINGULAR included), the parameter block's layout, argument errors, injected allocation failures,
    Prep.icp and both results' normal caches, pipeline.gicp_reg, register_clouds(refine={"metric": "gicp"}), and the `-m gpu`
    test functions of tests/test_zz9_gicp_gpu.py on small clouds."""
import ctypes as C
import math
import os
import subprocess
import sys

import numpy as np
import pytest

import gicp_oracle as go
from test_icp import OPTIONS, cases, clouds, ge, pose, rot_angle, same  # noqa: F401  (ge: fixture)
from test_icp_plane import rt_of, three_planes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EPS = 1e-3   # PCL's gicp_epsilon


def knn_cov_svd(X, k):
    """numpy: per point, the float64 covariance of its k_eff nearest (d2, index) neighbours with its singular values replaced
    by (1, 1, EPS), U diag(1, 1, EPS) U^T, as PCL's GICP builds it."""
    ke = min(k, len(X))
    out = np.empty((len(X), 3, 3))
    for j in range(len(X)):
        d = X - X[j]
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        nb = np.lexsort((np.arange(len(X)), d2))[:ke]
        U, _, _ = np.linalg.svd(np.cov(X[nb].astype(np.float64).T))
        out[j] = U @ np.diag([1.0, 1.0, EPS]) @ U.T
    return out


def cov_of(n):
    n = np.asarray(n, np.float64)
    return np.eye(3)[None] - (1.0 - EPS) * n[:, :, None] * n[:, None, :]


def pcl_delta(a, b, eps_t=1e-8, eps_r=1e-6):
    """PCL's GICP convergence measure between two float32 transforms, restated."""
    d = np.abs(np.asarray(a, np.float32) - np.asarray(b, np.float32)).astype(np.float64)
    r = np.full((4, 4), 1.0 / eps_t)
    r[:3, :3] = 1.0 / eps_r
    return float((r * d).max())


def move64(X, T):
    return X.astype(np.float64) @ T[:3, :3].T + T[:3, 3]


def jittered_planes(n, seed):
    P = three_planes(n, seed).astype(np.float64)
    P += np.random.default_rng(seed + 100).normal(0.0, 0.002, P.shape)
    return P.astype(np.float32)


# ---- the oracle against independent restatements --------------------------------------------------------------------------
def test_covariances_and_metric_equal_numpy():
    Q = jittered_planes(150, 1)
    P = jittered_planes(120, 2)
    _, o = go.gicp(P, Q, max_iterations=1, normal_k=20, steps=True)
    for X, N in ((Q, o["normals_t"]), (P, o["normals_s"])):
        assert np.abs(cov_of(N) - knn_cov_svd(X, 20)).max() <= 1e-5
    # M = inv(R C_s R^T + C_t), R a float32 rotation widened to double, against numpy's inverse
    R = pose(7.0, [0, 0, 0])[:3, :3].astype(np.float32).astype(np.float64)
    rng = np.random.default_rng(3)
    ns = o["normals_s"][rng.integers(0, len(P), 400)]
    nt = o["normals_t"][rng.integers(0, len(Q), 400)]
    M = go.mahalanobis(R, ns, nt)
    want = np.linalg.inv(R[None] @ cov_of(ns) @ R.T[None] + cov_of(nt))
    assert (np.abs(M - want).max(axis=(1, 2)) / np.abs(want).max(axis=(1, 2))).max() <= 1e-12
    assert np.all(np.linalg.eigvalsh(M) > 0.0)


def pcl_objective(P, Qc, M, F0):
    """PCL's f for fixed pairs and metric over x = (rx, ry, rz, tx, ty, tz): T(x) = constructTransformationMatrix(x) F0."""
    W0 = move64(P, F0.astype(np.float64))

    def f(x):
        r = move64(W0, rt_of(x)) - Qc
        return float(np.einsum("ni,nij,nj->", r, M, r)) / len(r)
    return f


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_inner_loop_ends_at_the_minimiser_of_pcls_objective(seed):
    """Where an inner loop ended on its tolerance, F is scipy's minimiser of PCL's objective for that iteration's pairs and
    metric, started from the same F, within 1e-6 rad / 1e-5 m.  (With gicp_reg's epsilons a float32 transform cannot resolve a
    1e-8 m change, and the loops end on a step that no longer lowers f instead; looser epsilons let them end on tolerance.)"""
    from scipy.optimize import minimize
    P, Q = clouds(300, 500, 40 + seed, deg=2.0)
    _, o = go.gicp(P, Q, max_iterations=4, transformation_epsilon=1e-6, rotation_epsilon=1e-5, normal_k=12, steps=True)
    checked = 0
    F_prev = np.eye(4, dtype=np.float32)
    for k in range(o["iterations"]):
        F_k = o["F"][k]
        if o["inner_end"][k] == "tolerance":
            corr = o["corr"][k]
            m = corr >= 0
            M = go.mahalanobis(F_prev[:3, :3].astype(np.float64), o["normals_s"][m], o["normals_t"][corr[m]])
            f = pcl_objective(P[m], Q[corr[m]].astype(np.float64), M, F_prev)
            res = minimize(f, np.zeros(6), method="BFGS", options=dict(gtol=1e-12, maxiter=2000))
            T = rt_of(res.x) @ F_prev.astype(np.float64)
            assert rot_angle(T[:3, :3], F_k[:3, :3].astype(np.float64)) <= 1e-6, k
            assert np.abs(T[:3, 3] - F_k[:3, 3]).max() <= 1e-5, k
            assert f(np.zeros(6)) >= f(res.x)
            checked += 1
        F_prev = F_k
    assert checked >= 1, o["inner_end"]


@pytest.mark.parametrize("eps", [(1e-8, 1e-6), (1e-5, 1e-3)])
def test_outer_stop_is_pcls_delta(eps):
    """A numpy restatement of PCL's criterion gives the oracle's state after every iteration: go on while k < max_iterations
    and delta(F before, F after) >= 1; ITERATIONS at max_iterations, else TRANSFORM."""
    eps_t, eps_r = eps
    P, Q = clouds(300, 500, 9, deg=2.0)
    for K in (3, 40):
        _, o = go.gicp(P, Q, max_iterations=K, transformation_epsilon=eps_t, rotation_epsilon=eps_r, normal_k=12, steps=True)
        F_prev = np.eye(4, dtype=np.float32)
        n = o["iterations"]
        for k in range(n):
            d = pcl_delta(F_prev, o["F"][k], eps_t, eps_r)
            if k < n - 1:
                assert k + 1 < K and d >= 1.0, (k, d)
            F_prev = o["F"][k]
        want = "ITERATIONS" if n == K else "TRANSFORM"
        assert o["state"] == want and (want == "ITERATIONS" or d < 1.0), (o["state"], n, d)
    assert o["state"] == "TRANSFORM" or eps == (1e-8, 1e-6)


def test_oracle_converges_to_the_truth_on_three_planes():
    Q = three_planes(700, 1)
    G = pose(2.0, [0.2, -0.2, 0.1])   # about 2 degrees, 0.3 m
    X = three_planes(400, 2).astype(np.float64)
    P = ((X - G[:3, 3]) @ G[:3, :3]).astype(np.float32)
    Rt, o = go.gicp(P, Q, max_iterations=50, normal_k=20)
    assert o["converged"], o["state"]
    assert rot_angle(Rt[:3, :3], G[:3, :3]) <= 1e-4 and np.abs(Rt[:3, 3] - G[:3, 3]).max() <= 1e-3
    print(dict(iterations=o["iterations"], state=o["state"], inner=o["inner_passes"].tolist(), rot=rot_angle(Rt[:3, :3], G[:3, :3]),
               t=float(np.abs(Rt[:3, 3] - G[:3, 3]).max())))


# ---- the emulated kernels through the C ABI --------------------------------------------------------------------------------
def gicp_cases():
    yield from cases()
    P, Q = clouds(500, 700, 11)
    B = P.copy()
    B[::20] += np.float32([2.0e6, 0.0, 0.0])   # beyond 1e6 m: their nearest target is > 1e12 m^2 away, the gate drops them
    yield "beyond", B, Q, None


@pytest.mark.parametrize("opt", range(4))
@pytest.mark.parametrize("name", ["random", "outside", "far", "utm", "ties", "nan", "beyond"])
def test_emulated_abi_equals_the_oracle(ge, name, opt):
    _, P, Q, G = next(c for c in gicp_cases() if c[0] == name)
    kw = dict(OPTIONS[opt], max_iterations=5)
    got = ge.cloud_icp(P, Q, G, return_moved=True, trace=True, metric="gicp", normal_k=20, **kw)
    want = go.gicp(P, Q, G, normal_k=20, **kw)
    same(got, want)
    assert got[1]["cells_visited"] > 0
    if name == "beyond":
        assert max(got[1]["cor_trace"]) <= len(P) - len(P[::20])


@pytest.mark.parametrize("k", [3, 32])
@pytest.mark.parametrize("opt", range(4))
def test_emulated_abi_equals_the_oracle_for_k(ge, opt, k):
    _, P, Q, G = next(cases())
    kw = dict(OPTIONS[opt], max_iterations=4)
    same(ge.cloud_icp(P, Q, G, return_moved=True, trace=True, metric="gicp", normal_k=k, **kw), go.gicp(P, Q, G, normal_k=k, **kw))


def test_emulated_abi_under_a_random_schedule(g, emu_library_path, tmp_path):
    """GHICP_EMU_SCHED: fibers visited in a fresh random order at every sweep (read once per process: a child process)."""
    _, P, Q, _ = next(cases())
    np.savez(tmp_path / "in.npz", P=P, Q=Q)
    code = ("import sys, numpy as np; sys.path.insert(0, %r); sys.path.insert(0, %r); import ghicp_b200 as g;"
            "from conftest import swap_in_library; swap_in_library(g, %r); a = np.load(%r);"
            "Rt, i = g.cloud_icp(a['P'], a['Q'], None, max_iterations=5, reciprocal=True, trim_ratio=0.8, trace=True,"
            " metric='gicp', normal_k=20);"
            "np.savez(%r, Rt=Rt, mse=i['mse_trace'], cor=i['cor_trace'], f=np.array([i['fitness']]))"
            % (ROOT, os.path.join(ROOT, "tests"), emu_library_path, str(tmp_path / "in.npz"), str(tmp_path / "out.npz")))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, GHICP_EMU_SCHED="11"))
    assert r.returncode == 0, r.stderr[-3000:]
    got = np.load(tmp_path / "out.npz")
    wRt, w = go.gicp(P, Q, None, max_iterations=5, reciprocal=True, trim_ratio=0.8, normal_k=20)
    assert np.array_equal(got["Rt"], wRt) and np.array_equal(got["mse"], w["mse_trace"]) and np.array_equal(got["cor"], w["cor_trace"])
    assert got["f"][0] == w["fitness"]


def test_convergence_states(ge):
    g = ge
    P, Q = clouds(400, 600, 13)
    gi = dict(metric="gicp", normal_k=20)
    Rt, i = g.cloud_icp(P, Q, max_iterations=1, trace=True, **gi)
    assert i["state"] == "ITERATIONS" and i["iterations"] == 1 and i["converged"] and i["warnings"] == 0
    Rt, i = g.cloud_icp(Q, Q, max_iterations=20, **gi)                 # from the truth: the step is exactly the identity
    assert i["state"] == "TRANSFORM" and i["iterations"] == 1 and i["mse"] == 0.0 and np.array_equal(Rt, np.eye(4))
    Rt, i = g.cloud_icp(P + np.float32([1.0e7, 0.0, 0.0]), Q, max_iterations=5, trace=True, **gi)   # every pair beyond the gate
    assert i["state"] == "NO_CORRESPONDENCES" and i["cor"] == 0 and not i["converged"]
    assert i["warnings"] == g.capi.GHICP_W_FEW_PAIRS and np.array_equal(Rt, np.eye(4))
    # points on the x axis: the rotation about it is unobservable, the first system is singular, F stays the guess
    rng = np.random.default_rng(4)
    Ql = np.zeros((300, 3), np.float32)
    Ql[:, 0] = rng.random(300) * 10.0
    Pl = Ql[rng.choice(300, 150, replace=False)].copy()
    Pl[:, 0] += np.float32(0.01)
    Rt, i = g.cloud_icp(Pl, Ql, None, max_iterations=5, trace=True, return_moved=True, **gi)
    assert i["state"] == "SINGULAR" and not i["converged"] and i["warnings"] == g.capi.GHICP_W_SINGULAR
    assert np.array_equal(Rt, np.eye(4)) and i["iterations"] == 1 and i["cor"] > 0
    same((Rt, i), go.gicp(Pl, Ql, None, max_iterations=5, normal_k=20))


def test_params_layout_and_zero_initialised_params(ge):
    """rotation_epsilon sits where reserved[2] was; a parameter block zeroed but for max_iterations is point-to-point, with
    the bits of capi.cloud_icp's metric="point"."""
    g = ge
    Pm = g.capi.IcpParams
    assert C.sizeof(Pm) == 48 and Pm.rotation_epsilon.offset == 40 and Pm.normal_k.offset == 36 and Pm.metric.offset == 32
    P, Q = clouds(60, 80, 17)
    fpp = C.POINTER(C.c_float)
    p = Pm()
    C.memset(C.byref(p), 0, C.sizeof(p))
    p.max_iterations = 5
    out = g.capi.IcpResult()
    moved = np.zeros_like(P)
    rc = g.capi.lib().ghicp_cloud_icp(0, P.ctypes.data_as(fpp), 60, Q.ctypes.data_as(fpp), 80, None, C.byref(p), C.byref(out),
                                      moved.ctypes.data_as(fpp), None, None)
    want = g.cloud_icp(P, Q, max_iterations=5, transformation_epsilon=0.0, fitness_epsilon=0.0, return_moved=True, metric="point")
    assert rc >= 0 and np.array_equal(np.array(out.Rt).reshape(4, 4).T, want[0]) and np.array_equal(moved, want[1]["moved"])
    assert out.iterations == want[1]["iterations"] and out.fitness == want[1]["fitness"]


def test_concurrent_swapped_prep_calls_do_not_deadlock(ge):
    """ghicp_prep_icp(a, b) and ghicp_prep_icp(b, a) with metric 2 from two host threads at once (ctypes releases the GIL during
    the call): each takes both results' locks together, so both finish, with the results of the same calls made one after
    the other.  (On the emulated library the kernels themselves run one call at a time: every launch is under the locks.)"""
    import threading
    g = ge
    T, S, R, t = g.synth.scan_pair(3000, seed=4)
    pt, ps = g.Prep(T, 0.3, 1.0, 1.5), g.Prep(S, 0.3, 1.0, 1.5)
    try:
        G = np.eye(4); G[:3, :3], G[:3, 3] = R, t
        G0, Gi = pose(1.0, [0.1, -0.1, 0.05]) @ G, np.linalg.inv(G)
        gi = dict(max_iterations=3, metric="gicp", normal_k=20)
        want_ab = g.cloud_icp(ps.down(), pt.down(), G0, **gi)[0]
        want_ba = g.cloud_icp(pt.down(), ps.down(), Gi, **gi)[0]
        got, errors_ = {}, []

        def run(name, a, b, guess):
            try:
                for r in range(3):
                    got[(name, r)] = a.icp(b, guess, **gi)[0]
            except Exception as e:   # noqa: BLE001  (reported by the main thread)
                errors_.append(e)
        th = [threading.Thread(target=run, args=("ab", ps, pt, G0), daemon=True),
              threading.Thread(target=run, args=("ba", pt, ps, Gi), daemon=True)]
        for x in th:
            x.start()
        for x in th:
            x.join(timeout=600)
        assert not any(x.is_alive() for x in th), "the swapped calls did not finish"
        assert not errors_, errors_
        for r in range(3):
            assert np.array_equal(got[("ab", r)], want_ab) and np.array_equal(got[("ba", r)], want_ba)
    finally:
        pt.close(); ps.close()


def test_argument_errors_write_nothing_and_metrics_0_1_ignore_rotation_epsilon(ge):
    g = ge
    P, Q = clouds(60, 80, 14)
    L = g.capi.lib()
    fpp = C.POINTER(C.c_float)
    p, q = P.ctypes.data_as(fpp), Q.ctypes.data_as(fpp)
    good = dict(max_iterations=5, reciprocal=0, trim_ratio=0.0, transformation_epsilon=1e-8, fitness_epsilon=1e-5, metric=2)
    moved = np.full((60, 3), 7.0, np.float32)
    cor = np.full(5, 7, np.int32)
    mse = np.full(5, 7.0)
    for bad in (dict(normal_k=2, rotation_epsilon=1e-6), dict(normal_k=33, rotation_epsilon=1e-6), dict(normal_k=20),
                dict(normal_k=20, rotation_epsilon=-1e-6), dict(normal_k=20, rotation_epsilon=float("nan")),
                dict(normal_k=20, rotation_epsilon=float("inf")), dict(normal_k=20, rotation_epsilon=-float("inf"))):
        out = g.capi.IcpResult()
        out.iterations = 12345
        rc = L.ghicp_cloud_icp(0, p, 60, q, 80, None, C.byref(g.capi.IcpParams(**good, **bad)), C.byref(out),
                               moved.ctypes.data_as(fpp), cor.ctypes.data_as(C.POINTER(C.c_int)),
                               mse.ctypes.data_as(C.POINTER(C.c_double)))
        assert rc == -1, (bad, rc)
        assert out.iterations == 12345 and np.all(moved == 7.0) and np.all(cor == 7) and np.all(mse == 7.0)
        assert "metric" in L.ghicp_last_error(None).decode()
    with pytest.raises(g.GhicpError):
        g.cloud_icp(P, Q, metric="gicpp")
    for metric in ("point", "plane"):
        want = g.cloud_icp(P, Q, max_iterations=5, return_moved=True, trace=True, metric=metric, normal_k=20)
        for re in (0.0, -1.0, float("nan"), float("inf"), 1e-6):
            got = g.cloud_icp(P, Q, max_iterations=5, return_moved=True, trace=True, metric=metric, normal_k=20, rotation_epsilon=re)
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
                               C.byref(g.capi.IcpParams(3, 1, 0.8, 1e-8, 1e-5, 2, 20, 1e-6)), C.byref(out), moved.ctypes.data_as(fpp),
                               None, None)
        L.ghicp_emu_fail_allocation(-1)
        assert L.ghicp_emu_live_allocations() == base, k
        if rc == 0:
            break
        failed += 1
        assert rc == -2, (k, rc)
        assert out.iterations == 12345 and np.all(moved == 7.0)
        assert "cloud_icp" in L.ghicp_last_error(None).decode()
    assert failed >= 16 and rc == 0


def test_prep_allocation_failure_returns_nomem_and_leaks_nothing(ge):
    """ghicp_prep_icp with metric 2 under the k-th allocation failing, k = 0, 1, ... until a call succeeds: GHICP_E_NOMEM,
    nothing written; the caches a failed call leaves are whole, and closing both results frees everything."""
    g = ge
    L = g.capi.lib()
    L.ghicp_emu_live_allocations.restype = C.c_longlong
    L.ghicp_emu_fail_allocation.argtypes = [C.c_longlong]
    base = L.ghicp_emu_live_allocations()
    T, S, R, t = g.synth.scan_pair(3000, seed=4)
    pt, ps = g.Prep(T, 0.3, 1.0, 1.5), g.Prep(S, 0.3, 1.0, 1.5)
    try:
        failed = 0
        for k in range(0, 2000):
            out = g.capi.IcpResult()
            out.iterations = 12345
            L.ghicp_emu_fail_allocation(k)
            rc = L.ghicp_prep_icp(ps.h, pt.h, None, C.byref(g.capi.IcpParams(3, 1, 0.8, 1e-8, 1e-5, 2, 20, 1e-6)), C.byref(out))
            L.ghicp_emu_fail_allocation(-1)
            if rc >= 0:
                break
            failed += 1
            assert rc == -2 and out.iterations == 12345, (k, rc)
            assert "prep_icp" in L.ghicp_last_error(None).decode()
        assert failed >= 10 and rc >= 0
        w = g.cloud_icp(ps.down(), pt.down(), None, max_iterations=3, reciprocal=True, trim_ratio=0.8, metric="gicp", normal_k=20)
        assert np.array_equal(np.array(out.Rt).reshape(4, 4).T, w[0])
    finally:
        pt.close(); ps.close()
    assert L.ghicp_emu_live_allocations() == base


def test_prep_icp_equals_the_stand_alone_call_and_caches_both_normals(ge):
    g = ge
    T, S, R, t = g.synth.scan_pair(6000, seed=4)
    pt, ps = g.Prep(T, 0.3, 1.0, 1.5), g.Prep(S, 0.3, 1.0, 1.5)
    try:
        G = np.eye(4); G[:3, :3], G[:3, 3] = R, t
        G0 = pose(2.0, [0.3, -0.2, 0.1]) @ G
        gi = dict(metric="gicp", normal_k=20)
        # (the emulator's events time nothing: tests/test_zz9_gicp_gpu.py checks the build times of the caches)
        a = ps.icp(pt, G0, max_iterations=4, reciprocal=True, trim_ratio=0.7, **gi)
        b = ps.icp(pt, G0, max_iterations=4, reciprocal=True, trim_ratio=0.7, **gi)
        w = g.cloud_icp(ps.down(), pt.down(), G0, max_iterations=4, reciprocal=True, trim_ratio=0.7, **gi)
        for x in (a, b):
            assert np.array_equal(x[0], w[0]) and x[1]["fitness"] == w[1]["fitness"] and x[1]["cor"] == w[1]["cor"]
            assert x[1]["iterations"] == w[1]["iterations"] and x[1]["cells_visited"] == w[1]["cells_visited"]
        assert np.array_equal(a[0], go.gicp(ps.down(), pt.down(), G0, max_iterations=4, reciprocal=True, trim_ratio=0.7)[0])
        c = ps.icp(pt, G0, max_iterations=4, metric="gicp", normal_k=8)   # another k: both results' normals are replaced
        assert np.array_equal(c[0], g.cloud_icp(ps.down(), pt.down(), G0, max_iterations=4, metric="gicp", normal_k=8)[0])
        d = ps.icp(pt, G0, max_iterations=4, metric="plane", normal_k=8)  # point-to-plane reads the target's k = 8 normals
        assert np.array_equal(d[0], g.cloud_icp(ps.down(), pt.down(), G0, max_iterations=4, metric="plane", normal_k=8)[0])
        Gi = np.linalg.inv(G0)   # the roles swapped: each result's normals serve as the other role's
        e = pt.icp(ps, Gi, max_iterations=4, **gi)
        assert np.array_equal(e[0], g.cloud_icp(pt.down(), ps.down(), Gi, max_iterations=4, **gi)[0])
        f = ps.icp(ps, None, max_iterations=3, **gi)   # source == target: one lock, one set of normals
        assert f[1]["state"] == "TRANSFORM" and np.array_equal(f[0], np.eye(4))
        assert np.array_equal(ps.icp(pt, G0, max_iterations=4, reciprocal=True, trim_ratio=0.7, **gi)[0], a[0])
    finally:
        pt.close(); ps.close()


def test_pipeline_gicp_reg(ge):
    g = ge
    P, Q = clouds(400, 600, 16)
    assert g.gicp_reg(P, Q + np.float32(100.0), 10, False, True, 0.1, 20, 0.3) is None      # no overlap at all
    Rt, info = g.gicp_reg(P, Q, 10, True, True, 0.1, 12, 0.0)
    assert info["overlap_ratio"] == g.cal_overlap(P, Q, 0.1)
    want = go.gicp(P, Q, None, max_iterations=10, normal_k=12)   # PCL's GICP: reciprocal and the rejector do not apply
    assert np.array_equal(Rt, want[0]) and np.array_equal(info["moved"], want[1]["moved"]) and info["fitness"] == want[1]["fitness"]
    Rt2, info2 = g.gicp_reg(P, Q, 10, False, False, 0.1, 12)
    assert np.array_equal(Rt2, Rt) and "overlap_ratio" not in info2


def test_register_clouds_refine_gicp(ge):
    g = ge
    T, S, _, _ = g.synth.scan_pair(6000, seed=4)
    kw = dict(corr_type=g.CT_NNR, feature_type=g.FT_FPFH, max_iter=20)
    Rt0, base = g.register_clouds(T, S, 0.3, 1.0, 1.5, **kw)
    ref = dict(max_iter=6, reciprocal=True, trimmed_thre_dis=0.3)
    Rt, info = g.register_clouds(T, S, 0.3, 1.0, 1.5, refine=dict(ref, metric="gicp", covariance_k=12), **kw)
    D_s, D_t = S[g.voxel_downsample(S, 0.3)], T[g.voxel_downsample(T, 0.3)]
    assert np.array_equal(info["icp"]["Rt_before"], Rt0)
    rho = g.cloud_overlap(D_s, D_t, Rt0, thre_dis=0.3, fitness=False)["ratio"]
    # the library's extension: reciprocal and the trimmed rejector honoured, as for the other metrics
    want = go.gicp(D_s, D_t, Rt0, max_iterations=6, reciprocal=True, trim_ratio=min(rho, 1.0), normal_k=12)
    assert np.array_equal(Rt, want[0]) and info["icp"]["fitness"] == want[1]["fitness"]
    for bad in (dict(ref, metric="gicpp"), dict(ref, metric="gicp", covariance_k=2)):
        with pytest.raises(g.GhicpError):
            g.register_clouds(T, S, 0.3, 1.0, 1.5, refine=bad, **kw)


@pytest.mark.parametrize("name,kw", [("test_equals_oracle", dict(n_points=3000)),
                                     ("test_million_points_equal_oracle_grid", dict(n_points=4000)),
                                     ("test_two_calls_are_identical", dict(n_points=3000)),
                                     ("test_cxx_gicp_reg_matches_python", dict(n_points=2000))])
def test_gpu_test_functions_on_the_emulated_library(ge, name, kw, tmp_path, emu_library_path, monkeypatch):
    import test_zz9_gicp_gpu as t
    fn = getattr(t, name)
    if name == "test_cxx_gicp_reg_matches_python":
        monkeypatch.setenv("LD_LIBRARY_PATH", os.path.dirname(emu_library_path) + os.pathsep + os.environ.get("LD_LIBRARY_PATH", ""))
        fn(ge, tmp_path, **kw)
    else:
        fn(ge, **kw)
