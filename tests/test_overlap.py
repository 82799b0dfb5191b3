"""CPU checks of the overlap and fitness evaluation (DESIGN.md §3.12).

  * the oracle (tests/harness/overlap_oracle.cpp, one thread) against a float32 numpy brute force, scipy's cKDTree, its own
    grid mode and analytic cases;
  * the product's kernels (ghicp_overlap.cu) through the C ABI of the emulated library (tests/harness/emu_library.cpp)
    against the oracle, bit for bit: random clouds, queries outside B's box, far outliers, UTM-like coordinates, finite and
    infinite max_range, the overlap-only mode, a random fiber schedule, Prep.overlap, argument errors, register_clouds, and
    the `-m gpu` test functions of tests/test_zz7_overlap_gpu.py on small clouds;
  * the work counter: far outliers add a bounded number of grid cells per outlier."""
import os
import subprocess
import sys

import numpy as np
import pytest
from scipy.spatial import cKDTree

import overlap_oracle as oo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INF = float("inf")


def rot(ax, ay, az):
    import ghicp_b200
    return np.asarray(ghicp_b200.synth.rot_xyz_deg(ax, ay, az))


def pose(deg, t):
    Rt = np.eye(4)
    Rt[:3, :3] = rot(0.3 * deg, -0.2 * deg, deg)
    Rt[:3, 3] = t
    return Rt


def clouds(n_a, n_b, seed, extent=10.0, offset=(0.0, 0.0, 0.0)):
    rng = np.random.default_rng(seed)
    B = (rng.random((n_b, 3)) * extent + offset).astype(np.float32)
    A = (B[rng.integers(0, n_b, n_a)] + rng.normal(0, 0.05 * extent / 10, (n_a, 3))).astype(np.float32)
    return A, B


# ---- the oracle against independent checks -------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", [0, 1])
def test_oracle_equals_numpy_brute_force(seed):
    A, B = clouds(700, 900, seed)
    Rt = pose(4.0, [0.3, -0.2, 0.1])
    o = oo.overlap(A, B, Rt, 0.3)
    assert np.array_equal(o["d2"], oo.numpy_d2(A, B, Rt))
    assert o["overlap"] == int((o["d2"] < np.float32(0.3) * np.float32(0.3)).sum())
    assert o["fit_sum"] == float(sum(float(x) for x in o["d2"]))


def test_oracle_matches_ckdtree():
    A, B = clouds(2000, 2500, 3)
    Rt = pose(3.0, [0.1, 0.2, 0.0])
    o = oo.overlap(A, B, Rt, 0.2)
    P = oo.move(A, Rt).astype(np.float64)
    dist, _ = cKDTree(B.astype(np.float64)).query(P)
    assert np.allclose(o["d2"], dist ** 2, rtol=2e-6, atol=1e-9)
    r2 = float(np.float32(0.2) * np.float32(0.2))
    away = np.abs(dist ** 2 - r2) > 1e-5 * r2
    assert int(((dist ** 2 < r2) & away).sum()) == int(((o["d2"] < r2) & away).sum())
    assert abs(o["fitness"] - float(np.mean(dist ** 2))) <= 1e-5 * o["fitness"]


@pytest.mark.parametrize("case", ["random", "outside", "far", "utm"])
def test_oracle_grid_mode_equals_brute_force(case):
    A, B = clouds(1500, 2000, 4)
    if case == "outside":
        A = A + np.float32([12.0, -3.0, 5.0])
    elif case == "far":
        A[::50] += np.float32([10000.0, 0.0, 0.0])
    elif case == "utm":
        A, B = A + np.float32([500000.0, 4400000.0, 50.0]), B + np.float32([500000.0, 4400000.0, 50.0])
        B[0] = 0.0
    for m in (INF, 0.5):
        a, b = oo.overlap(A, B, None, 0.25, m), oo.overlap(A, B, None, 0.25, m, grid=True)
        assert np.array_equal(a["d2"], b["d2"]) and a["fit_sum"] == b["fit_sum"] and a["overlap"] == b["overlap"]


def test_oracle_analytic_cases():
    rng = np.random.default_rng(5)
    B = (rng.random((500, 3)) * 4).astype(np.float32)
    o = oo.overlap(B, B, None, 0.1)
    assert o["overlap"] == 500 and o["ratio"] == np.float32((0.01 + 500) / 500) and o["fitness"] == 0.0
    Rt = np.eye(4); Rt[:3, 3] = [0.0, 0.0, 0.5]            # a translated copy, far beyond the spacing
    o = oo.overlap(B, B, Rt, 0.1)
    assert o["n_fit"] == 500 and o["fitness"] > 0
    o = oo.overlap(B + np.float32(100), B, None, 1.0)        # disjoint
    assert o["overlap"] == 0 and o["ratio"] == np.float32(0.01 / 500) and np.isnan(o["overlap_rmse"])
    o = oo.overlap(B + np.float32(100), B, None, 1.0, max_range=1.0)
    assert o["n_fit"] == 0 and o["fitness"] == sys.float_info.max and np.all(np.isinf(o["d2"]))
    o = oo.overlap(B[:1], B[:1], None, 0.5)                  # n = 1
    assert o["overlap"] == 1 and o["ratio"] == np.float32(1.01)
    D = np.repeat(B[:10], 5, axis=0)                         # duplicates
    assert oo.overlap(D, B[:10], None, 0.01)["overlap"] == 50
    r = np.float32(0.3)                                      # planted at exactly d2 == r * r: not counted
    P = np.array([[0, 0, 0]], np.float32)
    Q = np.array([[r, 0, 0]], np.float32)
    o = oo.overlap(P, Q, None, float(r))
    assert o["d2"][0] == r * r and o["overlap"] == 0 and o["n_fit"] == 1


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
    assert np.array_equal(got["d2"], want["d2"])
    assert (got["overlap"], got["n_fit"], got["ratio"]) == (want["overlap"], want["n_fit"], want["ratio"])
    for k in ("fitness", "overlap_rmse"):
        a, b = got[k], want[k]
        assert (np.isnan(a) and np.isnan(b)) or abs(a - b) <= 1e-12 * abs(b), (k, a, b)


def cases():
    A, B = clouds(1200, 1500, 6)
    yield "random", A, B, pose(3.0, [0.2, -0.1, 0.0])
    yield "outside", A + np.float32([15.0, 2.0, -4.0]), B, None
    F = A.copy(); F[::40] += np.float32([3000.0, -2000.0, 500.0])
    yield "far", F, B, None
    U = np.float32([500000.0, 4400000.0, 50.0])
    B2 = B + U; B2[0] = 0.0
    yield "utm", A + U, B2, None


@pytest.mark.parametrize("name", ["random", "outside", "far", "utm"])
def test_emulated_abi_equals_the_oracle(ge, name):
    g = ge
    _, A, B, Rt = next(c for c in cases() if c[0] == name)
    for r, m in ((0.1, INF), (0.3, 0.05), (0.05, 2.0), (0.3, 0.0)):
        got = g.cloud_overlap(A, B, Rt, thre_dis=r, max_range=m, return_d2=True)
        same(got, oo.overlap(A, B, Rt, r, m))
        ov = g.cloud_overlap(A, B, Rt, thre_dis=r, max_range=m, fitness=False)
        assert ov["overlap"] == got["overlap"] and ov["ratio"] == got["ratio"] and ov["n_fit"] == 0
        assert np.isnan(ov["fitness"]) and ov["cells_visited"] <= got["cells_visited"]


def test_emulated_abi_cell_order_equals_input_order(ge, monkeypatch):
    g = ge
    _, A, B, Rt = next(cases())
    a = g.cloud_overlap(A, B, Rt, thre_dis=0.2, return_d2=True)
    monkeypatch.setenv("GHICP_OVERLAP_ORDER", "cell")
    b = g.cloud_overlap(A, B, Rt, thre_dis=0.2, return_d2=True)
    monkeypatch.setenv("GHICP_OVERLAP_ORDER", "input")
    c = g.cloud_overlap(A, B, Rt, thre_dis=0.2, return_d2=True)
    for x in (b, c):
        assert np.array_equal(a["d2"], x["d2"]) and a["fitness"] == x["fitness"] and a["cells_visited"] == x["cells_visited"]


def test_emulated_abi_under_a_random_schedule(g, emu_library_path, tmp_path):
    """GHICP_EMU_SCHED: fibers visited in a fresh random order at every sweep (read once per process: a child process)."""
    _, A, B, Rt = next(cases())
    np.savez(tmp_path / "in.npz", A=A, B=B, Rt=Rt)
    code = ("import sys, numpy as np; sys.path.insert(0, %r); sys.path.insert(0, %r); import ghicp_b200 as g;"
            "from conftest import swap_in_library; swap_in_library(g, %r); a = np.load(%r);"
            "r = g.cloud_overlap(a['A'], a['B'], a['Rt'], thre_dis=0.2, max_range=0.5, return_d2=True);"
            "np.savez(%r, d2=r['d2'], v=np.array([r['overlap'], r['n_fit']]), f=np.array([r['fitness'], r['overlap_rmse']]))"
            % (ROOT, os.path.join(ROOT, "tests"), emu_library_path, str(tmp_path / "in.npz"), str(tmp_path / "out.npz")))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, GHICP_EMU_SCHED="7"))
    assert r.returncode == 0, r.stderr[-3000:]
    got = np.load(tmp_path / "out.npz")
    want = oo.overlap(A, B, Rt, 0.2, 0.5)
    assert np.array_equal(got["d2"], want["d2"]) and got["v"].tolist() == [want["overlap"], want["n_fit"]]
    assert abs(got["f"][0] - want["fitness"]) <= 1e-12 * want["fitness"]


def test_emulated_abi_prep_overlap_keeps_the_grid(ge):
    g = ge
    T, S, R, t = g.synth.scan_pair(6000, seed=4)
    pt, ps = g.Prep(T, 0.3, 1.0, 1.5), g.Prep(S, 0.3, 1.0, 1.5)
    try:
        G = np.eye(4); G[:3, :3], G[:3, 3] = R, t
        a = ps.overlap(pt, G, thre_dis=0.3)
        b = ps.overlap(pt, G, thre_dis=0.3)
        assert b["stage_ms"]["grid"] == 0.0
        want = oo.overlap(ps.down(), pt.down(), G, 0.3)
        for x in (a, b):
            assert (x["overlap"], x["n_fit"], x["ratio"]) == (want["overlap"], want["n_fit"], want["ratio"])
            assert abs(x["fitness"] - want["fitness"]) <= 1e-12 * want["fitness"]
        assert np.float64(a["fitness"]).tobytes() == np.float64(b["fitness"]).tobytes()
        c = ps.overlap(pt, None, thre_dis=0.6, max_range=1.0)          # another threshold on the same grid
        w = oo.overlap(ps.down(), pt.down(), None, 0.6, 1.0)
        assert (c["overlap"], c["n_fit"]) == (w["overlap"], w["n_fit"]) and c["stage_ms"]["grid"] == 0.0
        d = ps.overlap(pt, G, thre_dis=0.3, fitness=False)
        assert d["overlap"] == a["overlap"] and np.isnan(d["fitness"])
    finally:
        pt.close(); ps.close()


def test_emulated_abi_non_finite_points_cost_nothing(ge):
    """NaN / inf points of A (the NaN returns of an organised scan) get d2 = +inf without a walk: they add no cell and no
    candidate.  Non-finite points of B are left out of it, as PCL's KdTreeFLANN leaves them out; a non-finite Rt is refused."""
    g = ge
    A, B = clouds(2000, 4000, 10)
    bad = np.arange(0, len(A), 50)
    An = A.copy()
    An[bad[::2], 0] = np.nan
    An[bad[1::2], 2] = np.inf
    for kw in (dict(), dict(fitness=False), dict(max_range=0.5)):
        a = g.cloud_overlap(A[np.setdiff1d(np.arange(len(A)), bad)], B, thre_dis=0.1, **kw)
        f = g.cloud_overlap(An, B, thre_dis=0.1, **kw)
        assert (f["cells_visited"], f["candidates"], f["overlap"]) == (a["cells_visited"], a["candidates"], a["overlap"])
    f = g.cloud_overlap(An, B, thre_dis=0.1, return_d2=True)
    want = oo.overlap(An, B, None, 0.1)
    same(f, want)
    assert np.all(np.isinf(f["d2"][bad])) and f["n_fit"] == len(A) - len(bad)
    Bn = B.copy()
    Bn[::7, 1] = np.nan
    Bn[3::7, 0] = -np.inf
    got = g.cloud_overlap(A, Bn, thre_dis=0.1, return_d2=True)
    fin = np.isfinite(Bn).all(axis=1)
    same(got, oo.overlap(A, Bn[fin], None, 0.1))
    same(got, oo.overlap(A, Bn, None, 0.1))                                    # the oracle's brute force skips them too
    for Rt in (np.full((4, 4), np.nan), np.where(np.eye(4) > 0, np.inf, 0.0)):
        with pytest.raises(g.GhicpError) as e:
            g.cloud_overlap(A, B, Rt, thre_dis=0.1)
        assert e.value.code == -1
    with pytest.raises(g.GhicpError) as e:
        g.cloud_overlap(A, np.full((10, 3), np.nan, np.float32), thre_dis=0.1)   # no finite point in B
    assert e.value.code == -1


def test_emulated_abi_argument_errors_write_nothing(ge):
    import ctypes as C
    g = ge
    A, B = clouds(50, 60, 7)
    L = g.capi.lib()
    fpp = C.POINTER(C.c_float)
    a, b = A.ctypes.data_as(fpp), B.ctypes.data_as(fpp)
    d2 = np.full(len(A), 7.0, np.float32)
    bad = [(a, 0, b, 60, 0.1, INF, 1, None), (a, 50, b, -1, 0.1, INF, 1, None), (None, 50, b, 60, 0.1, INF, 1, None),
           (a, 50, None, 60, 0.1, INF, 1, None), (a, 50, b, 60, 0.0, INF, 1, None), (a, 50, b, 60, -1.0, INF, 1, None),
           (a, 50, b, 60, float("nan"), INF, 1, None), (a, 50, b, 60, 0.1, -1.0, 1, None), (a, 50, b, 60, 0.1, float("nan"), 1, None),
           (a, 50, b, 60, 0.1, INF, 0, d2.ctypes.data_as(fpp))]
    for pa, na, pb, nb, r, m, fit, pd in bad:
        out = g.capi.OverlapResult()
        out.overlap = 12345
        assert L.ghicp_cloud_overlap(0, pa, na, pb, nb, None, r, m, fit, C.byref(out), pd) == -1
        assert out.overlap == 12345 and np.all(d2 == 7.0)
    assert L.ghicp_cloud_overlap(0, a, 50, b, 60, None, 0.1, INF, 1, None, None) == -1
    with pytest.raises(g.GhicpError):
        g.cloud_overlap(A, B)                                            # no threshold


def test_emulated_abi_register_clouds_evaluation(ge):
    g = ge
    T, S, _, _ = g.synth.scan_pair(6000, seed=4)
    kw = dict(corr_type=g.CT_NNR, feature_type=g.FT_FPFH, max_iter=20)
    _, base = g.register_clouds(T, S, 0.3, 1.0, 1.5, **kw)
    assert "evaluation" not in base
    Rt, info = g.register_clouds(T, S, 0.3, 1.0, 1.5, evaluate=dict(thre_dis=0.3), initial_alignment="fpfh_sac",
                                 sac=dict(iterations=40), **kw)
    e = info["evaluation"]
    D_s, D_t = S[g.voxel_downsample(S, 0.3)], T[g.voxel_downsample(T, 0.3)]
    want = oo.overlap(D_s, D_t, Rt, 0.3)
    assert (e["overlap"], e["n_fit"]) == (want["overlap"], want["n_fit"]) and abs(e["fitness"] - want["fitness"]) <= 1e-12 * want["fitness"]
    assert info["sac"]["evaluation"]["overlap"] == oo.overlap(D_s, D_t, info["sac"]["Rt"], 0.3)["overlap"]
    # the features= path scores the same transform with capi.cloud_overlap
    base_kw = dict(kw, feature_type=g.FT_NONE)
    Rt2, info2 = g.register_clouds(T, S, 0.3, 1.0, 1.5, evaluate=dict(thre_dis=0.3, max_range=0.5), **base_kw,
                                   features=lambda td, tk, sd, sk: g.Keypoints().setCoordinate(sd[sk], td[tk]))
    want2 = oo.overlap(D_s, D_t, Rt2, 0.3, 0.5)
    assert (info2["evaluation"]["overlap"], info2["evaluation"]["n_fit"]) == (want2["overlap"], want2["n_fit"])
    with pytest.raises(g.GhicpError):
        g.register_clouds(T, S, 0.3, 1.0, 1.5, evaluate=dict(max_range=1.0), **kw)


def far_outlier_cost(g, behind, seed=9):
    """Extra B-grid cells per outlier when 1 % of A (3 000 points near B) is moved 10 km beyond B's +x face.  B is a 20 m
    cube of 3 000 random points, plus `behind` metres of the same density behind it (-x, away from the outliers): the side
    facing the outliers is the same.  Returns (extra cells per outlier, cells per in-box query)."""
    rng = np.random.default_rng(seed)
    B = (rng.random((3000, 3)) * 20.0).astype(np.float32)
    A = (B[rng.integers(0, 3000, 3000)] + rng.normal(0, 0.1, (3000, 3))).astype(np.float32)
    if behind > 0:
        n = int(round(3000 * behind / 20.0))
        B = np.concatenate([B, (rng.random((n, 3)) * np.array([behind, 20.0, 20.0]) - np.array([behind, 0, 0])).astype(np.float32)])
    F = A.copy()
    far = np.arange(0, len(A), 100)
    F[far] += np.float32([10000.0, 0.0, 0.0])
    for kw in (dict(fitness=False), dict(max_range=25.0)):          # rejected at B's box: no cell at all
        a = g.cloud_overlap(A, B, thre_dis=0.3, **kw)
        f = g.cloud_overlap(F, B, thre_dis=0.3, **kw)
        assert f["cells_visited"] <= a["cells_visited"] and f["candidates"] <= a["candidates"]
    a = g.cloud_overlap(A, B, thre_dis=0.3)
    f = g.cloud_overlap(F, B, thre_dis=0.3, return_d2=True)
    assert np.array_equal(f["d2"], oo.overlap(F, B, None, 0.3)["d2"])
    return (f["cells_visited"] - a["cells_visited"]) / len(far), a["cells_visited"] / len(A)


def test_far_outliers_add_a_bounded_number_of_cells(ge):
    """The overlap-only mode and a finite max_range reject far outliers at B's box (no cell).  With max_range = inf an outlier
    10 km out must read the first layers of B's facing side — its exact nearest point can lie anywhere on that side, since
    rho^2 / 2D is below 2 cm there — and nothing behind them: the same cube with nine more cubes of points behind it has ten
    times the cells, but the outliers' cost stays that of one or two layers of the facing side (how many depends on where the
    face falls inside its cells, which moves with the grid's origin)."""
    short, q_short = far_outlier_cost(ge, 0.0)
    long_, q_long = far_outlier_cost(ge, 180.0)
    print(dict(short=short, long=long_, cells_per_query=(q_short, q_long)))
    # about 14 x 14 cells of 1.4 m face the outliers; the walk reads about 126 of them per outlier
    assert short <= 140
    assert long_ <= 2.5 * short   # a walk through the grid behind the face would cost about ten times as much


@pytest.mark.parametrize("name,kw", [("test_equals_oracle", dict(n_points=2000)),
                                     ("test_small_clouds_equal_oracle", dict(n_points=1500)),
                                     ("test_million_points_equal_oracle_grid", dict(n_points=3000)),
                                     ("test_two_calls_are_identical", dict(n_points=2000)),
                                     ("test_prep_overlap_equals_the_stand_alone_call", dict(n_points=6000, res=0.3)),
                                     ("test_the_true_pose_scores_best", dict(n_points=4000)),
                                     ("test_cxx_mirror_matches_python", dict(n_points=1500))])
def test_gpu_test_functions_on_the_emulated_library(ge, name, kw, tmp_path, emu_library_path, monkeypatch):
    import test_zz7_overlap_gpu as t
    fn = getattr(t, name)
    if name == "test_cxx_mirror_matches_python":
        monkeypatch.setenv("LD_LIBRARY_PATH", os.path.dirname(emu_library_path) + os.pathsep + os.environ.get("LD_LIBRARY_PATH", ""))
        fn(ge, tmp_path, **kw)
    else:
        fn(ge, **kw)
