"""CPU checks of the FPFH estimator over radius neighbourhoods (DESIGN.md §3.10, "Radius neighbourhoods").

  * the oracle (tests/harness/fpfh_radius_oracle.cpp, brute force, one thread) against an independent numpy brute force of
    the float32 rule, scipy's cKDTree.query_ball_point away from the r2 boundary, a vectorised numpy restatement of normals /
    SPFH / FPFH, and analytic cases;
  * the product's kernels (ghicp_prep.cu: prep_fpfh_radius) run through the host emulation shim
    (tests/harness/fpfh_radius_emu_harness.cpp) against the oracle, bit for bit;
  * the C ABI over the emulated kernels (tests/harness/emu_library.cpp): argument checks, the list budget, register_clouds
    with fpfh_radius, coarsereg_fpfh_sac, and the `-m gpu` test functions of tests/test_zz6_fpfh_radius_gpu.py on smaller
    clouds."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
from scipy.spatial import cKDTree

import fpfh_radius_oracle as fro
from test_prep_oracle import scan_like_cloud

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
f32 = np.float32


def dup_cloud(n, seed):
    P = scan_like_cloud(n, seed, extent=(10.0, 10.0, 3.0))
    rng = np.random.default_rng(seed)
    return np.concatenate([P, P[rng.choice(n, n // 20, replace=False)], P[:1]]).astype(np.float32)


def outlier_cloud(n, seed):
    P = scan_like_cloud(n, seed, extent=(10.0, 10.0, 3.0))
    far = np.array([[400.0, 380.0, 90.0], [-250.0, 10.0, 3.0], [12.0, -600.0, -40.0], [10.0, 10.0, 300.0]], np.float32)
    return np.concatenate([P, far]).astype(np.float32)


CLOUDS = {
    "random": lambda s: np.random.default_rng(s).random((900, 3)).astype(np.float32) * np.float32(5.0),
    "scan": lambda s: scan_like_cloud(1200, s, extent=(10.0, 10.0, 3.0)),
    "dups": lambda s: dup_cloud(900, s),
    "outliers": lambda s: outlier_cloud(1000, s),
}


# ---- an independent numpy restatement --------------------------------------------------------------------------------------
def np_d2(P):
    d = P[:, None, :] - P[None, :, :]                                      # q - p, float32
    return (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]


def np_lists(P, r):
    """Padded N_r lists: (idx [n][kmax] (-1 padding), d2 [n][kmax], counts [n]), ascending (d2, index)."""
    D2 = np_d2(P)
    inside = D2 < f32(r) * f32(r)
    key = np.where(inside, D2, np.inf)
    order = np.argsort(key, axis=1, kind="stable")                         # stable: ties by ascending index
    cnt = inside.sum(axis=1)
    kmax = max(int(cnt.max()), 1)
    order = order[:, :kmax]
    d2 = np.take_along_axis(D2, order, axis=1)
    valid = np.arange(kmax)[None, :] < cnt[:, None]
    return np.where(valid, order, -1).astype(np.int32), np.where(valid, d2, 0).astype(np.float32), cnt


def np_fpfh_radius(P, rn, rf):
    """Whole-cloud FPFH and normals over radius neighbourhoods, vectorised (the definition of DESIGN.md §3.10)."""
    from test_fpfh_estimator import np_jacobi
    P = np.asarray(P, np.float32)
    n = len(P)
    rows = np.arange(n)
    nb, _, cn = np_lists(P, rn)
    sd, sdd = np.zeros((n, 3)), np.zeros((n, 6))
    for j in range(nb.shape[1]):
        ok = (nb[:, j] >= 0)[:, None]
        e = np.where(ok, (P[np.maximum(nb[:, j], 0)] - P).astype(np.float64), 0.0)
        a, b, c = e[:, 0], e[:, 1], e[:, 2]
        sd += e
        sdd += np.stack([a * a, a * b, a * c, b * b, b * c, c * c], axis=1)
    with np.errstate(divide="ignore", invalid="ignore"):
        inv_n, alpha = 1.0 / cn, 1.0 / (cn - 1)
        pr = [(0, 0), (0, 1), (0, 2), (1, 1), (1, 2), (2, 2)]
        cv = np.stack([((sdd[:, i] - sd[:, u] * sd[:, v] * inv_n) * alpha) for i, (u, v) in enumerate(pr)], axis=1).astype(f32)
    cv[cn < 3] = 0
    A = cv[:, [0, 1, 2, 1, 3, 4, 2, 4, 5]].astype(np.float64).reshape(n, 3, 3)
    w, V = np_jacobi(A)
    jm = np.argmin(w, axis=1)
    v = V[rows, :, jm]
    ln = np.sqrt((v[:, 0] * v[:, 0] + v[:, 1] * v[:, 1]) + v[:, 2] * v[:, 2])
    nrm = (v / ln[:, None]).astype(f32)
    s = ((-P[:, 0]) * nrm[:, 0] + (-P[:, 1]) * nrm[:, 1]) + (-P[:, 2]) * nrm[:, 2]
    nrm[s < 0] = -nrm[s < 0]
    nrm[cn < 3] = np.nan

    def dot(x, y):
        return (x[..., 0] * y[..., 0] + x[..., 1] * y[..., 1]) + x[..., 2] * y[..., 2]

    def cross(x, y):
        return np.stack([x[..., 1] * y[..., 2] - x[..., 2] * y[..., 1], x[..., 2] * y[..., 0] - x[..., 0] * y[..., 2],
                         x[..., 0] * y[..., 1] - x[..., 1] * y[..., 0]], axis=-1)

    nb, d2, cf = np_lists(P, rf)
    spfh = np.zeros((n, 33), np.float32)
    with np.errstate(divide="ignore", invalid="ignore"):
        incr = (f32(100.0) / (cf - 1).astype(f32)).astype(f32)
        inv2pi = f32(1.0) / (f32(2.0) * f32(np.pi))
        for j in range(nb.shape[1]):
            qi = np.maximum(nb[:, j], 0)
            npp, nq = nrm, nrm[qi]
            dp = P[qi] - P
            f4 = np.sqrt(dot(dp, dp))
            a1, a2 = dot(npp, dp) / f4, dot(nq, dp) / f4
            sw = (np.abs(a1) < np.abs(a2))[:, None]
            u, other = np.where(sw, nq, npp), np.where(sw, npp, nq)
            dpp = np.where(sw, -dp, dp)
            f3 = np.where(sw[:, 0], -a2, a1)
            vv = cross(dpp, u)
            vn = np.sqrt(dot(vv, vv))
            vv = vv / vn[:, None]
            wv = cross(u, vv)
            f2 = dot(vv, other)
            f1 = np.arctan2(dot(wv, other).astype(np.float64), dot(u, other).astype(np.float64)).astype(f32)
            ok = (nb[:, j] >= 0) & (qi != rows) & (cf > 1) & ~np.isnan(npp[:, 0]) & ~np.isnan(nq[:, 0]) & (f4 != 0) & (vn != 0)
            for off, x in ((0, (f1.astype(np.float64) + np.pi) * np.float64(inv2pi)), (11, (f2.astype(np.float64) + 1.0) * 0.5),
                           (22, (f3.astype(np.float64) + 1.0) * 0.5)):
                h = np.clip(np.nan_to_num(np.floor(11 * x), nan=0.0), 0, 10).astype(np.int64)
                spfh[rows[ok], off + h[ok]] += incr[ok]
    hist, tot = np.zeros((n, 33), np.float32), np.zeros((n, 3))
    with np.errstate(divide="ignore"):
        for j in range(nb.shape[1]):
            ok = (nb[:, j] >= 0) & (d2[:, j] != 0)
            wgt = f32(1.0) / d2[:, j]
            val = spfh[np.maximum(nb[:, j], 0)] * wgt[:, None]
            hist[ok] += val[ok]
            for b in range(33):
                tot[ok, b // 11] += val[ok, b].astype(np.float64)
    scale = np.ones((n, 3), np.float32)
    nz = tot != 0
    scale[nz] = (100.0 / tot[nz]).astype(f32)
    out = np.where(np.repeat(nz, 11, axis=1), hist * np.repeat(scale, 11, axis=1), hist)
    return out, nrm, cn, cf


# ---- oracle vs numpy / scipy / analytic ------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind,r", [("random", 0.4), ("scan", 0.5), ("dups", 0.7), ("outliers", 0.6)])
def test_oracle_lists_equal_brute_force_and_ckdtree(kind, r):
    P = CLOUDS[kind](3)
    counts, idx, d2 = fro.lists(P, r)
    nb, wd2, cnt = np_lists(P, r)
    assert np.array_equal(counts, cnt)
    valid = nb >= 0
    assert np.array_equal(idx, nb[valid]) and np.array_equal(d2, wd2[valid])
    tree = cKDTree(P.astype(np.float64))
    D = np.sqrt(np_d2(P).astype(np.float64))
    off = np.concatenate([[0], np.cumsum(counts)])
    balls = tree.query_ball_point(P.astype(np.float64), r)
    for i in range(len(P)):
        far_from_boundary = np.abs(D[i] - r) > 1e-4 * r
        mine = set(idx[off[i]:off[i + 1]].tolist())
        theirs = set(balls[i])
        assert {q for q in mine if far_from_boundary[q]} == {q for q in theirs if far_from_boundary[q]}, i
    assert counts.min() >= 1                                                # the query itself


@pytest.mark.parametrize("kind,seed,rn,rf", [("random", 1, 0.45, 0.9), ("scan", 2, 0.4, 0.8), ("scan", 3, 0.6, 0.6),
                                             ("dups", 4, 0.8, 0.5), ("outliers", 5, 0.5, 1.0)])
def test_oracle_equals_numpy_restatement(kind, seed, rn, rf):
    P = CLOUDS[kind](seed)
    got, nrm, st, comp = fro.fpfh(P, None, rn, rf)
    want, wn, cn, _ = np_fpfh_radius(P, rn, rf)
    assert (comp & 2).all()
    assert np.array_equal(st, np.where(cn < 3, 1, 0))
    assert np.array_equal(nrm, wn, equal_nan=True)
    assert np.array_equal(got, want)


def test_plane_normals_face_the_origin():
    rng = np.random.default_rng(7)
    P = np.zeros((700, 3), np.float32)
    P[:, :2] = rng.random((700, 2)) * 8 - 4
    P[:, 2] = 2.0
    f, nrm, st, _ = fro.fpfh(P, None, 0.6, 1.2)
    assert np.array_equal(nrm, np.tile(np.float32([0, 0, -1]), (700, 1))) and (st == 0).all()
    other = np.delete(np.arange(33), [5, 16, 27])
    assert (f[:, other] == 0).all() and np.allclose(f[:, [5, 16, 27]], 100.0, rtol=1e-5, atol=0)


@pytest.mark.parametrize("kind", ["random", "scan", "dups"])
def test_every_block_sums_to_100(kind):
    f, _, _, _ = fro.fpfh(CLOUDS[kind](9), None, 0.8, 1.6)
    s = f.reshape(-1, 3, 11).astype(np.float64).sum(axis=2)
    nonempty = s > 0
    assert nonempty.mean() > 0.95
    assert np.allclose(s[nonempty], 100.0, rtol=2e-5)


def test_isolated_point_duplicates_and_a_radius_larger_than_the_cloud():
    P = scan_like_cloud(500, 11, extent=(6.0, 6.0, 2.0))
    D = np.concatenate([P, P[:1], P[:1], np.float32([[50.0, 50.0, 50.0]])]).astype(np.float32)
    iso = len(D) - 1
    f, nrm, st, _ = fro.fpfh(D, None, 0.5, 1.0)
    assert np.isnan(nrm[iso]).all() and st[iso] == 1 and (f[iso] == 0).all()   # its own only neighbour
    counts, idx, d2 = fro.lists(D, 1.0)
    off = np.concatenate([[0], np.cumsum(counts)])
    row0 = idx[off[0]:off[1]]
    assert sorted(row0[:3].tolist()) == [0, 500, 501] and (d2[off[0]:off[0] + 3] == 0).all()   # duplicates counted
    assert np.array_equal(f[0], f[500]) and np.array_equal(f[0], f[501])
    counts, _, _ = fro.lists(P, 100.0)
    assert (counts == len(P)).all()
    f, nrm, st, _ = fro.fpfh(P, None, 100.0, 100.0)
    want, wn, _, _ = np_fpfh_radius(P, 100.0, 100.0)
    assert np.array_equal(f, want) and np.array_equal(nrm, wn)


def test_subset_equals_rows_of_the_whole_cloud():
    P = CLOUDS["scan"](12)
    full, fn, _, _ = fro.fpfh(P, None, 0.4, 0.8)
    idx = np.random.default_rng(1).choice(len(P), 30, replace=False).astype(np.int32)
    sub, sn, _, comp = fro.fpfh(P, idx, 0.4, 0.8, all_normals=False)
    assert np.array_equal(sub, full[idx]) and (comp != 7).any()
    done = (comp & 2) != 0
    assert np.array_equal(sn[done], fn[done], equal_nan=True)


# ---- the product's kernels on the CPU (host emulation shim) ----------------------------------------------------------------
@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    out = os.path.join(str(tmp_path_factory.mktemp("fpfh_radius_emu")), "libfpfh_radius_emu_harness.so")
    src = os.path.join(ROOT, "tests", "harness", "fpfh_radius_emu_harness.cpp")
    extra = os.environ.get("GHICP_EMU_CXXFLAGS", "").split()
    r = subprocess.run(["g++", "-O1", "-g", "-std=c++17", "-fPIC", "-ffp-contract=off", "-DGHICP_EMU_HOST"] + extra +
                       ["-I" + os.path.join(ROOT, "tests", "harness", "cuda_emu"), "-x", "c++", "-shared", "-o", out, src],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return out


def emu_run(path, P, idx=None, rn=0.5, rf=1.0, nb_max=0):
    L = C.CDLL(path)
    fp, ip, lp = C.POINTER(C.c_float), C.POINTER(C.c_int), C.POINTER(C.c_longlong)
    P = np.ascontiguousarray(P, np.float32)
    n = len(P)
    ia = None if idx is None else np.ascontiguousarray(idx, np.int32)
    m = n if ia is None else len(ia)
    f, nrm, st = np.zeros((m, 33), np.float32), np.zeros((n, 3), np.float32), np.zeros(n, np.int32)
    stats, cell = np.zeros(8, np.int64), C.c_float(0)
    L.emu_fpfh_radius.argtypes = [fp, C.c_int, ip, C.c_int, C.c_float, C.c_float, C.c_longlong, fp, fp, ip, lp, fp]
    rc = L.emu_fpfh_radius(P.ctypes.data_as(fp), n, None if ia is None else ia.ctypes.data_as(ip), m, rn, rf, nb_max,
                           f.ctypes.data_as(fp), nrm.ctypes.data_as(fp), st.ctypes.data_as(ip), stats.ctypes.data_as(lp),
                           C.byref(cell))
    return dict(rc=rc, fpfh=f, normals=nrm, status=st, nb_n=int(stats[0]), nb_f=int(stats[1]), spfh_points=int(stats[2]),
                rings_n=int(stats[3]), rings_f=int(stats[4]), needed=int(stats[5]), budget=int(stats[6]), cell=cell.value)


@pytest.mark.parametrize("kind,rn,rf", [("random", 0.3, 0.6), ("scan", 0.4, 0.8), ("scan", 0.6, 0.6), ("scan", 0.9, 0.45),
                                        ("dups", 0.5, 1.0), ("outliers", 0.5, 1.0), ("outliers", 1.2, 0.6)])
def test_emulated_kernels_equal_the_oracle(harness, kind, rn, rf):
    P = CLOUDS[kind](21)
    want, wn, wst, _ = fro.fpfh(P, None, rn, rf)
    got = emu_run(harness, P, None, rn, rf)
    assert got["rc"] == 0
    assert np.array_equal(got["normals"], wn, equal_nan=True) and np.array_equal(got["status"], wst)
    assert np.array_equal(got["fpfh"], want)
    cn, _, _ = fro.lists(P, rn)
    cf, _, _ = fro.lists(P, rf)
    assert got["nb_n"] == cn.sum() and got["nb_f"] == cf.sum() and got["spfh_points"] == len(P)
    assert got["rings_n"] == 1 and got["rings_f"] == 1                       # cell = 1.02 max(rn, rf): one ring
    idx = np.random.default_rng(3).choice(len(P), 25, replace=False).astype(np.int32)
    sub = emu_run(harness, P, idx, rn, rf)
    assert sub["rc"] == 0 and np.array_equal(sub["fpfh"], want[idx])
    done = sub["status"] != 2
    assert np.array_equal(sub["normals"][done], wn[done], equal_nan=True) and np.isnan(sub["normals"][~done]).all()
    assert sub["nb_f"] < got["nb_f"] and sub["spfh_points"] < len(P)


def test_emulated_kernels_at_the_cell_clamp(harness):
    """A far point makes the extent / 2^20 floor larger than the cell the radii ask for: the walk covers more rings."""
    P = scan_like_cloud(800, 5, extent=(4.0, 4.0, 1.0))
    P = np.concatenate([P, np.float32([[400000.0, 0.0, 0.0]])]).astype(np.float32)
    rn, rf = 0.05, 0.1
    want, wn, wst, _ = fro.fpfh(P, None, rn, rf)
    got = emu_run(harness, P, None, rn, rf)
    assert got["rc"] == 0 and got["cell"] > 1.02 * rf and got["rings_f"] >= 2
    assert np.array_equal(got["normals"], wn, equal_nan=True) and np.array_equal(got["status"], wst)
    assert np.array_equal(got["fpfh"], want)


def test_emulated_kernels_over_the_budget_write_nothing(harness):
    P = CLOUDS["scan"](4)
    ok = emu_run(harness, P, None, 0.4, 0.8)
    over = emu_run(harness, P, None, 0.4, 0.8, nb_max=ok["nb_f"] - 1)           # the feature lists alone do not fit
    assert over["rc"] != 0 and over["needed"] == ok["nb_f"] and (over["fpfh"] == 0).all() and (over["normals"] == 0).all()
    over = emu_run(harness, P, None, 0.4, 0.8, nb_max=ok["nb_f"] + ok["nb_n"] - 1)   # both lists together do not
    assert over["rc"] != 0 and over["needed"] == ok["nb_f"] + ok["nb_n"] and (over["fpfh"] == 0).all()
    exact = emu_run(harness, P, None, 0.4, 0.8, nb_max=ok["nb_f"] + ok["nb_n"])
    assert exact["rc"] == 0 and np.array_equal(exact["fpfh"], ok["fpfh"])


def test_emulated_kernels_under_a_random_schedule(harness, tmp_path):
    """GHICP_EMU_SCHED: fibers visited in a fresh random order at every sweep (read once per process: a child process)."""
    P = CLOUDS["outliers"](22)
    np.save(tmp_path / "P.npy", P)
    code = ("import sys, numpy as np; sys.path.insert(0, %r); import test_fpfh_radius as t; r = t.emu_run(%r, np.load(%r), None, 0.5, 1.0);"
            "np.savez(%r, **{k: v for k, v in r.items() if isinstance(v, np.ndarray)})"
            % (os.path.join(ROOT, "tests"), harness, str(tmp_path / "P.npy"), str(tmp_path / "out.npz")))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True,
                       env=dict(os.environ, GHICP_EMU_SCHED="7", PYTHONPATH=os.path.join(ROOT, "tests")))
    assert r.returncode == 0, r.stderr[-3000:]
    got = np.load(tmp_path / "out.npz")
    want, wn, _, _ = fro.fpfh(P, None, 0.5, 1.0)
    assert np.array_equal(got["normals"], wn, equal_nan=True) and np.array_equal(got["fpfh"], want)


# ---- the C ABI over the emulated kernels ------------------------------------------------------------------------------------
@pytest.fixture()
def ge(g, emu_library_path):
    from conftest import swap_in_library
    real = swap_in_library(g, emu_library_path)
    try:
        yield g
    finally:
        g.capi._lib = real


def test_emulated_abi_extract_bad_arguments_and_budget(ge, monkeypatch):
    g = ge
    P = CLOUDS["dups"](5)
    want, wn, wst, _ = fro.fpfh(P, None, 0.5, 1.0)
    f, nrm, st = g.fpfh_extract_radius(P, normal_radius=0.5, feature_radius=1.0)
    assert np.array_equal(f, want) and np.array_equal(nrm, wn, equal_nan=True) and np.array_equal(st, wst)
    for bad in (dict(normal_radius=0.0, feature_radius=1.0), dict(normal_radius=0.5, feature_radius=-1.0),
                dict(normal_radius=float("nan"), feature_radius=1.0), dict(normal_radius=0.5, feature_radius=float("inf")),
                dict(normal_radius=1e-30, feature_radius=1.0), dict(normal_radius=0.5, feature_radius=1.0, idx=np.array([len(P)], np.int32)),
                dict(normal_radius=0.5, feature_radius=1.0, idx=np.array([-1], np.int32))):
        with pytest.raises(g.GhicpError) as e:
            g.fpfh_extract_radius(P, **bad)
        assert e.value.code == -1, bad                                         # GHICP_E_ARG
    monkeypatch.setenv("GHICP_FPFH_NB_MAX", "1000")
    with pytest.raises(g.GhicpError) as e:
        g.fpfh_extract_radius(P, normal_radius=0.5, feature_radius=1.0)
    assert e.value.code == -2 and "entries" in str(e.value)                   # GHICP_E_NOMEM with the entry count
    monkeypatch.delenv("GHICP_FPFH_NB_MAX")
    f2, nrm2, st2 = g.fpfh_extract_radius(P, normal_radius=0.5, feature_radius=1.0)
    assert np.array_equal(f2, want) and np.array_equal(st2, wst)


def test_emulated_abi_prep_over_the_budget_keeps_the_previous_histograms(ge, monkeypatch):
    g = ge
    T, _, _, _ = g.synth.scan_pair(6000, seed=4)
    p = g.Prep(T, 0.3, 1.0, 1.5)
    try:
        p.fpfh_radius(0.6, 1.2)
        before = p.get_fpfh()
        monkeypatch.setenv("GHICP_FPFH_NB_MAX", "10")
        with pytest.raises(g.GhicpError) as e:
            p.fpfh_radius(0.9, 1.8)
        assert e.value.code == -2
        monkeypatch.delenv("GHICP_FPFH_NB_MAX")
        assert np.array_equal(p.get_fpfh(), before)
    finally:
        p.close()


def test_emulated_abi_register_clouds_and_coarsereg(ge):
    g = ge
    T, S, _, _ = g.synth.scan_pair(6000, seed=4)
    Rt, info = g.register_clouds(T, S, 0.3, 1.0, 1.5, corr_type=g.CT_NNR, feature_type=g.FT_FPFH, max_iter=40,
                                 fpfh_radius=(0.6, 1.2))
    assert info["n_source_kp"] > 10 and set(info["fpfh_ms"]["source"]) == {"lists", "normals", "spfh_fpfh", "total"}
    assert np.isfinite(Rt).all() and abs(np.linalg.det(Rt[:3, :3]) - 1.0) < 1e-5
    D = [X[g.voxel_downsample(X, 0.5)] for X in (S, T)]
    Rt, info = g.coarsereg_fpfh_sac(D[0], D[1], 0.75, sac=dict(iterations=50))
    assert np.isfinite(Rt).all() and info["best_hypothesis"] >= 0 and np.isfinite(info["fitness"])


@pytest.mark.parametrize("name,kw", [("test_extract_equals_oracle", dict(n=1500, seed=1)),
                                     ("test_sample_of_indices_computes_only_what_it_needs", dict(n_points=6000)),
                                     ("test_two_calls_are_identical", dict(n=1500)),
                                     ("test_prep_fpfh_radius_equals_standalone_and_registers", dict(n_points=6000)),
                                     ("test_coarsereg_equals_the_sac_oracle", dict(n_points=6000, iterations=40, voxel=0.4)),
                                     ("test_cxx_mirror_coarsereg_matches_python", dict(n_points=6000, voxel=0.4))])
def test_gpu_test_functions_on_the_emulated_library(ge, name, kw, tmp_path, emu_library_path, monkeypatch):
    import test_zz6_fpfh_radius_gpu as t
    fn = getattr(t, name)
    if name == "test_cxx_mirror_coarsereg_matches_python":
        monkeypatch.setenv("LD_LIBRARY_PATH", os.path.dirname(emu_library_path) + os.pathsep + os.environ.get("LD_LIBRARY_PATH", ""))
        fn(ge, tmp_path, **kw)
    else:
        fn(ge, **kw)
