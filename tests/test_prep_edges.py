"""The raw-cloud pre-processing (ghicp_prep.cu: voxel filter, radius PCA + keypoint NMS, both FPFH estimators, BSC) against
references that share nothing with its grid, on the clouds where such code goes wrong: organised scans with non-finite rows,
far outliers, large offsets, exact ties and degenerate clouds.

The rule under test (DESIGN.md §3.8, "Non-finite points"): non-finite points take no part in any pre-processing stage.  Every stage returns on a
cloud with non-finite rows what it returns on the cloud's finite rows, indices mapped back (pcl::removeNaNFromPointCloud, then
the reference).  A non-finite point gets pt_num 0, eigenvalues and curvature 0 and is never a keypoint; a NaN normal, status 1
and a zero histogram in both FPFH estimators; a zero BSC descriptor and status 1 as a keypoint.

The references:
  voxel filter  include/filter.hpp's float32 (x - min) * inv and floor, voxel ids modulo 2^64 (the reference's arithmetic,
                wrap included), the first index per id, the phantom entry (the first finite point) in front
  radius PCA    neighbour sets from cKDTree with the radius widened by 1e-5, kept where the float32 d2 < r^2 in the kernel's
                operation order; pt_num exact, eigenvalues / curvature against float64 eigvalsh within a float32 tolerance
  NMS           the greedy definition run sequentially over (curvature descending, index ascending) on the kernel's own
                curvatures and float32 distances
  FPFH          metamorphic: a cloud with non-finite rows inserted gives the clean cloud's results bit for bit, mapped back
The kernels run here through the emulated library (tests/harness/emu_library.cpp); tests/test_zz9_prep_edges_gpu.py runs
the same checks on the device."""
import os

import numpy as np
import pytest
from scipy.spatial import cKDTree

from test_prep_oracle import scan_like_cloud

NONFINITE = np.array([[np.nan, 1, 1], [1, np.nan, 1], [1, 1, np.nan], [1, 1, -np.nan], [np.inf, 1, 1], [1, -np.inf, 1],
                      [1, 1, np.inf]], np.float32)


# ---- clouds --------------------------------------------------------------------------------------------------------------
def edge_cloud(kind, n, seed):
    """The clouds of this file, all float32 [n'][3]; every one finite except through with_nonfinite."""
    rng = np.random.default_rng(seed)
    if kind == "scan":
        return scan_like_cloud(n, seed)
    if kind == "far":         # 1 % of the points 10 km away
        P = scan_like_cloud(n, seed)
        P[rng.choice(n, max(n // 100, 1), replace=False)] += np.float32([1e4, -7e3, 2e3])
        return P
    if kind == "far1e7":      # one point past 2^22 cells of 1 m: its cell key aliases
        P = scan_like_cloud(n, seed)
        P[n // 3] = [1e7, 2.0, 1.0]
        return P
    if kind == "far1e10":     # one point past int range in cell_coord
        P = scan_like_cloud(n, seed)
        P[n // 3] = [1e10, 2.0, 1.0]
        return P
    if kind == "offset":
        return (scan_like_cloud(n, seed).astype(np.float64) + [3e5, 4e5, 50.0]).astype(np.float32)
    if kind == "lattice":     # exact multiples of 0.25 m: points on voxel faces, neighbours at exactly d2 == r^2
        m = max(int(round(n ** (1 / 3))), 2)
        g = np.arange(m, dtype=np.float32) * np.float32(0.25)
        L = np.stack(np.meshgrid(g, g, g[: max(m // 3, 1)], indexing="ij"), axis=-1).reshape(-1, 3)
        return np.ascontiguousarray(L[rng.permutation(len(L))], np.float32)
    if kind == "triple":      # every point three times: exact curvature ties across NMS
        P = scan_like_cloud(max(n // 3, 8), seed)
        return np.ascontiguousarray(np.repeat(P, 3, axis=0))
    if kind == "patches":     # two identical patches far apart
        P = scan_like_cloud(max(n // 2, 8), seed, extent=(6.0, 6.0, 2.0))
        return np.concatenate([P, P + np.float32([1000.0, 0.0, 0.0])])
    if kind == "plane":       # lambda3 = 0
        P = (rng.random((n, 3)) * [8.0, 8.0, 0.0]).astype(np.float32)
        return P
    if kind == "line":        # lambda2 = lambda3 = 0: ratio2 = 0 / 0
        t = rng.random(n).astype(np.float32) * np.float32(8.0)
        return np.stack([t, np.zeros_like(t), np.zeros_like(t)], axis=1)
    if kind == "same":        # every point identical
        return np.tile(np.float32([[1.5, -2.0, 0.5]]), (n, 1))
    raise ValueError(kind)


def with_nonfinite(C, frac, seed, first=True):
    """C with non-finite rows (every kind of NONFINITE) inserted at random positions, row 0 among them when `first`.
    Returns (D, pos): pos[i] = the row of D that holds C[i]."""
    rng = np.random.default_rng(seed)
    n = len(C)
    m = max(int(round(frac * n)), 1)
    bad = np.zeros(n + m, bool)
    bad[rng.choice(n + m, m, replace=False)] = True
    if first and not bad[0]:
        bad[np.flatnonzero(bad)[-1]] = False
        bad[0] = True
    D = np.empty((n + m, 3), np.float32)
    D[bad] = NONFINITE[rng.integers(0, len(NONFINITE), m)]
    pos = np.flatnonzero(~bad)
    D[pos] = C
    return D, pos


# ---- brute-force references ------------------------------------------------------------------------------------------------
def voxel_ref(P, v):
    """CFilter::voxelfilter on the finite rows of P (include/filter.hpp:28-88), ids modulo 2^64 as the reference computes them."""
    fin = np.flatnonzero(np.isfinite(P).all(axis=1))
    if len(fin) == 0:
        return np.zeros(0, np.int32)
    F = P[fin]
    inv = np.float32(1.0) / np.float32(v)
    mn, mx = F.min(axis=0), F.max(axis=0)
    gap = (mx - mn).astype(np.float32)
    max_vy = int(np.float32(np.ceil(np.float32(gap[1] * inv))) + np.float32(1.0))
    max_vz = int(np.float32(np.ceil(np.float32(gap[2] * inv))) + np.float32(1.0))
    V = np.floor(((F - mn).astype(np.float32) * inv).astype(np.float32)).astype(np.float64)
    M = 1 << 64
    ids = [(int(x) * ((max_vy * max_vz) % M) + int(y) * max_vz + int(z)) % M for x, y, z in V]
    first = {}
    for i, key in enumerate(ids):
        first.setdefault(key, i)
    out = [0] + [first[key] for key in sorted(first) if key != 0]   # the phantom {voxel 0, point 0} absorbs voxel 0
    return fin[np.asarray(out)].astype(np.int32)


def d2_f32(Q, P):
    """(ex*ex + ey*ey) + ez*ez in float32, e = P - Q, every operation rounded (the kernels' order, no contraction)."""
    E = (P.astype(np.float32) - Q.astype(np.float32)).astype(np.float32)
    return ((E[..., 0] * E[..., 0] + E[..., 1] * E[..., 1]).astype(np.float32) + E[..., 2] * E[..., 2]).astype(np.float32)


def radius_sets(P, r, queries=None):
    """Neighbour lists {q: ascending indices p with d2_f32(q, p) < r*r (float32)}, finite rows only."""
    fin = np.flatnonzero(np.isfinite(P).all(axis=1))
    r2 = np.float32(np.float32(r) * np.float32(r))
    tree = cKDTree(P[fin].astype(np.float64))
    qs = fin if queries is None else np.asarray(queries)
    cands = tree.query_ball_point(P[qs].astype(np.float64), float(r) * (1 + 1e-5))
    out = {}
    for q, c in zip(qs, cands):
        c = fin[np.sort(np.asarray(c, np.int64))]
        out[int(q)] = c[d2_f32(P[q], P[c]) < r2]
    return out


def pca_ref(P, r):
    """(pt_num, eigenvalues descending [n][3] float64, curvature) of every row by brute force."""
    n = len(P)
    cnt, lam, curv = np.zeros(n, np.int64), np.zeros((n, 3)), np.zeros(n)
    for q, nb in radius_sets(P, r).items():
        cnt[q] = len(nb)
        if len(nb) >= 3:
            E = P[nb].astype(np.float64) - P[q].astype(np.float64)
            w = np.linalg.eigvalsh(np.cov(E.T, ddof=1))[::-1]
            lam[q] = w
            curv[q] = w[2] / w.sum() if w.sum() != 0 else 0.0
    return cnt, lam, curv


def nms_ref(P, lam, curv, cnt, ratio_max, min_pts, nms_radius):
    """pruneUnstablePoints + the greedy nonMaximaSuppression, sequential, on the kernel's own eigenvalues and curvatures."""
    with np.errstate(divide="ignore", invalid="ignore"):
        r1 = (lam[:, 1].astype(np.float64) / lam[:, 0].astype(np.float64)).astype(np.float32)
        r2 = (lam[:, 2].astype(np.float64) / lam[:, 1].astype(np.float64)).astype(np.float32)
    cand = np.flatnonzero((r1 < np.float32(ratio_max)) & (r2 < np.float32(ratio_max)) & (cnt > min_pts))
    order = cand[np.lexsort((cand, -curv[cand]))]
    if len(order) == 0:
        return np.zeros(0, np.int32)
    near = radius_sets(P, nms_radius, order)
    is_cand = np.zeros(len(P), bool)
    is_cand[cand] = True
    visited = np.zeros(len(P), bool)
    keep = []
    for q in order:
        if visited[q]:
            continue
        keep.append(q)
        nb = near[int(q)]
        visited[nb[is_cand[nb]]] = True
        visited[q] = True
    return np.asarray(keep, np.int32)


# ---- the checks (shared with the GPU file, which runs them at larger sizes) ----------------------------------------------
def check_voxel(g, orc, P, v):
    want = voxel_ref(P, v)
    assert np.array_equal(g.voxel_downsample(P, v), want)
    assert np.array_equal(orc.voxel_downsample(P, v), want)


def check_keypoints(g, P, r, nms, lam_tol=2e-5):
    """pt_num exact, eigenvalues / curvature within lam_tol of float64 (relative to the largest eigenvalue), non-finite rows
    zero, the keypoint list equal to the sequential greedy NMS."""
    kp, lam, curv, cnt = g.detect_keypoints(P, r, 0.65, 20, nms)
    rcnt, rlam, rcurv = pca_ref(P, r)
    assert np.array_equal(cnt, rcnt)
    scale = np.maximum(rlam[:, :1], 1e-30)
    assert np.all(np.abs(lam - rlam) <= lam_tol * scale), np.max(np.abs(lam - rlam) / scale)
    assert np.all(np.abs(curv - rcurv) <= lam_tol)
    bad = ~np.isfinite(P).all(axis=1)
    assert np.all(cnt[bad] == 0) and np.all(lam[bad] == 0) and np.all(curv[bad] == 0)
    assert np.array_equal(kp, nms_ref(P, lam, curv, cnt, 0.65, 20, nms))
    assert not np.any(bad[kp])
    return kp, lam, curv, cnt


def check_fpfh_metamorphic(g, fo, fro, C, seed, k=20, rn=0.6, rf=1.0):
    """Both estimators (and both oracles) on C with non-finite rows inserted: the clean results bit for bit, mapped back; the
    non-finite rows: NaN normal, status 1, zero histogram."""
    D, pos = with_nonfinite(C, 0.05, seed)
    bad = np.ones(len(D), bool)
    bad[pos] = False
    idx = np.arange(0, len(C), 7, dtype=np.int32)
    didx = np.concatenate([pos[idx], np.flatnonzero(bad)[:5]]).astype(np.int32)   # keypoints, some of them non-finite
    runs = [("knn", lambda X, i: g.fpfh_extract(X, i, k=k)),
            ("radius", lambda X, i: g.fpfh_extract_radius(X, i, normal_radius=rn, feature_radius=rf))]
    if fo is not None:
        runs.append(("knn oracle", lambda X, i: fo.fpfh(X, i, k=k)[:3]))
        runs.append(("radius oracle", lambda X, i: fro.fpfh(X, i, rn=rn, rf=rf)[:3]))
    for name, run in runs:
        for ci, di in ((None, None), (idx, didx)):
            f0, n0, s0 = run(C, ci)
            f1, n1, s1 = run(D, di)
            rows = pos if ci is None else np.arange(len(idx))
            assert np.array_equal(f1[rows], f0), name
            assert np.array_equal(n1[pos], n0, equal_nan=True) and np.array_equal(s1[pos], s0), name
            assert np.all(np.isnan(n1[bad])) and np.all(s1[bad] == 1), name
            zero = np.flatnonzero(bad) if ci is None else np.arange(len(idx), len(didx))
            assert np.all(f1[zero] == 0), name


def check_prep_metamorphic(g, C, seed, voxel=0.1, radius=1.0, nms=1.2):
    """ghicp_prep_run on C with non-finite rows: n_down, the down-sampled cloud, keypoints, bbx_magnitude, BSC and both FPFH
    estimators bit for bit as on C."""
    D, _ = with_nonfinite(C, 0.05, seed)
    a = g.capi.Prep(C, voxel, radius, nms, bsc_radius=radius, dof_type=6)
    b = g.capi.Prep(D, voxel, radius, nms, bsc_radius=radius, dof_type=6)
    assert a.n_down == b.n_down and a.n_kp == b.n_kp and a.n_kp > 0
    assert np.array_equal(a.down(), b.down())
    for x, y in zip(a.keypoints(), b.keypoints()):
        assert np.array_equal(x, y)
    assert np.array_equal(a.bbox_min, b.bbox_min) and np.array_equal(a.bbox_max, b.bbox_max)
    assert np.isfinite(b.bbx_magnitude) and a.bbx_magnitude == b.bbx_magnitude
    assert np.array_equal(a.bsc(), b.bsc())
    a.fpfh(20); b.fpfh(20)
    assert np.array_equal(a.get_fpfh(), b.get_fpfh())
    assert a.fpfh_stats["fallbacks"] == b.fpfh_stats["fallbacks"]
    a.fpfh_radius(0.5, 1.0); b.fpfh_radius(0.5, 1.0)
    assert np.array_equal(a.get_fpfh(), b.get_fpfh())


def check_far_fallbacks(g, P, n_out, voxel=0.1):
    """The k-NN estimator's exhaustive scans stay bounded by the number of far outliers."""
    p = g.capi.Prep(P, voxel, 1.0, 1.2)
    p.fpfh(20)
    assert p.fpfh_stats["fallbacks"] <= n_out


def check_bsc_nonfinite_keypoint(g, C, seed, R=1.0):
    D, pos = with_nonfinite(C, 0.05, seed)
    bad = np.flatnonzero(~np.isin(np.arange(len(D)), pos))
    kp = np.arange(0, len(C), 31, dtype=np.int32)
    f0, l0, s0 = g.bsc_extract(C, kp, R)
    f1, l1, s1 = g.bsc_extract(D, np.concatenate([pos[kp], bad[:4]]).astype(np.int32), R)
    m = len(kp)
    assert np.array_equal(f1[:, :m], f0) and np.array_equal(l1[:m], l0) and np.array_equal(s1[:m], s0)
    assert np.all(f1[:, m:] == 0) and np.all(s1[m:] == 1)


# ---- CPU tests: the emulated kernels and the oracles ---------------------------------------------------------------------
@pytest.fixture()
def ge(g, emu_library_path):
    from conftest import swap_in_library
    real = swap_in_library(g, emu_library_path)
    try:
        yield g
    finally:
        g.capi._lib = real


@pytest.fixture(scope="module")
def fo():
    import fpfh_oracle
    return fpfh_oracle


@pytest.fixture(scope="module")
def fro():
    import fpfh_radius_oracle
    return fpfh_radius_oracle


def test_with_nonfinite_covers_every_kind_and_row_zero():
    D, pos = with_nonfinite(scan_like_cloud(400, 1), 0.05, 2)
    bad = np.setdiff1d(np.arange(len(D)), pos)
    assert 0 in bad and not np.isfinite(D[bad]).all(axis=1).any() and np.isfinite(D[pos]).all()
    assert len(bad) == 20


def test_voxel_reference_restates_the_oracle_on_clean_scans(orc):
    """The brute-force reference agrees with the oracle where both were written independently (finite clouds)."""
    for seed, v in ((1, 0.4), (2, 0.05), (3, 3.0)):
        P = scan_like_cloud(3000, seed)
        assert np.array_equal(voxel_ref(P, v), orc.voxel_downsample(P, v))


VOXEL_CASES = [("scan", 4000, 0.4), ("far", 3000, 0.25), ("far1e7", 2000, 0.5), ("offset", 3000, 0.25), ("lattice", 1500, 0.25),
               ("triple", 2400, 0.3), ("patches", 2000, 0.2), ("plane", 500, 0.5), ("line", 300, 0.5), ("same", 50, 0.5)]


@pytest.mark.parametrize("kind,n,v", VOXEL_CASES)
@pytest.mark.parametrize("nonfinite", [False, True])
def test_voxel_filter_equals_brute_force(ge, orc, kind, n, v, nonfinite):
    P = edge_cloud(kind, n, 5)
    if nonfinite:
        P, _ = with_nonfinite(P, 0.05, 6)
    check_voxel(ge, orc, P, v)


@pytest.mark.parametrize("n", [1, 2, 3])
def test_voxel_filter_tiny_and_all_nonfinite(ge, orc, n):
    P = scan_like_cloud(8, 7)[:n]
    check_voxel(ge, orc, P, 0.5)
    D, _ = with_nonfinite(P, 1.0, 8)
    check_voxel(ge, orc, D, 0.5)
    assert len(ge.voxel_downsample(NONFINITE, 0.5)) == 0 and len(orc.voxel_downsample(NONFINITE, 0.5)) == 0


KP_CASES = [("scan", 3000, 1.0, 1.5), ("far", 2000, 1.0, 1.2), ("far1e7", 1500, 1.0, 1.0), ("offset", 2000, 1.0, 1.5),
            ("lattice", 1500, 0.5, 0.5), ("triple", 1500, 0.8, 1.0), ("patches", 1600, 1.0, 1.0), ("plane", 400, 1.5, 1.0),
            ("line", 200, 1.0, 1.0), ("same", 30, 0.5, 0.5)]


@pytest.mark.parametrize("kind,n,r,nms", KP_CASES)
@pytest.mark.parametrize("nonfinite", [False, True])
def test_keypoints_equal_brute_force(ge, orc, kind, n, r, nms, nonfinite):
    P = edge_cloud(kind, n, 9)
    if nonfinite:
        P, _ = with_nonfinite(P, 0.05, 10)
    kp, lam, curv, cnt = check_keypoints(ge, P, r, nms)
    okp, olam, ocurv, ocnt = orc.detect_keypoints(P, r, 0.65, 20, nms)
    assert np.array_equal(cnt, ocnt) and np.array_equal(lam, olam) and np.array_equal(curv, ocurv) and np.array_equal(kp, okp)


def test_keypoints_tiny_clouds(ge):
    for n in (1, 2, 3):
        P = scan_like_cloud(8, 11)[:n]
        kp, lam, curv, cnt = check_keypoints(ge, P, 50.0, 50.0)   # every point within the radius of every other
        assert len(kp) == 0 and np.all(cnt == n)


def test_every_stage_on_a_cloud_without_a_finite_point(ge, fo, fro):
    """Nothing finite: no voxel, no neighbour, no keypoint; NaN normals, status 1 and zero rows from both FPFH estimators
    (requested rows included); zero BSC descriptors; ghicp_prep_run refuses the cloud with GHICP_E_ARG."""
    D = np.concatenate([NONFINITE, NONFINITE[::-1]])
    n = len(D)
    assert len(ge.voxel_downsample(D, 0.5)) == 0
    kp, lam, curv, cnt = ge.detect_keypoints(D, 1.0, 0.65, 20, 1.0)
    assert len(kp) == 0 and np.all(cnt == 0) and np.all(lam == 0) and np.all(curv == 0)
    idx = np.array([3, 0, 5], np.int32)
    for run in (lambda i: ge.fpfh_extract(D, i, k=20), lambda i: fo.fpfh(D, i, k=20)[:3],
                lambda i: ge.fpfh_extract_radius(D, i, normal_radius=0.5, feature_radius=1.0),
                lambda i: fro.fpfh(D, i, rn=0.5, rf=1.0)[:3]):
        for i in (None, idx):
            f, nrm, st = run(i)
            assert f.shape == (n if i is None else len(i), 33) and np.all(f == 0)
            assert np.all(np.isnan(nrm)) and np.all(st == 1)
    feats, _, st = ge.bsc_extract(D, idx, 1.0)
    assert np.all(feats == 0) and np.all(st == 1)
    with pytest.raises(ge.GhicpError) as e:
        ge.capi.Prep(D, 0.1, 1.0, 1.2, bsc_radius=1.0, dof_type=6)
    assert e.value.code == -1 and "no finite point" in str(e.value)                  # GHICP_E_ARG


def test_neighbours_at_exactly_r_are_excluded(ge):
    """Lattice spacing 0.25, radius 0.5: the axis neighbours two steps away sit at d2 == r^2 exactly and are not counted."""
    g1 = np.arange(7, dtype=np.float32) * np.float32(0.25)
    L = np.stack(np.meshgrid(g1, g1, g1, indexing="ij"), axis=-1).reshape(-1, 3).astype(np.float32)
    _, _, _, cnt = ge.detect_keypoints(L, 0.5, 0.65, 20, 0.5)
    c = np.flatnonzero((L == np.float32(0.75)).all(axis=1))[0]
    assert cnt[c] == 1 + 6 + 12 + 8   # |e| < 2 steps: the point, 6 faces, 12 edges (d2 = 2), 8 corners (d2 = 3)


@pytest.mark.parametrize("kind", ["scan", "offset", "triple", "patches"])
def test_fpfh_nonfinite_rows_change_nothing(ge, fo, fro, kind):
    check_fpfh_metamorphic(ge, fo, fro, edge_cloud(kind, 900, 12), 13)


def test_fpfh_fewer_finite_points_than_k(ge, fo, fro):
    """k_eff = min(k, finite points): 10 finite points and 12 non-finite ones with k = 20 are the 10-point cloud."""
    check_fpfh_metamorphic(ge, fo, fro, scan_like_cloud(10, 14), 15, k=20)
    D, pos = with_nonfinite(scan_like_cloud(10, 14), 1.2, 16)
    f, nrm, st = ge.fpfh_extract(D, k=20)
    f0, n0, s0 = ge.fpfh_extract(scan_like_cloud(10, 14), k=20)
    assert np.array_equal(f[pos], f0) and np.array_equal(nrm[pos], n0, equal_nan=True)


def test_bsc_nonfinite_keypoints(ge):
    check_bsc_nonfinite_keypoint(ge, scan_like_cloud(1500, 17), 18)


@pytest.mark.parametrize("kind", ["scan", "offset"])
def test_prep_run_nonfinite_rows_change_nothing(ge, kind):
    check_prep_metamorphic(ge, edge_cloud(kind, 6000, 19), 20)


def test_prep_far_outliers_bound_the_fallbacks(ge):
    P = edge_cloud("far", 3000, 21)
    check_far_fallbacks(ge, P, 30)


@pytest.mark.parametrize("name,kw", [("test_voxel_filter", dict(n=3000)), ("test_keypoints", dict(n=2000)),
                                     ("test_fpfh_metamorphic", dict(n=800)), ("test_prep_run", dict(n=5000)),
                                     ("test_far_outlier_1e10", dict(n=1500)), ("test_pcd_with_nan_rows_end_to_end", dict(n=8000))])
def test_gpu_test_functions_on_the_emulated_library(ge, orc, name, kw, tmp_path, emu_library_path, monkeypatch):
    import test_zz9_prep_edges_gpu as t
    if name == "test_pcd_with_nan_rows_end_to_end":   # ghicp_cli finds the emulated libghicp_b200.so through the loader path
        monkeypatch.setenv("LD_LIBRARY_PATH", os.path.dirname(emu_library_path) + os.pathsep + os.environ.get("LD_LIBRARY_PATH", ""))
        kw = dict(kw, tmp_path=tmp_path)
    getattr(t, name)(ge, orc, **kw)
