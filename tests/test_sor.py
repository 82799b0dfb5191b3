"""CPU checks of the statistical outlier removal (CFilter::SORFilter, DESIGN.md §3.16).

  * the oracle (tests/harness/sor_oracle.cpp, one thread) against an independent formulation (scipy's cKDTree with a margin
    of extra neighbours, float32 d2 recomputed in numpy in the definition's order, square roots added column by column),
    bit for bit, in its brute-force and grid modes; PCL's one-pass variance going negative on a lattice;
  * the product's kernels (ghicp_prep.cu) through the C ABI of the emulated library (tests/harness/emu_library.cpp) against
    the oracle: distances bit for bit, statistics within 1e-12, the same kept points; edge cases, far outliers, a random
    fiber schedule, argument errors, allocation failures;
  * the pipeline: Prep(sor=...) equals the hand-chained stand-alone calls, and register_clouds(sor=None) is unchanged."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
from scipy.spatial import cKDTree

import sor_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KS = [1, 2, 31, 32, 33, 50, 128]


def cloud(n, seed, outliers=0, dup=0):
    """points on two noisy planes of a 10 m box, `outliers` scattered in a 3x larger box, `dup` exact duplicates"""
    rng = np.random.default_rng(seed)
    a = rng.random((n, 3)) * 10.0
    a[: n // 2, 2] = rng.normal(0.0, 0.02, n // 2)
    a[n // 2:, 0] = 10.0 + rng.normal(0.0, 0.02, n - n // 2)
    P = a.astype(np.float32)
    if outliers:
        P = np.concatenate([P, (rng.random((outliers, 3)) * 30.0 - 10.0).astype(np.float32)])
    if dup:
        P = np.concatenate([P, P[rng.integers(0, len(P), dup)]])
    return P[rng.permutation(len(P))]


def numpy_sor(P, mean_k, std_mul, margin=8):
    """The definition through cKDTree candidates: float32 d2 in (dx*dx + dy*dy) + dz*dz order, (d2, index) order, the square
    roots added column by column in double (np.sum would add pairwise)."""
    P = np.asarray(P, np.float32)
    fin = np.flatnonzero(np.isfinite(P).all(axis=1))
    F = P[fin]
    nf = len(F)
    k = min(mean_k, nf - 1) if nf else 0
    dist = np.full(len(P), np.nan, np.float32)
    if k == 0:
        dist[fin] = 0.0
    else:
        m = min(nf, k + 1 + margin)
        _, nb = cKDTree(F.astype(np.float64)).query(F.astype(np.float64), k=m)
        nb = nb.reshape(nf, m)
        dx, dy, dz = (F[:, None, a] - F[nb, a] for a in range(3))
        d2 = (dx * dx + dy * dy) + dz * dz
        d2 = np.where(nb == np.arange(nf)[:, None], np.float32(np.inf), d2)          # not its own neighbour (by index)
        order = np.lexsort((fin[nb], d2), axis=-1)
        d2s = np.take_along_axis(d2, order, axis=1)[:, :k]
        s = np.zeros(nf)
        for j in range(k):
            s = s + np.sqrt(d2s[:, j].astype(np.float64))
        dist[fin] = (s / k).astype(np.float32)
    d = dist[fin].astype(np.float64)
    mean = 0.0
    for v in d:
        mean += v
    mean = mean / nf if nf else 0.0
    ss = 0.0
    for v in d:
        ss += (v - mean) * (v - mean)
    sd = float(np.sqrt(ss / (nf - 1))) if nf > 1 else 0.0
    thr = mean + std_mul * sd
    kept = fin[~(d > thr)]
    return dict(distances=dist, kept=kept, mean=mean, stddev=sd, threshold=thr)


def inputs():
    yield "random", cloud(600, 1)
    yield "outliers", cloud(600, 2, outliers=12)
    yield "duplicates", cloud(500, 3, dup=80)


# ---- the oracle against an independent formulation -----------------------------------------------------------------------
@pytest.mark.parametrize("mean_k", KS)
@pytest.mark.parametrize("name", ["random", "outliers", "duplicates"])
def test_oracle_equals_ckdtree_formulation(name, mean_k):
    P = dict(inputs())[name]
    want = numpy_sor(P, mean_k, 1.0)
    for grid in (False, True):
        o = so.sor(P, mean_k, 1.0, grid=grid)
        assert np.array_equal(o["distances"].view(np.uint32), want["distances"].view(np.uint32)), grid
        assert np.array_equal(o["kept"], want["kept"])
        assert o["mean"] == want["mean"] and o["stddev"] == want["stddev"] and o["threshold"] == want["threshold"]


def test_oracle_grid_mode_with_far_outliers_and_non_finite_rows():
    P = cloud(800, 4, outliers=5)
    P[::97] += np.float32([1e4, 0.0, 0.0])
    P[5::131] = np.nan
    P[7::151, 1] = np.inf
    for k in (8, 50):
        a, b = so.sor(P, k, 2.0), so.sor(P, k, 2.0, grid=True)
        assert np.array_equal(a["distances"].view(np.uint32), b["distances"].view(np.uint32)) and np.array_equal(a["kept"], b["kept"])


def lattice(m=24):
    """points (i, j, 0) with i + j even: every point's nearest neighbour is a diagonal one, d = float(sqrt(2))"""
    i, j = np.meshgrid(np.arange(m), np.arange(m), indexing="ij")
    sel = (i + j) % 2 == 0
    return np.stack([i[sel], j[sel], np.zeros(sel.sum())], axis=1).astype(np.float32)


def test_one_pass_variance_goes_negative_on_a_lattice():
    """PCL's (sq_sum - sum^2 / n) / (n - 1), with float squares, is negative here (a NaN stddev); the two-pass form gives 0
    and keeps every point."""
    P = lattice()
    o = so.sor(P, 1, 1.0)
    d = o["distances"]
    assert np.all(d == np.float32(np.sqrt(2.0)))
    s, sq = 0.0, 0.0
    for v in d:
        s += float(v)
        sq += float(np.float32(v) * np.float32(v))
    n = len(d)
    assert (sq - s * s / n) / (n - 1) < 0.0
    assert o["stddev"] == 0.0 and len(o["kept"]) == n


# ---- the emulated kernels through the C ABI --------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def ge(g, emu_library_path):
    from conftest import swap_in_library
    real = swap_in_library(g, emu_library_path)
    try:
        yield g
    finally:
        g.capi._lib = real


def near_threshold(d, thr):
    d = d.astype(np.float64)
    return np.flatnonzero(~np.isnan(d) & (np.abs(d - thr) <= 1e-9 * max(abs(thr), 1e-300)))


def same(got_idx, info, want):
    """distances bit for bit, statistics within 1e-12 relative, kept sets equal away from the threshold (none near it here)"""
    d = info["distances"]
    assert np.array_equal(d.view(np.uint32), want["distances"].view(np.uint32))
    for key in ("mean", "stddev", "threshold"):
        a, b = info[key], want[key]
        assert a == b or abs(a - b) <= 1e-12 * abs(b), (key, a, b)
    if info["threshold"] != want["threshold"]:   # equal thresholds decide every point alike (on a lattice d == threshold)
        near = near_threshold(d, want["threshold"])
        assert len(near) == 0, near
    assert np.array_equal(got_idx, want["kept"])
    assert info["n_kept"] == len(got_idx) and info["n_finite"] == want["n_finite"] and info["k_eff"] == want["k_eff"]


@pytest.mark.parametrize("mean_k", KS)
def test_emulated_abi_equals_the_oracle(ge, mean_k):
    P = cloud(700, 5, outliers=10, dup=20)
    for std_mul in (1.0, -0.5):
        idx, info = ge.sor_filter(P, mean_k, std_mul, return_distances=True)
        same(idx, info, so.sor(P, mean_k, std_mul))
        assert info["fallbacks"] >= 0 and info["candidates"] >= info["n_finite"] * info["k_eff"]


@pytest.mark.parametrize("mean_k", [1, 2, 20, 31])
def test_emulated_abi_both_distance_paths(ge, mean_k, monkeypatch):
    """k_eff <= 31 runs k_knn + k_sor_listmean; GHICP_SOR_FORCE_WARP=1 runs the warp kernel of larger k instead: both equal the
    oracle bit for bit (duplicates included, where the point itself may fall out of k_knn's list)"""
    P = cloud(600, 13, outliers=8, dup=60)
    P = np.concatenate([P, np.repeat(P[:1], 40, axis=0)])   # more copies of one point than the list holds
    want = so.sor(P, mean_k, 1.0)
    a, ia = ge.sor_filter(P, mean_k, 1.0, return_distances=True)
    monkeypatch.setenv("GHICP_SOR_FORCE_WARP", "1")
    b, ib = ge.sor_filter(P, mean_k, 1.0, return_distances=True)
    for idx, info in ((a, ia), (b, ib)):
        same(idx, info, want)


@pytest.mark.parametrize("n", [0, 1, 2, 3, 20])
def test_emulated_abi_small_clouds(ge, n):
    P = cloud(20, 6)[:n]
    for k in (1, 2, 19, 50):
        idx, info = ge.sor_filter(P, k, 1.0, return_distances=True)
        want = so.sor(P, k, 1.0)
        if n == 0:
            assert len(idx) == 0 and info["n_finite"] == 0 and info["k_eff"] == 0
            continue
        same(idx, info, want)
        assert info["k_eff"] == min(k, n - 1)
    if n == 1:
        idx, info = ge.sor_filter(P, 5, 1.0, return_distances=True)
        assert info["distances"][0] == 0.0 and idx.tolist() == [0] and info["stddev"] == 0.0


def test_emulated_abi_non_finite_rows(ge):
    """the result equals the finite-only result mapped back; non-finite rows have NaN distances and are never kept"""
    P = cloud(600, 7, outliers=6)
    Q = P.copy()
    bad = np.arange(3, len(P), 37)
    Q[bad[::3], 0] = np.nan
    Q[bad[1::3], 1] = np.inf
    Q[bad[2::3], 2] = -np.inf
    fin = np.setdiff1d(np.arange(len(P)), bad)
    for k in (8, 50):
        idx, info = ge.sor_filter(Q, k, 1.0, return_distances=True)
        i2, info2 = ge.sor_filter(P[fin], k, 1.0, return_distances=True)
        assert np.array_equal(idx, fin[i2])
        assert np.array_equal(info["distances"][fin].view(np.uint32), info2["distances"].view(np.uint32))
        assert np.all(np.isnan(info["distances"][bad]))
        same(idx, info, so.sor(Q, k, 1.0))
    idx, info = ge.sor_filter(np.full((9, 3), np.nan, np.float32), 5, 1.0, return_distances=True)
    assert len(idx) == 0 and info["n_finite"] == 0 and np.all(np.isnan(info["distances"]))


def test_emulated_abi_far_outliers(ge):
    P = cloud(600, 8)
    P[17] = [1e4, 0.0, 0.0]
    P[301] = [0.0, 1e7, 5.0]
    P[450] = [-1e4, -1e4, 3.0]
    idx, info = ge.sor_filter(P, 20, 1.0, return_distances=True)
    same(idx, info, so.sor(P, 20, 1.0))
    assert info["fallbacks"] > 0
    assert 301 not in idx              # the 10^7 m return; it inflates stddev enough to mask the two at 10 km (as in PCL)


def test_emulated_abi_lattice(ge):
    P = lattice(20)
    for k in (1, 4, 12):
        idx, info = ge.sor_filter(P, k, 1.0, return_distances=True)
        same(idx, info, so.sor(P, k, 1.0))
    idx, info = ge.sor_filter(P, 1, 1.0)
    assert info["stddev"] == 0.0 and len(idx) == len(P)


def test_emulated_abi_under_a_random_schedule(g, emu_library_path, tmp_path):
    """GHICP_EMU_SCHED: fibers visited in a fresh random order at every sweep (read once per process: a child process)."""
    P = cloud(500, 9, outliers=8, dup=10)
    np.save(tmp_path / "in.npy", P)
    code = ("import sys, numpy as np; sys.path.insert(0, %r); sys.path.insert(0, %r); import ghicp_b200 as g;"
            "from conftest import swap_in_library; swap_in_library(g, %r); P = np.load(%r);"
            "i, r = g.sor_filter(P, 40, 1.0, return_distances=True);"
            "np.savez(%r, i=i, d=r['distances'], s=np.array([r['mean'], r['stddev'], r['threshold']]))"
            % (ROOT, os.path.join(ROOT, "tests"), emu_library_path, str(tmp_path / "in.npy"), str(tmp_path / "out.npz")))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, GHICP_EMU_SCHED="11"))
    assert r.returncode == 0, r.stderr[-3000:]
    got = np.load(tmp_path / "out.npz")
    want = so.sor(P, 40, 1.0)
    assert np.array_equal(got["d"].view(np.uint32), want["distances"].view(np.uint32)) and np.array_equal(got["i"], want["kept"])
    assert abs(got["s"][2] - want["threshold"]) <= 1e-12 * abs(want["threshold"])


def test_emulated_abi_argument_errors(ge):
    g = ge
    L = g.capi.lib()
    fpp, ip = C.POINTER(C.c_float), C.POINTER(C.c_int)
    P = cloud(40, 10)
    out = np.full(40, -7, np.int32)
    x, o = P.ctypes.data_as(fpp), out.ctypes.data_as(ip)
    r = g.capi.SorResult()
    bad = [(x, 40, 0, 1.0, o, C.byref(r)), (x, 40, 129, 1.0, o, C.byref(r)), (x, 40, 5, float("nan"), o, C.byref(r)),
           (x, 40, 5, float("inf"), o, C.byref(r)), (x, 40, 5, -float("inf"), o, C.byref(r)), (None, 40, 5, 1.0, o, C.byref(r)),
           (x, 40, 5, 1.0, None, C.byref(r)), (x, 40, 5, 1.0, o, None), (x, -1, 5, 1.0, o, C.byref(r))]
    for px, n, k, s, po, pr in bad:
        assert L.ghicp_sor_filter(0, px, n, k, s, po, None, pr) == -1
        assert np.all(out == -7)
    for k, s in ((0, 1.0), (129, 1.0), (5, float("nan"))):
        with pytest.raises(g.GhicpError):
            g.sor_filter(P, k, s)
        with pytest.raises(g.GhicpError) as e:                 # refused before any pipeline work (mean_k 0 = "no filter")
            g.Prep(P, 0.3, 1.0, 1.5, sor=(k, s))
        assert "sor: mean_k must be in 1..128" in str(e.value)
        with pytest.raises(g.GhicpError) as e:
            g.register_clouds(P, P, 0.3, 1.0, 1.5, sor=(k, s))
        assert "sor: mean_k must be in 1..128" in str(e.value)
    idx, info = g.sor_filter(P, 5, -3.0)                       # a negative std_mul is allowed, as in PCL
    assert np.array_equal(idx, so.sor(P, 5, -3.0)["kept"])
    p = g.Prep(cloud(400, 11), 0.3, 1.0, 1.5)
    try:
        assert p.sor_info is None
        assert L.ghicp_prep_sor_info(p.h, None, None, None) == -1   # made without the filter
    finally:
        p.close()


# ---- allocation failures -------------------------------------------------------------------------------------------------
def test_allocation_failures(ge):
    from test_alloc_failures import sweep
    g = ge
    L = g.capi.lib()
    L.ghicp_emu_live_allocations.restype = C.c_longlong
    L.ghicp_emu_fail_allocation.argtypes = [C.c_longlong]
    fpp, ip = C.POINTER(C.c_float), C.POINTER(C.c_int)
    P = cloud(300, 12, outliers=4)
    want = so.sor(P, 10, 1.0)
    out = np.full(len(P), -7, np.int32)
    dist = np.zeros(len(P), np.float32)

    def call():
        r = g.capi.SorResult()
        return L.ghicp_sor_filter(0, P.ctypes.data_as(fpp), len(P), 10, 1.0, out.ctypes.data_as(ip), dist.ctypes.data_as(fpp),
                                  C.byref(r))

    def untouched(k):
        assert np.all(out == -7)

    k, rc = sweep(L, "sor_filter", call, untouched)
    assert rc == 0 and k > 5
    assert np.array_equal(out[:len(want["kept"])], want["kept"])

    T, _, _, _ = g.synth.scan_pair(3000, seed=3)
    T = np.ascontiguousarray(T, np.float32)
    params = g.capi.PrepParams(0.3, 1.0, 0.65, 5, 1.5, 0.0, 7, 0)
    handles = []

    def prep_call():
        h = C.c_void_p()
        rc = L.ghicp_prep_run_sor(0, T.ctypes.data_as(fpp), len(T), C.byref(params), None, 20, 1.0, C.byref(h))
        if rc >= 0:
            handles.append(h)
        else:
            assert not h.value
        return rc

    k, rc = sweep(L, "prep_run", prep_call)
    assert rc == 0 and k > 10
    h = handles[0]
    r, nv = g.capi.SorResult(), C.c_int(0)
    assert L.ghicp_prep_sor_info(h, C.byref(r), C.byref(nv), None) == 0
    assert nv.value > r.n_kept > 0
    L.ghicp_prep_destroy(h)


# ---- the pipeline ----------------------------------------------------------------------------------------------------------
def test_prep_sor_equals_the_hand_chained_calls(ge):
    """voxel -> gather -> sor_filter -> gather -> detect_keypoints -> BSC, bit for bit"""
    g = ge
    T, _, _, _ = g.synth.scan_pair(5000, seed=5)
    T = np.concatenate([T, np.float32([[60.0, -40.0, 9.0], [0.5, 80.0, -30.0]])]).astype(np.float32)
    p = g.Prep(T, 0.3, 1.0, 1.5, bsc_radius=1.5, dof_type=6, min_pts=5, sor=(20, 1.0))
    try:
        D = T[g.voxel_downsample(T, 0.3)]
        kept, info = g.sor_filter(D, 20, 1.0)
        F = D[kept]
        assert np.array_equal(p.down(), F)
        assert p.n_down == len(F) and p.sor_info["n_voxel"] == len(D) and p.sor_info["n_kept"] == len(F)
        for key in ("mean", "stddev", "threshold", "candidates", "fallbacks", "k_eff", "n_finite"):
            assert p.sor_info[key] == info[key], key
        assert np.array_equal(p.bbox_min, F.min(axis=0)) and np.array_equal(p.bbox_max, F.max(axis=0))
        kp, _, _, _ = g.detect_keypoints(F, 1.0, 0.65, 5, 1.5)
        idx, _ = p.keypoints()
        assert np.array_equal(idx, kp)
        bits, _, _ = g.bsc_extract(F, kp, 1.5, dof_type=6)
        assert np.array_equal(p.bsc(), bits)
        assert len(D) - len(F) >= 2                                      # the two planted returns at least
    finally:
        p.close()


def test_register_clouds_sor(ge):
    g = ge
    T, S, _, _ = g.synth.scan_pair(5000, seed=4)
    kw = dict(corr_type=g.CT_NNR, feature_type=g.FT_NONE, max_iter=15)
    Rt0, base = g.register_clouds(T, S, 0.3, 1.0, 1.5, **kw)
    Rt1, same_ = g.register_clouds(T, S, 0.3, 1.0, 1.5, sor=None, **kw)
    assert np.array_equal(Rt0, Rt1) and "sor" not in same_ and set(same_) == set(base)
    Rt2, info = g.register_clouds(T, S, 0.3, 1.0, 1.5, sor=(20, 2.0), **kw)
    for side in ("target", "source"):
        s = info["sor"][side]
        assert s["n_voxel"] >= s["n_kept"] > 0
    assert info["n_source_down"] == info["sor"]["source"]["n_kept"]
    # the features= branch filters the same clouds
    Rt3, info3 = g.register_clouds(T, S, 0.3, 1.0, 1.5, sor=(20, 2.0), **kw,
                                   features=lambda td, tk, sd, sk: g.Keypoints().setCoordinate(sd[sk], td[tk]))
    assert info3["n_source_down"] == info["n_source_down"] and info3["bbx_magnitude"] == info["bbx_magnitude"]
    assert info3["sor"]["source"]["threshold"] == info["sor"]["source"]["threshold"]
    assert set(info3["sor"]["source"]) == set(info["sor"]["source"])   # the same keys on both branches
    with pytest.raises(g.GhicpError):
        g.register_clouds(T, S, 0.3, 1.0, 1.5, sor=(20,), **kw)
