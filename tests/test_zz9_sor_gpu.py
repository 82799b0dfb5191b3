"""GPU tests of the statistical outlier removal (CFilter::SORFilter, DESIGN.md §3.16) through the C ABI against the oracle
(tests/harness/sor_oracle.cpp): per-point distances bit for bit, statistics within 1e-12 relative, the same kept points.
Also determinism, planted outliers, the edge cases of tests/test_sor.py on hardware, a full registration with outliers and a
far return, and the C++ mirror."""
import os
import subprocess

import numpy as np
import pytest
from scipy.spatial import cKDTree

import sor_oracle as so
from test_sor import cloud, lattice, same

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def scans(g, n_points=1000000, voxel=0.05):
    T, _, _, _ = g.synth.scan_pair(n_points, seed=6)
    raw = np.ascontiguousarray(T, np.float32)
    return dict(raw=raw, voxel=np.ascontiguousarray(raw[g.voxel_downsample(raw, voxel)]))


@pytest.fixture(scope="module")
def scan_set(g):
    return scans(g)


@pytest.mark.parametrize("which", ["raw", "voxel"])
@pytest.mark.parametrize("mean_k", [8, 50, 128])
def test_scan_equals_oracle(g, scan_set, which, mean_k):
    P = scan_set[which]
    want = so.sor(P, mean_k, 1.0, grid=True)
    for std_mul in (1.0, 2.0):
        idx, info = g.sor_filter(P, mean_k, std_mul, return_distances=True)
        same(idx, info, so.with_std_mul(want, std_mul))
        print(dict(which=which, n=len(P), mean_k=mean_k, std_mul=std_mul, kept=len(idx), stage_ms=info["stage_ms"],
                   candidates_per_query=info["candidates"] / max(info["n_finite"], 1), fallbacks=info["fallbacks"]))


@pytest.mark.parametrize("mean_k", [8, 31])
def test_both_distance_paths_agree(g, scan_set, mean_k, monkeypatch):
    """k_eff <= 31 runs k_knn's register top-k; GHICP_SOR_FORCE_WARP=1 runs the warp kernel of larger k on the same input"""
    P = scan_set["voxel"]
    a, ia = g.sor_filter(P, mean_k, 1.0, return_distances=True)
    monkeypatch.setenv("GHICP_SOR_FORCE_WARP", "1")
    b, ib = g.sor_filter(P, mean_k, 1.0, return_distances=True)
    assert np.array_equal(a, b) and np.array_equal(ia["distances"].view(np.uint32), ib["distances"].view(np.uint32))
    assert ia["threshold"] == ib["threshold"]


def test_two_runs_are_identical(g, scan_set):
    P = scan_set["voxel"]
    a, ia = g.sor_filter(P, 50, 1.0, return_distances=True)
    b, ib = g.sor_filter(P, 50, 1.0, return_distances=True)
    assert np.array_equal(a, b) and np.array_equal(ia["distances"].view(np.uint32), ib["distances"].view(np.uint32))
    for k in ("mean", "stddev", "threshold"):
        assert np.float64(ia[k]).tobytes() == np.float64(ib[k]).tobytes()


def planted(P, frac=0.005, min_dist=1.0, seed=3):
    """P plus frac * len(P) points scattered in its box, each at least min_dist from every point of P"""
    rng = np.random.default_rng(seed)
    tree = cKDTree(P.astype(np.float64))
    lo, hi = P.min(axis=0).astype(np.float64), P.max(axis=0).astype(np.float64)
    want, out = int(frac * len(P)), []
    for _ in range(100):
        c = lo + rng.random((20 * want, 3)) * (hi - lo)
        d, _ = tree.query(c)
        out.append(c[d >= min_dist])
        if sum(len(o) for o in out) >= want:
            break
    O = np.concatenate(out)[:want].astype(np.float32)
    assert len(O) == want, "the box has too little room at this clearance"
    return np.concatenate([P, O]), np.arange(len(P), len(P) + len(O))


def test_planted_outliers_are_removed(g, scan_set):
    """0.5 % of points scattered in the scan's box, at least 10 voxels (0.5 m) from every scan point: mean_k 50, std_mul 1
    removes every one of them.  The synthetic scan fills its box densely: no point of the box lies farther than 0.83 m from
    it, and about 1 % lie 0.5 m away or more."""
    P = scan_set["raw"]
    Q, out_idx = planted(P, 0.005, 10 * 0.05)
    idx, info = g.sor_filter(Q, 50, 1.0)
    assert not np.isin(out_idx, idx).any()
    print(dict(n=len(Q), planted=len(out_idx), kept=len(idx), threshold=info["threshold"], stage_ms=info["stage_ms"]))


def test_edge_cases(g):
    P = cloud(3000, 7, outliers=20, dup=200)
    Q = P.copy()
    bad = np.arange(3, len(P), 37)
    Q[bad[::2], 0] = np.nan
    Q[bad[1::2], 2] = np.inf
    Q[11] = [1e4, 0.0, 0.0]
    Q[1234] = [0.0, 1e7, 5.0]
    fin = np.setdiff1d(np.arange(len(P)), bad)
    for k in (1, 32, 33, 128):
        idx, info = g.sor_filter(Q, k, 1.0, return_distances=True)
        same(idx, info, so.sor(Q, k, 1.0))
        i2, _ = g.sor_filter(Q[fin], k, 1.0)
        assert np.array_equal(idx, fin[i2]) and np.all(np.isnan(info["distances"][bad]))
        assert info["fallbacks"] > 0
    for n in (0, 1, 2):
        idx, info = g.sor_filter(P[:n], 50, 1.0, return_distances=True)
        assert len(idx) == n and info["k_eff"] == max(n - 1, 0)
    idx, info = g.sor_filter(lattice(30), 1, 1.0)
    assert info["stddev"] == 0.0 and len(idx) == len(lattice(30))


def test_registration_with_outliers(g, n_points=60000):
    """register_clouds(sor=(50, 1.0)) on a scan pair whose source carries 0.5 % planted outliers and one return 1 km away
    (not at index 0: the voxel filter's phantom entry is the first finite point): the pose moves towards the ground truth as
    the pipeline tests require, and bbx_magnitude is that of the filtered down-sampled source, whose box lies inside the box of
    the source without the far return."""
    T, S, R_gt, t_gt = g.synth.scan_pair(n_points, seed=4)
    S = np.ascontiguousarray(S, np.float32)
    S2, _ = planted(S, 0.005, 0.5)
    S2 = np.insert(S2, 17, np.float32([1000.0, 0.0, 0.0]), axis=0)
    res, nms = 0.1, 1.2
    Rt, info = g.register_clouds(T, S2, res, 0.6, nms, corr_type=g.CT_NNR, feature_type=g.FT_FPFH, max_iter=60, sor=(50, 1.0))
    assert g.synth.rot_angle(Rt[:3, :3], R_gt) < g.synth.rot_angle(np.eye(3), R_gt)
    ps = g.Prep(S2, res, 0.6, nms, sor=(50, 1.0))
    try:
        D = ps.down()
        assert info["bbx_magnitude"] == ps.bbx_magnitude and info["n_source_down"] == ps.n_down
        assert np.all(D.min(axis=0) >= S.min(axis=0)) and np.all(D.max(axis=0) <= S.max(axis=0))
        assert info["sor"]["source"]["n_voxel"] > info["sor"]["source"]["n_kept"]
    finally:
        ps.close()
    _, plain = g.register_clouds(T, S2, res, 0.6, nms, corr_type=g.CT_NNR, feature_type=g.FT_FPFH, max_iter=60)
    assert plain["bbx_magnitude"] > 900.0 > info["bbx_magnitude"]   # without the filter the far return sets the scale


CXX_MAIN = r"""
// CFilter::voxelfilter and CFilter::SORFilter of the C++ mirror
#include <fstream>
#include "filter.h"
using namespace ghicp;
static Cloud read_xyz(const char *path) { std::ifstream f(path, std::ios::binary); Cloud c; float v[3];
  while (f.read((char *)v, sizeof(v))) c.push(v[0], v[1], v[2]); return c; }
static void write_xyz(const char *path, const Cloud &c) { std::ofstream f(path, std::ios::binary);
  f.write((const char *)c.xyz.data(), c.xyz.size() * sizeof(float)); }
int main(int argc, char **argv) {
  Cloud in = read_xyz(argv[1]), down, sor;
  CFilter<> f;
  f.voxelfilter(in, down, 0.1f);
  f.SORFilter(down, sor, 50, 2.0);
  write_xyz(argv[2], down);
  write_xyz(argv[3], sor);
  return 0;
}
"""


def test_cxx_mirror_matches_python(g, tmp_path, n_points=100000):
    T, _, _, _ = g.synth.scan_pair(n_points, seed=8)
    P = np.ascontiguousarray(T, np.float32)
    P.tofile(tmp_path / "in.bin")
    (tmp_path / "main.cpp").write_text(CXX_MAIN)
    pkg = os.path.join(ROOT, "gh-icp_b200")
    exe = str(tmp_path / "filter_main")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-I" + os.path.join(pkg, "cxx"), str(tmp_path / "main.cpp"), "-o", exe,
                        "-L" + pkg, "-lghicp_b200", "-Wl,-rpath," + pkg, "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "down.bin"), str(tmp_path / "sor.bin")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "Downsample done" in r.stdout
    down = np.fromfile(tmp_path / "down.bin", np.float32).reshape(-1, 3)
    sor = np.fromfile(tmp_path / "sor.bin", np.float32).reshape(-1, 3)
    D = P[g.voxel_downsample(P, 0.1)]
    assert np.array_equal(down, D)
    kept, _ = g.sor_filter(D, 50, 2.0)
    assert np.array_equal(sor, D[kept])
