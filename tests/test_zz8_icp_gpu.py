"""GPU tests of point-to-point ICP on the dense clouds (ghicp_icp.cu, DESIGN.md §3.13) through the C ABI against the oracle
(tests/harness/icp_oracle.cpp): the transform, traces, state, fitness and moved cloud bit for bit, with all four option
combinations.  Also determinism, the known-pose scan pairs, register_clouds(refine=...) and the C++ icp_reg.
tests/test_icp.py runs these functions on the emulated library with smaller clouds."""
import math
import os
import subprocess

import numpy as np
import pytest

import icp_oracle as io

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OPTIONS = [dict(), dict(reciprocal=True), dict(trim_ratio=0.8), dict(reciprocal=True, trim_ratio=0.7)]


def pose(deg, t):
    g = __import__("ghicp_b200")
    Rt = np.eye(4)
    Rt[:3, :3] = g.synth.rot_xyz_deg(0.3 * deg, -0.2 * deg, deg)
    Rt[:3, 3] = t
    return Rt


def truth(R, t):
    G = np.eye(4)
    G[:3, :3], G[:3, 3] = R, t
    return G


def same(got, want):
    Rt, info = got
    wRt, w = want
    assert np.array_equal(Rt, wRt)
    for k in ("iterations", "state", "converged", "cor"):
        assert info[k] == w[k], (k, info[k], w[k])
    assert np.array_equal(info["cor_trace"], w["cor_trace"]) and np.array_equal(info["mse_trace"], w["mse_trace"], equal_nan=True)
    assert np.float64(info["fitness"]).tobytes() == np.float64(w["fitness"]).tobytes()
    assert np.array_equal(info["moved"], w["moved"], equal_nan=True)


def errors(Rt, G):
    """(rotation error in degrees, translation error in m) of Rt against the truth G; the angle from the skew part of
    Rt^T G, which stays accurate near 0 where acos of the trace does not."""
    M = Rt[:3, :3].T @ G[:3, :3]
    v = 0.5 * np.array([M[2, 1] - M[1, 2], M[0, 2] - M[2, 0], M[1, 0] - M[0, 1]])
    return math.degrees(math.asin(min(1.0, float(np.linalg.norm(v))))), float(np.linalg.norm(Rt[:3, 3] - G[:3, 3]))


def scan(g, n_points, seed):
    T, S, R, t = g.synth.scan_pair(n_points, seed=seed)
    return np.asarray(S, np.float32), np.asarray(T, np.float32), truth(R, t)


def test_equals_oracle(g, n_points=60000):
    S, T, G = scan(g, n_points, 1)
    G0 = pose(2.0, [0.3, -0.2, 0.1]) @ G
    for kw in OPTIONS:
        got = g.cloud_icp(S, T, G0, max_iterations=10, return_moved=True, trace=True, **kw)
        same(got, io.icp(S, T, G0, max_iterations=10, grid=True, **kw))


def test_million_points_equal_oracle_grid(g, n_points=1000000):
    """A million-point scan against a shuffled copy of itself with 1 cm of noise, started 0.3 degrees / 5 cm off: every query
    has a near neighbour, which keeps the one-thread oracle's grid search to minutes."""
    T = np.asarray(g.synth.scan_pair(n_points, seed=5)[0], np.float32)
    rng = np.random.default_rng(5)
    S = (T[rng.permutation(len(T))] + rng.normal(0.0, 0.01, T.shape)).astype(np.float32)
    G0 = pose(0.3, [0.03, -0.03, 0.02])
    for kw in (OPTIONS[0], OPTIONS[3]):
        got = g.cloud_icp(S, T, G0, max_iterations=3, return_moved=True, trace=True, **kw)
        same(got, io.icp(S, T, G0, max_iterations=3, grid=True, **kw))
        i = got[1]
        print(dict(n=len(S), opt=kw, ms=i["stage_ms"], iterations=i["iterations"],
                   cells_per_query=i["cells_visited"] / (len(S) * i["iterations"])))


def test_two_calls_are_identical(g, n_points=60000):
    S, T, G = scan(g, n_points, 6)
    G0 = pose(3.0, [0.5, 0.2, 0.0]) @ G
    a = g.cloud_icp(S, T, G0, max_iterations=8, reciprocal=True, trim_ratio=0.8, return_moved=True, trace=True)
    b = g.cloud_icp(S, T, G0, max_iterations=8, reciprocal=True, trim_ratio=0.8, return_moved=True, trace=True)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1].pop("moved"), b[1].pop("moved"))
    for x in (a[1], b[1]):
        x.pop("stage_ms")
    assert np.array_equal(a[1].pop("mse_trace"), b[1].pop("mse_trace")) and np.array_equal(a[1].pop("cor_trace"), b[1].pop("cor_trace"))
    assert a[1] == b[1]


def test_scan_pairs_converge_towards_the_truth(g, n_points=200000, res=0.05):
    """Started 2 degrees / 0.5 m off the truth on the down-sampled scan pair, ICP with the trimmed rejector (ratio = calOverlap
    at the start, as icp_reg sets it) ends closer to the truth than it started, with and without reciprocal correspondences;
    register_clouds(refine=...) gives a fitness no worse than the unrefined transform.  Without the rejector the 40 % of the
    source the target never saw pull the pose away (printed, not asserted): that is what the rejector is for."""
    T, S, R, t = g.synth.scan_pair(n_points, seed=4)
    G = truth(R, t)
    pt, ps = g.Prep(T, res, 1.0, 1.5), g.Prep(S, res, 1.0, 1.5)
    try:
        G0 = pose(2.0, [0.3, -0.3, 0.25]) @ G
        e0 = errors(G0, G)
        rho = min(ps.overlap(pt, G0, thre_dis=0.3, fitness=False)["ratio"], 1.0)
        for recip in (False, True):
            for trim in (0.0, rho):
                Rt, info = ps.icp(pt, G0, max_iterations=50, reciprocal=recip, trim_ratio=trim)
                e = errors(Rt, G)
                print(dict(reciprocal=recip, trim_ratio=trim, start=e0, end=e, iterations=info["iterations"], state=info["state"],
                           fitness=info["fitness"]))
                assert info["converged"]
                if trim > 0:
                    assert e[0] < e0[0] and e[1] < e0[1]
        Rt, info = ps.icp(pt, G, max_iterations=50)
        print(dict(start="truth", end=errors(Rt, G), iterations=info["iterations"], state=info["state"]))
    finally:
        pt.close(); ps.close()
    # scored within 1 m (max_range = 1 m^2): over every point the fitness also averages the 40 % of the source the target never
    # saw, which the true pose places beyond the target's end (DESIGN.md §3.12)
    kw = dict(corr_type=g.CT_NNR, feature_type=g.FT_FPFH, max_iter=30)
    ev = dict(thre_dis=0.3, max_range=1.0)
    Rt0, i0 = g.register_clouds(T, S, 0.3, 1.0, 1.5, evaluate=ev, **kw)
    Rt1, i1 = g.register_clouds(T, S, 0.3, 1.0, 1.5, evaluate=ev, refine=dict(max_iter=30, reciprocal=False, trimmed_thre_dis=0.3),
                                **kw)
    print(dict(ghicp=(errors(Rt0, G), i0["evaluation"]["fitness"]), refined=(errors(Rt1, G), i1["evaluation"]["fitness"]),
               icp=dict(iterations=i1["icp"]["iterations"], state=i1["icp"]["state"], trim_ratio=i1["icp"]["trim_ratio"])))
    assert np.array_equal(i1["icp"]["Rt_before"], Rt0)
    assert i1["evaluation"]["fitness"] <= i0["evaluation"]["fitness"]


CXX_MAIN = r"""
// CRegistration::icp_reg of the C++ mirror
#include <fstream>
#include "common_reg.h"
using namespace ghicp;
static Cloud read_xyz(const char *path) { std::ifstream f(path, std::ios::binary); Cloud c; float v[3];
  while (f.read((char *)v, sizeof(v))) c.push(v[0], v[1], v[2]); return c; }
int main(int argc, char **argv) {
  Cloud S = read_xyz(argv[1]), T = read_xyz(argv[2]), moved;
  Matrix4f m;
  CRegistration<> reg;
  const bool ok = reg.icp_reg(S, T, moved, m, 20, true, true, 0.3f, 0.1f);
  Cloud none;
  Matrix4f m2;
  const bool refused = !reg.icp_reg(S, T, none, m2, 20, false, true, 0.3f, 1.5f);   // the ratio is below 1.5: not done
  std::ofstream out(argv[3], std::ios::binary);
  const double fit = reg.getFitnessScore();
  out.write((const char *)&fit, sizeof(fit));
  out.write((const char *)m.data(), 16 * sizeof(float));
  out.write((const char *)moved.xyz.data(), moved.xyz.size() * sizeof(float));
  return ok && refused ? 0 : 3;
}
"""


def test_cxx_icp_reg_matches_python(g, tmp_path, n_points=20000):
    S, T, G = scan(g, n_points, 8)
    S = io_move(S, G)   # the C++ icp_reg starts from the identity: hand it a source already close to the target
    S.tofile(tmp_path / "s.bin"); T.tofile(tmp_path / "t.bin")
    (tmp_path / "main.cpp").write_text(CXX_MAIN)
    pkg = os.path.join(ROOT, "gh-icp_b200")
    exe = str(tmp_path / "icp_main")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-I" + os.path.join(pkg, "cxx"), str(tmp_path / "main.cpp"), "-o", exe,
                        "-L" + pkg, "-lghicp_b200", "-Wl,-rpath," + pkg, "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([exe, str(tmp_path / "s.bin"), str(tmp_path / "t.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "Point-to-Point ICP done in " in r.stdout and "The fitness score of this registration is " in r.stdout
    assert "The overlap ratio is too small. This registration would not be done." in r.stdout
    raw = np.fromfile(tmp_path / "out.bin", np.uint8)
    fit = np.frombuffer(raw[:8].tobytes(), np.float64)[0]
    m = np.frombuffer(raw[8:72].tobytes(), np.float32).reshape(4, 4).T
    moved = np.frombuffer(raw[72:].tobytes(), np.float32).reshape(-1, 3)
    Rt, info = g.icp_reg(S, T, 20, True, True, 0.3, 0.1)
    assert np.array_equal(m.astype(np.float64), Rt) and fit == info["fitness"] and np.array_equal(moved, info["moved"])


def io_move(A, G):
    G = np.asarray(G, np.float32)
    return np.stack([((G[r, 0] * A[:, 0] + G[r, 1] * A[:, 1]) + G[r, 2] * A[:, 2]) + G[r, 3] for r in range(3)], axis=1)
