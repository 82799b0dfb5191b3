"""GPU tests of Generalized ICP on the dense clouds (ghicp_icp.cu, metric 2, DESIGN.md §3.15) through the C ABI against the
oracle (tests/harness/gicp_oracle.cpp): the transform, traces, state, fitness and moved cloud bit for bit, with all four option
combinations.  Also determinism, both results' normal caches, the known-pose scan pair next to point-to-point and
point-to-plane, and the C++ gicp_reg.  tests/test_gicp.py runs these functions on the emulated library with smaller clouds."""
import os
import subprocess

import numpy as np
import pytest

import gicp_oracle as go
from test_zz8_icp_gpu import OPTIONS, errors, io_move, pose, same, scan, truth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GICP = dict(metric="gicp", normal_k=20)


def test_equals_oracle(g, n_points=60000):
    S, T, G = scan(g, n_points, 1)
    G0 = pose(2.0, [0.3, -0.2, 0.1]) @ G
    for kw in OPTIONS:
        got = g.cloud_icp(S, T, G0, max_iterations=8, return_moved=True, trace=True, **GICP, **kw)
        want = go.gicp(S, T, G0, max_iterations=8, grid=True, normal_k=20, **kw)
        same(got, want)
        print(dict(opt=kw, iterations=got[1]["iterations"], state=got[1]["state"], inner_passes=want[1]["inner_passes"].tolist()))


def test_million_points_equal_oracle_grid(g, n_points=1000000):
    """A million-point scan against a shuffled copy of itself with 1 cm of noise, started 0.3 degrees / 5 cm off (the
    one-thread oracle's grid search and both clouds' k-NN normals stay within minutes)."""
    T = np.asarray(g.synth.scan_pair(n_points, seed=5)[0], np.float32)
    rng = np.random.default_rng(5)
    S = (T[rng.permutation(len(T))] + rng.normal(0.0, 0.01, T.shape)).astype(np.float32)
    G0 = pose(0.3, [0.03, -0.03, 0.02])
    for kw in (OPTIONS[0], OPTIONS[3]):
        got = g.cloud_icp(S, T, G0, max_iterations=2, return_moved=True, trace=True, **GICP, **kw)
        want = go.gicp(S, T, G0, max_iterations=2, grid=True, normal_k=20, **kw)
        same(got, want)
        i = got[1]
        print(dict(n=len(S), opt=kw, ms=i["stage_ms"], iterations=i["iterations"], inner_passes=want[1]["inner_passes"].tolist()))


def test_two_calls_are_identical(g, n_points=60000):
    S, T, G = scan(g, n_points, 6)
    G0 = pose(3.0, [0.5, 0.2, 0.0]) @ G
    a = g.cloud_icp(S, T, G0, max_iterations=6, reciprocal=True, trim_ratio=0.8, return_moved=True, trace=True, **GICP)
    b = g.cloud_icp(S, T, G0, max_iterations=6, reciprocal=True, trim_ratio=0.8, return_moved=True, trace=True, **GICP)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1].pop("moved"), b[1].pop("moved"))
    for x in (a[1], b[1]):
        x.pop("stage_ms")
    assert np.array_equal(a[1].pop("mse_trace"), b[1].pop("mse_trace")) and np.array_equal(a[1].pop("cor_trace"), b[1].pop("cor_trace"))
    assert a[1] == b[1]


def test_scan_pairs_converge_towards_the_truth(g, n_points=200000, res=0.05):
    """Started 2 degrees / 0.5 m off the truth on the down-sampled scan pair, GICP with the trimmed rejector (ratio =
    calOverlap at the start) ends closer to the truth than it started, with and without reciprocal correspondences.
    Iterations, states, final errors and ms per iteration are printed next to point-to-point's and point-to-plane's."""
    T, S, R, t = g.synth.scan_pair(n_points, seed=4)
    G = truth(R, t)
    pt, ps = g.Prep(T, res, 1.0, 1.5), g.Prep(S, res, 1.0, 1.5)
    try:
        G0 = pose(2.0, [0.3, -0.3, 0.25]) @ G
        e0 = errors(G0, G)
        rho = min(ps.overlap(pt, G0, thre_dis=0.3, fitness=False)["ratio"], 1.0)
        for recip in (False, True):
            for trim in (0.0, rho):
                res_ = {}
                for metric in ("point", "plane", "gicp"):
                    Rt, info = ps.icp(pt, G0, max_iterations=50, reciprocal=recip, trim_ratio=trim, metric=metric, normal_k=20)
                    res_[metric] = (errors(Rt, G), info["iterations"], info["state"], info["stage_ms"]["iterations"] / info["iterations"])
                print(dict(reciprocal=recip, trim_ratio=trim, start=e0, **res_))
                if trim > 0:
                    e = res_["gicp"][0]
                    assert e[0] < e0[0] and e[1] < e0[1]
    finally:
        pt.close(); ps.close()


def test_prep_keeps_both_normals_per_k(g, n_points=200000, res=0.05):
    """Prep.icp(metric="gicp") builds the target's grid and both results' normals on the first call (stage_ms["grid"] > 0),
    reuses them for the same k (0), rebuilds them for another k, and a point-to-plane call with that k reuses the target's;
    every result equals the stand-alone call's."""
    T, S, R, t = g.synth.scan_pair(n_points, seed=4)
    G = truth(R, t)
    pt, ps = g.Prep(T, res, 1.0, 1.5), g.Prep(S, res, 1.0, 1.5)
    try:
        G0 = pose(1.0, [0.1, -0.1, 0.05]) @ G
        ms = []
        for k in (20, 20, 8, 8, 20):
            Rt, info = ps.icp(pt, G0, max_iterations=5, metric="gicp", normal_k=k)
            ms.append(info["stage_ms"]["grid"])
            w = g.cloud_icp(ps.down(), pt.down(), G0, max_iterations=5, metric="gicp", normal_k=k)
            assert np.array_equal(Rt, w[0]) and info["fitness"] == w[1]["fitness"]
        plane_ms = ps.icp(pt, G0, max_iterations=2, metric="plane", normal_k=20)[1]["stage_ms"]["grid"]
        print(dict(n_source_down=ps.n_down, n_target_down=pt.n_down, grid_and_normals_ms=ms, plane_after_gicp_ms=plane_ms))
        assert ms[0] > 0.0 and ms[1] == 0.0 and ms[2] > 0.0 and ms[3] == 0.0 and ms[4] > 0.0 and plane_ms == 0.0
    finally:
        pt.close(); ps.close()


CXX_MAIN = r"""
// CRegistration::gicp_reg of the C++ mirror
#include <fstream>
#include "common_reg.h"
using namespace ghicp;
static Cloud read_xyz(const char *path) { std::ifstream f(path, std::ios::binary); Cloud c; float v[3];
  while (f.read((char *)v, sizeof(v))) c.push(v[0], v[1], v[2]); return c; }
int main(int argc, char **argv) {
  Cloud S = read_xyz(argv[1]), T = read_xyz(argv[2]), moved;
  Matrix4f m;
  CRegistration<> reg;
  const bool ok = reg.gicp_reg(S, T, moved, m, 20, true, true, 0.3f, 20, 0.1f);
  Cloud none;
  Matrix4f m2;
  const bool refused = !reg.gicp_reg(S, T, none, m2, 20, false, true, 0.3f, 20, 1.5f);   // the ratio is below 1.5
  std::ofstream out(argv[3], std::ios::binary);
  const double fit = reg.getFitnessScore();
  out.write((const char *)&fit, sizeof(fit));
  out.write((const char *)m.data(), 16 * sizeof(float));
  out.write((const char *)moved.xyz.data(), moved.xyz.size() * sizeof(float));
  return ok && refused ? 0 : 3;
}
"""


def test_cxx_gicp_reg_matches_python(g, tmp_path, n_points=20000):
    S, T, G = scan(g, n_points, 8)
    S = io_move(S, G)   # the C++ gicp_reg starts from the identity: hand it a source already close to the target
    S.tofile(tmp_path / "s.bin"); T.tofile(tmp_path / "t.bin")
    (tmp_path / "main.cpp").write_text(CXX_MAIN)
    pkg = os.path.join(ROOT, "gh-icp_b200")
    exe = str(tmp_path / "gicp_main")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-I" + os.path.join(pkg, "cxx"), str(tmp_path / "main.cpp"), "-o", exe,
                        "-L" + pkg, "-lghicp_b200", "-Wl,-rpath," + pkg, "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([exe, str(tmp_path / "s.bin"), str(tmp_path / "t.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    lines = r.stdout.splitlines()
    assert any(x.startswith("GICP done in ") and x.endswith(" s") for x in lines)
    assert "The fitness score of this registration is " in r.stdout
    assert "-" * 77 in lines
    assert "The overlap ratio is too small. This registration would not be done." in r.stdout
    raw = np.fromfile(tmp_path / "out.bin", np.uint8)
    fit = np.frombuffer(raw[:8].tobytes(), np.float64)[0]
    m = np.frombuffer(raw[8:72].tobytes(), np.float32).reshape(4, 4).T
    moved = np.frombuffer(raw[72:].tobytes(), np.float32).reshape(-1, 3)
    Rt, info = g.gicp_reg(S, T, 20, True, True, 0.3, 20, 0.1)
    assert np.array_equal(m.astype(np.float64), Rt) and fit == info["fitness"] and np.array_equal(moved, info["moved"])
    assert g.gicp_reg(S, T, 20, False, True, 0.3, 20, 1.5) is None
