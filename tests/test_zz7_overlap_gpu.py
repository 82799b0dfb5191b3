"""GPU tests of the overlap and fitness evaluation (ghicp_overlap.cu, DESIGN.md §3.12) through the C ABI against the oracle
(tests/harness/overlap_oracle.cpp): d2 bit for bit, counts identical, sums within 1e-12 relative.  Also determinism,
Prep.overlap against the stand-alone call, the scores of known poses on the synthetic scan pairs, and the C++ mirror.
tests/test_overlap.py runs these functions on the emulated library with smaller clouds."""
import os
import subprocess

import numpy as np
import pytest

import overlap_oracle as oo

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def pose(deg, t):
    g = __import__("ghicp_b200")
    Rt = np.eye(4)
    Rt[:3, :3] = g.synth.rot_xyz_deg(0.3 * deg, -0.2 * deg, deg)
    Rt[:3, 3] = t
    return Rt


def same(got, want, d2=True):
    assert got["overlap"] == want["overlap"] and got["n_fit"] == want["n_fit"] and got["ratio"] == want["ratio"]
    for k in ("fitness", "overlap_rmse"):
        a, b = got[k], want[k]
        assert (np.isnan(a) and np.isnan(b)) or abs(a - b) <= 1e-12 * abs(b), (k, a, b)
    if d2:
        assert np.array_equal(got["d2"], want["d2"])


def scan_clouds(g, n_points, seed):
    T, S, _, _ = g.synth.scan_pair(n_points, seed=seed)
    return np.asarray(S, np.float32), np.asarray(T, np.float32)


def test_equals_oracle(g, n_points=60000, seeds=(1,)):
    for seed in seeds:
        S, T = scan_clouds(g, n_points, seed)
        for Rt, r, m in ((None, 0.1, float("inf")), (pose(2.0, [0.5, -0.3, 0.1]), 0.25, 4.0), (pose(30.0, [3, 1, 0]), 0.5, 0.01)):
            got = g.cloud_overlap(S, T, Rt, thre_dis=r, max_range=m, return_d2=True)
            same(got, oo.overlap(S, T, Rt, r, m))
            ov = g.cloud_overlap(S, T, Rt, thre_dis=r, max_range=m, fitness=False)
            assert ov["overlap"] == got["overlap"] and ov["ratio"] == got["ratio"] and ov["cells_visited"] <= got["cells_visited"]


def test_small_clouds_equal_oracle(g, n_points=3000):
    test_equals_oracle(g, n_points, seeds=(2, 3))


def test_million_points_equal_oracle_grid(g, n_points=1000000):
    S, T = scan_clouds(g, n_points, 5)
    Rt = pose(2.0, [0.5, -0.3, 0.1])
    got = g.cloud_overlap(S, T, Rt, thre_dis=0.1, return_d2=True)
    want = oo.overlap(S, T, Rt, 0.1, grid=True)
    same(got, want)
    print(dict(n=n_points, grid_ms=got["stage_ms"]["grid"], query_ms=got["stage_ms"]["queries"],
               cells_per_query=got["cells_visited"] / n_points, candidates_per_query=got["candidates"] / n_points))


def test_two_calls_are_identical(g, n_points=60000):
    S, T = scan_clouds(g, n_points, 6)
    Rt = pose(5.0, [1.0, 0.5, 0.0])
    a = g.cloud_overlap(S, T, Rt, thre_dis=0.2, return_d2=True)
    b = g.cloud_overlap(S, T, Rt, thre_dis=0.2, return_d2=True)
    assert np.array_equal(a.pop("d2"), b.pop("d2"))
    a.pop("stage_ms"); b.pop("stage_ms")
    assert a == b and np.float64(a["fitness"]).tobytes() == np.float64(b["fitness"]).tobytes()


def test_prep_overlap_equals_the_stand_alone_call(g, n_points=60000, res=0.1):
    T, S, _, _ = g.synth.scan_pair(n_points, seed=7)
    pt, ps = g.Prep(T, res, 0.6, 1.2), g.Prep(S, res, 0.6, 1.2)
    try:
        Rt = pose(2.0, [0.2, 0.1, 0.0])
        a = ps.overlap(pt, Rt, thre_dis=0.15, max_range=1.0)
        b = ps.overlap(pt, Rt, thre_dis=0.15, max_range=1.0)
        want = g.cloud_overlap(ps.down(), pt.down(), Rt, thre_dis=0.15, max_range=1.0)
        # the first call builds the target's grid, the second reuses it (event times are 0 on the emulated library)
        assert b["stage_ms"]["grid"] == 0 and (a["stage_ms"]["grid"] > 0 or a["stage_ms"]["total"] == 0)
        for x in (a, b):
            x = dict(x); x.pop("stage_ms")
            w = dict(want); w.pop("stage_ms")
            assert x == w
        c = ps.overlap(pt, None, thre_dis=0.3, fitness=False)
        assert c["overlap"] == g.cloud_overlap(ps.down(), pt.down(), None, thre_dis=0.3)["overlap"]
    finally:
        pt.close(); ps.close()


def yaw(deg):
    return np.asarray(__import__("ghicp_b200").synth.rot_xyz_deg(0.0, 0.0, deg))


def test_the_true_pose_scores_best(g, n_points=60000):
    """On the known-pose scan pairs of test_zz5_sac_gpu.py the ground-truth pose has the higher ratio and the lower fitness than
    the identity and than a 90 / 180-degree yaw start.  The fitness is taken within 1 m (max_range = 1 m^2): over every point
    it also averages the 40 % of the source the target never saw, which the true pose places beyond the target's end."""
    for deg in (None, 90.0, 180.0):
        if deg is None:
            T, S, R, t = g.synth.scan_pair(n_points, seed=4)
        else:
            T, S, R, t = g.synth.scan_pair(n_points, seed=4, R_gt=yaw(deg))
        G = np.eye(4)
        G[:3, :3], G[:3, 3] = R, t
        S_down, T_down = S[g.voxel_downsample(S, 0.1)], T[g.voxel_downsample(T, 0.1)]
        true = g.evaluate_registration(S_down, T_down, G, thre_dis=0.2, max_range=1.0)
        ident = g.evaluate_registration(S_down, T_down, np.eye(4), thre_dis=0.2, max_range=1.0)
        start = np.eye(4)
        start[:3, :3] = yaw(90.0 if deg is None else deg)
        wrong = g.evaluate_registration(S_down, T_down, start, thre_dis=0.2, max_range=1.0)
        print(dict(yaw=deg, true=(true["ratio"], true["fitness"]), identity=(ident["ratio"], ident["fitness"]),
                   start=(wrong["ratio"], wrong["fitness"])))
        for other in (ident, wrong):
            assert true["ratio"] > other["ratio"] and true["fitness"] < other["fitness"]
        assert g.cal_overlap(S_down, T_down, 0.2) == ident["ratio"]


CXX_MAIN = r"""
// CRegistration::calOverlap, transformcloud and invTransform of the C++ mirror
#include <fstream>
#include "common_reg.h"
using namespace ghicp;
static Cloud read_xyz(const char *path) { std::ifstream f(path, std::ios::binary); Cloud c; float v[3];
  while (f.read((char *)v, sizeof(v))) c.push(v[0], v[1], v[2]); return c; }
int main(int argc, char **argv) {
  Cloud A = read_xyz(argv[1]), B = read_xyz(argv[2]), moved;
  Matrix4f m, inv;
  std::ifstream mf(argv[3], std::ios::binary); mf.read((char *)m.data(), 16 * sizeof(float));
  CRegistration<> reg;
  reg.transformcloud(A, moved, m);
  const float ratio = reg.calOverlap(moved, B, 0.2f);
  reg.invTransform(m, inv);
  std::ofstream out(argv[4], std::ios::binary);
  out.write((const char *)&ratio, sizeof(ratio));
  out.write((const char *)inv.data(), 16 * sizeof(float));
  out.write((const char *)moved.xyz.data(), moved.xyz.size() * sizeof(float));
  return 0;
}
"""


def test_cxx_mirror_matches_python(g, tmp_path, n_points=20000):
    S, T = scan_clouds(g, n_points, 8)
    Rt = pose(3.0, [0.4, -0.2, 0.05]).astype(np.float32)
    S.tofile(tmp_path / "a.bin"); T.tofile(tmp_path / "b.bin")
    np.ascontiguousarray(Rt.T).tofile(tmp_path / "m.bin")   # column-major, as Matrix4f::data()
    (tmp_path / "main.cpp").write_text(CXX_MAIN)
    pkg = os.path.join(ROOT, "gh-icp_b200")
    exe = str(tmp_path / "overlap_main")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-I" + os.path.join(pkg, "cxx"), str(tmp_path / "main.cpp"), "-o", exe,
                        "-L" + pkg, "-lghicp_b200", "-Wl,-rpath," + pkg, "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([exe, str(tmp_path / "a.bin"), str(tmp_path / "b.bin"), str(tmp_path / "m.bin"), str(tmp_path / "out.bin")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "The estimated approximate overlap ratio of Cloud 1 is" in r.stdout and "Transform done ..." in r.stdout
    raw = np.fromfile(tmp_path / "out.bin", np.uint8)
    ratio = np.frombuffer(raw[:4].tobytes(), np.float32)[0]
    inv = np.frombuffer(raw[4:68].tobytes(), np.float32).reshape(4, 4).T
    moved = np.frombuffer(raw[68:].tobytes(), np.float32).reshape(-1, 3)
    assert np.array_equal(moved, oo.move(S, Rt.astype(np.float64)))
    assert ratio == np.float32(g.cal_overlap(moved, T, 0.2))
    assert ratio == np.float32(g.cloud_overlap(S, T, Rt.astype(np.float64), thre_dis=0.2)["ratio"])
    want = np.eye(4, dtype=np.float32)
    want[:3, :3] = Rt[:3, :3].T
    want[:3, 3] = -Rt[:3, 3]   # the reference's inverse negates the translation only
    assert np.array_equal(inv, want)
