"""GPU tests of SAC-IA (ghicp_sac.cu, DESIGN.md §3.11) through the C ABI against the oracle (tests/harness/sac_oracle.cpp), bit
for bit: transform, error, fitness, inliers, h*, invalid count.  Also determinism, the recovery of large rotations by
register_clouds(initial_alignment="fpfh_sac"), and the C++ mirror's fpfhalign.  tests/test_sac_ia.py runs these functions
on the emulated library with smaller clouds."""
import os
import subprocess

import numpy as np
import pytest

import sac_oracle as so

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def same_result(Rt, info, o):
    assert info["best_hypothesis"] == o["best"] and info["invalid_hypotheses"] == o["invalid"]
    assert np.array_equal(Rt, o["Rt"]), "the device's Umeyama (or a sample / correspondence) differs from the oracle's"
    assert info["error"] == o["error"] and info["inliers"] == o["inliers"] and info["fitness"] == o["fitness"]


def keypoint_clouds(g, n_kp, n_points=60000, seed=4):
    """n_kp points of each down-sampled synthetic scan with their FPFH histograms (k = 20 on the down-sampled cloud)."""
    T, S, _, _ = g.synth.scan_pair(n_points, seed=seed)
    out = []
    rng = np.random.default_rng(seed)
    for X in (S, T):
        D = X[g.voxel_downsample(X, 0.1)]
        idx = np.sort(rng.choice(len(D), min(n_kp, len(D)), replace=False)).astype(np.int32)
        f, _, _ = g.fpfh_extract(D, idx)
        out += [D[idx], f]
    return out   # P, Fs, Q, Ft


def test_keypoints_equal_oracle(g, n_kp=2000, iterations=1000):
    P, Fs, Q, Ft = keypoint_clouds(g, n_kp)
    for kw in (dict(threshold=1.44), dict(threshold=1.0, k=15, min_sample_distance=0.5, seed=3)):
        Rt, info = g.sac_ia(P, Fs, Q, Ft, iterations=iterations, **kw)
        same_result(Rt, info, so.sac(P, Fs, Q, Ft, iterations=iterations, **kw))
        assert info["best_hypothesis"] >= 0 and info["inliers"] > 0


def test_whole_cloud_equals_oracle(g, n_points=60000, iterations=200):
    T, S, _, _ = g.synth.scan_pair(n_points, seed=7)
    fs, _, _ = g.fpfh_extract(S)
    ft, _, _ = g.fpfh_extract(T)
    Rt, info = g.sac_ia(S, fs, T, ft, iterations=iterations, threshold=0.25)
    same_result(Rt, info, so.sac(S, fs, T, ft, iterations=iterations, threshold=0.25))


def test_two_calls_are_identical(g, n_kp=2000):
    P, Fs, Q, Ft = keypoint_clouds(g, n_kp, seed=5)
    a, ia = g.sac_ia(P, Fs, Q, Ft, threshold=1.44)
    b, ib = g.sac_ia(P, Fs, Q, Ft, threshold=1.44)
    assert np.array_equal(a, b)
    ia.pop("stage_ms"); ib.pop("stage_ms")
    assert ia == ib


def yaw(deg):
    return np.asarray(__import__("ghicp_b200").synth.rot_xyz_deg(0.0, 0.0, deg))


def register_without_sac(g, T, S, res, nbr, nms, ct, max_iter):
    """register_clouds' device pipeline, but the pose after max_iter iterations even when the loop has not converged (ghicp_run
    reports that as an error)."""
    pt, ps = g.Prep(T, res, nbr, nms), g.Prep(S, res, nbr, nms)
    try:
        pt.fpfh(); ps.fpfh()
        Ef = g.Energyfunction().init(ps.n_kp, pt.n_kp, ps.bbx_magnitude)
        reg = g.GHRegistration((ps, pt), Ef, g.FT_FPFH, ct, nms, max_iter=max_iter)
        Rt, _ = reg.ghicp_reg(track_matches=True)
        reg.close()
    finally:
        pt.close(); ps.close()
    return Rt


_ROWS = {}


def rotation_rows(g, n_points=60000):
    """Rotation error (degrees) of the default 2-degree pair and of 90 / 180-degree yaw pairs, with FPFH and NNR / KM: GH-ICP
    alone, SAC-IA alone and SAC-IA + GH-ICP (register_clouds(initial_alignment="fpfh_sac"), its defaults)."""
    if n_points in _ROWS:
        return _ROWS[n_points]
    res, nbr, nms = 0.1, 0.6, 1.2
    T, S, R_gt, _ = g.synth.scan_pair(n_points, seed=4)
    rows = []
    for ct in (g.CT_NNR, g.CT_KM):
        Rt, _ = g.register_clouds(T, S, res, nbr, nms, corr_type=ct, feature_type=g.FT_FPFH, max_iter=60)
        base = np.degrees(g.synth.rot_angle(Rt[:3, :3], R_gt))
        for deg in (90.0, 180.0):
            T2, S2, R2, _ = g.synth.scan_pair(n_points, seed=4, R_gt=yaw(deg))
            Rn = register_without_sac(g, T2, S2, res, nbr, nms, ct, 60)
            Rs, info = g.register_clouds(T2, S2, res, nbr, nms, corr_type=ct, feature_type=g.FT_FPFH, max_iter=60,
                                         initial_alignment="fpfh_sac")
            rows.append(dict(corr=int(ct), yaw=deg, default_2deg=float(base),
                             without_sac=float(np.degrees(g.synth.rot_angle(Rn[:3, :3], R2))),
                             sac_only=float(np.degrees(g.synth.rot_angle(info["sac"]["Rt"][:3, :3], R2))),
                             with_sac=float(np.degrees(g.synth.rot_angle(Rs[:3, :3], R2))), sac_inliers=info["sac"]["inliers"]))
    print(rows)
    _ROWS[n_points] = rows
    return rows


def test_large_rotations_need_the_coarse_stage(g, n_points=60000):
    """GH-ICP alone does not leave a 90 or 180 degree start."""
    for r in rotation_rows(g, n_points):
        assert r["without_sac"] > 20.0, r


@pytest.mark.xfail(strict=True, reason="finding: on this synthetic pair (about 110 keypoints per scan, scan_world's walls and "
                   "poles repeat along the axes) 1000 hypotheses with the NMS-radius-squared threshold choose a pose about 170 "
                   "degrees off (an aliased, nearly symmetric pose) on the 90 and the 180 degree pair; 10000 hypotheses land within 2 - 8 "
                   "degrees.  Recorded, not tuned away.")
def test_large_rotations_are_recovered(g, n_points=60000):
    """With SAC-IA first the loop ends as close to the ground truth as from the 2-degree start of the default pair (within 1
    degree).  scan_world repeats structures: a wrong, aliased pose picked by SAC-IA fails here."""
    for r in rotation_rows(g, n_points):
        assert r["with_sac"] <= r["default_2deg"] + 1.0, r


CXX_MAIN = r"""
// the reference's fpfhalign call (src/ghicp_reg.cpp:1643, include/fpfh.hpp:117-133) on the C++ mirror, then GH-ICP from it
#include <cstdio>
#include <fstream>
#include "fpfh_feature.h"
#include "ghicp_reg.h"
using namespace ghicp;
static Cloud read_xyz(const char *path) { std::ifstream f(path, std::ios::binary); Cloud c; float v[3];
  while (f.read((char *)v, sizeof(v))) c.push(v[0], v[1], v[2]); return c; }
static void read_fpfh(const char *path, fpfhFeaturePtr f) { std::ifstream in(path, std::ios::binary); FPFHSignature33 h;
  while (in.read((char *)h.histogram, sizeof(h.histogram))) f->points.push_back(h); }
int main(int argc, char **argv) {
  Cloud CloudS = read_xyz(argv[1]), CloudT = read_xyz(argv[2]), reg;
  fpfhFeaturePtr source_fpfh(new fpfhFeature), target_fpfh(new fpfhFeature);
  read_fpfh(argv[3], source_fpfh); read_fpfh(argv[4], target_fpfh);
  FPFHfeature<float> fpfh0(1.2);
  bool ok = fpfh0.fpfhalign(CloudS, CloudT, source_fpfh, target_fpfh, reg);
  std::ofstream out(argv[5], std::ios::binary);
  out.write((const char *)fpfh0.getFinalTransformation().data(), 16 * sizeof(double));
  const double fit = fpfh0.getFitnessScore();
  out.write((const char *)&fit, sizeof(fit));
  out.write((const char *)reg.xyz.data(), reg.xyz.size() * sizeof(float));
  return ok ? 0 : 1;
}
"""


def test_cxx_mirror_matches_python(g, tmp_path, n_kp=2000):
    P, Fs, Q, Ft = keypoint_clouds(g, n_kp, seed=6)
    for name, a in (("s.bin", P), ("t.bin", Q), ("fs.bin", Fs), ("ft.bin", Ft)):
        np.ascontiguousarray(a, np.float32).tofile(tmp_path / name)
    (tmp_path / "main.cpp").write_text(CXX_MAIN)
    pkg = os.path.join(ROOT, "gh-icp_b200")
    exe = str(tmp_path / "sac_main")
    r = subprocess.run(["g++", "-O2", "-std=c++17", "-I" + os.path.join(pkg, "cxx"), str(tmp_path / "main.cpp"), "-o", exe,
                        "-L" + pkg, "-lghicp_b200", "-Wl,-rpath," + pkg, "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64"],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    r = subprocess.run([exe] + [str(tmp_path / f) for f in ("s.bin", "t.bin", "fs.bin", "ft.bin", "out.bin")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    raw = np.fromfile(tmp_path / "out.bin", np.uint8)
    Rt = np.frombuffer(raw[:128].tobytes(), np.float64).reshape(4, 4).T
    fit = np.frombuffer(raw[128:136].tobytes(), np.float64)[0]
    moved = np.frombuffer(raw[136:].tobytes(), np.float32).reshape(-1, 3)
    want, info = g.sac_ia(P, Fs, Q, Ft, k=6, threshold=100.0)   # the reference's settings: randomness 6, PCL's defaults
    assert np.array_equal(Rt, want) and fit == info["fitness"]
    R, t = want[:3, :3].astype(np.float32), want[:3, 3].astype(np.float32)
    P = np.asarray(P, np.float32)
    mv = np.stack([((R[r, 0] * P[:, 0] + R[r, 1] * P[:, 1]) + R[r, 2] * P[:, 2]) + t[r] for r in range(3)], axis=1)
    assert np.array_equal(moved, mv)
