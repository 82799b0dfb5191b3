"""GPU tests of the FPFH estimator over radius neighbourhoods (ghicp_prep.cu: prep_fpfh_radius; DESIGN.md §3.10, "Radius
neighbourhoods") through the C ABI against the oracle (tests/harness/fpfh_radius_oracle.cpp), of Prep.fpfh_radius /
register_clouds(fpfh_radius=...) and of coarsereg_fpfh_sac (CRegistration::Coarsereg_FPFHSAC) and its C++ mirror.  Normals and
status are bit-identical to the oracle; histograms meet §3.10's atan2 allowance (at most 1e-4 of them differ, each with
correlation >= 0.999).  tests/test_fpfh_radius.py runs these functions on the emulated library with smaller clouds."""
import os
import subprocess

import numpy as np
import pytest

import fpfh_radius_oracle as fro
import sac_oracle as so
from test_prep_oracle import scan_like_cloud

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def agree(got, want, what):
    diff = np.flatnonzero(~np.all(got == want, axis=1))
    assert len(diff) <= max(1e-4 * len(want), 0), f"{what}: {len(diff)} of {len(want)} histograms differ"
    for i in diff:
        assert np.corrcoef(got[i], want[i])[0, 1] >= 0.999, f"{what}: histogram {i}"


def radius_cloud(n, seed):
    """Scan-like, with duplicates and a far outlier; radii that give tens of neighbours per point."""
    P = scan_like_cloud(n, seed, extent=(20.0, 20.0, 5.0) if n < 30000 else (40.0, 40.0, 6.0))
    return np.concatenate([P, P[:5], np.float32([[300.0, -200.0, 50.0]])]).astype(np.float32)


RADII = {3000: (0.8, 1.6), 20000: (0.35, 0.7), 60000: (0.4, 0.6), 1500: (1.0, 2.0)}


@pytest.mark.parametrize("n,seed", [(3000, 1), (20000, 2), (60000, 3)])
def test_extract_equals_oracle(g, n, seed):
    P = radius_cloud(n, seed)
    rn, rf = RADII[n]
    want, wn, wst, _ = fro.fpfh(P, None, rn, rf)
    got, nrm, st = g.fpfh_extract_radius(P, normal_radius=rn, feature_radius=rf)
    assert np.array_equal(st, wst) and np.array_equal(nrm, wn, equal_nan=True)
    agree(got, want, f"n {n}")
    idx = np.random.default_rng(seed).choice(len(P), min(500, len(P)), replace=False).astype(np.int32)
    sub, snrm, sst = g.fpfh_extract_radius(P, idx, normal_radius=rn, feature_radius=rf)
    assert np.array_equal(sub, got[idx])
    done = sst != 2
    assert np.array_equal(snrm[done], nrm[done], equal_nan=True) and np.isnan(snrm[~done]).all()


def test_sample_of_indices_computes_only_what_it_needs(g, n_points=200000):
    """40 indices of a raw scan: the same rows as the whole-cloud call, with normals computed only around them."""
    T, _, _, _ = g.synth.scan_pair(n_points, seed=6)
    idx = np.random.default_rng(2).choice(len(T), 40, replace=False).astype(np.int32)
    rn, rf = 0.1, 0.2
    full, fn, fst = g.fpfh_extract_radius(T, normal_radius=rn, feature_radius=rf)
    sub, sn, sst = g.fpfh_extract_radius(T, idx, normal_radius=rn, feature_radius=rf)
    assert np.array_equal(sub, full[idx])
    done = sst != 2
    assert 0 < done.sum() < len(T) // 4 and (fst != 2).all()
    assert np.array_equal(sn[done], fn[done], equal_nan=True) and np.array_equal(sst[done], fst[done])
    want, wn, _, comp = fro.fpfh(T, idx[:4], rn, rf, all_normals=False)   # a few rows against the oracle as well
    agree(sub[:4], want, "200k scan")


def test_two_calls_are_identical(g, n=50000):
    P = radius_cloud(n, 8)
    a = g.fpfh_extract_radius(P, normal_radius=0.4, feature_radius=0.8)
    b = g.fpfh_extract_radius(P, normal_radius=0.4, feature_radius=0.8)
    for x, y in zip(a, b):
        assert np.array_equal(x, y, equal_nan=True)


def test_prep_fpfh_radius_equals_standalone_and_registers(g, n_points=60000):
    """Prep.fpfh_radius = the stand-alone call on the down-sampled cloud at the keypoints; set_from_prep then runs the loop in
    lock-step with the oracle's; register_clouds(fpfh_radius=...) converges with NNR and with KM."""
    import oracle
    oracle.build()
    T, S, R_gt, t_gt = g.synth.scan_pair(n_points, seed=4)
    res, nms, radii = 0.1, 1.2, (0.25, 0.5)
    pt, ps = g.Prep(T, res, 0.6, nms), g.Prep(S, res, 0.6, nms)
    try:
        for p in (pt, ps):
            ms = p.fpfh_radius(*radii)
            assert ms["total"] >= 0 and 0 < p.fpfh_work["spfh_points"] <= p.n_down
            assert p.fpfh_work["feature_entries"] > 0 and p.fpfh_work["normal_entries"] > 0
            kp, _ = p.keypoints()
            want, _, _ = g.fpfh_extract_radius(p.down(), kp, *radii)
            assert np.array_equal(p.get_fpfh(), want)
        fs, ft = ps.get_fpfh(), pt.get_fpfh()
        (skp, sxyz), (tkp, txyz) = ps.keypoints(), pt.keypoints()
        bbx = ps.bbx_magnitude
        Ef = g.Energyfunction().init(ps.n_kp, pt.n_kp, bbx)
        reg = g.GHRegistration((ps, pt), Ef, g.FT_FPFH, g.CT_NNR, nms, max_iter=60)
        o = oracle.Oracle(oracle.FT_FPFH, oracle.CT_NNR, bbx_magnitude=bbx, nonmax=nms, solve_mode=1, max_iter=60)
        o.set_keypoints(sxyz, txyz); o.set_fpfh(fs, ft); o.build_fd()
        for it in range(60):
            a, b = reg.iterate(), o.iterate()
            assert np.array_equal(reg.pairs()[0], o.pairs()[0]) and np.array_equal(reg.pairs()[1], o.pairs()[1]), it
            if a.converged or b.converged:
                break
        assert a.converged and b.converged
        Rt_step = reg.Rt_tillnow()
        reg.close()
    finally:
        pt.close(); ps.close()
    for ct in (g.CT_NNR, g.CT_KM):
        Rt, info = g.register_clouds(T, S, res, 0.6, nms, corr_type=ct, feature_type=g.FT_FPFH, max_iter=60, fpfh_radius=radii)
        assert info["fpfh_ms"]["source"]["total"] >= 0 and info["iterations"] < 60
        if ct == g.CT_NNR:
            assert np.allclose(Rt, Rt_step, atol=1e-12)
        assert np.isfinite(Rt).all() and abs(np.linalg.det(Rt[:3, :3]) - 1.0) < 1e-5


def down_pair(g, n_points, voxel, seed=4, R_gt=None):
    T, S, R, t = g.synth.scan_pair(n_points, seed=seed, R_gt=R_gt)
    return S[g.voxel_downsample(S, voxel)], T[g.voxel_downsample(T, voxel)], R


def test_coarsereg_equals_the_sac_oracle(g, n_points=60000, iterations=300, voxel=0.4):
    """coarsereg_fpfh_sac = sac_oracle on the same GPU histograms, bit for bit."""
    S, T, _ = down_pair(g, n_points, voxel)
    r = 2.0 * voxel
    Rt, info = g.coarsereg_fpfh_sac(S, T, r, sac=dict(iterations=iterations))
    fs, _, _ = g.fpfh_extract_radius(S, normal_radius=r, feature_radius=2 * r)
    ft, _, _ = g.fpfh_extract_radius(T, normal_radius=r, feature_radius=2 * r)
    o = so.sac(S, fs, T, ft, iterations=iterations, k=15, threshold=100.0)
    assert info["best_hypothesis"] == o["best"] and info["invalid_hypotheses"] == o["invalid"]
    assert np.array_equal(Rt, o["Rt"]) and info["error"] == o["error"] and info["fitness"] == o["fitness"]


CXX_MAIN = r"""
// CRegistration::Coarsereg_FPFHSAC (src/common_reg.cpp:393-423) on the C++ mirror
#include <cstdio>
#include <fstream>
#include "common_reg.h"
using namespace ghicp;
static Cloud read_xyz(const char *path) { std::ifstream f(path, std::ios::binary); Cloud c; float v[3];
  while (f.read((char *)v, sizeof(v))) c.push(v[0], v[1], v[2]); return c; }
int main(int argc, char **argv) {
  Cloud S = read_xyz(argv[1]), T = read_xyz(argv[2]), moved;
  CRegistration<float> reg;
  Matrix4f m;
  reg.Coarsereg_FPFHSAC(S, T, moved, m, (float)atof(argv[3]));
  std::ofstream out(argv[4], std::ios::binary);
  out.write((const char *)m.data(), 16 * sizeof(float));
  const double fit = reg.getFitnessScore();
  out.write((const char *)&fit, sizeof(fit));
  out.write((const char *)moved.xyz.data(), moved.xyz.size() * sizeof(float));
  return 0;
}
"""


def test_cxx_mirror_coarsereg_matches_python(g, tmp_path, n_points=60000, voxel=0.2):
    S, T, _ = down_pair(g, n_points, voxel, seed=5)
    r = 2.0 * voxel
    S.tofile(tmp_path / "s.bin"); T.tofile(tmp_path / "t.bin")
    (tmp_path / "main.cpp").write_text(CXX_MAIN)
    pkg = os.path.join(ROOT, "gh-icp_b200")
    exe = str(tmp_path / "coarse_main")
    c = subprocess.run(["g++", "-O2", "-std=c++17", "-I" + os.path.join(pkg, "cxx"), str(tmp_path / "main.cpp"), "-o", exe,
                        "-L" + pkg, "-lghicp_b200", "-Wl,-rpath," + pkg, "-L/usr/local/cuda/lib64", "-Wl,-rpath,/usr/local/cuda/lib64"],
                       capture_output=True, text=True)
    assert c.returncode == 0, c.stderr[-3000:]
    c = subprocess.run([exe, str(tmp_path / "s.bin"), str(tmp_path / "t.bin"), repr(float(np.float32(r))), str(tmp_path / "out.bin")],
                       capture_output=True, text=True)
    assert c.returncode == 0, c.stdout[-2000:] + c.stderr[-2000:]
    raw = np.fromfile(tmp_path / "out.bin", np.uint8)
    m = np.frombuffer(raw[:64].tobytes(), np.float32).reshape(4, 4).T
    fit = np.frombuffer(raw[64:72].tobytes(), np.float64)[0]
    moved = np.frombuffer(raw[72:].tobytes(), np.float32).reshape(-1, 3)
    want, info = g.coarsereg_fpfh_sac(S, T, float(np.float32(r)))
    assert np.array_equal(m, want.astype(np.float32)) and fit == info["fitness"]
    R, t = m[:3, :3], m[:3, 3]
    mv = np.stack([((R[k, 0] * S[:, 0] + R[k, 1] * S[:, 1]) + R[k, 2] * S[:, 2]) + t[k] for k in range(3)], axis=1)
    assert np.array_equal(moved, mv)


_ROWS = {}


def radius_rotation_rows(g, n_points=60000, pairs=((0.25, 0.5), (0.5, 1.0))):
    """The rotation rows of test_zz5_sac_gpu.rotation_rows (90 / 180-degree yaw pairs, FPFH, NNR / KM, register_clouds with
    initial_alignment="fpfh_sac" and its defaults) with the histograms of the radius estimator at each (normal, feature)
    radius pair: rotation error in degrees of SAC-IA alone and of SAC-IA + GH-ICP."""
    key = (n_points, pairs)
    if key in _ROWS:
        return _ROWS[key]
    from test_zz5_sac_gpu import yaw
    res, nbr, nms = 0.1, 0.6, 1.2
    rows = []
    for radii in pairs:
        for ct in (g.CT_NNR, g.CT_KM):
            for deg in (90.0, 180.0):
                T2, S2, R2, _ = g.synth.scan_pair(n_points, seed=4, R_gt=yaw(deg))
                Rs, info = g.register_clouds(T2, S2, res, nbr, nms, corr_type=ct, feature_type=g.FT_FPFH, max_iter=60,
                                             initial_alignment="fpfh_sac", fpfh_radius=radii)
                rows.append(dict(radii=radii, corr=int(ct), yaw=deg,
                                 sac_only=float(np.degrees(g.synth.rot_angle(info["sac"]["Rt"][:3, :3], R2))),
                                 with_sac=float(np.degrees(g.synth.rot_angle(Rs[:3, :3], R2))),
                                 sac_inliers=info["sac"]["inliers"]))
    print(rows)
    _ROWS[key] = rows
    return rows


@pytest.mark.xfail(strict=True, reason="finding: with radius histograms (0.25 / 0.5 m and 0.5 / 1.0 m on the 0.1 m voxel cloud) "
                   "SAC-IA no longer picks the aliased pose about 170 degrees off that the k = 20 histograms give, but it lands 9.6 "
                   "(90 deg) and 23.9 (180 deg) degrees off at 0.25 / 0.5 m and 23.5 / 33.3 degrees off at 0.5 / 1.0 m, and GH-ICP "
                   "from there ends 9.6 - 28.6 degrees off (H100, 1000 hypotheses, register_clouds' defaults).  Recorded, not tuned "
                   "away.")
def test_large_rotations_are_recovered_with_radius_histograms(g, n_points=60000):
    """test_zz5_sac_gpu.test_large_rotations_are_recovered with fpfh_radius: SAC-IA + GH-ICP ends within 1 degree of what the
    loop reaches from the 2-degree start of the default pair."""
    from test_zz5_sac_gpu import rotation_rows
    base = {r["corr"]: r["default_2deg"] for r in rotation_rows(g, n_points)}
    for r in radius_rotation_rows(g, n_points):
        assert r["with_sac"] <= base[r["corr"]] + 1.0, r
