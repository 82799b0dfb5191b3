"""The raw-cloud pre-processing on the device against the brute-force references of tests/test_prep_edges.py: organised scans
with non-finite rows, far outliers (one of them past int range in cell_coord, where the device's saturating float-to-int
conversion differs from the host's), large offsets, ties and degenerate clouds.  tests/test_prep_edges.py runs these
functions at small sizes on the emulated library."""
import os
import subprocess

import numpy as np
import pytest

import fpfh_oracle as fo
import fpfh_radius_oracle as fro
from test_prep_oracle import scan_like_cloud
from test_prep_edges import (VOXEL_CASES, KP_CASES, edge_cloud, with_nonfinite, check_voxel, check_keypoints,
                             check_fpfh_metamorphic, check_prep_metamorphic, check_far_fallbacks, check_bsc_nonfinite_keypoint)

pytestmark = pytest.mark.gpu


def test_voxel_filter(g, orc, n=60000):
    for kind, m, v in VOXEL_CASES:
        P = edge_cloud(kind, max(m, n // 4) if kind not in ("same", "line", "plane") else m, 31)
        check_voxel(g, orc, P, v)
        D, _ = with_nonfinite(P, 0.05, 32)
        check_voxel(g, orc, D, v)


def test_keypoints(g, orc, n=20000):
    for kind, m, r, nms in KP_CASES:
        P = edge_cloud(kind, max(m, n // 4) if kind not in ("same", "line", "plane") else m, 33)
        D, _ = with_nonfinite(P, 0.05, 34)
        for X in (P, D):
            kp, lam, curv, cnt = check_keypoints(g, X, r, nms)
            okp, olam, ocurv, ocnt = orc.detect_keypoints(X, r, 0.65, 20, nms)
            assert np.array_equal(cnt, ocnt) and np.array_equal(lam, olam) and np.array_equal(kp, okp), kind


def test_fpfh_metamorphic(g, orc, n=6000):
    for kind in ("scan", "offset", "triple", "patches"):
        check_fpfh_metamorphic(g, fo if n <= 6000 else None, fro if n <= 6000 else None, edge_cloud(kind, n, 35), 36)
    check_bsc_nonfinite_keypoint(g, edge_cloud("scan", n, 37), 38)


def test_prep_run(g, orc, n=200000):
    for kind in ("scan", "offset"):
        check_prep_metamorphic(g, edge_cloud(kind, n, 39), 40)
    P = edge_cloud("far", n, 41)
    check_far_fallbacks(g, P, max(n // 100, 1))


def test_far_outlier_1e10(g, orc, n=20000):
    """One point 1e10 m away: past int range in cell_coord at r = 1 m.  It stays a voxel of its own, has itself as its only
    neighbour, and changes nothing for the other points."""
    P = edge_cloud("far1e10", n, 42)
    far = n // 3
    check_voxel(g, orc, P, 0.25)
    kp, lam, curv, cnt = check_keypoints(g, P, 1.0, 1.2)
    assert cnt[far] == 1
    rest = np.delete(np.arange(n), far)
    kp0, lam0, curv0, cnt0 = g.detect_keypoints(P[rest], 1.0, 0.65, 20, 1.2)
    assert np.array_equal(cnt[rest], cnt0) and np.array_equal(lam[rest], lam0)
    assert np.array_equal(kp, rest[kp0])
    f, nrm, st = g.fpfh_extract_radius(P, normal_radius=0.6, feature_radius=1.0)
    f0, n0, s0 = g.fpfh_extract_radius(P[rest], normal_radius=0.6, feature_radius=1.0)
    assert np.array_equal(f[rest], f0) and np.array_equal(nrm[rest], n0, equal_nan=True) and st[far] == 1
    check_far_fallbacks(g, P, 1)


def test_pcd_with_nan_rows_end_to_end(g, orc, tmp_path, n=40000):
    """An organised scan's NaN and inf rows, kept in the .pcd files as cloud_io.h reads them, change no transform: ghicp_cli with
    BSC features and register_clouds with BSC, k-NN FPFH and radius FPFH features give on the files with those rows exactly
    what they give on the cleaned files."""
    from test_cli_io import CLI, ROOT, write_pcd
    assert subprocess.run(["make", "-C", os.path.join(ROOT, "gh-icp_b200", "cxx"), "ghicp_cli"], capture_output=True).returncode == 0
    s = float(np.sqrt(n / 40000.0))                       # the density of a 40 000-point, 20 m x 20 m scan at every size
    T = scan_like_cloud(n, 21, extent=(20.0 * s, 20.0 * s, 5.0))
    R = g.synth.rot_xyz_deg(0.5, -0.3, 1.5)
    S = ((T.astype(np.float64) - [0.3, -0.2, 0.1]) @ R).astype(np.float32)
    Tn, _ = with_nonfinite(T, 0.05, 50)
    Sn, _ = with_nonfinite(S, 0.05, 51)
    out = {}
    for name, (A, B) in (("clean", (T, S)), ("nan", (Tn, Sn))):
        ft, fs, fr = (str(tmp_path / f"{name}_{x}.pcd") for x in ("t", "s", "reg"))
        write_pcd(ft, A, True); write_pcd(fs, B, True)
        r = subprocess.run([CLI, ft, fs, fr, "B", "R", "0.25", "1.0", "1.2", "1.1", "0.1", "6", "0.5", "0"], capture_output=True,
                           text=True, cwd=str(tmp_path), env=dict(os.environ, GHICP_MAX_ITER="80"))
        assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
        out[name] = [np.loadtxt(fr + ".Rt.txt")]
        for kw in (dict(feature_type=g.FT_BSC), dict(feature_type=g.FT_FPFH), dict(feature_type=g.FT_FPFH, fpfh_radius=(0.6, 1.2))):
            out[name].append(g.register_clouds(A, B, 0.25, 1.0, 1.2, corr_type=g.CT_NNR, max_iter=80, **kw)[0])
    for a, b in zip(out["clean"], out["nan"]):
        assert np.all(np.isfinite(b)) and np.array_equal(a, b)
