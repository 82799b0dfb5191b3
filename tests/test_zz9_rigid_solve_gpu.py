"""GPU tests of the float32 Umeyama solve (umeyama_from_moments_f32 -> svd3_f32, gh-icp_b200/csrc/ghicp_device.cuh) against a
float64 Kabsch, through every device entry point that reaches it: the stand-alone fits (k_solve<false>, k_solve_alt), the
in-loop solve (k_solve<true>, with more than 65536 keypoints so the full cooperative grid merges its per-CTA partials),
point-to-point cloud_icp on a million points in millimetres, and SAC-IA on a 60 000-point scene in millimetres.  The table of
cases and the checks live in tests/test_rigid_solve.py, which runs these functions on the emulated library with smaller
clouds."""
import numpy as np
import pytest

import icp_oracle as io
import sac_oracle as so
from test_rigid_solve import (CASES, check_case, check_pow2, check_rotation, kabsch, pose, rot_angle, solvers_capi,
                              translation_floor)

pytestmark = pytest.mark.gpu


def test_table_through_the_stand_alone_fits(g):
    """Every case of the table through ghicp_rigid_fit and ghicp_rigid_fit_ex (SVD and WEIGHTED_SVD)."""
    for name, fit in solvers_capi(g).items():
        for case in CASES:
            check_case(case, fit, name)


def test_power_of_two_scalings_through_the_stand_alone_fits(g):
    for name, fit in solvers_capi(g).items():
        check_pow2(fit, name)


def loop_scene(g, n):
    return g.synth.gen_points(n, n, overlap=0.9, extent=(100.0, 100.0, 20.0), noise=0.02, seed=21)


def test_loop_solve_equals_kabsch_on_its_pairs(g, n=70000, iterations=3):
    """The in-loop solve (NN correspondences, no feature) of each iteration against a float64 Kabsch on that iteration's own
    pairs and source, on a 100 m x 100 m x 20 m scene in metres and the same scene x 4096 (~4e5 units: beyond the range where
    the unscaled Jacobi sweep's alpha * beta stays finite)."""
    from ghicp_b200 import registration as reg_mod
    base = loop_scene(g, n)
    for f in (1.0, 4096.0):
        sc = loop_scene(g, n)
        sc.S, sc.T = np.asfortranarray(base.S * f), np.asfortranarray(base.T * f)
        sc.bbx_magnitude = base.bbx_magnitude * f
        reg = reg_mod.from_scene(sc, g.FT_NONE, g.CT_NN)
        try:
            for k in range(iterations):
                src = reg.source().copy()
                st = reg.iterate()
                sp, tp = reg.pairs()
                assert st.cor == len(sp) >= 3
                Rt = st.Rt_np()
                check_rotation(Rt[:3, :3], (f, k))
                A, B = src[sp], np.asarray(sc.T)[tp]
                Rk, tk = kabsch(A, B)
                assert rot_angle(Rt[:3, :3], Rk) < 1e-5, (f, k, rot_angle(Rt[:3, :3], Rk))
                assert np.abs(Rt[:3, 3] - tk).max() <= translation_floor(A, B), (f, k, Rt[:3, 3] - tk)
        finally:
            reg.close()


def box_clouds(n, seed, extent=(300.0, 300.0, 30.0)):
    """Target: n random points in a box (metres); source: the target moved by the inverse of a small motion with 1 cm of
    noise, so point-to-point ICP from the identity should return that motion."""
    rng = np.random.default_rng(seed)
    Q = rng.random((n, 3)) * np.asarray(extent)
    G = pose(0.02, [0.04, -0.03, 0.02])
    P = (Q - G[:3, 3]) @ G[:3, :3] + rng.normal(0.0, 0.01, Q.shape)
    return P, Q, G


def test_cloud_icp_in_millimetres(g, n_points=1000000, max_iterations=30):
    """Point-to-point cloud_icp on a 300 m x 300 m x 30 m box, in metres and in millimetres: a rotation both times, the same
    motion up to the scale, and within 1 mm / 1e-5 rad of the truth."""
    P, Q, G = box_clouds(n_points, 31)
    out = {}
    for f in (1.0, 1000.0):
        Rt, info = g.cloud_icp((P * f).astype(np.float32), (Q * f).astype(np.float32), max_iterations=max_iterations)
        check_rotation(Rt[:3, :3], f)
        assert rot_angle(Rt[:3, :3], G[:3, :3]) < 1e-5, (f, rot_angle(Rt[:3, :3], G[:3, :3]))
        assert np.abs(Rt[:3, 3] / f - G[:3, 3]).max() < 1e-3, (f, Rt[:3, 3] / f - G[:3, 3])
        out[f] = Rt
    assert rot_angle(out[1.0][:3, :3], out[1000.0][:3, :3]) < 1e-5


def sac_scene(g, n_points, n_kp, seed=4):
    """n_kp FPFH keypoints of each cloud of a synthetic scan pair spread over ~300 m x 200 m (metres)."""
    T, S, _, _ = g.synth.scan_pair(n_points, seed=seed, density=n_points / 60000.0)
    rng = np.random.default_rng(seed)
    out = []
    for X in (S, T):
        idx = np.sort(rng.choice(len(X), min(n_kp, len(X)), replace=False)).astype(np.int32)
        f, _, _ = g.fpfh_extract(X, idx)
        out += [X[idx], f]
    return out   # P, Fs, Q, Ft


def test_sac_ia_in_millimetres(g, n_points=60000, n_kp=2000, iterations=1000):
    """SAC-IA on the same keypoints and histograms in metres and in millimetres (thresholds scaled to match): both equal the
    oracle bit for bit, both results are rotations, and they pick the same hypothesis and the same motion up to the scale."""
    P, Fs, Q, Ft = sac_scene(g, n_points, n_kp)
    got = {}
    for f in (1.0, 1000.0):
        kw = dict(iterations=iterations, threshold=4.0 * f * f, min_sample_distance=2.0 * f, k=6)
        Pf, Qf = (P * np.float32(f)).astype(np.float32), (Q * np.float32(f)).astype(np.float32)
        Rt, info = g.sac_ia(Pf, Fs, Qf, Ft, **kw)
        o = so.sac(Pf, Fs, Qf, Ft, **kw)
        assert np.array_equal(Rt, o["Rt"]) and info["best_hypothesis"] == o["best"], f
        check_rotation(Rt[:3, :3], f)
        got[f] = (Rt, info)
    (a, ia), (b, ib) = got[1.0], got[1000.0]
    assert ia["best_hypothesis"] == ib["best_hypothesis"]
    assert rot_angle(a[:3, :3], b[:3, :3]) < 1e-5
    assert np.abs(b[:3, 3] / 1000.0 - a[:3, 3]).max() < 1e-3


def test_cloud_icp_steps_equal_kabsch_in_millimetres(g, n_points=200000, max_iterations=3):
    """Each step T_k of the oracle's ICP in millimetres, the same text as the kernels, against a float64 Kabsch on its pairs;
    the kernels' result equal to the oracle's bit for bit."""
    P, Q, _ = box_clouds(n_points, 32)
    P, Q = (P * 1000.0).astype(np.float32), (Q * 1000.0).astype(np.float32)
    Rt, _ = g.cloud_icp(P, Q, max_iterations=max_iterations)
    wRt, o = io.icp(P, Q, max_iterations=max_iterations, grid=True, steps=True)
    assert np.array_equal(Rt, wRt)
    W = P.astype(np.float64)
    for k in range(o["iterations"]):
        m = o["corr"][k] >= 0
        A, B = W[m], Q[o["corr"][k][m]].astype(np.float64)
        Rk, _ = kabsch(A, B)
        T = o["T"][k].astype(np.float64)
        check_rotation(T[:3, :3], k)
        assert rot_angle(Rk, T[:3, :3]) < 1e-5, (k, rot_angle(Rk, T[:3, :3]))
        W = io_move(W.astype(np.float32), o["T"][k]).astype(np.float64)


def io_move(A, T):
    A, T = np.asarray(A, np.float32), np.asarray(T, np.float32)
    return np.stack([((T[r, 0] * A[:, 0] + T[r, 1] * A[:, 1]) + T[r, 2] * A[:, 2]) + T[r, 3] for r in range(3)], axis=1)
