"""CPU checks of SAC-IA (DESIGN.md §3.11).

  * the oracle (tests/harness/sac_oracle.cpp, one thread) against independent numpy / scipy restatements and an exact
    synthetic case;
  * the product's kernels (ghicp_sac.cu) run through the host emulation shim (tests/harness/sac_emu_harness.cpp) against the
    oracle, bit for bit: samples, correspondences, per-hypothesis transforms and integer errors, h*, fitness, invalid count;
  * the C ABI over the emulated kernels (tests/harness/emu_library.cpp): capi.sac_ia, Prep.sac_ia, set_initial_transform,
    register_clouds(initial_alignment="fpfh_sac"), and the `-m gpu` test functions of tests/test_zz5_sac_gpu.py on small
    clouds."""
import os
import subprocess
import sys

import numpy as np
import pytest
from scipy.spatial import cKDTree

import sac_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MASK64 = (1 << 64) - 1


def np_draw(seed, h, d):
    """SplitMix64 output h * 2^32 + d of the stream started at mix(seed) (ghicp_sac.h), in Python integers."""
    def mix(z):
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & MASK64
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & MASK64
        return z ^ (z >> 31)
    c = (h << 32) | d
    return mix((mix(seed) + (c + 1) * 0x9E3779B97F4A7C15) & MASK64)


def problem(n_s, n_t, seed, extent=20.0, noise=0.0, rot_deg=30.0):
    """Target: random points with random histograms; source: a rigid motion of a subset with the same histograms (+ noise)."""
    rng = np.random.default_rng(seed)
    Q = (rng.random((n_t, 3)) * np.float32(extent)).astype(np.float32)
    Ft = (rng.random((n_t, 33)) * 10).astype(np.float32)
    idx = rng.choice(n_t, min(n_s, n_t), replace=False) if n_s <= n_t else rng.integers(0, n_t, n_s)
    a = np.radians(rot_deg)
    R = np.array([[np.cos(a), -np.sin(a), 0], [np.sin(a), np.cos(a), 0], [0, 0, 1]]) @ \
        np.array([[1, 0, 0], [0, np.cos(a / 3), -np.sin(a / 3)], [0, np.sin(a / 3), np.cos(a / 3)]])
    t = np.array([1.5, -2.0, 0.5])
    P = ((Q[idx].astype(np.float64) - t) @ R + rng.normal(0, noise, (len(idx), 3))).astype(np.float32)   # R p + t = q
    return P, Ft[idx].copy(), Q, Ft, R, t


# ---- the oracle against numpy / scipy -----------------------------------------------------------------------------------
def test_draws_match_a_python_splitmix64():
    P, Fs, Q, Ft, _, _ = problem(50, 80, 1)
    o = so.sac(P, Fs, Q, Ft, iterations=20, k=1, threshold=1.0, seed=12345)
    for h in range(20):   # msd 0, 50 distinct points: the first draws that give new indices are the samples
        want, d = [], 0
        while len(want) < 3:
            c = ((np_draw(12345, h, d) >> 32) * 50) >> 32
            d += 1
            if c not in want:
                want.append(c)
        assert o["samples"][h].tolist() == want


@pytest.mark.parametrize("msd", [0.0, 3.0, 8.0])
def test_samples_are_distinct_and_far_enough(msd):
    P, Fs, Q, Ft, _, _ = problem(300, 400, 2)
    o = so.sac(P, Fs, Q, Ft, iterations=200, samples=4, min_sample_distance=msd, threshold=1.0)
    ok = o["valid"] == 1
    assert ok.any()
    for s in o["samples"][ok]:
        assert len(set(s.tolist())) == 4
        for i in range(4):
            for j in range(i):
                d = P[s[i]] - P[s[j]]
                assert np.sqrt(np.float32((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])) >= np.float32(msd)


def test_feature_knn_equals_numpy_bin_serial():
    rng = np.random.default_rng(3)
    Fs, Ft = (rng.random((40, 33)) * 5).astype(np.float32), (rng.random((500, 33)) * 5).astype(np.float32)
    Ft[7] = Ft[9]                                             # a tie: ascending index
    Fs[0] = Ft[9]
    d = np.zeros((40, 500), np.float32)
    for b in range(33):                                       # float32, bins in order, no fused operations
        t = Fs[:, None, b] - Ft[None, :, b]
        d = d + t * t
    want = np.argsort(d, axis=1, kind="stable")[:, :6]
    got = so.feat_knn(Fs, np.arange(40), Ft, 6)
    assert np.array_equal(got, want) and got[0, :2].tolist() == [7, 9]


@pytest.mark.parametrize("thr", [0.05, 1.0, 30.0])
def test_errors_match_ckdtree(thr):
    P, Fs, Q, Ft, _, _ = problem(400, 600, 4, noise=0.05)
    o = so.sac(P, Fs, Q, Ft, iterations=30, k=4, threshold=thr)
    tree = cKDTree(Q.astype(np.float64))
    for h in np.flatnonzero(o["valid"]):
        rt = o["rt"][h]
        R, t = rt[:9].reshape(3, 3), rt[9:]
        X = np.stack([((R[r, 0] * P[:, 0] + R[r, 1] * P[:, 1]) + R[r, 2] * P[:, 2]) + t[r] for r in range(3)], axis=1)
        dd, _ = tree.query(X.astype(np.float64))
        d2 = dd * dd
        want = np.where(d2 <= thr, d2 / thr, 1.0).sum()
        assert abs(o["err"][h] / 2.0 ** 32 - want) <= 1e-6 * max(want, 1.0), h
    assert o["error"] == o["err"][o["best"]] / 2.0 ** 32
    assert o["err"][o["best"]] == o["err"][o["valid"] == 1].min()


@pytest.mark.parametrize("rot", [10.0, 95.0, 180.0])
def test_exact_case_recovers_the_motion(rot):
    P, Fs, Q, Ft, R, t = problem(300, 500, 5, rot_deg=rot)
    o = so.sac(P, Fs, Q, Ft, iterations=20, k=1, threshold=0.01)
    assert o["invalid"] == 0 and o["inliers"] == len(P)
    assert np.abs(o["Rt"][:3, :3] - R).max() < 1e-5 and np.abs(o["Rt"][:3, 3] - t).max() < 1e-4
    assert o["error"] < 1e-6 and o["fitness"] < 1e-9


# ---- the kernels on the CPU (host emulation shim) -----------------------------------------------------------------------------
@pytest.fixture(scope="module")
def harness(tmp_path_factory):
    return so.build_emu_harness(tmp_path_factory.mktemp("sac_emu"))


def same(got, want):
    for k in ("samples", "valid", "corr", "rt", "err"):
        assert np.array_equal(got[k], want[k]), k
    for k in ("Rt", "error", "fitness", "inliers", "best", "invalid"):
        assert np.array_equal(got[k], want[k]), k


CASES = {
    "n1": (dict(n_s=1, n_t=1), dict(iterations=5)),
    "n2": (dict(n_s=2, n_t=2), dict(iterations=5)),
    "n3": (dict(n_s=3, n_t=3), dict(iterations=20, threshold=1.0)),
    "n17": (dict(n_s=17, n_t=17), dict(iterations=40, threshold=2.0, samples=5)),
    "n1000": (dict(n_s=1000, n_t=1000, noise=0.02), dict(iterations=60, threshold=0.5)),
    "n5000": (dict(n_s=5000, n_t=5000, extent=60.0, noise=0.02), dict(iterations=8, threshold=1.0)),
    "k_above_nt": (dict(n_s=40, n_t=12), dict(iterations=30, k=32, threshold=4.0)),
    "msd_rejects_all": (dict(n_s=200, n_t=300), dict(iterations=10, min_sample_distance=1e4)),
    "msd_some": (dict(n_s=200, n_t=300), dict(iterations=50, min_sample_distance=6.0, samples=8, k=3)),
    "tiny_thr": (dict(n_s=300, n_t=400, noise=0.05), dict(iterations=30, threshold=1e-6)),
    "huge_thr": (dict(n_s=300, n_t=400, noise=0.05), dict(iterations=30, threshold=1e7)),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_emulated_kernels_equal_the_oracle(harness, case):
    pk, kw = CASES[case]
    P, Fs, Q, Ft, _, _ = problem(seed=11, **pk)
    want = so.sac(P, Fs, Q, Ft, **kw)
    got = so.emu(harness, P, Fs, Q, Ft, **kw)
    same(got, want)
    if case in ("n1", "n2", "msd_rejects_all"):
        assert want["best"] == -1 and want["invalid"] == kw["iterations"] and np.array_equal(want["Rt"], np.eye(4))
    else:
        assert want["best"] >= 0


def test_identical_hypotheses_tie_to_the_smaller_index(harness):
    """Three source points only, k = 1 and identical histograms: every hypothesis draws the same set and fits the same
    transform, so all errors tie and h* must be 0."""
    P, Fs, Q, Ft, _, _ = problem(3, 3, 12)
    want = so.sac(P, Fs, Q, Ft, iterations=25, k=1, threshold=1.0)
    got = so.emu(harness, P, Fs, Q, Ft, iterations=25, k=1, threshold=1.0)
    same(got, want)
    assert len(set(want["err"].tolist())) == 1 and want["best"] == 0


def test_emulated_kernels_under_a_random_schedule(harness, tmp_path):
    """GHICP_EMU_SCHED: fibers visited in a fresh random order at every sweep (read once per process: a child process)."""
    P, Fs, Q, Ft, _, _ = problem(700, 800, 13, noise=0.03)
    np.savez(tmp_path / "in.npz", P=P, Fs=Fs, Q=Q, Ft=Ft)
    code = ("import sys, numpy as np; sys.path.insert(0, %r); import sac_oracle as so; a = np.load(%r);"
            "r = so.emu(%r, a['P'], a['Fs'], a['Q'], a['Ft'], iterations=40, threshold=0.5);"
            "np.savez(%r, **{k: np.asarray(v) for k, v in r.items()})"
            % (os.path.join(ROOT, "tests"), str(tmp_path / "in.npz"), harness, str(tmp_path / "out.npz")))
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, env=dict(os.environ, GHICP_EMU_SCHED="5"))
    assert r.returncode == 0, r.stderr[-3000:]
    got = dict(np.load(tmp_path / "out.npz"))
    same(got, so.sac(P, Fs, Q, Ft, iterations=40, threshold=0.5))


# ---- the C ABI over the emulated kernels --------------------------------------------------------------------------------------
@pytest.fixture()
def ge(g, emu_library_path):
    from conftest import swap_in_library
    real = swap_in_library(g, emu_library_path)
    try:
        yield g
    finally:
        g.capi._lib = real


def test_emulated_abi_sac_ia_and_bad_arguments(ge):
    g = ge
    P, Fs, Q, Ft, _, _ = problem(500, 600, 14, noise=0.02)
    kw = dict(iterations=40, samples=4, k=5, min_sample_distance=1.0, threshold=0.3, seed=9)
    Rt, info = g.sac_ia(P, Fs, Q, Ft, **kw)
    o = so.sac(P, Fs, Q, Ft, **kw)
    assert np.array_equal(Rt, o["Rt"]) and info["error"] == o["error"] and info["fitness"] == o["fitness"]
    assert (info["inliers"], info["best_hypothesis"], info["invalid_hypotheses"]) == (o["inliers"], o["best"], o["invalid"])
    for bad in (dict(iterations=0), dict(samples=2), dict(samples=9), dict(k=0), dict(k=33), dict(min_sample_distance=-1.0),
                dict(threshold=0.0), dict(threshold=float("inf"))):
        with pytest.raises(g.GhicpError) as e:
            g.sac_ia(P, Fs, Q, Ft, **bad)
        assert e.value.code == -1


def test_emulated_abi_prep_sac_ia_equals_the_oracle(ge):
    g = ge
    T, S, _, _ = g.synth.scan_pair(6000, seed=4)
    pt, ps = g.Prep(T, 0.3, 1.0, 1.5), g.Prep(S, 0.3, 1.0, 1.5)
    try:
        with pytest.raises(g.GhicpError):
            ps.sac_ia(pt)                                           # no histograms yet
        pt.fpfh(); ps.fpfh()
        Rt, info = ps.sac_ia(pt, iterations=30, threshold=2.25)
        (_, sxyz), (_, txyz) = ps.keypoints(), pt.keypoints()
        o = so.sac(sxyz.astype(np.float32), ps.get_fpfh(), txyz.astype(np.float32), pt.get_fpfh(), iterations=30, threshold=2.25)
        assert np.array_equal(Rt, o["Rt"]) and info["error"] == o["error"] and info["best_hypothesis"] == o["best"]
    finally:
        pt.close(); ps.close()


def k_apply(S, Rt):
    """the update k_apply runs on the source keypoints (double, ((R0 x + R1 y) + R2 z) + t)."""
    x, y, z = S[:, 0], S[:, 1], S[:, 2]
    return np.asfortranarray(np.stack([((Rt[r, 0] * x + Rt[r, 1] * y) + Rt[r, 2] * z) + Rt[r, 3] for r in range(3)], axis=1))


@pytest.mark.parametrize("ft,ct", [("NONE", "NN"), ("FPFH", "NNR"), ("FPFH", "KM")])
def test_emulated_abi_initial_transform_equals_premoved_source(ge, ft, ct):
    g = ge
    sc = g.synth.add_fpfh(g.synth.gen_points(300, 280, overlap=0.7, extent=(40, 40, 8), noise=0.03, seed=21))
    G = np.eye(4)
    G[:3, :3] = g.synth.rot_xyz_deg(1.0, -0.5, 3.0)
    G[:3, 3] = [0.3, -0.2, 0.1]
    Ft, Ct = getattr(g, "FT_" + ft), getattr(g, "CT_" + ct)
    a = g.registration.from_scene(sc, Ft, Ct)
    a.set_initial_transform(G)
    assert np.array_equal(a.Rt_tillnow(), G)
    b = g.registration.from_scene(sc, Ft, Ct)
    b.set_keypoints(k_apply(np.asarray(sc.S), G), sc.T)
    assert np.array_equal(a.source(), b.source())
    for it in range(4):
        sa, sb = a.iterate(), b.iterate()
        assert np.array_equal(a.pairs()[0], b.pairs()[0]) and np.array_equal(a.pairs()[1], b.pairs()[1]), it
        assert np.array_equal(sa.Rt_np(), sb.Rt_np())
    want = b.Rt_tillnow() @ G
    assert np.allclose(a.Rt_tillnow(), want, rtol=0, atol=1e-12)
    with pytest.raises(g.GhicpError) as e:
        a.set_initial_transform(G)                                  # after iteration 0
    assert e.value.code == -1
    a.close(); b.close()


def test_emulated_abi_register_clouds_with_sac(ge):
    g = ge
    T, S, R_gt, t_gt = g.synth.scan_pair(6000, seed=4)
    for ft in (g.FT_FPFH, g.FT_BSC):
        Rt, info = g.register_clouds(T, S, 0.3, 1.0, 1.5, corr_type=g.CT_NNR, feature_type=ft, max_iter=20,
                                     initial_alignment="fpfh_sac", sac=dict(iterations=40))
        assert "sac" in info and info["sac"]["best_hypothesis"] >= 0
        assert np.isfinite(Rt).all() and abs(np.linalg.det(Rt[:3, :3]) - 1.0) < 1e-5
    with pytest.raises(g.GhicpError):
        g.register_clouds(T, S, 0.3, 1.0, 1.5, initial_alignment="ransac")


@pytest.mark.parametrize("name,kw", [("test_keypoints_equal_oracle", dict(n_kp=300, iterations=30)),
                                     ("test_whole_cloud_equals_oracle", dict(n_points=3000, iterations=6)),
                                     ("test_two_calls_are_identical", dict(n_kp=300)),
                                     ("test_cxx_mirror_matches_python", dict(n_kp=200))])
def test_gpu_test_functions_on_the_emulated_library(ge, name, kw, tmp_path, emu_library_path, monkeypatch):
    import test_zz5_sac_gpu as t
    fn = getattr(t, name)
    if name == "test_cxx_mirror_matches_python":
        monkeypatch.setenv("LD_LIBRARY_PATH", os.path.dirname(emu_library_path) + os.pathsep + os.environ.get("LD_LIBRARY_PATH", ""))
        fn(ge, tmp_path, **kw)
    else:
        fn(ge, **kw)
