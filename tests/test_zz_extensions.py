"""GPU tests of the paths added last in round 1 (file name sorts last on purpose: these kernels were written after the
round's GPU budget was spent, so a failure here must not mask the verified suites under `pytest -x`):

  * matrix-free FPFH (gh-icp_b200/csrc/ghicp_fpfh.cu): must be BIT-IDENTICAL to the stored-plane kernels,
  * opt-in estimators (ghicp_solvers.cu): against the oracle's restatements (parity unpinned by the reference).
"""
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


# ---- matrix-free FPFH -------------------------------------------------------------------------------------------
def fpfh_scene(g, N, M, seed):
    return g.synth.add_fpfh(g.synth.gen_points(N, M, overlap=0.7, extent=(60, 60, 12), noise=0.03, seed=seed))


@pytest.mark.parametrize("N,M", [(100, 77), (33, 260), (257, 1000)])
def test_fpfh_matrix_free_fd_identical(g, orc, N, M):
    sc = fpfh_scene(g, N, M, N + M)
    mf = g.registration.from_scene(sc, g.FT_FPFH, g.CT_NN, fpfh_matrix_free=1)
    pl = g.registration.from_scene(sc, g.FT_FPFH, g.CT_NN, fpfh_matrix_free=-1)
    a, b = mf.fd(), pl.fd()
    assert np.array_equal(a, b)
    o = orc.Oracle(orc.FT_FPFH, orc.CT_NN, bbx_magnitude=sc.bbx_magnitude)
    o.set_keypoints(sc.S, sc.T); o.set_fpfh(sc.fpfh_s, sc.fpfh_t); o.build_fd()
    assert np.array_equal(a.astype(np.float32), o.fd().astype(np.float32))


@pytest.mark.parametrize("N,M", [(777, 1501), (300, 4500), (5, 3)])   # (300, 4500): two column chunks per row block
def test_fpfh_matrix_free_rowmin_identical(g, N, M):
    sc = fpfh_scene(g, N, M, 3 * N + M)
    mf = g.registration.from_scene(sc, g.FT_FPFH, g.CT_NN, fpfh_matrix_free=1)
    pl = g.registration.from_scene(sc, g.FT_FPFH, g.CT_NN, fpfh_matrix_free=-1)
    for it in (0, 1, 3):
        mf.set_state(it, 0.7, 0.5, 0.2, 1.0, 1.0)
        pl.set_state(it, 0.7, 0.5, 0.2, 1.0, 1.0)
        ia, ca, ma, sa, pa = mf.probe_rowmin()
        ib, cb, mb, sb, pb = pl.probe_rowmin()
        assert np.array_equal(ia, ib)
        assert np.array_equal(ca, cb)                      # same FD floats, same double arithmetic: identical bits
        assert ma == pytest.approx(mb, rel=1e-12)          # only the summation order of the statistics differs
        assert pa == pytest.approx(pb, rel=1e-12)


@pytest.mark.parametrize("Ct", ["nn", "nnr", "km"])
def test_fpfh_matrix_free_exact_loop_identical(g, Ct):
    """force_exact: the matrix-free sweeps with the all-double arithmetic == the stored-plane kernels, bit for bit."""
    N, M = (600, 500) if Ct != "km" else (220, 260)
    sc = fpfh_scene(g, N, M, 17)
    ct = {"nn": g.CT_NN, "nnr": g.CT_NNR, "km": g.CT_KM}[Ct]
    mf = g.registration.from_scene(sc, g.FT_FPFH, ct, fpfh_matrix_free=1, force_exact=True)
    pl = g.registration.from_scene(sc, g.FT_FPFH, ct, fpfh_matrix_free=-1)
    for it in range(12):
        a, b = mf.iterate(), pl.iterate()
        sp, tp = mf.pairs()
        osp, otp = pl.pairs()
        same = np.array_equal(sp, osp) and np.array_equal(tp, otp)
        if Ct == "km" and not same:
            # the CD mean (hence the penalty, hence every gain) may differ in its last bits between the two sweeps' reduction
            # orders (rel 1e-12 below); an eps-optimal matching is then free to differ: compare the objective and stop —
            # from here on the two loops are legitimately on different trajectories
            assert a.nnz == b.nnz and a.penalty == pytest.approx(b.penalty, rel=1e-12)
            assert abs(a.km_energy - b.km_energy) <= max(N, M) * 0.01 + 1e-6 * abs(b.km_energy)
            assert it >= 1                                             # iteration 0 has no geometry in the metric: identical
            break
        assert same, f"iteration {it}"
        assert np.array_equal(np.array(a.Rt), np.array(b.Rt))          # same pairs -> bit-identical solve
        assert a.fdm == b.fdm and a.fdstd == b.fdstd                   # FD of the pairs recomputed identically
        assert a.cd_mean == pytest.approx(b.cd_mean, rel=1e-12)
        assert a.stream_passes == 0
        if Ct == "km":
            assert a.nnz == b.nnz
        if a.converged:
            break


@pytest.mark.parametrize("Ct,N,M", [("nn", 600, 500), ("nnr", 600, 500), ("nnr", 2300, 1700), ("nnr", 40, 1500)])
def test_fpfh_fast_path_equals_exact_path(g, Ct, N, M):
    """FP32 filter + exact refinement (the default with fpfh_matrix_free=1) against the all-double stored-plane path:
    identical correspondence sets and transforms every iteration.  NN only takes the fast path from iteration 2 on (its
    penalty depends on the CD mean before that); the CD mean itself is the filter's estimate on fast iterations."""
    sc = fpfh_scene(g, N, M, 23)
    ct = {"nn": g.CT_NN, "nnr": g.CT_NNR}[Ct]
    fast = g.registration.from_scene(sc, g.FT_FPFH, ct, fpfh_matrix_free=1)
    slow = g.registration.from_scene(sc, g.FT_FPFH, ct, fpfh_matrix_free=-1)
    n_fast = 0
    for it in range(14):
        a, b = fast.iterate(), slow.iterate()
        sp, tp = fast.pairs()
        osp, otp = slow.pairs()
        assert np.array_equal(sp, osp) and np.array_equal(tp, otp), f"iteration {it}"
        assert np.array_equal(np.array(a.Rt), np.array(b.Rt))
        assert a.fdm == b.fdm and a.rmse == b.rmse
        assert a.exact_fallback == 0
        on_fast = Ct == "nnr" or it >= 2
        assert (a.stream_passes >= 1) == on_fast
        if on_fast:
            n_fast += 1
            assert a.candidates >= N                                   # at least the minimum of every row is refined
            assert a.candidates <= 8 * (N + M) + 64                    # ... and not much more than that
            # the CD mean is only an ESTIMATE here: ED / FD^ex is heavy-tailed (a handful of near-zero correlations carry
            # most of the sum) and no decision depends on it on these iterations
            assert 0.3 * b.cd_mean < a.cd_mean < 3.0 * b.cd_mean
        else:
            assert a.cd_mean == pytest.approx(b.cd_mean, rel=1e-12)
            assert a.penalty == pytest.approx(b.penalty, rel=1e-12)
        if a.converged:
            break
    assert n_fast >= 1


def test_fpfh_auto_mode_and_overrides(g, monkeypatch):
    sc = fpfh_scene(g, 64, 80, 5)
    auto = g.registration.from_scene(sc, g.FT_FPFH, g.CT_NNR)         # auto: NN / NNR go matrix-free + fast path
    plane = g.registration.from_scene(sc, g.FT_FPFH, g.CT_NNR, fpfh_matrix_free=-1)
    monkeypatch.setenv("GHICP_FPFH_EXACT", "1")                       # matrix-free, but the all-double sweeps
    exact = g.registration.from_scene(sc, g.FT_FPFH, g.CT_NNR)
    e = exact.iterate()
    monkeypatch.delenv("GHICP_FPFH_EXACT")
    a, b = auto.iterate(), plane.iterate()
    assert a.stream_passes >= 1 and b.stream_passes == 0 and e.stream_passes == 0
    for r in (auto, exact):
        assert np.array_equal(r.pairs()[0], plane.pairs()[0]) and np.array_equal(r.pairs()[1], plane.pairs()[1])
    assert np.array_equal(np.array(a.Rt), np.array(b.Rt)) and np.array_equal(np.array(e.Rt), np.array(b.Rt))
    assert e.cd_mean == pytest.approx(b.cd_mean, rel=1e-12)
    km = g.registration.from_scene(sc, g.FT_FPFH, g.CT_KM, fpfh_matrix_free=-1)   # the stored float plane
    km_mf = g.registration.from_scene(sc, g.FT_FPFH, g.CT_KM)                       # auto: matrix-free for KM as well
    x, y = km_mf.iterate(), km.iterate()
    assert x.nnz == y.nnz and abs(x.km_energy - y.km_energy) <= 80 * 0.01 + 1e-9 * abs(y.km_energy)


def test_fpfh_km_filter_gate_gives_the_exact_graph(g, monkeypatch):
    """FPFH + KM from iteration 2 on (penalty = RMS*para1*scale*para2): the FP32 filter with every row's threshold at the
    penalty + exact evaluation of its hits must produce the SAME candidate graph as the all-double sweeps, hence (same
    deterministic auction) the same matching and transform, iteration by iteration."""
    N, M = 700, 640
    sc = fpfh_scene(g, N, M, 21)
    fast = g.registration.from_scene(sc, g.FT_FPFH, g.CT_KM)
    monkeypatch.setenv("GHICP_FPFH_EXACT", "1")
    slow = g.registration.from_scene(sc, g.FT_FPFH, g.CT_KM)
    n_gate = 0
    for it in range(8):
        monkeypatch.delenv("GHICP_FPFH_EXACT", raising=False)
        a = fast.iterate()
        monkeypatch.setenv("GHICP_FPFH_EXACT", "1")
        b = slow.iterate()
        assert b.stream_passes == 0
        n_gate += 1 if a.stream_passes >= 1 else 0
        assert (a.nnz, a.cor) == (b.nnz, b.cor), it
        assert a.penalty == b.penalty
        assert a.km_energy == pytest.approx(b.km_energy, rel=1e-12)
        pa, pb = fast.pairs(), slow.pairs()
        assert np.array_equal(pa[0], pb[0]) and np.array_equal(pa[1], pb[1]), it
        assert np.array_equal(np.array(a.Rt), np.array(b.Rt)), it
        if a.converged:
            break
    assert n_gate >= 1, "the filter's KM gate was never taken"


# ---- opt-in estimators --------------------------------------------------------------------------------------------
def rot_zyx(rx, ry, rz):
    cx, sx, cy, sy, cz, sz = math.cos(rx), math.sin(rx), math.cos(ry), math.sin(ry), math.cos(rz), math.sin(rz)
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rz @ Ry @ Rx


def unit_normals(n, seed):
    v = np.random.default_rng(seed).normal(size=(n, 3))
    return v / np.linalg.norm(v, axis=1, keepdims=True)


@pytest.mark.parametrize("n", [3, 10, 1000, 50000])
def test_weighted_svd_unit_weights_bit_equal_to_rigid_fit(g, n):
    rng = np.random.default_rng(n)
    S = rng.random((n, 3)) * [100, 100, 20]
    T = S @ rot_zyx(0.01, -0.02, 0.04).T + [0.8, -1.2, 0.3] + rng.normal(0, 0.02, S.shape)
    a = g.rigid_fit(S, T)
    b, rc = g.rigid_fit_ex(S, T, g.SOLVER_WEIGHTED_SVD, weights=np.ones(n))
    c, _ = g.rigid_fit_ex(S, T, g.SOLVER_SVD)
    assert rc == 0
    assert np.array_equal(a, b) and np.array_equal(a, c)


@pytest.mark.parametrize("n", [40, 5000])
def test_estimators_match_oracle(g, orc, n):
    rng = np.random.default_rng(n + 1)
    S = rng.random((n, 3)) * [80, 60, 15]
    w = rng.random(n) + 0.1
    # weighted point-to-point (float32 SVD core on both sides: compare to the north-star tolerance, measured ~1e-7)
    T = S @ rot_zyx(0.01, -0.02, 0.04).T + [0.8, -1.2, 0.3] + rng.normal(0, 0.02, S.shape)
    a, _ = g.rigid_fit_ex(S, T, g.SOLVER_WEIGHTED_SVD, weights=w)
    b, _ = orc.rigid_fit_ex(S, T, 1, weights=w)
    assert g.synth.rot_angle(a[:3, :3], b[:3, :3]) < 1e-5 and np.linalg.norm(a[:3, 3] - b[:3, 3]) < 1e-4
    # point-to-plane (all double)
    Nn = unit_normals(n, n)
    T2 = S @ rot_zyx(0.004, -0.003, 0.006).T + [0.05, -0.03, 0.02]
    for weights in (None, w):
        a, rca = g.rigid_fit_ex(S, T2, g.SOLVER_POINT_TO_PLANE, normals=Nn, weights=weights)
        b, rcb = orc.rigid_fit_ex(S, T2, 2, normals=Nn, weights=weights)
        assert rca == 0 and rcb == 0
        assert np.allclose(a, b, atol=1e-9)
    # yaw-only
    T3 = S @ rot_zyx(0, 0, math.radians(11.0)).T + [1.5, -2.0, 0.4] + rng.normal(0, 0.03, S.shape)
    for weights in (None, w):
        a, rca = g.rigid_fit_ex(S, T3, g.SOLVER_YAW_4DOF, weights=weights)
        b, rcb = orc.rigid_fit_ex(S, T3, 3, weights=weights)
        assert rca == 0 and rcb == 0
        assert np.allclose(a, b, atol=1e-9)


def test_estimators_degenerate_and_errors(g):
    P = np.tile([[1.0, 2.0, 3.0]], (10, 1))
    Rt, rc = g.rigid_fit_ex(P, P, g.SOLVER_YAW_4DOF)
    assert rc == g.capi.GHICP_W_FEW_PAIRS and np.array_equal(Rt, np.eye(4))
    with pytest.raises(g.GhicpError):
        g.rigid_fit_ex(P, P, g.SOLVER_POINT_TO_PLANE)                 # normals missing
    sc = g.synth.config1(100, 100)
    with pytest.raises(g.GhicpError):
        g.registration.from_scene(sc, g.FT_NONE, g.CT_NN, solver=g.SOLVER_WEIGHTED_SVD)   # stand-alone only
    reg = g.registration.from_scene(sc, g.FT_NONE, g.CT_NN, solver=g.SOLVER_POINT_TO_PLANE)
    with pytest.raises(g.GhicpError):
        reg.iterate()                                                  # normals not set


@pytest.mark.parametrize("solver", ["yaw", "plane"])
def test_loop_with_opt_in_estimator_lockstep_with_oracle(g, orc, solver):
    if solver == "yaw":
        sc = g.synth.gen_points(900, 800, overlap=0.85, extent=(70, 70, 12), noise=0.01,
                                R_gt=g.synth.rot_xyz_deg(0, 0, 2.0), t_gt=(0.5, -0.4, 0.2), seed=8)
        kw, osolver, normals = dict(solver=g.SOLVER_YAW_4DOF), 3, None
    else:
        sc = g.synth.gen_points(900, 800, overlap=0.85, extent=(70, 70, 12), noise=0.01,
                                R_gt=g.synth.rot_xyz_deg(0.3, -0.2, 0.5), t_gt=(0.1, -0.1, 0.05), seed=9)
        normals = unit_normals(800, 4)
        kw, osolver = dict(solver=g.SOLVER_POINT_TO_PLANE, target_normals=normals), 2
    reg = g.registration.from_scene(sc, g.FT_NONE, g.CT_NN, max_iter=40, **kw)
    o = orc.Oracle(orc.FT_NONE, orc.CT_NN, bbx_magnitude=sc.bbx_magnitude, solve_mode=1, max_iter=40)
    o.set_keypoints(sc.S, sc.T)
    o.set_solver(osolver, normals)
    for it in range(40):
        a, b = reg.iterate(), o.iterate()
        sp, tp = reg.pairs()
        osp, otp = o.pairs()
        assert np.array_equal(sp, osp) and np.array_equal(tp, otp), f"iteration {it}"
        assert np.allclose(np.array(a.Rt), np.array(b.Rt), atol=1e-9)
        assert a.rmse_after == pytest.approx(b.rmse_after, rel=1e-7, abs=1e-10)
        if a.converged or b.converged:
            assert a.converged == b.converged
            break
    Ra = a.Rt_tillnow_np()
    if solver == "yaw":
        assert Ra[2, 2] == pytest.approx(1.0, abs=1e-15) and abs(Ra[0, 2]) < 1e-15


# ---- committed loop fixtures (tests/golden/loop_golden.npz) ------------------------------------------------------------
@pytest.mark.parametrize("name", ["none_nn", "none_nnr", "bsc_nn", "bsc_nnr", "bsc_km", "bsc_nn_dof4", "fpfh_nn", "fpfh_nnr"])
def test_cuda_path_reproduces_committed_loop_fixture(g, scratch_cwd, name):
    """The CUDA path against vectors committed to the repository (generated by the oracle in the build container, see
    tests/golden/make_loop_golden.py): identical correspondence lists every iteration for NN / NNR, transforms to the
    north-star tolerance; KM to the n*KM_eps energy bound (eps-optimal matchings are not unique)."""
    from test_oracle_golden import load_loop_case
    c = load_loop_case(name)
    ft, ct, dof, max_it, n_it = (int(v) for v in c["meta"])
    Kp = g.Keypoints().setCoordinate(c["S"], c["T"])
    if "bsc_s" in c:
        Kp.setBSCfeature(c["bsc_s"], c["bsc_t"], 441)
    if "fpfh_s" in c:
        Kp.setFPFHfeature(c["fpfh_s"], c["fpfh_t"])
    Ef = g.Energyfunction().init(Kp.kps_num, Kp.kpt_num, float(c["bbx"]))
    reg = g.GHRegistration(Kp, Ef, ft, ct, dof_type=dof, max_iter=max_it)
    n = max(Kp.kps_num, Kp.kpt_num)
    mismatched = 0
    for it in range(n_it):
        st = reg.iterate()
        b, e = c["off"][it], c["off"][it + 1]
        if ct == g.CT_KM:
            assert abs(st.km_energy - float(c["km_energy"][it])) <= n * 0.01 + 1e-6 * abs(float(c["km_energy"][it]))
            break   # later iterations depend on which eps-optimal matching was chosen
        sp, tp = reg.pairs()
        same = np.array_equal(sp, c["sp"][b:e]) and np.array_equal(tp, c["tp"][b:e])
        if ft == g.FT_FPFH and not same:
            mismatched += 1      # CUDA pow() vs glibc pow(): last-ulp differences of CD can flip an exact near-tie
            continue
        assert same, (name, it)
        assert np.allclose(np.array(st.Rt), c["Rt"][it], atol=1e-5)
    assert mismatched <= 1   # none observed on the stored-plane path (tests/test_gpu_parity.py allows the same)
    if ct != g.CT_KM and mismatched == 0:
        Ra, Rb = reg.Rt_tillnow(), np.array(c["Rt_final"]).reshape(4, 4).T
        assert g.synth.rot_angle(Ra[:3, :3], Rb[:3, :3]) < 1e-4 and np.linalg.norm(Ra[:3, 3] - Rb[:3, 3]) < 1e-3


# ---- the reference's own per-pair feature distances (tests/golden/feat_golden.npz) -------------------------------------
@pytest.mark.parametrize("bits", [441, 672, 9, 64, 2048])
def test_fd_bsc_equals_reference_hamming_fixture(g, bits):
    """The FD build (wgmma / POPC) against Hamming distances produced by the REFERENCE's own
    StereoBinaryFeature::hammingDistance (compiled verbatim in the build container, outputs committed)."""
    from test_oracle_golden import load_feat_golden
    z = load_feat_golden()
    S, T, H = z[f"bsc{bits}/S"], z[f"bsc{bits}/T"], z[f"bsc{bits}/H"]
    _, V, N, M = (int(v) for v in z[f"bsc{bits}/meta"])
    for dof, nv in ((6, 4), (4, 2)):
        if V < nv:
            continue
        Kp = g.Keypoints().setCoordinate(np.zeros((N, 3)), np.zeros((M, 3))).setBSCfeature(S, T, bits)
        reg = g.GHRegistration(Kp, g.Energyfunction().init(N, M, 10.0), g.FT_BSC, g.CT_NN, dof_type=dof)
        assert np.array_equal(reg.fd(), H[:nv].min(axis=0).astype(np.float64))


@pytest.mark.parametrize("mf", [1, -1])
def test_fd_fpfh_equals_reference_fixture(g, mf):
    from test_oracle_golden import load_feat_golden
    z = load_feat_golden()
    fs, ft, D = z["fpfh/S"], z["fpfh/T"], z["fpfh/D"]
    Kp = g.Keypoints().setCoordinate(np.zeros((len(fs), 3)), np.zeros((len(ft), 3))).setFPFHfeature(fs, ft)
    reg = g.GHRegistration(Kp, g.Energyfunction().init(len(fs), len(ft), 10.0), g.FT_FPFH, g.CT_NN, fpfh_matrix_free=mf)
    assert np.array_equal(reg.fd().astype(np.float32), D, equal_nan=True)
