"""GPU parity tests proper: the CUDA path (through the C ABI) against the CPU oracle on the same
seeded inputs.  Bit-exact for integer / index work, stated tolerances for floating point."""
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ROT_TOL = 1e-4    # rad   (BASELINE.json north_star)
TRANS_TOL = 1e-3  # m


def make_pair(g, orc, scene, Ft, Ct, dof=6, solve_mode=1, **kw):
    reg = g.registration.from_scene(scene, Ft, Ct, dof=dof, **kw)
    kw = {k: v for k, v in kw.items() if k != "force_exact"}
    o = orc.Oracle(Ft, Ct, dof=dof, bbx_magnitude=scene.bbx_magnitude, solve_mode=solve_mode,
                   max_iter=kw.get("max_iter", 0))
    o.set_keypoints(scene.S, scene.T)
    if Ft == g.FT_BSC:
        o.set_bsc(scene.bsc_s, scene.bsc_t, scene.bits)
    elif Ft == g.FT_FPFH:
        o.set_fpfh(scene.fpfh_s, scene.fpfh_t)
    o.build_fd()
    return reg, o


# ---- one-time FD build ---------------------------------------------------------------------------
# 672 / 700 bits: wgmma kernel with a 256-row B tile; 1000 / 1400: 128 rows; 2048 (the fp16 plane's limit): 64 rows
@pytest.mark.parametrize("bits,V,dof", [(441, 4, 6), (672, 4, 6), (441, 2, 4), (64, 4, 6), (9, 2, 4), (672, 2, 4), (700, 4, 6),
                                        (1000, 4, 6), (1400, 2, 4), (2048, 4, 6)])
@pytest.mark.parametrize("N,M", [(257, 131), (64, 300)])
def test_fd_bsc_bit_exact(g, orc, bits, V, dof, N, M):
    sc = g.synth.add_bsc(g.synth.gen_points(N, M, seed=bits + N), bits=bits, V=V)
    reg, o = make_pair(g, orc, sc, g.FT_BSC, g.CT_NN, dof=dof)
    assert np.array_equal(reg.fd(), o.fd())


def test_fd_bsc_672_many_tiles_equals_popc_kernel(g, orc, monkeypatch):
    """672-bit descriptors at a size with many A tiles and several CTAs: the K-chunked tensor-core build against the oracle and
    against the XOR + POPC kernel (GHICP_FD_POPC=1)."""
    sc = g.synth.add_bsc(g.synth.gen_points(700, 1500, seed=672), bits=672, V=4)
    reg, o = make_pair(g, orc, sc, g.FT_BSC, g.CT_NN, dof=6)
    a = reg.fd()
    assert np.array_equal(a, o.fd())
    monkeypatch.setenv("GHICP_FD_POPC", "1")
    reg2 = g.registration.from_scene(sc, g.FT_BSC, g.CT_NN, dof=6)
    reg2.build_fd()
    assert np.array_equal(reg2.fd(), a)


@pytest.mark.parametrize("N,M", [(100, 77), (33, 260)])
def test_fd_fpfh_float_exact(g, orc, N, M):
    sc = g.synth.add_fpfh(g.synth.gen_points(N, M, seed=N))
    reg, o = make_pair(g, orc, sc, g.FT_FPFH, g.CT_NN)
    a, b = reg.fd(), o.fd()
    # same float32 operation order as include/fpfh.hpp:135-165 → identical floats
    assert np.array_equal(a.astype(np.float32), b.astype(np.float32))


# ---- cost build + row scan (single stage, identical inputs) -----------------------------------------
@pytest.mark.parametrize("Ft", ["none", "bsc", "fpfh"])
@pytest.mark.parametrize("N,M", [(2000, 2000), (777, 1501), (5, 3)])
def test_rowmin_identical_indices(g, orc, Ft, N, M):
    sc = g.synth.gen_points(N, M, seed=N + M)
    ft = {"none": g.FT_NONE, "bsc": g.FT_BSC, "fpfh": g.FT_FPFH}[Ft]
    if Ft == "bsc":
        g.synth.add_bsc(sc, bits=441, V=4)
    if Ft == "fpfh":
        g.synth.add_fpfh(sc)
    reg, o = make_pair(g, orc, sc, ft, g.CT_NN)
    for it in (0, 1, 3):
        reg.set_state(it, 0.7, 30.0, 8.0, 1.0, 1.0)
        o.set_state(it, 0.7, 30.0, 8.0, 1.0, 1.0)
        idx, cd, mean, std, pen = reg.probe_rowmin()
        st = o.iterate()  # advances the oracle; reset below
        CD = o.cd()
        ref_idx = np.argmin(CD, axis=1)  # first minimum, like the strict '<' scan (src/ghicp_reg.cpp:719)
        assert np.array_equal(idx, ref_idx.astype(np.int32))
        if Ft != "fpfh":
            assert np.array_equal(cd, CD[np.arange(N), ref_idx])  # bit-identical doubles
        else:
            assert np.allclose(cd, CD[np.arange(N), ref_idx], rtol=1e-13, atol=0)
        assert mean == pytest.approx(st.cd_mean, rel=1e-11)
        assert std == pytest.approx(st.cd_std, rel=1e-8, abs=1e-12)
        assert pen == pytest.approx(st.penalty, rel=1e-8)
        # restore the oracle's geometry for the next probe
        o.set_keypoints(sc.S, sc.T)
        if Ft == "bsc":
            o.set_bsc(sc.bsc_s, sc.bsc_t, sc.bits)
        if Ft == "fpfh":
            o.set_fpfh(sc.fpfh_s, sc.fpfh_t)
        o.build_fd()


# ---- rigid solve ------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [3, 10, 1000, 50000])
def test_rigid_fit(g, orc, n):
    rng = np.random.default_rng(n)
    S = rng.random((n, 3)) * [200, 200, 40]
    R = g.synth.rot_xyz_deg(1.0, -0.7, 3.0)
    T = S @ R.T + [0.8, -1.2, 0.3] + rng.normal(0, 0.05, (n, 3))
    a = g.rigid_fit(S, T)
    b1 = orc.rigid_fit(S, T, 1)
    b0 = orc.rigid_fit(S, T, 0)
    assert g.synth.rot_angle(a[:3, :3], b1[:3, :3]) < 1e-6 and np.linalg.norm(a[:3, 3] - b1[:3, 3]) < 1e-4
    assert g.synth.rot_angle(a[:3, :3], b0[:3, :3]) < ROT_TOL and np.linalg.norm(a[:3, 3] - b0[:3, 3]) < TRANS_TOL


# ---- full loop, NN (config 1) ----------------------------------------------------------------------
def run_lockstep(g, reg, o, max_it=80):
    """Iterate both; return per-iteration records."""
    recs = []
    for _ in range(max_it):
        a = reg.iterate()
        b = o.iterate()
        recs.append((a, b, reg.pairs(), o.pairs()))
        if a.converged or b.converged:
            break
    return recs


@pytest.mark.parametrize("force_exact", [False, True])
def test_config1_nn_identical_pairs_every_iteration(g, orc, force_exact):
    sc = g.synth.config1()  # 2k x 2k, NN, no feature, 6-DoF
    reg, o = make_pair(g, orc, sc, g.FT_NONE, g.CT_NN, solve_mode=1, force_exact=force_exact)
    # statistics: all-double kernels agree to summation order; the streaming path accumulates FP32 pair
    # values in FP64 (documented tolerance 1e-6; decisions inside that band fall back to the exact kernels)
    pen_tol = 1e-10 if force_exact else 1e-6
    recs = run_lockstep(g, reg, o)
    assert len(recs) >= 3
    for a, b, (sp, tp), (osp, otp) in recs:
        assert a.iteration == b.iteration
        assert a.cor == b.cor
        assert np.array_equal(sp, osp) and np.array_equal(tp, otp)
        assert a.penalty == pytest.approx(b.penalty, rel=pen_tol)
        assert a.rmse == pytest.approx(b.rmse, rel=1e-9)
    a, b = recs[-1][0], recs[-1][1]
    assert a.converged == b.converged == 1
    Ra, Rb = a.Rt_tillnow_np(), np.array(b.Rt_tillnow).reshape(4, 4).T
    assert g.synth.rot_angle(Ra[:3, :3], Rb[:3, :3]) < ROT_TOL
    assert np.linalg.norm(Ra[:3, 3] - Rb[:3, 3]) < TRANS_TOL


def test_config1_final_transform_vs_pcl_like_oracle(g, orc):
    """Against the float32-accumulating (PCL-like) oracle the final transform agrees to the north_star
    tolerance; iteration counts may differ by one (SURVEY.md §7.4-6)."""
    sc = g.synth.config1()
    reg = g.registration.from_scene(sc, g.FT_NONE, g.CT_NN, max_iter=100)
    Rt, it = reg.ghicp_reg()
    o = orc.Oracle(orc.FT_NONE, orc.CT_NN, bbx_magnitude=sc.bbx_magnitude, solve_mode=0, max_iter=100)
    o.set_keypoints(sc.S, sc.T)
    Ro, ito, rc = o.run()
    assert rc == 0 and abs(it - ito) <= 1
    assert g.synth.rot_angle(Rt[:3, :3], Ro[:3, :3]) < ROT_TOL
    assert np.linalg.norm(Rt[:3, 3] - Ro[:3, 3]) < TRANS_TOL


@pytest.mark.parametrize("Ft,Ct", [("bsc", "nn"), ("bsc", "nnr"), ("none", "nnr"), ("fpfh", "nn"), ("fpfh", "nnr")])
def test_loop_nn_nnr_features(g, orc, Ft, Ct):
    sc = g.synth.gen_points(600, 500, overlap=0.7, extent=(60, 60, 12), noise=0.03, seed=17)
    ft = {"none": g.FT_NONE, "bsc": g.FT_BSC, "fpfh": g.FT_FPFH}[Ft]
    ct = {"nn": g.CT_NN, "nnr": g.CT_NNR}[Ct]
    if Ft == "bsc":
        g.synth.add_bsc(sc, bits=441, V=4)
    if Ft == "fpfh":
        g.synth.add_fpfh(sc)
    reg, o = make_pair(g, orc, sc, ft, ct, solve_mode=1)
    recs = run_lockstep(g, reg, o, max_it=40)
    n_mismatch = 0
    for a, b, (sp, tp), (osp, otp) in recs:
        if not (np.array_equal(sp, osp) and np.array_equal(tp, otp)):
            n_mismatch += 1
    if Ft == "fpfh":
        assert n_mismatch <= 1  # pow() differs in the last ulp between CUDA and glibc
    else:
        assert n_mismatch == 0
    a, b = recs[-1][0], recs[-1][1]
    Ra, Rb = a.Rt_tillnow_np(), np.array(b.Rt_tillnow).reshape(4, 4).T
    assert g.synth.rot_angle(Ra[:3, :3], Rb[:3, :3]) < ROT_TOL
    assert np.linalg.norm(Ra[:3, 3] - Rb[:3, 3]) < TRANS_TOL


# ---- streaming (FP32 filter + FP64 refine) path against the all-double kernels ---------------------------
@pytest.mark.parametrize("Ft", ["none", "bsc"])
@pytest.mark.parametrize("Ct", ["nn", "nnr"])
def test_streaming_path_equals_all_double_path(g, Ft, Ct):
    N, M = 5000, 4309  # ragged: partial column panels, partial row blocks
    sc = g.synth.gen_points(N, M, overlap=0.6, extent=(90, 90, 18), noise=0.04, seed=23)
    ft = {"none": g.FT_NONE, "bsc": g.FT_BSC}[Ft]
    ct = {"nn": g.CT_NN, "nnr": g.CT_NNR}[Ct]
    if Ft == "bsc":
        g.synth.add_bsc(sc, bits=441, V=4)
    fast = g.registration.from_scene(sc, ft, ct)
    slow = g.registration.from_scene(sc, ft, ct, force_exact=True)
    n_fallback = 0
    for it in range(8):
        a, b = fast.iterate(), slow.iterate()
        n_fallback += a.exact_fallback
        assert b.exact_fallback == 0
        sp, tp = fast.pairs()
        osp, otp = slow.pairs()
        assert np.array_equal(sp, osp) and np.array_equal(tp, otp), f"iteration {it}"
        assert a.cd_mean == pytest.approx(b.cd_mean, rel=2e-6)
        assert a.penalty == pytest.approx(b.penalty, rel=1e-5)
        assert np.array_equal(np.array(a.Rt), np.array(b.Rt))  # same pairs -> bit-identical solve
        if a.converged:
            break
    assert n_fallback <= 2


def test_streaming_path_km_candidates(g):
    N, M = 3000, 3300
    sc = g.synth.add_bsc(g.synth.gen_points(N, M, overlap=0.6, extent=(80, 80, 16), noise=0.04, seed=29), bits=441, V=4)
    fast = g.registration.from_scene(sc, g.FT_BSC, g.CT_KM)
    slow = g.registration.from_scene(sc, g.FT_BSC, g.CT_KM, force_exact=True)
    for it in range(5):
        a, b = fast.iterate(), slow.iterate()
        assert a.penalty == pytest.approx(b.penalty, rel=1e-5)
        assert abs(a.nnz - b.nnz) <= max(2, 1e-4 * b.nnz)   # gate flips only inside the statistics error band
        assert abs(a.km_energy - b.km_energy) <= max(N, M) * 0.01 + 1e-6 * abs(b.km_energy)
        # keep the trajectories together (eps-optimal matchings are not unique)
        slow.set_keypoints(fast.source(), sc.T)
        slow.set_state(a.iteration + 1, a.rmse, a.fdm, a.fdstd, a.para1, a.para2)


def test_km_edge_list_equals_fill_pass(g, monkeypatch):
    """The KM count pass appends its gate hits to an edge list (one stream over the plane); the two-pass
    count + fill route is the overflow fallback.  Both must give the same graph and the same matching."""
    N, M = 2500, 2100
    sc = g.synth.add_bsc(g.synth.gen_points(N, M, overlap=0.6, extent=(70, 70, 14), noise=0.04, seed=31), bits=441, V=4)
    one = g.registration.from_scene(sc, g.FT_BSC, g.CT_KM)
    monkeypatch.setenv("GHICP_KM_FILL", "1")
    two = g.registration.from_scene(sc, g.FT_BSC, g.CT_KM)
    for it in range(6):
        monkeypatch.delenv("GHICP_KM_FILL", raising=False)
        a = one.iterate()
        monkeypatch.setenv("GHICP_KM_FILL", "1")
        b = two.iterate()
        # the list is switched on from the previous iteration's edge count (off while the graph is dense)
        assert b.stream_passes - a.stream_passes in (0, 1)
        saved = b.stream_passes - a.stream_passes
        assert (a.nnz, a.cor, a.penalty) == (b.nnz, b.cor, b.penalty)
        assert a.km_energy == b.km_energy
        pa, pb = one.pairs(), two.pairs()
        assert np.array_equal(pa[0], pb[0]) and np.array_equal(pa[1], pb[1])
        assert np.array_equal(one.source(), two.source())
    assert saved == 1   # a settled loop streams the plane once per iteration


# ---- KM -----------------------------------------------------------------------------------------------
def test_km_golden_g1_g2(g, orc):
    from golden_vectors import G1_W, G2_CD
    m, e, _ = g.km_solve(G1_W, eps=0.01, penalty=1000.0)
    assert m.tolist() == [0, 2, 1]
    G = orc.km_graph(G2_CD, 30.0)
    m, e, _ = g.km_solve(G, sp=7, tp=6, eps=0.01, penalty=30.0)
    kept = [(int(m[y]), y) for y in range(7) if m[y] >= 0]
    # E_min = 106 is attained by exactly two matchings (brute force): the figure's / the reference DFS's
    # {S6-T2, S2-T4} and its mirror {S2-T2, S6-T4}; an eps-optimal solver may return either.
    assert kept in ([(0, 0), (1, 1), (6, 2), (4, 3), (2, 4)], [(0, 0), (1, 1), (2, 2), (4, 3), (6, 4)])
    assert e == 106.0


@pytest.mark.parametrize("n,m,pen,seed", [(60, 60, 20.0, 0), (300, 250, 12.0, 1), (200, 320, 25.0, 2), (1000, 1000, 6.0, 3)])
def test_km_within_n_eps_of_optimum_and_reference(g, orc, scratch_cwd, n, m, pen, seed):
    from scipy.optimize import linear_sum_assignment
    rng = np.random.default_rng(seed)
    CD = rng.random((n, m)) * 50.0
    G = orc.km_graph(CD, pen)
    size = max(n, m)
    eps = 0.01
    match, energy, rounds = g.km_solve(G, sp=n, tp=m, eps=eps, penalty=pen)
    # valid partial matching on candidate edges only
    used = [x for x in match if x >= 0]
    assert len(used) == len(set(used))
    for y, x in enumerate(match):
        if x >= 0:
            assert CD[x, y] < pen
    r, c = linear_sum_assignment(-G)
    e_opt = -G[r, c].sum()
    assert energy >= e_opt - 1e-9
    assert energy <= e_opt + size * eps
    mo = orc.km_solve(G, eps, "port")
    _, _, _, _, e_ref = orc.km_output(G, n, m, pen, mo)
    assert abs(energy - e_ref) <= size * eps


def test_km_integer_costs_with_ties(g, orc, scratch_cwd):
    """Iteration 0 of BSC mode has CD = FD exactly (integers): masses of ties."""
    from scipy.optimize import linear_sum_assignment
    rng = np.random.default_rng(9)
    CD = rng.integers(150, 230, size=(400, 400)).astype(np.float64)
    pen = 171.3
    G = orc.km_graph(CD, pen)
    match, energy, rounds = g.km_solve(G, sp=400, tp=400, eps=0.01, penalty=pen)
    r, c = linear_sum_assignment(-G)
    e_opt = -G[r, c].sum()
    assert e_opt - 1e-9 <= energy <= e_opt + 400 * 0.01


@pytest.mark.parametrize("N,M", [(300, 300), (260, 340)])
def test_loop_km_bsc(g, orc, scratch_cwd, N, M):
    sc = g.synth.add_bsc(g.synth.gen_points(N, M, overlap=0.6, extent=(40, 40, 8), noise=0.03, seed=5), bits=441, V=4)
    reg, o = make_pair(g, orc, sc, g.FT_BSC, g.CT_KM, solve_mode=1, max_iter=40)
    n = max(N, M)
    for _ in range(40):
        a = reg.iterate()
        b = o.iterate()
        # same penalty rule input → same candidate graph; energies within n*KM_eps
        assert a.penalty == pytest.approx(b.penalty, rel=1e-6)
        assert abs(a.km_energy - b.km_energy) <= n * 0.01 + 1e-6 * abs(b.km_energy)
        if a.converged or b.converged:
            break
        # keep the two loops on the same trajectory: eps-optimal matchings are not unique
        S = reg.source()
        o.set_keypoints(S, sc.T)
        o.set_bsc(sc.bsc_s, sc.bsc_t, sc.bits)
        o.build_fd()
        o.set_state(a.iteration + 1, a.rmse, a.fdm, a.fdstd, a.para1, a.para2)
    Rt = reg.Rt_tillnow()
    assert g.synth.rot_angle(Rt[:3, :3], sc.R_gt) < 5e-3  # registration succeeded


def test_error_paths(g):
    sc = g.synth.gen_points(50, 40, seed=1)
    reg = g.registration.from_scene(sc, g.FT_NONE, g.CT_NN)
    reg.close()
    Kp = g.Keypoints().setCoordinate(sc.S, sc.T)
    Ef = g.Energyfunction().init(50, 40, sc.bbx_magnitude)
    with pytest.raises(g.GhicpError):
        g.GHRegistration(Kp, Ef, 1, g.CT_NN)  # RoPS: "Not passed yet" in the reference


# ---- ragged / tiny shapes (partial column panels, partial row blocks, fewer than 3 pairs) ----------------
@pytest.mark.parametrize("N,M", [(1, 1), (2, 5), (3, 700), (700, 3), (257, 255), (513, 2049)])
@pytest.mark.parametrize("Ft,Ct", [("none", "nn"), ("bsc", "nn"), ("bsc", "nnr"), ("bsc", "km")])
def test_ragged_and_tiny_shapes(g, orc, scratch_cwd, N, M, Ft, Ct):
    sc = g.synth.gen_points(N, M, overlap=0.7, extent=(20, 20, 4), noise=0.02, seed=N * 7 + M)
    ft = {"none": g.FT_NONE, "bsc": g.FT_BSC}[Ft]
    ct = {"nn": g.CT_NN, "nnr": g.CT_NNR, "km": g.CT_KM}[Ct]
    if Ft == "bsc":
        g.synth.add_bsc(sc, bits=441, V=4)
    reg, o = make_pair(g, orc, sc, ft, ct, solve_mode=1)
    for it in range(3):
        a, b = reg.iterate(), o.iterate()
        assert a.penalty == pytest.approx(b.penalty, rel=1e-6, nan_ok=True)
        if ct != g.CT_KM:
            sp, tp = reg.pairs()
            osp, otp = o.pairs()
            assert np.array_equal(sp, osp) and np.array_equal(tp, otp), (it, N, M)
            assert np.allclose(np.array(a.Rt), np.array(b.Rt), atol=1e-5)
        else:
            assert abs(a.km_energy - b.km_energy) <= max(N, M) * 0.01 + 1e-6 * abs(b.km_energy)
            o.set_keypoints(reg.source(), sc.T)
            o.set_bsc(sc.bsc_s, sc.bsc_t, sc.bits)
            o.build_fd()
            o.set_state(a.iteration + 1, a.rmse, a.fdm, a.fdstd, a.para1, a.para2)
        if a.converged or b.converged:
            break


def test_dof4_two_variants_loop(g, orc):
    """dof != 6 uses only the first two BSC source variants (src/ghicp_reg.cpp:181-182)."""
    sc = g.synth.add_bsc(g.synth.gen_points(500, 450, overlap=0.7, extent=(50, 50, 10), noise=0.03, seed=77), bits=441, V=4)
    reg, o = make_pair(g, orc, sc, g.FT_BSC, g.CT_NN, dof=4, solve_mode=1)
    assert np.array_equal(reg.fd(), o.fd())
    for _ in range(4):
        a, b = reg.iterate(), o.iterate()
        sp, tp = reg.pairs()
        osp, otp = o.pairs()
        assert np.array_equal(sp, osp) and np.array_equal(tp, otp)


def test_bsc_672_bits_loop(g, orc):
    """BASELINE.json names 672-bit BSC; 672 bits take the tensor-core FD kernel with its widest B tile."""
    sc = g.synth.add_bsc(g.synth.gen_points(400, 420, overlap=0.7, extent=(50, 50, 10), noise=0.03, seed=78), bits=672, V=4)
    reg, o = make_pair(g, orc, sc, g.FT_BSC, g.CT_NNR, solve_mode=1)
    assert np.array_equal(reg.fd(), o.fd())
    for _ in range(4):
        a, b = reg.iterate(), o.iterate()
        sp, tp = reg.pairs()
        osp, otp = o.pairs()
        assert np.array_equal(sp, osp) and np.array_equal(tp, otp)


def test_page_locked_caller_buffers_give_identical_results(g):
    """ghicp_host_alloc: coordinates uploaded from and results read into page-locked caller buffers (one DMA each, no staging
    copy inside the library) — same pairs, same transform, same updated source as with pageable numpy arrays."""
    sc = g.synth.add_bsc(g.synth.gen_points(900, 1100, overlap=0.6, extent=(50, 50, 10), noise=0.04, seed=77), bits=441, V=4)
    a = g.registration.from_scene(sc, g.FT_BSC, g.CT_NN)
    b = g.registration.from_scene(sc, g.FT_BSC, g.CT_NN)
    S_pin = g.capi.pinned_copy(np.asfortranarray(sc.S, dtype=np.float64), order="F")
    T_pin = g.capi.pinned_copy(np.asfortranarray(sc.T, dtype=np.float64), order="F")
    sp_buf = g.capi.pinned_empty(1100, np.int32)
    tp_buf = g.capi.pinned_empty(1100, np.int32)
    S_a = np.asfortranarray(sc.S, dtype=np.float64)
    for it in range(4):
        a.set_keypoints(S_a, np.asfortranarray(sc.T, dtype=np.float64))
        b.set_keypoints(S_pin, T_pin)
        sa, sb = a.iterate(), b.iterate()
        assert np.array_equal(np.array(sa.Rt), np.array(sb.Rt)) and sa.cor == sb.cor
        pa = a.pairs()
        pb = b.pairs(out=(sp_buf, tp_buf))
        assert np.array_equal(pa[0], pb[0]) and np.array_equal(pa[1], pb[1])
        S_a = a.source()
        b.source(out=S_pin)
        assert np.array_equal(S_a, S_pin)
