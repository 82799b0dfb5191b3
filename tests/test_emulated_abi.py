"""The WHOLE C ABI on the CPU: tests/harness/emu_library.cpp builds ghicp_capi.cu (context, iteration orchestration, every
extern "C" entry point) on top of the product's own kernels through the host emulation shim — CUDA threads as fibers, device
memory = the heap — the TMA streaming kernel of ghicp_stream.cu and the wgmma FD build of ghicp_fdtc.cu included (their
PTX statements have host stand-ins: mbarriers, bulk copies, packed arithmetic, tensor memory as an int32 array).

This module loads that library IN PLACE OF libghicp_b200.so for the duration of a test (the product never does: it has no CPU
path) and runs, on a machine without a GPU:
  * the Python mirror (GHRegistration, register_clouds), the ctypes binding, __graft_entry__.smoke() and bench.py's own arm;
  * the command-line driver and the C++ mirror (ghicp_cli finds the emulated library through LD_LIBRARY_PATH);
  * the `-m gpu` test FUNCTIONS of tests/test_zz*.py themselves — written after the round's GPU budget was spent — with the
    emulated library as their `g`.  (This is how a missing `build_fd()` and a too small iteration cap in two of them were
    found before any GPU run.)
What it cannot show: code generation, memory ordering, asynchrony (copies and MMAs complete at once), performance."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture()
def ge(g, emu_library_path):
    """The product package with the emulated library swapped in for this test only."""
    from conftest import swap_in_library
    real = swap_in_library(g, emu_library_path)
    try:
        yield g
    finally:
        g.capi._lib = real


@pytest.fixture()
def cli_env(emu_library_path):
    return {"LD_LIBRARY_PATH": os.path.dirname(emu_library_path) + os.pathsep + os.environ.get("LD_LIBRARY_PATH", "")}


def test_emulated_library_exports_the_whole_abi_and_reports_one_device(ge, g, emu_library_path):
    L = C.CDLL(emu_library_path)
    for s in g.capi.EXPORTS:                       # tests/test_abi.py checks EXPORTS == the header's declarations
        assert hasattr(L, s), s
    assert ge.device_count() == 1
    assert ge.capi.lib() is not None and g.capi._lib is not None


# ---- the hot path through the ABI: lock-step with the oracle -------------------------------------------------------------
@pytest.mark.parametrize("ft,ct,dof", [("none", "nn", 6), ("none", "nnr", 6), ("bsc", "nn", 6), ("bsc", "nnr", 4), ("bsc", "km", 6),
                                       ("fpfh", "nn", 6), ("fpfh", "nnr", 6)])   # FPFH + KM: the ORACLE's Kuhn-Munkres
# (slack steps of eps = 0.01 on float costs of order 1e4) takes minutes per iteration; that pair has its -m gpu test
def test_registration_through_the_abi_in_lock_step_with_the_oracle(ge, orc, ft, ct, dof):
    g = ge
    FT = {"none": g.FT_NONE, "bsc": g.FT_BSC, "fpfh": g.FT_FPFH}[ft]
    CT = {"nn": g.CT_NN, "nnr": g.CT_NNR, "km": g.CT_KM}[ct]
    N, M, iters = (110, 100, 8) if ct == "km" else (260, 230, 30)   # every emulated auction round runs ~1000 fibers: keep KM small
    sc = g.synth.gen_points(N, M, overlap=0.9, seed=11)
    if ft == "bsc":
        g.synth.add_bsc(sc, V=4 if dof == 6 else 2)
    if ft == "fpfh":
        g.synth.add_fpfh(sc)
    reg = g.registration.from_scene(sc, FT, CT, dof=dof, max_iter=iters)
    o = orc.Oracle(FT, CT, dof=dof, bbx_magnitude=sc.bbx_magnitude, solve_mode=1, max_iter=iters)
    o.set_keypoints(sc.S, sc.T)
    if ft == "bsc":
        o.set_bsc(sc.bsc_s, sc.bsc_t, sc.bits)
    if ft == "fpfh":
        o.set_fpfh(sc.fpfh_s, sc.fpfh_t)
    o.build_fd()
    for it in range(iters):
        a, b = reg.iterate(), o.iterate()
        if ct == "km":      # eps-optimal matchings are not unique: compare the objective, keep both on one trajectory
            assert abs(a.km_energy - b.km_energy) <= N * 0.01 + 1e-6 * abs(b.km_energy)
            o.set_keypoints(reg.source(), sc.T)
            if ft == "bsc":
                o.set_bsc(sc.bsc_s, sc.bsc_t, sc.bits)
            if ft == "fpfh":
                o.set_fpfh(sc.fpfh_s, sc.fpfh_t)
            o.build_fd()
            o.set_state(a.iteration + 1, a.rmse, a.fdm, a.fdstd, a.para1, a.para2)
        else:
            assert np.array_equal(reg.pairs()[0], o.pairs()[0]) and np.array_equal(reg.pairs()[1], o.pairs()[1]), it
            assert a.cor == b.cor and a.rmse == pytest.approx(b.rmse, rel=1e-6)
        if a.converged or b.converged:
            break
    if a.converged:
        assert g.synth.rot_angle(reg.Rt_tillnow()[:3, :3], sc.R_gt) < 2e-2
    reg.close()


def test_settled_km_block_overflow_falls_back_to_the_general_route(ge, monkeypatch):
    """The settled KM iteration carries each rank's candidates in a fixed-size block; when a block overflows (flag travels with
    the statistics, the keypoints are left alone) the host repeats the iteration on the general route.  GHICP_KM_XUSE_MAX = 8
    forces that on every settled iteration: results must equal the general route's (GHICP_KM_GENERAL) and the default's."""
    g = ge
    sc = g.synth.add_bsc(g.synth.gen_points(110, 100, overlap=0.9, seed=11), V=4)
    runs = {}
    for name, env in (("default", {}), ("overflow", {"GHICP_KM_XUSE_MAX": "8"}), ("general", {"GHICP_KM_GENERAL": "1"})):
        for k, v in env.items():
            monkeypatch.setenv(k, v)
        reg = g.registration.from_scene(sc, g.FT_BSC, g.CT_KM, max_iter=5)
        out = []
        for it in range(5):      # the settled route is eligible from iteration 2 on
            st = reg.iterate()
            out.append((st.cor, st.nnz, st.km_energy, np.array(st.Rt), reg.pairs(), reg.source(), st.exact_fallback))
        runs[name] = out
        for k in env:
            monkeypatch.delenv(k)
    # bit 1 of exact_fallback = "the settled iteration's block overflowed, re-ran on the general route": never by default, on
    # every settled-eligible iteration (2, 3, 4) under the hook
    assert all(r[6] == 0 for r in runs["default"]) and all(r[6] == 0 for r in runs["general"])
    assert [r[6] for r in runs["overflow"]] == [0, 0, 2, 2, 2]
    for name in ("overflow", "general"):
        for a, b in zip(runs["default"], runs[name]):
            assert a[0] == b[0] and a[1] == b[1] and a[2] == b[2], name
            assert np.array_equal(a[3], b[3]) and np.array_equal(a[5], b[5]), name
            assert np.array_equal(a[4][0], b[4][0]) and np.array_equal(a[4][1], b[4][1]), name


def test_smoke_entry_point(ge):
    import __graft_entry__ as entry
    entry.smoke()


# ---- the `-m gpu` test functions of tests/test_zz*.py, on the emulated library ------------------------------------------
def test_zz2_functions(ge, orc, tmp_path, cli_env):
    import test_zz2_prep_gpu as z
    z.test_voxel_filter_equals_oracle(ge, orc, 5000, 0.4, 4)
    z.test_voxel_filter_equals_oracle(ge, orc, 1, 1.0, 6)
    z.test_keypoint_detection_equals_oracle(ge, orc, 1500, 0.6, 0.6, 9)
    z.test_prep_error_paths(ge)
    z.test_pipeline_raw_cloud_to_registration(ge, orc, n_points=12000)
    z.test_command_line_driver_registers_two_files(ge, orc, tmp_path, n_points=12000, cli_env=cli_env)


def test_zz2_python_pipeline_helper(ge, orc, monkeypatch):
    import test_zz2_prep_gpu as z
    small = z.scan_like_cloud
    monkeypatch.setattr(z, "scan_like_cloud", lambda n, seed, **kw: small(min(n, 12000), seed, **kw))
    z.test_python_pipeline_helper(ge, orc)


def test_zz3_functions(ge, orc):
    import test_zz3_bsc_gpu as z
    for dof, V in ((0, 1), (4, 2), (6, 4)):
        z.test_golden_vectors_of_the_reference_build(ge, dof, V)
    z.test_equals_oracle(ge, orc, 3000, 40, 1.0, 7, 1)
    z.test_equals_oracle(ge, orc, 2500, 16, 1.2, 9, 5)
    z.test_isolated_keypoints_borders_and_bad_arguments(ge, orc)


def test_zz3_pipeline_and_command_line_with_bsc_features(ge, orc, tmp_path, cli_env):
    import test_zz3_bsc_gpu as z
    z.test_raw_clouds_to_transform_with_bsc_features(ge, orc, n_points=7000)
    z.test_command_line_driver_with_bsc_features(ge, tmp_path, n_points=7000, cli_env=cli_env)


@pytest.mark.parametrize("name", ["none_nn", "bsc_nnr", "bsc_km", "bsc_nn_dof4", "fpfh_nnr"])
def test_zz_loop_fixture_functions(ge, scratch_cwd, name):
    import test_zz_extensions as z
    z.test_cuda_path_reproduces_committed_loop_fixture(ge, scratch_cwd, name)


def test_zz_feature_distance_fixture_functions(ge):
    import test_zz_extensions as z
    for bits in (441, 9, 2048):
        z.test_fd_bsc_equals_reference_hamming_fixture(ge, bits)
    for mf in (1, -1):
        z.test_fd_fpfh_equals_reference_fixture(ge, mf)


def test_zz_extension_functions(ge, orc, monkeypatch):
    import test_zz_extensions as z
    z.test_fpfh_matrix_free_fd_identical(ge, orc, 100, 77)
    z.test_fpfh_matrix_free_rowmin_identical(ge, 5, 3)
    z.test_fpfh_fast_path_equals_exact_path(ge, "nnr", 600, 500)
    z.test_fpfh_auto_mode_and_overrides(ge, monkeypatch)
    z.test_weighted_svd_unit_weights_bit_equal_to_rigid_fit(ge, 1000)
    z.test_estimators_match_oracle(ge, orc, 40)
    z.test_estimators_degenerate_and_errors(ge)
    for solver in ("yaw", "plane"):
        z.test_loop_with_opt_in_estimator_lockstep_with_oracle(ge, orc, solver)


# ---- bench.py's own arm, end to end (the numbers mean nothing here; the contract does) --------------------------------------
@pytest.mark.parametrize("workload", ["config2", "config3"])
def test_bench_line_contract_on_the_emulated_library(ge, capsys, monkeypatch, workload):
    import json
    import runpy
    import sys
    monkeypatch.setattr(sys, "argv", ["bench.py", "--workload", workload, "--n", "200", "--steps", "3", "--warmup", "3",
                                      "--cpu-sample", "200"])
    runpy.run_path(os.path.join(ROOT, "bench.py"), run_name="__main__")
    lines = [l for l in capsys.readouterr().out.splitlines() if l.startswith("{")]
    assert len(lines) == 1
    d = json.loads(lines[0])
    for k in ("metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling", "vs_baseline",
              "dtype", "data", "config", "roofline", "cpu_baseline", "e2e", "clocks", "gpu_launches"):
        assert k in d, k
    assert d["metric"] == "ICP iterations/sec" and d["steps"] == 3 and d["warmup"] == 3 and d["n_gpus"] == 1
    assert set(("bound", "achieved", "peak", "unit", "frac", "traffic")) <= set(d["roofline"])
    assert set(("value", "unit", "cores", "kind", "sample")) <= set(d["cpu_baseline"])
    assert set(("value", "unit", "h2d_bytes_per_step", "d2h_bytes_per_step")) <= set(d["e2e"])
    assert d["e2e"]["h2d_bytes_per_step"] > 0 and d["e2e"]["d2h_bytes_per_step"] > 0
    assert d["gpu_launches"] > 0 and d["vs_baseline"] is None
    assert "workload" in d["config"] and "model" not in d["config"]


# ---- odd sizes: every feature x correspondence mode at N, M around the warp / tile / chunk boundaries ---------------------
def test_random_odd_sizes_in_lock_step_with_the_oracle(ge, orc):
    """Sizes 1, 2, 3, 31..33, 63..65, 257 ... on either side, 4- and 6-DoF, 9- to 672-bit descriptors: the ABI's host logic
    (workspace sizes, chunking, degenerate pair counts) on shapes nobody benchmarks.  200 such trials ran clean under
    ASan + UBSan; 30 run here."""
    g = ge
    rng = np.random.default_rng(2026)
    for trial in range(30):
        N = int(rng.choice([1, 2, 3, 4, 7, 31, 32, 33, 64, 65, 100, 257])); M = int(rng.choice([1, 2, 3, 5, 8, 31, 32, 33, 63, 64, 129, 300]))
        ft = str(rng.choice(["none", "bsc", "fpfh"])); ct = str(rng.choice(["nn", "nnr", "km"]))
        if ft == "fpfh" and ct == "km":
            ct = "nnr"                                  # the oracle's Kuhn-Munkres on float costs is too slow (see above)
        dof = int(rng.choice([4, 6]))
        FT = {"none": g.FT_NONE, "bsc": g.FT_BSC, "fpfh": g.FT_FPFH}[ft]
        CT = {"nn": g.CT_NN, "nnr": g.CT_NNR, "km": g.CT_KM}[ct]
        sc = g.synth.gen_points(N, M, overlap=float(rng.choice([0.3, 0.9, 1.0])), seed=int(rng.integers(1 << 30)))
        if ft == "bsc":
            g.synth.add_bsc(sc, bits=int(rng.choice([9, 64, 441, 672])), V=4 if dof == 6 else 2)
        if ft == "fpfh":
            g.synth.add_fpfh(sc)
        reg = g.registration.from_scene(sc, FT, CT, dof=dof, max_iter=6)
        o = orc.Oracle(FT, CT, dof=dof, bbx_magnitude=sc.bbx_magnitude, solve_mode=1, max_iter=6)
        o.set_keypoints(sc.S, sc.T)
        if ft == "bsc":
            o.set_bsc(sc.bsc_s, sc.bsc_t, sc.bits)
        if ft == "fpfh":
            o.set_fpfh(sc.fpfh_s, sc.fpfh_t)
        o.build_fd()
        what = (trial, N, M, ft, ct, dof)
        for it in range(6):
            a, b = reg.iterate(), o.iterate()
            if ct == "km":
                assert abs(a.km_energy - b.km_energy) <= max(N, M) * 0.01 + 1e-6 * abs(b.km_energy), what
                break
            assert np.array_equal(reg.pairs()[0], o.pairs()[0]) and np.array_equal(reg.pairs()[1], o.pairs()[1]), what + (it,)
            if a.converged or b.converged:
                break
        reg.close()


def test_random_odd_clouds_through_the_preprocessing_abi(ge, orc):
    """1-, 2-, 3-point clouds, exact planes and lines, coincident points, centimetre to 50 m scales, offsets of +-1000 m, grids of
    1 x 1 to 9 x 9 cells: voxel filter, keypoint detector and BSC encoder through the ABI against the oracle.  Voxel indices,
    eigenvalues, curvatures, counts, keypoints and encoder status must be identical; descriptors are compared on the generic
    clouds (a 2 x 2 grid on 3 points is decided by rounding noise in the reference too).  300 trials ran clean under ASan."""
    from test_bsc_encoder import hamming
    g = ge
    rng = np.random.default_rng(3)
    tot = diff = 0
    for trial in range(60):
        n = int(rng.choice([1, 2, 3, 5, 17, 100, 700, 3000]))
        kind = str(rng.choice(["uniform", "plane", "dups", "line", "clusters"]))
        scale = float(rng.choice([0.01, 1.0, 50.0]))
        P = rng.random((n, 3)) * scale
        if kind == "plane":
            P[:, 2] = 0.3 * scale + 1e-4 * scale * rng.standard_normal(n)
        if kind == "dups":
            P = P[rng.integers(0, max(1, n // 3), n)]
        if kind == "line":
            P[:, 1:] = 0.5 * scale
        if kind == "clusters":
            P = P[rng.integers(0, max(1, n // 10), n)] + 0.02 * scale * rng.standard_normal((n, 3))
        P = (P + float(rng.choice([0.0, -100.0, 1000.0]))).astype(np.float32)
        what = (trial, n, kind, scale)
        vox = float(rng.choice([0.001, 0.05, 0.3, 2.0])) * scale
        assert np.array_equal(g.voxel_downsample(P, vox), orc.voxel_downsample(P, vox)), what
        rad = float(rng.choice([0.02, 0.1, 0.4, 3.0])) * scale
        nms = float(rng.choice([0.05, 0.3, 1.0])) * scale
        minp = int(rng.choice([3, 20]))
        kp, lam, curv, cnt = g.detect_keypoints(P, rad, 0.65, minp, nms)
        okp, olam, ocurv, ocnt = orc.detect_keypoints(P, rad, 0.65, minp, nms)
        assert np.array_equal(cnt, ocnt) and np.array_equal(lam, olam) and np.array_equal(curv, ocurv) and np.array_equal(kp, okp), what
        side = int(rng.choice([1, 2, 3, 7, 9])); dof = int(rng.choice([0, 3, 6]))
        kpi = rng.choice(n, int(min(n, rng.choice([1, 2, 9]))), replace=False).astype(np.int32)
        pairs = np.stack([rng.integers(0, side * side, side * side), rng.integers(0, side * side, side * side)], axis=1).astype(np.int32)
        R = float(rng.choice([0.05, 0.3, 2.0])) * scale
        got, _, st = g.bsc_extract(P, kpi, R, dof, side, pairs)
        want, _, wst = orc.bsc_extract(P, kpi, R, pairs, side, dof)
        assert np.array_equal(st, wst), what
        ok = wst == 0
        assert got[:, ~ok].sum() == 0
        if kind in ("uniform", "clusters") and ok.any() and side >= 7 and n >= 100:
            h = hamming(got[:, ok], want[:, ok]); tot += h.size; diff += int((h > 0).sum())
    assert tot > 0 and diff <= 0.02 * tot + 1


def test_cpp_dropin_demo_on_the_emulated_library(ge, orc, tmp_path, monkeypatch, cli_env):
    """gh-icp_b200/cxx/dropin_demo (Keypoints / Energyfunction / GHRegistration constructed like test/ghicp_main.cpp:143-151,
    BSC descriptors uploaded through the C++ mirror) resolves libghicp_b200.so through LD_LIBRARY_PATH: the emulated one."""
    import test_gpu_dropin as z
    monkeypatch.setenv("LD_LIBRARY_PATH", cli_env["LD_LIBRARY_PATH"])
    z.test_cpp_dropin_matches_oracle(ge, orc, tmp_path, "bsc-nn")


def test_python_mirror_public_members(ge):
    """energy / rmse / rmseafter / cor / RMS from the iterations run; ghicp_reg(track_matches=True) adds pre / rec / matchlist
    (src/ghicp_reg.cpp:443-460) and returns the same transform as the default ghicp_run path."""
    g = ge
    sc = g.synth.add_bsc(g.synth.gen_points(110, 100, overlap=0.9, seed=11), V=4)
    a = g.registration.from_scene(sc, g.FT_BSC, g.CT_KM, max_iter=6)
    assert a.RMS == 99999.0 and a.cor == []
    Rt_a, it_a = a.ghicp_reg(track_matches=True)
    assert it_a == len(a.cor) == len(a.energy) == len(a.rmse) == len(a.rmseafter) == len(a.pre) == len(a.rec)
    assert a.matchlist.shape == (110, it_a) and a.RMS == a.rmse[-1]
    for it in range(it_a):
        assert int((a.matchlist[:, it] >= 0).sum()) == a.cor[it]
        assert 0.0 <= a.rec[it] <= a.pre[it] <= 1.0
    sp, tp = a.pairs()
    assert np.array_equal(a.matchlist[sp, -1], tp)
    b = g.registration.from_scene(sc, g.FT_BSC, g.CT_KM, max_iter=6)
    try:
        Rt_b, it_b = b.ghicp_reg()
    except g.capi.GhicpError:      # GHICP_E_NOCONV: max_iter reached; the transform so far is what is compared
        Rt_b, it_b = b.Rt_tillnow(), it_a
    assert it_b == it_a and np.array_equal(Rt_a, Rt_b)
    a.close(); b.close()


@pytest.mark.skipif(not os.environ.get("GHICP_EMU_SLOW"), reason="minutes on the emulator: set GHICP_EMU_SLOW=1")
def test_cpp_dropin_demo_km_full_size_on_the_emulated_library(ge, orc, tmp_path, monkeypatch, cli_env):
    """The `-m gpu` KM drop-in test function itself (700 x 640 keypoints) on the emulated library."""
    import test_gpu_dropin as z
    monkeypatch.setenv("LD_LIBRARY_PATH", cli_env["LD_LIBRARY_PATH"])
    z.test_cpp_dropin_matches_oracle(ge, orc, tmp_path, "bsc-km")


def test_cpp_mirror_fills_matchlist_pre_rec_in_km_mode(ge, tmp_path, monkeypatch, cli_env):
    """Public members of the reference's GHRegistration that its KM branch fills every iteration (src/ghicp_reg.cpp:440-460,
    src/km.cpp:159,226-227): cor, energy, pre, rec and one matchlist column.  The C++ mirror (dropin_demo) and the Python mirror
    run the same library on the same scene, so their iterations are identical: the demo's values must be the ones computed here
    from the Python mirror's pair lists."""
    import test_gpu_dropin as z
    g = ge
    monkeypatch.setenv("LD_LIBRARY_PATH", cli_env["LD_LIBRARY_PATH"])
    assert subprocess.run(["make", "-C", os.path.join(ROOT, "gh-icp_b200", "cxx")], capture_output=True).returncode == 0
    sc = g.synth.add_bsc(g.synth.gen_points(110, 100, overlap=0.9, seed=11), V=4)
    # make the identity a frequent true match so that pre / rec are not trivially zero: the generator pairs source i with
    # target perm[i]; reorder the targets (coordinates and descriptors) so that the pairing is the identity
    order = np.concatenate([sc.perm, np.setdiff1d(np.arange(100), sc.perm)])
    sc.T, sc.bsc_t = np.asfortranarray(sc.T[order]), np.ascontiguousarray(sc.bsc_t[order])
    p = str(tmp_path / "scene.bin")
    z.write_scene(p, sc, 0, 2)
    r = subprocess.run([z.DEMO, p, "6"], capture_output=True, text=True, cwd=str(tmp_path))
    assert r.returncode == 0, r.stderr
    lines = r.stdout.strip().splitlines()
    km = [ln.split() for ln in lines[5:] if ln.startswith("km ")]
    reg = g.registration.from_scene(sc, g.FT_BSC, g.CT_KM, max_iter=6)
    reg.build_fd()
    n_it = int(lines[4].split()[1])
    assert len(km) == n_it >= 1
    seen_exact = 0
    for it in range(n_it):
        st = reg.iterate()
        sp, tp = reg.pairs()
        exact = int((sp == tp).sum())
        assert int(km[it][1]) == it == st.iteration
        assert int(km[it][4]) == int(km[it][5]) == st.cor == len(sp)
        assert float(km[it][2]) == exact / st.cor and float(km[it][3]) == exact / 110
        assert float(km[it][6]) == st.km_energy
        seen_exact = max(seen_exact, exact)
    assert seen_exact >= 45, "the scene pairs source i with target i on 90 keypoints: identity matches expected"
    reg.close()


# ---- stress modes of the emulator: scheduling order and asynchronous copies -------------------------------------------------
@pytest.mark.parametrize("env,expect_ok", [({}, True),
                                           ({"GHICP_EMU_SCHED": "1"}, True),
                                           ({"GHICP_EMU_TMA_DELAY": "7"}, True),
                                           ({"GHICP_EMU_SCHED": "5", "GHICP_EMU_TMA_DELAY": "40"}, True),
                                           ({"GHICP_EMU_NEGCTL_NOWAIT": "1", "GHICP_EMU_TMA_DELAY": "7"}, False)])
def test_tma_and_tcgen05_kernels_under_random_scheduling_and_delayed_copies(emu_library_path, env, expect_ok):
    """The streaming kernel and the wgmma FD build must not depend on which fiber runs first (GHICP_EMU_SCHED: a fresh
    random order every scheduling sweep) nor on a bulk copy having landed before its mbarrier says so (GHICP_EMU_TMA_DELAY: the
    destination is poisoned and the bytes land 1..n ticks later).  Negative control: with every mbarrier wait turned into a no-op
    the same check must FAIL — the modes can see a forgotten wait."""
    import sys
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "harness", "emu_stress_check.py"), emu_library_path],
                       env=dict(os.environ, **env), capture_output=True, text=True)
    assert r.returncode in (0, 1), r.stderr[-2000:]
    assert (r.returncode == 0) == expect_ok, (env, r.stdout[-500:], r.stderr[-1500:])
