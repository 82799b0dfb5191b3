"""The float32 Umeyama solve (svd3_f32 / umeyama_from_moments_f32) pinned to a float64 Kabsch over one table of cases.

Every transform the project returns comes out of that solve: the GH-ICP loop (k_solve<true>), the stand-alone fits
(k_solve<false>, k_solve_alt), point-to-point ICP (k_icp_solve), the SAC-IA hypotheses (k_sac_estimate) and the BSC local
frame.  The kernels are checked bit for bit against CPU restatements of the same text (oracle/ghicp_oracle.cpp,
tests/harness/sac_oracle.cpp, which icp_oracle.cpp includes), so a flaw shared by the copies would pass every parity test.
Here each copy and the kernels meet an independent float64 reference instead:

  * the table (CASES) through both CPU restatements (orc.rigid_fit modes 0 / 1, orc.rigid_fit_ex solvers 0 / 1, the harness
    oracle's Umeyama on float64 moments) and through the C ABI of the emulated library (rigid_fit, rigid_fit_ex SVD /
    WEIGHTED_SVD): R orthonormal with det +1, the residual no worse than the optimum plus a float32 floor, R within 1e-5 rad of
    Kabsch where the optimum is unique, the degenerate flag where there is nothing to solve;
  * power-of-two scalings 2^k, k = -40 .. 40, of one scene: R bit-identical and t exactly 2^k t (the SVD divides sigma by a
    power of two first, like Eigen's JacobiSVD divides by its largest entry);
  * the in-loop solve, cloud_icp and sac_ia on the emulated library in metres and at 1e5 - 1e6 units, through the `-m gpu` test
    functions of tests/test_zz9_rigid_solve_gpu.py on small clouds.

Before the scaling, points spread over more than ~6e4 units (a 300 m site in millimetres) overflowed the sweep's
alpha * beta, every rotation was skipped and R came out 2-15 degrees off and not a rotation, without any error."""
import math
from dataclasses import dataclass

import numpy as np
import pytest

import icp_oracle as io
import sac_oracle as so

EPS32 = 2.0 ** -23
POW2 = range(-40, 41)


# ---- the float64 reference -------------------------------------------------------------------------------------------------
def kabsch(S, T, w=None):
    """(R, t) minimising sum w_i |R s_i + t - t_i|^2 over rotations, in float64 (det-sign correction of Umeyama)."""
    S, T = np.asarray(S, np.float64), np.asarray(T, np.float64)
    w = np.ones(len(S)) if w is None else np.asarray(w, np.float64)
    ms, mt = (w @ S) / w.sum(), (w @ T) / w.sum()
    H = ((T - mt) * w[:, None]).T @ (S - ms)
    U, _, Vt = np.linalg.svd(H)
    D = np.diag([1.0, 1.0, np.sign(np.linalg.det(U) * np.linalg.det(Vt)) or 1.0])
    R = U @ D @ Vt
    return R, mt - R @ ms


def residual(R, t, S, T, w=None):
    """Weighted RMS of R s + t - t_i, in float64."""
    S, T = np.asarray(S, np.float64), np.asarray(T, np.float64)
    w = np.ones(len(S)) if w is None else np.asarray(w, np.float64)
    e = S @ np.asarray(R, np.float64).T + np.asarray(t, np.float64) - T
    return math.sqrt(float(w @ (e * e).sum(axis=1)) / float(w.sum()))


def rot_angle(Ra, Rb):
    """Angle of Ra^T Rb in rad from its skew part (accurate near 0, unlike acos of the trace)."""
    M = np.asarray(Ra, np.float64).T @ np.asarray(Rb, np.float64)
    v = 0.5 * np.array([M[2, 1] - M[1, 2], M[0, 2] - M[2, 0], M[1, 0] - M[0, 1]])
    return math.atan2(float(np.linalg.norm(v)), 0.5 * (np.trace(M) - 1.0))


def check_rotation(R, ctx=None):
    """R orthonormal with det +1 to float32 precision: every entry of R^T R - I and det R - 1 within 2e-6 (~17 ulp of 1)."""
    R = np.asarray(R, np.float64)
    assert np.all(np.isfinite(R)), (ctx, R)
    assert np.abs(R.T @ R - np.eye(3)).max() <= 2e-6, (ctx, np.abs(R.T @ R - np.eye(3)).max())
    assert abs(np.linalg.det(R) - 1.0) <= 2e-6, (ctx, np.linalg.det(R))


def translation_floor(S, T, w=None, float32_sums=False):
    """Float32 bound on |t - t_Kabsch| per coordinate, and on the residual above the optimum: t = mu_d - R mu_s is formed from
    means rounded to float32 (PCL's float clouds force that on the reference), so it is off by up to ~1 ulp of the largest
    |mu| (0.5 m at a northing of 4.4e6: measured 0.19 m, and 0.35 m of extra residual RMS), plus the rotation's float32 error
    (~1e-7 rad) over the extent.  Bound: 2 ulp(max |mu|) + 4 * 2^-23 * extent."""
    S, T = np.asarray(S, np.float64), np.asarray(T, np.float64)
    w = np.ones(len(S)) if w is None else np.asarray(w, np.float64)
    mu = max(np.abs((w @ S) / w.sum()).max(), np.abs((w @ T) / w.sum()).max())
    extent = max(np.ptp(S, axis=0).max(), np.ptp(T, axis=0).max())
    floor = 2.0 * float(np.spacing(np.float32(mu))) + 4.0 * EPS32 * extent
    if float32_sums:   # PCL's float path sums n float32 points for each mean: ~sqrt(n) more roundings
        floor += 4.0 * math.sqrt(len(S)) * EPS32 * (mu + extent)
    return floor


# ---- the table ---------------------------------------------------------------------------------------------------------------
def rot(ax, ay, az):
    from ghicp_b200.synth import rot_xyz_deg
    return np.asarray(rot_xyz_deg(ax, ay, az))


def pose(deg, t):
    Rt = np.eye(4)
    Rt[:3, :3] = rot(0.3 * deg, -0.2 * deg, deg)
    Rt[:3, 3] = t
    return Rt


def axis_rot(axis, deg):
    a = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    th = math.radians(deg)
    return np.eye(3) + math.sin(th) * K + (1 - math.cos(th)) * K @ K


R0, T0 = rot(1.0, -0.7, 3.0), np.array([0.5, -0.25, 0.1])


def moved(S, R=R0, t=T0, noise=0.01, seed=0):
    rng = np.random.default_rng(seed)
    return S @ R.T + t + (rng.normal(0.0, noise, S.shape) if noise else 0.0)


def generic(n=2000, seed=1, extent=(60.0, 60.0, 12.0)):
    S = np.random.default_rng(seed).random((n, 3)) * np.asarray(extent)
    return S, moved(S, seed=seed + 100)


@dataclass
class Case:
    name: str
    why: str
    S: np.ndarray
    T: np.ndarray
    w: np.ndarray = None        # None: unweighted (every solver); else only the weighted solvers
    unique: bool = True         # the optimum is unique by a margin: R within 1e-5 rad of Kabsch
    degenerate: bool = False    # nothing to solve: identity and the degenerate flag


def make_cases():
    c = []
    S, T = generic()
    c.append(Case("generic", "a 60 m x 60 m x 12 m scene with 1 cm of noise: the baseline", S, T))
    S = np.random.default_rng(2).random((3000, 3)) * [3e5, 3e5, 3e4]
    c.append(Case("site_mm", "a 300 m site in millimetres: alpha * beta of the unscaled sweep overflows", S,
                  moved(S, t=T0 * 1000, noise=10.0, seed=3)))
    S = np.random.default_rng(4).random((3000, 3)) * [1e6, 1e6, 1e5]
    c.append(Case("km_mm", "a 1 km site in millimetres", S, moved(S, t=T0 * 1000, noise=10.0, seed=5)))
    S = np.random.default_rng(6).random((2000, 3)) * [4e5, 4e5, 30]
    c.append(Case("flat_mm", "a flat 400 m site in millimetres: one small extent, two that overflow", S,
                  moved(S, t=T0 * 1000, noise=10.0, seed=7)))
    S, T = generic(seed=8)
    S, T = S * 2e-12, T * 2e-12
    c.append(Case("tiny", "extents of ~1e-10: the unscaled sweep's products underflow", S, T))
    S, T = generic(seed=9)
    U = np.array([5e5, 4.4e6, 100.0])
    c.append(Case("utm", "a georeferenced offset: the translation carries the float32 rounding of the means", S + U, T + U))
    S = np.array([[0.0, 0.0, 0.0], [3.0, 0.5, 0.2], [0.7, 2.5, -0.4]])
    c.append(Case("n3", "three points: the minimal non-collinear set", S, moved(S, noise=0.0)))
    S = np.random.default_rng(10).random((500, 3)) * [40.0, 30.0, 0.0]
    c.append(Case("planar_exact", "exactly planar source (z = 0), exact motion: sigma has rank 2", S, moved(S, noise=0.0)))
    c.append(Case("planar_noisy", "planar source with noise on the target", S, moved(S, noise=0.005, seed=11)))
    rng = np.random.default_rng(12)
    S = rng.random((300, 3)) * [10.0, 10.0, 0.0]
    S[:, 2] = rng.normal(0.0, 1e-3, 300)
    T = S.copy()
    T[:, 2] = -S[:, 2]
    c.append(Case("reflection", "coplanar, noisy, mirrored: the unconstrained optimum is a reflection (det-sign branch)", S, T))
    u = np.array([1.0, 2.0, 0.5])
    S = np.linspace(-20.0, 30.0, 200)[:, None] * u + [3.0, -1.0, 2.0]
    c.append(Case("collinear", "collinear points (sigma_2 ~ 0): the rotation about the line is free", S, moved(S, noise=0.0),
                  unique=False))
    S = np.tile([[12.5, -3.0, 7.25]], (50, 1))
    c.append(Case("identical", "all points identical: sigma = 0", S, moved(S, noise=0.0), unique=False))
    S = np.array([[x, y, z] for x in (-1.0, 1.0) for y in (-1.0, 1.0) for z in (-1.0, 1.0)]) * 5.0
    c.append(Case("cube", "cube corners: three equal singular values", S, moved(S, noise=0.0)))
    S = np.array([[1.0, 1.0, 1.0], [1.0, -1.0, -1.0], [-1.0, 1.0, -1.0], [-1.0, -1.0, 1.0]]) * 3.0
    c.append(Case("tetrahedron", "a regular tetrahedron: three equal singular values", S, moved(S, noise=0.0)))
    S, _ = generic(n=800, seed=13)
    for name, axis, deg in [("rot180_x", (1, 0, 0), 180.0), ("rot180_y", (0, 1, 0), 180.0), ("rot180_z", (0, 0, 1), 180.0),
                            ("rot180_generic", (0.3, -0.5, 0.8), 180.0), ("rot179.99", (0.3, -0.5, 0.8), 179.99)]:
        c.append(Case(name, "a half turn: sigma's symmetric part changes sign", S, moved(S, R=axis_rot(axis, deg), seed=14)))
    S, T = generic(n=500, seed=15)
    w = np.zeros(len(S)); w[[3, 111, 402]] = 1.0
    T2 = T.copy(); T2[w == 0] += np.random.default_rng(16).normal(0.0, 50.0, ((w == 0).sum(), 3))
    c.append(Case("weights_three", "zero weight everywhere except three points", S, T2, w))
    w = 10.0 ** np.random.default_rng(17).uniform(-12.0, 12.0, len(S))
    c.append(Case("weights_span", "weights spanning 1e-12 .. 1e12", S, T, w))
    c.append(Case("weights_outlier", "a far outlier of weight 0 appended: changes nothing", np.vstack([S, [[1e4, -2e4, 5e3]]]),
                  np.vstack([T, [[-3e4, 1e4, 0.0]]]), np.append(np.ones(len(S)), 0.0)))
    c.append(Case("weights_zero", "total weight 0: the degenerate flag", S, T, np.zeros(len(S)), degenerate=True))
    c.append(Case("two_points", "fewer than three pairs: identity and the degenerate flag", S[:2], T[:2], degenerate=True))
    return c


CASES = make_cases()
NAMES = [c.name for c in CASES]


def check_case(case, fit, solver=None):
    """fit(S, T, w) -> (R, t, degenerate flag or None).  w is None for the unweighted cases; weighted cases are skipped by
    solvers without weights (fit.weighted False)."""
    if case.w is not None and not getattr(fit, "weighted", False):
        return
    ctx = (case.name, solver)
    R, t, flag = fit(case.S, case.T, case.w)
    if case.degenerate:
        assert np.array_equal(R, np.eye(3)) and np.array_equal(t, np.zeros(3)), ctx
        assert flag in (None, True), ctx
        return
    assert flag in (None, False), ctx
    check_rotation(R, ctx)
    Rk, tk = kabsch(case.S, case.T, case.w)
    floor = translation_floor(case.S, case.T, case.w, getattr(fit, "float32_sums", False))
    opt = residual(Rk, tk, case.S, case.T, case.w)
    got = residual(R, t, case.S, case.T, case.w)
    assert got <= opt + floor, (ctx, got, opt, floor)
    if case.unique:
        assert rot_angle(R, Rk) < 1e-5, (ctx, rot_angle(R, Rk))
        assert np.abs(t - tk).max() <= floor, (ctx, t - tk, floor)
    if case.name == "weights_outlier":      # the same bits as without the outlier
        R1, t1, _ = fit(case.S[:-1], case.T[:-1], np.ones(len(case.S) - 1))
        assert np.array_equal(R, R1) and np.array_equal(t, t1), ctx


def check_pow2(fit, solver=None):
    """Scaling both clouds by 2^k returns the same R bit for bit and exactly 2^k t, for k = -40 .. 40."""
    S, T = generic(n=500, seed=18)
    R0_, t0_, _ = fit(S, T, None)
    check_rotation(R0_, (solver, 0))
    for k in POW2:
        f = 2.0 ** k
        R, t, _ = fit(S * f, T * f, None)
        assert np.array_equal(R, R0_), (solver, k, rot_angle(R, R0_), np.linalg.det(R))
        assert np.array_equal(t, t0_ * f), (solver, k, t / f - t0_)


# ---- the solvers -------------------------------------------------------------------------------------------------------------
def _split(Rt):
    return np.asarray(Rt[:3, :3], np.float64), np.asarray(Rt[:3, 3], np.float64)


def _solver(fn, weighted):
    fn.weighted = weighted
    return fn


def solvers_oracle(orc):
    def fit(mode):
        return lambda S, T, w: (*_split(orc.rigid_fit(S, T, mode)), None)

    def fit_ex(solver, weighted):
        def f(S, T, w):
            Rt, rc = orc.rigid_fit_ex(S, T, solver, weights=w if weighted else None)
            return (*_split(Rt), rc != 0)
        return _solver(f, weighted)

    mode0 = _solver(fit(0), False)
    mode0.float32_sums = True
    return {"orc.rigid_fit(0)": mode0, "orc.rigid_fit(1)": _solver(fit(1), False),
            "orc.rigid_fit_ex(0)": fit_ex(0, False), "orc.rigid_fit_ex(1)": fit_ex(1, True)}


def harness_fit(S, T, w):
    """tests/harness/sac_oracle.cpp's Umeyama (also icp_oracle.cpp's) on float64 (weighted) moments rounded once to float32,
    as its callers form them."""
    S, T = np.asarray(S, np.float64), np.asarray(T, np.float64)
    w = np.ones(len(S)) if w is None else np.asarray(w, np.float64)
    if len(S) < 3 or not w.sum() > 0:
        return np.eye(3), np.zeros(3), True
    ms, mt = (w @ S) / w.sum(), (w @ T) / w.sum()
    sigma = ((T - mt) * w[:, None]).T @ (S - ms) / w.sum()
    R, t = so.umeyama(ms.astype(np.float32), mt.astype(np.float32), sigma.astype(np.float32))
    return R.astype(np.float64), t.astype(np.float64), False


harness_fit.weighted = True


def solvers_capi(g):
    def fit(S, T, w):
        return (*_split(g.rigid_fit(S, T)), None)

    def fit_ex(solver, weighted):
        def f(S, T, w):
            Rt, rc = g.rigid_fit_ex(S, T, solver, weights=w if weighted else None)
            return (*_split(Rt), rc == g.capi.GHICP_W_FEW_PAIRS)
        return _solver(f, weighted)

    return {"rigid_fit": _solver(fit, False), "rigid_fit_ex(SVD)": fit_ex(g.capi.SOLVER_SVD, False),
            "rigid_fit_ex(WEIGHTED_SVD)": fit_ex(g.capi.SOLVER_WEIGHTED_SVD, True)}


# ---- the CPU restatements ----------------------------------------------------------------------------------------------------
ORACLE_SOLVERS = ["orc.rigid_fit(0)", "orc.rigid_fit(1)", "orc.rigid_fit_ex(0)", "orc.rigid_fit_ex(1)"]


@pytest.mark.parametrize("solver,name", [(s, n) for s in ORACLE_SOLVERS for n in NAMES
                                         # mode 0 restates PCL's float clouds: points and means in float32, so at a 4.4e6
                                         # offset its input is already quantised to 0.5 m (the kernels use mode 1's moments)
                                         if not (s == "orc.rigid_fit(0)" and n == "utm")])
def test_oracle_against_kabsch(orc, solver, name):
    check_case(next(c for c in CASES if c.name == name), solvers_oracle(orc)[solver], solver)


@pytest.mark.parametrize("name", NAMES)
def test_harness_oracle_against_kabsch(name):
    check_case(next(c for c in CASES if c.name == name), harness_fit, "harness")


@pytest.mark.parametrize("solver", ORACLE_SOLVERS)
def test_oracle_power_of_two_scalings(orc, solver):
    check_pow2(solvers_oracle(orc)[solver], solver)


def test_harness_oracle_power_of_two_scalings():
    check_pow2(harness_fit, "harness")


def test_copies_agree_bit_for_bit(orc):
    """orc.rigid_fit_ex(1) and the harness's Umeyama fed the same float32 moments give the same bits on every case: the two
    restatements of the solve cannot drift apart."""
    for case in CASES:
        if case.degenerate:
            continue
        S, T = np.asarray(case.S, np.float64), np.asarray(case.T, np.float64)
        w = np.ones(len(S)) if case.w is None else case.w
        Rt, rc = orc.rigid_fit_ex(S, T, 1, weights=w)
        # the oracle's moments, in its summation order
        sw = 0.0
        ms, md = np.zeros(3), np.zeros(3)
        for i in range(len(S)):
            sw += w[i]; ms += w[i] * S[i]; md += w[i] * T[i]
        mus, mud = ms / sw, md / sw
        acc = np.zeros((3, 3))
        for i in range(len(S)):
            acc += w[i] * np.outer(T[i] - mud, S[i] - mus)
        R, t = so.umeyama(mus.astype(np.float32), mud.astype(np.float32), (acc / sw).astype(np.float32))
        assert rc == 0 and np.array_equal(Rt[:3, :3], R.astype(np.float64)) and np.array_equal(Rt[:3, 3], t.astype(np.float64)), \
            case.name


def test_icp_oracle_in_millimetres():
    """The ICP oracle's steps on a 300 m x 300 m x 30 m box in millimetres are rotations within 1e-5 rad of a float64 Kabsch on
    their own pairs, and the result reaches the motion found in metres."""
    import test_zz9_rigid_solve_gpu as t
    P, Q, G = t.box_clouds(3000, 33)
    out = {}
    for f in (1.0, 1000.0):
        Pf, Qf = (P * f).astype(np.float32), (Q * f).astype(np.float32)
        Rt, o = io.icp(Pf, Qf, max_iterations=10, steps=True)
        W = Pf
        for k in range(o["iterations"]):
            m = o["corr"][k] >= 0
            Rk, _ = kabsch(W[m], Qf[o["corr"][k][m]])
            check_rotation(o["T"][k][:3, :3], (f, k))
            assert rot_angle(Rk, o["T"][k][:3, :3]) < 1e-5, (f, k)
            W = t.io_move(W, o["T"][k])
        check_rotation(Rt[:3, :3], f)
        out[f] = Rt
    assert rot_angle(out[1.0][:3, :3], out[1000.0][:3, :3]) < 1e-5
    assert np.abs(out[1000.0][:3, 3] / 1000.0 - out[1.0][:3, 3]).max() < 1e-3


# ---- the emulated kernels through the C ABI ----------------------------------------------------------------------------------
@pytest.fixture()
def ge(g, emu_library_path):
    from conftest import swap_in_library
    real = swap_in_library(g, emu_library_path)
    try:
        yield g
    finally:
        g.capi._lib = real


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("solver", ["rigid_fit", "rigid_fit_ex(SVD)", "rigid_fit_ex(WEIGHTED_SVD)"])
def test_emulated_abi_against_kabsch(ge, solver, name):
    check_case(next(c for c in CASES if c.name == name), solvers_capi(ge)[solver], solver)


@pytest.mark.parametrize("solver", ["rigid_fit", "rigid_fit_ex(SVD)", "rigid_fit_ex(WEIGHTED_SVD)"])
def test_emulated_abi_power_of_two_scalings(ge, solver):
    check_pow2(solvers_capi(ge)[solver], solver)


@pytest.mark.parametrize("name,kw", [("test_loop_solve_equals_kabsch_on_its_pairs", dict(n=600, iterations=2)),
                                     ("test_cloud_icp_in_millimetres", dict(n_points=4000)),
                                     ("test_sac_ia_in_millimetres", dict(n_points=6000, n_kp=300, iterations=200)),
                                     ("test_cloud_icp_steps_equal_kabsch_in_millimetres", dict(n_points=3000))])
def test_gpu_test_functions_on_the_emulated_library(ge, name, kw):
    import test_zz9_rigid_solve_gpu as t
    getattr(t, name)(ge, **kw)
