"""The error bounds of the two FP32 correspondence filters, restated in numpy and checked over whole scenes, and the near-tie
scenes that make those bounds matter, run through the emulated library against the all-double route and the oracle.

  * k_stream (gh-icp_b200/csrc/ghicp_stream.cu, Ft = None / BSC): d2' = S.w + T.w + S.x T.x + S.y T.y + S.z T.z (1 FADD,
    3 FFMA in the kernel's order), dist = sqrt.approx(d2'), cd32 = fma(fd, b, dist).  k_margin promises
    |cd32 - kappa * cd64| <= margin inside the window of stream_in_window (ghicp_internal.h); outside it the iteration takes
    the all-double route (exact_fallback bit 2).
  * k_ff_sweep (gh-icp_b200/csrc/ghicp_fpfh.cu, FPFH): fd32 = |<h_s, h_t>| of the L2-normalised centred histograms (three
    11-term FMA chains), dist from hi/lo-split centred coordinates, cd32 = dist * ex2(-ex lg2(fd32)).  It promises
    |fd32 - FD_reference| <= FF_G and LB = cd32 (1 - FF_D0 - 1.5 ex FF_G / fd32) <= CD_exact.

Every float32 rounding of the kernels is reproduced exactly (fma32: the product of two float32 is exact in float64, the sum
is rounded once with its TwoSum tail breaking float32 ties).  The approximate MUFU operations cannot be reproduced: each is
its exact value times (1 +- its error), with the figures of the PTX ISA manual below, and the bound is checked at both ends
of that interval (tests/test_zz9_filter_margins_gpu.py measures the three instructions on the H100 against those figures).
"""
import copy
import math

import numpy as np
import pytest

from test_filter_redo import codes, lockstep, oracle_for

F32 = np.float32
U = 2.0 ** -24                 # float32 unit roundoff
# PTX ISA manual, "Floating Point Instructions": sqrt.approx.f32 maximum relative error 2^-23; lg2.approx.f32 maximum
# absolute error 2^-22 (the manual's figure, 2^-22.6, is for the mantissa's logarithm: the float result adds up to an ulp of
# itself, 7.6e-6 near |lg2| = 100, so the model is LG2_ABS * (1 + |lg2 x|)); ex2.approx.f32 maximum relative error 2^-22
# (manual: 2^-22.5).  The .ftz forms flush subnormal inputs and results to zero.  Measured on an H100 over the inputs the
# filters use: 2^-23.25, 2^-16.97 absolute (at lg2 ~ -100), 2^-22.71.
SQRT_REL = 2.0 ** -23
LG2_ABS = 2.0 ** -22
EX2_REL = 2.0 ** -22


def _fpfh_constant(name):
    """FF_D0 / FF_G as ghicp_fpfh.cu defines them: the bounds are checked for the values the kernel uses."""
    import os
    import re
    src = open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "gh-icp_b200", "csrc", "ghicp_fpfh.cu")).read()
    return float(F32(re.search(r"constexpr float %s = ([0-9.eE+-]+)f;" % name, src).group(1)))


FF_D0 = _fpfh_constant("FF_D0")
FF_G = _fpfh_constant("FF_G")
WINDOW_LO, WINDOW_HI = 2.0 ** -80, 2.0 ** 120     # ghicp_internal.h, stream_in_window
SCALES = [-40, -32, -24, -20, -16, -8, -4, 0, 4, 8, 16, 20, 24, 32, 40]


# ---- exact float32 arithmetic ------------------------------------------------------------------------------------------
def _round32(s, e):
    """float32(s + e) for s = RN64(s + e): s rounds like s + e unless s is a float32 midpoint, where the tail decides."""
    r = s.astype(F32)
    lo = np.where(r.astype(np.float64) > s, np.nextafter(r, F32(-np.inf)), r)
    hi = np.nextafter(lo, F32(np.inf))
    mid = 0.5 * (lo.astype(np.float64) + hi.astype(np.float64))
    return np.where((s == mid) & (e != 0), np.where(e > 0, hi, lo), r)


def add32(a, b):
    return (np.asarray(a, F32) + np.asarray(b, F32)).astype(F32)


def fma32(a, b, c):
    """fmaf(a, b, c) with one rounding."""
    p = np.asarray(a, F32).astype(np.float64) * np.asarray(b, F32).astype(np.float64)
    c = np.asarray(c, F32).astype(np.float64)
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)
    return _round32(s, e)


def f32_ru(x):
    """__double2float_ru"""
    r = np.asarray(x, np.float64).astype(F32)
    return np.where(r.astype(np.float64) < x, np.nextafter(r, F32(np.inf)), r)


def serial_mean(v):
    return np.cumsum(v, axis=0)[-1] / v.shape[0]


# ---- k_stream ----------------------------------------------------------------------------------------------------------
def stream_weights(ft, it, bbx):
    """(a, b, kappa, scale, WED, WFD) of launch_stream_prep (ghicp_stream.cu)."""
    scale = float(F32(0.005 * bbx))
    WFD = math.exp(-it / 6.0)
    WED = 1.0 - WFD
    if ft == "none":
        return scale, 0.0, 1.0, scale, WED, WFD
    whf = float(np.float16(F32(WFD)))
    if WFD >= 6.2e-5 and whf > 0.0:
        kappa, b = whf / WFD, whf
    else:
        kappa, b = 1.0, float(F32(WFD))
    return scale * WED * kappa, b, kappa, scale, WED, WFD


def stream_in_window(A, R2):
    if not (2.0 ** -100 <= R2 <= 2.0 ** 100):
        return False
    if A == 0.0:
        return True
    P = A * R2
    return WINDOW_LO <= P <= WINDOW_HI and 4.0 * A * A * R2 <= 2.0 ** 240


def stream_prep(S, T, a):
    """k_prep: S4, T4 centred on the target centroid, and R2 (rounded up)."""
    c = serial_mean(T)
    A = a * a
    xs, xt = S - c, T - c
    ns = (xs[:, 0] * xs[:, 0] + xs[:, 1] * xs[:, 1]) + xs[:, 2] * xs[:, 2]
    nt = (xt[:, 0] * xt[:, 0] + xt[:, 1] * xt[:, 1]) + xt[:, 2] * xt[:, 2]
    S4 = np.column_stack([xs.astype(F32), (A * ns).astype(F32)])
    T4 = np.column_stack([((-2.0 * A) * xt).astype(F32), (A * nt).astype(F32)])
    R2 = float(max(f32_ru(ns).max(), f32_ru(nt).max()))
    return S4, T4, A, R2


def stream_d2(S4, T4):
    """d2' of every pair, the kernel's order: Tw + Sw, then the z, y, x FFMAs."""
    acc = add32(T4[None, :, 3], S4[:, None, 3])
    for k in (2, 1, 0):
        acc = fma32(S4[:, None, k], T4[None, :, k], acc)
    return acc


def stream_margin(A, a, b, fdmax, R2):
    E = 32.0 * U * A * R2
    return float(f32_ru(math.sqrt(E) * 1.001 + 2.0 ** -20 * (2.0 * a * math.sqrt(R2) + b * fdmax) + 1e-30))


def stream_cd32_interval(d2, fd, b):
    """[lo, hi] of cd32 over every outcome of sqrt.approx.ftz (relative SQRT_REL; a subnormal d2' is flushed to 0)."""
    with np.errstate(invalid="ignore", over="ignore"):
        r = np.sqrt(np.abs(d2.astype(np.float64)))
        sub = np.abs(d2) < 2.0 ** -126
        dlo = np.where(sub, 0.0, r * (1.0 - SQRT_REL))
        dhi = np.where(sub, 0.0, r * (1.0 + SQRT_REL))
        bf = fd * b
        return (bf + dlo) * (1.0 - U), (bf + dhi) * (1.0 + U)   # the FFMA rounds once


def cd64_stream(S, T, ft, fd, scale, WED, WFD):
    d = S[:, None, :] - T[None, :, :]
    ed = scale * np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])
    return WED * ed + WFD * fd if ft == "bsc" else ed


def check_stream_bound(S, T, ft, it, bbx, fd=None, bits=0):
    """Returns (in_window, worst |cd32 - kappa cd64| / margin)."""
    a, b, kappa, scale, WED, WFD = stream_weights(ft, it, bbx)
    S4, T4, A, R2 = stream_prep(S, T, a)
    fdv = np.zeros((len(S), len(T))) if fd is None else fd
    m = stream_margin(A, a, b if ft == "bsc" else 0.0, float(bits), R2)
    lo, hi = stream_cd32_interval(stream_d2(S4, T4), fdv, b if ft == "bsc" else 0.0)
    ref = kappa * cd64_stream(S, T, ft, fdv, scale, WED, WFD)
    with np.errstate(invalid="ignore"):
        err = np.maximum(np.abs(lo - ref), np.abs(hi - ref))
    worst = float(np.nanmax(err)) if np.isfinite(err).all() else math.inf
    return stream_in_window(A, R2), worst / m


def scaled(sc0, k):
    sc = copy.deepcopy(sc0)
    f = 2.0 ** k
    sc.S, sc.T, sc.bbx_magnitude = np.asfortranarray(sc0.S * f), np.asfortranarray(sc0.T * f), sc0.bbx_magnitude * f
    return sc


def scan_scene(g, n, seed=4):
    tgt, src, _, _ = g.synth.scan_pair(4 * n, seed=seed)
    rng = np.random.default_rng(seed)
    S = src[rng.choice(len(src), n, replace=False)].astype(np.float64)
    T = tgt[rng.choice(len(tgt), n, replace=False)].astype(np.float64)
    ext = (S.max(axis=0) - S.min(axis=0)).astype(F32)
    return g.synth.Scene(S=np.asfortranarray(S), T=np.asfortranarray(T), bbx_magnitude=float(F32(ext.sum())), R_gt=np.eye(3),
                         t_gt=np.zeros(3), n_overlap=0, perm=np.zeros(0, np.int64), meta=dict(seed=seed))


@pytest.mark.parametrize("kind", ["gen_points", "scan_like"])
@pytest.mark.parametrize("k", SCALES)
def test_stream_bound_across_scales(g, kind, k):
    """Ft = None at iteration 0 (the ED term alone): inside the window the bound holds with room to spare; outside it the
    window says so (at 2^40 S.w overflows, at 2^-40 every product is subnormal)."""
    sc0 = g.synth.gen_points(150, 140, overlap=0.9, seed=7) if kind == "gen_points" else scan_scene(g, 150)
    sc = scaled(sc0, k)
    inside, ratio = check_stream_bound(sc.S, sc.T, "none", 0, sc.bbx_magnitude)
    if inside:
        assert ratio <= 1.0, (k, ratio)
    assert inside or k != 0
    if abs(k) == 40:
        assert not inside and not ratio <= 1.0, (k, ratio)     # the window is needed: the bound really fails out there


def test_stream_bound_far_outlier_utm_and_coincident_points(g):
    from test_filter_redo import UTM
    sc = g.synth.gen_points(150, 139, overlap=0.9, extent=(100, 100, 20), seed=3)
    far = np.vstack([sc.T, (sc.T.mean(axis=0) + [4e4, 0.0, 0.0]).astype(F32)])
    utm_s = (sc.S + UTM).astype(F32).astype(np.float64)
    utm_t = np.vstack([(sc.T + UTM).astype(F32).astype(np.float64), [0.0, 0.0, 0.0]])
    near = sc.T[:139] + np.random.default_rng(1).normal(0.0, 1e-6, (139, 3))     # sources on top of the targets
    for S, T in ((sc.S, far), (utm_s, utm_t), (near, sc.T)):
        for it in (0, 1, 3, 12):
            inside, ratio = check_stream_bound(S, T, "none", it, sc.bbx_magnitude)
            assert inside and ratio <= 1.0, (it, ratio)


@pytest.mark.parametrize("bits", [441, 511, 1000, 1023, 2048])
def test_stream_bound_bsc_at_the_largest_fd_code(g, bits):
    """BSC with FD up to the largest code of the plane width (fd_hb: 9 / 10 / 12 bits), the weights of iterations 0-40."""
    sc = g.synth.gen_points(120, 110, overlap=0.9, seed=5)
    rng = np.random.default_rng(bits)
    fd = rng.integers(0, bits + 1, (120, 110)).astype(np.float64)
    fd[:, :8] = bits
    for it in (0, 1, 2, 5, 20, 40, 60, 80):
        inside, ratio = check_stream_bound(sc.S, sc.T, "bsc", it, sc.bbx_magnitude, fd=fd, bits=bits)
        assert inside and ratio <= 1.0, (it, ratio)


# ---- k_ff_sweep --------------------------------------------------------------------------------------------------------
def fpfh_center(h):
    """k_fpfh_center2 (no FMA contraction in ghicp_fpfh.cu): centred histogram and its serial sum of squares."""
    h = np.asarray(h, F32)
    mean = np.zeros(len(h), F32)
    for k in range(33):
        mean = (mean + h[:, k]).astype(F32)
    mean = (mean / F32(33)).astype(F32)
    c = (h - mean[:, None]).astype(F32)
    d = np.zeros(len(h), F32)
    for k in range(33):
        d = (d + (c[:, k] * c[:, k]).astype(F32)).astype(F32)
    return c, d


def fpfh_fd_reference(cs, ds, ct, dt):
    """fpfh_fd_pair: the float FD every exact path (and the oracle) uses."""
    up = np.zeros((len(cs), len(ct)), F32)
    for k in range(33):
        up = (up + (cs[:, None, k] * ct[None, :, k]).astype(F32)).astype(F32)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.abs((up / np.sqrt((ds[:, None] * dt[None, :]).astype(F32))).astype(F32))


def fpfh_fd32(cs, ds, ct, dt):
    """k_ff_normalise + the three 11-term FMA chains of k_ff_sweep: fd32 before its 1e-30 floor."""
    def norm(c, d):
        inv = np.where(d > 0, (F32(1.0) / np.sqrt(d)).astype(F32), F32(0.0))
        return (c * inv[:, None]).astype(F32)
    ns, nt = norm(cs, ds), norm(ct, dt)
    part = []
    for q in range(3):
        acc = np.zeros((len(cs), len(ct)), F32)
        for k in range(11):
            acc = fma32(ns[:, None, 11 * q + k], nt[None, :, 11 * q + k], acc)
        part.append(acc)
    return np.abs(add32(add32(part[0], part[1]), part[2]))


def fpfh_dist32(S, T, scalef):
    """k_ff_prep's hi/lo split and the sweep's difference, FMA chain and scale (sqrt.approx.ftz: interval)."""
    c = serial_mean(T)

    def split(X):
        x = X - c
        hi = x.astype(F32)
        return hi, (x - hi.astype(np.float64)).astype(F32)
    sh, sl = split(S)
    th, tl = split(T)
    d = [add32(add32(sh[:, None, k], -th[None, :, k]), add32(sl[:, None, k], -tl[None, :, k])) for k in range(3)]
    d2 = fma32(d[2], d[2], fma32(d[1], d[1], (d[0] * d[0]).astype(F32)))
    r = np.sqrt(d2.astype(np.float64))
    r = np.where(d2 < 2.0 ** -126, 0.0, r)
    return r * (1.0 - SQRT_REL) * scalef * (1.0 - U), r * (1.0 + SQRT_REL) * scalef * (1.0 + U), d2


def check_fpfh_bound(S, T, hs, ht, bbx, exs):
    """|fd32 - FD_ref| <= FF_G, and the largest LB (or rare-path bound) any MUFU outcome gives <= CD_exact.  Returns the worst
    |fd32 - FD_ref| / FF_G and the worst LB / CD_exact."""
    cs, ds = fpfh_center(hs)
    ct, dt = fpfh_center(ht)
    ref = fpfh_fd_reference(cs, ds, ct, dt).astype(np.float64)
    fd32 = fpfh_fd32(cs, ds, ct, dt).astype(np.float64)
    ok = np.isfinite(ref) & (ref > 0)
    err = float(np.max(np.abs(fd32 - ref)[ok]))
    g_ratio = err / FF_G if FF_G > 0 else (math.inf if err > 0 else 0.0)
    scale = float(F32(0.005 * bbx))
    d = S[:, None, :] - T[None, :, :]
    ed = scale * np.sqrt((d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2])
    _, dist_hi, _ = fpfh_dist32(S, T, float(F32(scale)))
    fdc = np.maximum(fd32, 1e-30)
    worst = 0.0
    for ex in exs:
        exf = float(F32(ex))
        with np.errstate(divide="ignore", over="ignore", invalid="ignore"):
            cd_exact = ed / np.power(ref, ex)
            l = np.log2(fdc)
            # largest cd32: lg2 low by LG2_ABS, every product and ex2 at the top of its interval
            dl = LG2_ABS * (1.0 + np.abs(l))
            y_hi = -exf * (l - dl) * (1.0 + U)
            cd_hi = dist_hi * np.exp2(y_hi) * (1.0 + EX2_REL) * (1.0 + U)
            rinv_lo = np.exp2(-(l + dl)) * (1.0 - EX2_REL)
            c1 = float(F32(1.5 * exf * FF_G))
            fac = (float(F32(1.0 - FF_D0)) - c1 * rinv_lo * (1.0 - U)) * (1.0 + U)
            lb = np.where(fdc < 8.0 * FF_G, -np.inf, cd_hi * fac * (1.0 + U))
            # rare path of ff_slow when FF_G > fd32 / 8: the bound through fd32 + FF_G
            l2 = np.log2(np.maximum(fdc + FF_G, 1e-30))
            lb2 = dist_hi * np.exp2(-exf * (l2 - LG2_ABS * (1.0 + np.abs(l2))) * (1.0 + U)) * (1.0 + EX2_REL) * float(F32(1.0 - FF_D0)) * (1.0 + U) ** 3
            lb = np.maximum(lb, np.where(FF_G > 0.125 * fdc, lb2, -np.inf))
            r = np.where(ok & (cd_exact > 0), lb / cd_exact, 0.0)
        worst = max(worst, float(np.nanmax(r)))
    return g_ratio, worst


EXS = [1.0 / (it + 1) for it in range(51)]


def hist_family(rng, n, kind):
    if kind == "gamma":
        h = rng.gamma(0.6, 1.0, size=(n, 3, 11))
        return (100.0 * h / h.sum(axis=2, keepdims=True)).reshape(n, 33)
    if kind == "near_constant":     # centring cancels: bins equal up to a few float32 ulps
        return 100.0 / 11.0 + rng.integers(-3, 4, (n, 33)) * 2.0 ** -20
    if kind == "one_hot":
        h = np.zeros((n, 33))
        h[np.arange(n), rng.integers(0, 33, n)] = 100.0
        return h + (rng.random((n, 33)) < 0.1) * 1e-3
    raise ValueError(kind)


@pytest.mark.parametrize("kind", ["gamma", "near_constant", "one_hot"])
def test_fpfh_bound_histogram_families(g, kind):
    rng = np.random.default_rng({"gamma": 1, "near_constant": 2, "one_hot": 3}[kind])
    sc = g.synth.gen_points(90, 80, overlap=0.9, seed=9)
    hs, ht = hist_family(rng, 90, kind).astype(F32), hist_family(rng, 80, kind).astype(F32)
    g_ratio, lb_ratio = check_fpfh_bound(sc.S, sc.T, hs, ht, sc.bbx_magnitude, EXS)
    print(f"\n{kind}: max |fd32 - FD_ref| = {g_ratio:.3f} FF_G, max LB / CD_exact = {lb_ratio:.9f}")
    assert g_ratio <= 1.0 and lb_ratio <= 1.0


def correlated_pairs(rng, rhos, n_each=8):
    """Histogram pairs whose centred correlation is rho: s = rho u + sqrt(1 - rho^2) v (u, v orthonormal, centred)."""
    hs, ht = [], []
    for rho in rhos:
        for _ in range(n_each):
            x = rng.normal(size=(2, 33))
            x -= x.mean(axis=1, keepdims=True)
            u = x[0] / np.linalg.norm(x[0])
            v = x[1] - (x[1] @ u) * u
            v /= np.linalg.norm(v)
            ht.append(5.0 + u)
            hs.append(5.0 + rho * u + math.sqrt(1.0 - rho * rho) * v)
    return np.array(hs, F32), np.array(ht, F32)


def test_fpfh_bound_correlation_around_8_ff_g(g):
    """|correlation| just above and below 8 FF_G, where the first-order bound hands over to ff_slow's fd32 + FF_G bound."""
    rng = np.random.default_rng(11)
    rhos = [8 * FF_G * f for f in (0.5, 0.9, 0.99, 0.999, 1.001, 1.01, 1.1, 2.0)]
    hs, ht = correlated_pairs(rng, rhos)
    pts = np.random.default_rng(12).random((len(hs), 3)) * 50.0
    S, T = pts.astype(F32).astype(np.float64), (pts + 0.5).astype(F32).astype(np.float64)
    g_ratio, lb_ratio = check_fpfh_bound(S, T, hs, ht, 150.0, EXS)
    cs, ds = fpfh_center(hs)
    ct, dt = fpfh_center(ht)
    fd = np.diag(fpfh_fd32(cs, ds, ct, dt)).astype(np.float64)
    assert (fd < 8 * FF_G).any() and (fd > 8 * FF_G).any()
    assert g_ratio <= 1.0 and lb_ratio <= 1.0, (g_ratio, lb_ratio)


@pytest.mark.parametrize("k", [-40, -20, 0, 20, 40])
def test_fpfh_bound_across_scales(g, k):
    sc = scaled(g.synth.add_fpfh(g.synth.gen_points(90, 80, overlap=0.9, seed=9)), k)
    g_ratio, lb_ratio = check_fpfh_bound(sc.S, sc.T, sc.fpfh_s, sc.fpfh_t, sc.bbx_magnitude, EXS[::5])
    assert g_ratio <= 1.0 and lb_ratio <= 1.0, (g_ratio, lb_ratio)


# ---- near-tie scenes ---------------------------------------------------------------------------------------------------
def nominal_filter(ft, S, T, c, bbx, it):
    """The filter's distance term of the pairs (S[k], T[k]) with an exact sqrt (c = the target centroid).  The FD term is
    shared by a decoy and its target (same descriptor), so this orders the pair's cd32 like the kernel does."""
    x_s, x_t = S - c, T - c
    if ft == "fpfh":
        def split(x):
            hi = x.astype(F32)
            return hi, (x - hi.astype(np.float64)).astype(F32)
        (sh, sl), (th, tl) = split(x_s), split(x_t)
        d = [add32(add32(sh[:, k], -th[:, k]), add32(sl[:, k], -tl[:, k])) for k in range(3)]
        return np.sqrt(fma32(d[2], d[2], fma32(d[1], d[1], (d[0] * d[0]).astype(F32))).astype(np.float64))
    a = stream_weights(ft, it, bbx)[0]
    A = a * a
    ns = (x_s[:, 0] * x_s[:, 0] + x_s[:, 1] * x_s[:, 1]) + x_s[:, 2] * x_s[:, 2]
    nt = (x_t[:, 0] * x_t[:, 0] + x_t[:, 1] * x_t[:, 1]) + x_t[:, 2] * x_t[:, 2]
    acc = add32((A * nt).astype(F32), (A * ns).astype(F32))
    for k in (2, 1, 0):
        acc = fma32(x_s[:, k].astype(F32), ((-2.0 * A) * x_t[:, k]).astype(F32), acc)
    return np.sqrt(np.abs(acc).astype(np.float64))


def _ed(a, b):
    d = a - b
    return np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])


def near_tie_scene(g, ft, N, it, seed=31, max_decoys=None):
    """A gen_points scene plus one decoy target per chosen source row: a copy of the row's nearest target (same descriptor)
    at a LOWER index, moved straight away from the source by a few float32 ulps of its centred coordinates (k_stream), or by
    eighths of an ulp of the pair distance (the FPFH filter, whose hi/lo coordinates resolve the distance to about an ulp) until the float filter ranks it at or
    below the true nearest target, whose exact CD stays the smaller.  Returns (scene, rows the restated filter misranks)."""
    from scipy.spatial import cKDTree
    sc = g.synth.gen_points(N, N, overlap=0.9, extent=(60, 60, 12), noise=0.03, seed=seed)
    if ft == "bsc":
        g.synth.add_bsc(sc, bits=441, V=4)
    if ft == "fpfh":
        g.synth.add_fpfh(sc)
    S, T = np.array(sc.S), np.array(sc.T)
    nearest = cKDTree(T).query(S[: sc.n_overlap])[1]
    rows = np.unique(nearest, return_index=True)[1][: (max_decoys or N)]
    js = nearest[rows]
    u = T[js] - S[rows]
    u /= np.linalg.norm(u, axis=1, keepdims=True)
    D = len(rows)
    unit = (np.spacing(np.abs(T[js] - serial_mean(T)).max(axis=1).astype(F32)).astype(np.float64) if ft != "fpfh"
            else np.spacing(_ed(S[rows], T[js]).astype(F32)).astype(np.float64) / 8.0)
    steps = np.ones(D)

    def evaluate():
        T2 = np.vstack([T[js] + u * (steps * unit)[:, None], T])
        c = serial_mean(T2)
        f_dec = nominal_filter(ft, S[rows], T2[:D], c, sc.bbx_magnitude, it)
        f_true = nominal_filter(ft, S[rows], T2[D + js], c, sc.bbx_magnitude, it)
        return T2, (f_dec <= f_true) & (_ed(S[rows], T2[:D]) > _ed(S[rows], T2[D + js]))
    for _ in range(6):
        T2, ok = evaluate()
        steps = np.where(ok, steps, steps + 1 + (np.arange(D) % 3))
    T2, ok = evaluate()
    sc.T = np.asfortranarray(T2)
    if ft == "bsc":
        sc.bsc_t = np.vstack([sc.bsc_t[js], sc.bsc_t])
    if ft == "fpfh":
        sc.fpfh_t = np.ascontiguousarray(np.vstack([sc.fpfh_t[js], sc.fpfh_t]))
    return sc, int(ok.sum())


# the iteration a near-tie scene is built for and started at: None from 0; BSC at 1 (iteration 0 has no ED term, the
# copies would tie exactly); FPFH at 2, the first iteration of the NN filter route
START = {"none": 0, "bsc": 1, "fpfh": 2}


def run_near_ties(g, orc, ft, ct, N, iters=2, scene=None, with_oracle=True):
    """Against the all-double route iteration by iteration (identical pairs, Rt bit for bit) and the oracle: identical pairs
    for NN / NNR, the KM energy within n * KM_eps on the first iteration (the auction is eps-optimal, and a decoy is far
    closer than eps to its target).  The oracle's KM (Hungarian) runs up to 1000 keypoints."""
    it = START[ft]
    sc, misranked = scene or near_tie_scene(g, ft, N, it)
    print(f"\nnear ties {ft}-{ct} {sc.S.shape[0]}x{sc.T.shape[0]}: {misranked} rows misranked by the float filter")
    assert misranked > 0
    state = (it, 99999.0, 0.0, 0.0, 1.0, 1.0) if it else None
    if ct == "km":
        # one iteration: the auction's eps-optimal matching is not unique (a decoy lies far closer than KM_eps to its
        # target), so the routes agree on the graph and the objective, not on the pair list (DESIGN §4)
        n_eps = max(sc.S.shape[0], sc.T.shape[0]) * 0.01
        FT, CT = codes(g, ft, ct)
        fast = g.registration.from_scene(sc, FT, CT)
        slow = g.registration.from_scene(sc, FT, CT, force_exact=True)
        try:
            if state:
                fast.set_state(*state)
                slow.set_state(*state)
            a, b = fast.iterate(), slow.iterate()
        finally:
            fast.close()
            slow.close()
        # the penalty comes from the filter's statistics (~1e-8 relative): edges at the penalty may flip (DESIGN §3.1)
        assert a.nnz > 0 and abs(a.nnz - b.nnz) <= max(1, 1e-7 * b.nnz) and a.exact_fallback & 5 == 0, (a.nnz, b.nnz)
        assert abs(a.km_energy - b.km_energy) <= n_eps + 1e-6 * abs(b.km_energy), (a.km_energy, b.km_energy)
        if with_oracle and N <= 1000:
            o = oracle_for(orc, sc, ft, ct, 6)
            if state:
                o.set_state(*state)
            c = o.iterate()
            assert abs(a.km_energy - c.km_energy) <= n_eps + 1e-6 * abs(c.km_energy), (a.km_energy, c.km_energy)
        return [a]
    stats = lockstep(g, orc, sc, ft, ct, 6, iters, state=state, with_oracle=with_oracle)
    assert stats[0].candidates > 0 and stats[0].exact_fallback == 0, (stats[0].candidates, stats[0].exact_fallback)
    return stats


@pytest.fixture()
def ge(g, emu_library_path):
    from conftest import swap_in_library
    real = swap_in_library(g, emu_library_path)
    try:
        yield g
    finally:
        g.capi._lib = real


@pytest.fixture(autouse=True)
def no_hooks(monkeypatch):
    for k in ("GHICP_CAND_CAP_MAX", "GHICP_FPFH_EXACT", "GHICP_FPFH_MATRIX_FREE", "GHICP_EMU_SCHED", "GHICP_KM_GENERAL",
              "GHICP_KM_FILL", "GHICP_KM_XUSE_MAX"):
        monkeypatch.delenv(k, raising=False)


NEAR_TIE_CASES = [("none", "nn"), ("none", "nnr"), ("none", "km"), ("bsc", "nn"), ("bsc", "nnr"), ("bsc", "km"),
                  ("fpfh", "nn"), ("fpfh", "nnr")]


@pytest.mark.parametrize("ft,ct", NEAR_TIE_CASES)
def test_emulated_near_ties(ge, orc, scratch_cwd, ft, ct):
    run_near_ties(ge, orc, ft, ct, N=220 if ct != "km" else 120)


# ---- the scale sweep through the library ---------------------------------------------------------------------------
SWEEP_K = [-40, -20, -8, 0, 8, 20, 40]


def run_scale_sweep(g, orc, ft, ct, N, iters, ks=SWEEP_K):
    """Ft = None: CD = ED scales by 4^k exactly, so pair lists equal the k = 0 run's and R is bit-identical, t = 2^k t, as
    long as the reference's own scans still see the CDs: they start at MAXVALIUE = 9e20 and keep (9e20, 0) for a row
    whose CDs all lie above, which happens at 2^40 (the library and the oracle then agree on that).  KM only where the
    penalty max(CDmean, 1) and KM_eps (scaled with the run) keep the assignment problem the same, k >= 0, and only up to
    2^8: at 2^20 the auction's objective (fast and all-double routes alike) is no longer 4^k times the k = 0 one.
    Every run is also checked against force_exact (and for NN / NNR the oracle); outside the window the all-double route
    takes every iteration (exact_fallback bit 2)."""
    sc0 = g.synth.gen_points(N, N - 20, overlap=0.9, seed=11)
    if ft == "bsc":
        g.synth.add_bsc(sc0)
    if ft == "fpfh":
        g.synth.add_fpfh(sc0)
    FT, CT = codes(g, ft, ct)
    runs = {}
    for k in ks:
        sc = scaled(sc0, k)
        eps = 0.01 * 4.0 ** max(k, 0) if ct == "km" else 0.0     # KM_eps is absolute: scaled with large CDs
        fast = g.registration.from_scene(sc, FT, CT, km_eps=eps)
        slow = g.registration.from_scene(sc, FT, CT, km_eps=eps, force_exact=True)
        o = oracle_for(orc, sc, ft, ct, 6) if ct != "km" else None
        rec = []
        try:
            for _ in range(iters):
                a, b = fast.iterate(), slow.iterate()
                sp, tp = fast.pairs()
                esp, etp = slow.pairs()
                if ct == "km":
                    # same graph and objective; the eps-optimal matching is not unique (DESIGN §4), so the two routes'
                    # trajectories part after the first iteration
                    n_eps = max(len(sc.S), len(sc.T)) * (eps or 0.01)
                    assert abs(a.nnz - b.nnz) <= max(1, 1e-7 * b.nnz), (k, a.iteration, a.nnz, b.nnz)
                    assert abs(a.km_energy - b.km_energy) <= n_eps + 1e-6 * abs(b.km_energy), (k, a.iteration)
                    assert bool(a.exact_fallback & 4) == (abs(k) == 40 and ft == "none"), (k, a.exact_fallback)
                    rec.append((a.nnz, a.km_energy, n_eps))
                    break
                assert np.array_equal(sp, esp) and np.array_equal(tp, etp), (k, a.iteration)
                assert [float(x).hex() for x in a.Rt] == [float(x).hex() for x in b.Rt], (k, a.iteration)
                if o is not None:
                    o.iterate()
                    osp, otp = o.pairs()
                    assert np.array_equal(sp, osp) and np.array_equal(tp, otp), (k, a.iteration)
                # BSC iteration 0 has no ED term (A = 0): inside the window at any scale; FPFH has no window
                outside = abs(k) == 40 and ft != "fpfh" and not (ft == "bsc" and a.iteration == 0)
                assert bool(a.exact_fallback & 4) == outside, (k, a.iteration, a.exact_fallback)
                rec.append((sp, tp, np.array(a.Rt).reshape(4, 4)))
        finally:
            fast.close()
            slow.close()
        runs[k] = rec
    if ft != "none":
        return runs
    for k in ks:
        if k > 20 or (ct == "km" and not 0 <= k <= 8):
            continue
        if ct == "km":     # iteration 0: the same graph, and the objective scaled by 4^k
            (nnz, e, n_eps), (nnz0, e0, _) = runs[k][0], runs[0][0]
            assert nnz == nnz0 and abs(e - 4.0 ** k * e0) <= 2 * n_eps + 1e-6 * abs(e), (k, nnz, nnz0, e, e0)
            continue
        for it, ((sp, tp, Rt), (sp0, tp0, Rt0)) in enumerate(zip(runs[k], runs[0])):
            assert np.array_equal(sp, sp0) and np.array_equal(tp, tp0), (k, it)
            assert np.array_equal(Rt[:3, :3], Rt0[:3, :3]), (k, it)
            assert np.array_equal(Rt[:3, 3], Rt0[:3, 3] * 2.0 ** k), (k, it)
    return runs


@pytest.mark.parametrize("ft,ct", [("none", "nn"), ("none", "nnr"), ("none", "km"), ("bsc", "nn"), ("fpfh", "nnr")])
def test_emulated_scale_sweep(ge, orc, scratch_cwd, ft, ct):
    run_scale_sweep(ge, orc, ft, ct, N=120, iters=3)
