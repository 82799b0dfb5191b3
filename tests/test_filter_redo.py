"""The all-double redo of the NN / NNR filter routes (gh-icp_b200/csrc/ghicp_capi.cu: nn_tail sets RouteResult::exact_redo,
iterate_impl then runs route_exact on the same iteration and reports bit 0 of ghicp_iter_stats.exact_fallback).  Two
triggers send an iteration there:
  * candidate-buffer overflow: more pairs within the filter margin of a row / column minimum than cand_cap holds
    (push_candidate / ff_push set StreamDev::overflow, k_publish / k_ff_publish hand it to k_penalty as
    DevIter::overflow_any);
  * the NN gate's error band (Stream route, Ft = None and BSC iterations 0-1): a row minimum within 1e-5 * max(1, |penalty|)
    of the penalty taken from the FP32-filtered statistics (k_select_count: DevIter::ambiguous).

Cases:
  a. GHICP_CAND_CAP_MAX=16 on the iteration-route scene: every filter iteration overflows (CPU and GPU);
  b. overflow from real ties: 8 sites x 512 exact target copies, no hook (GPU);
  c. one row minimum planted at penalty * (1 +- 1e-9), with controls at 0.5e-5 (still in the band) and 2e-5 (outside);
     the KM counterpart, which has no redo (CPU and GPU);
  d. far outliers (a target keypoint 2 km / 40 km out, or UTM-like coordinates with a glitch point at the origin): the filter
     margin grows with the cloud's radius and the candidate counts with it (CPU at small size, GPU at 3000 x 3000);
  e. more than 2^31 candidate pushes in one pass: the saturating counters keep the slot index in range (GPU).

Comparison rule: against the library's own all-double run (force_exact) iteration by iteration, identical pair lists,
bit-identical Rt, Rt_tillnow and moved source, and on every redone iteration cd_mean, cd_std and penalty equal as float.hex
(both runs then take route_exact on the same inputs); against the oracle, identical pair lists (FPFH: at most one iteration
may differ, CUDA and glibc pow differ in the last ulp)."""
import math

import numpy as np
import pytest

CAP = 16                      # GHICP_CAND_CAP_MAX of case a
RESIDENT = 132 * 2048         # threads resident at once on an H100 (132 SMs x 2048): the saturating counters' overshoot bound
ITERS = 8


def _hex(xs):
    return [float(x).hex() for x in xs]


def cand_cap(N, M):
    """The candidate buffer's capacity on one GPU (ghicp_capi.cu, next to its allocation)."""
    return min(96 * max(N, M) + (1 << 20), 1 << 28)


def codes(m, ft, ct):
    return ({"none": m.FT_NONE, "bsc": m.FT_BSC, "fpfh": m.FT_FPFH}[ft], {"nn": m.CT_NN, "nnr": m.CT_NNR, "km": m.CT_KM}[ct])


def oracle_for(orc, sc, ft, ct, dof):
    FT, CT = codes(orc, ft, ct)
    o = orc.Oracle(FT, CT, dof=dof, bbx_magnitude=sc.bbx_magnitude, solve_mode=1)
    o.set_keypoints(sc.S, sc.T)
    if ft == "bsc":
        o.set_bsc(sc.bsc_s, sc.bsc_t, sc.bits)
    if ft == "fpfh":
        o.set_fpfh(sc.fpfh_s, sc.fpfh_t)
    o.build_fd()
    return o


def check_against_all_double(a, b, fast, slow, at):
    """The comparison rule against the force_exact run; returns the fast run's pairs."""
    sp, tp = fast.pairs()
    esp, etp = slow.pairs()
    assert np.array_equal(sp, esp) and np.array_equal(tp, etp), at
    assert a.cor == b.cor, at
    assert _hex(a.Rt) == _hex(b.Rt) and _hex(a.Rt_tillnow) == _hex(b.Rt_tillnow), at
    assert np.array_equal(fast.source(), slow.source()), at
    assert b.exact_fallback == 0, at
    if a.exact_fallback & 1:      # redone: route_exact's statistics, not the filter's
        assert _hex((a.cd_mean, a.cd_std, a.penalty)) == _hex((b.cd_mean, b.cd_std, b.penalty)), at
    return sp, tp


def lockstep(g, orc, sc, ft, ct, dof, iters, state=None, with_oracle=True, on_pairs=None):
    """fast (default routes), slow (force_exact) and the oracle side by side; returns the fast run's stats per iteration."""
    FT, CT = codes(g, ft, ct)
    fast = g.registration.from_scene(sc, FT, CT, dof=dof)
    slow = g.registration.from_scene(sc, FT, CT, dof=dof, force_exact=True)
    o = oracle_for(orc, sc, ft, ct, dof) if with_oracle else None
    out, n_mismatch = [], 0
    try:
        if state is not None:
            for r in (fast, slow) + ((o,) if o else ()):
                r.set_state(*state)
        for _ in range(iters):
            a, b = fast.iterate(), slow.iterate()
            at = (ft, ct, dof, a.iteration)
            sp, tp = check_against_all_double(a, b, fast, slow, at)
            if on_pairs:
                on_pairs(a, sp, tp)
            if o is not None:
                o.iterate()
                osp, otp = o.pairs()
                if not (np.array_equal(sp, osp) and np.array_equal(tp, otp)):
                    n_mismatch += 1
            out.append(a)
    finally:
        fast.close()
        slow.close()
    assert n_mismatch <= (1 if ft == "fpfh" else 0), n_mismatch
    return out


def is_filter_iteration(ft, ct, it):
    """FPFH NN takes the all-double route in iterations 0-1 (its penalty needs the CD mean there)."""
    return not (ft == "fpfh" and ct == "nn" and it < 2)


# ---- a. forced overflow ------------------------------------------------------------------------------------------------------
# the scene of tests/test_iteration_routes.py
REDO_CASES = {
    "none_nn": ("none", "nn", 6), "none_nnr": ("none", "nnr", 6),
    "bsc_nn": ("bsc", "nn", 6), "bsc_nnr": ("bsc", "nnr", 6), "bsc_nn_dof4": ("bsc", "nn", 4), "bsc_nnr_dof4": ("bsc", "nnr", 4),
    "fpfh_nn": ("fpfh", "nn", 6), "fpfh_nnr": ("fpfh", "nnr", 6),
}


def route_scene(g, ft, dof, N=260, M=230):
    sc = g.synth.gen_points(N, M, overlap=0.9, seed=11)
    if ft == "bsc":
        g.synth.add_bsc(sc, V=4 if dof == 6 else 2)
    if ft == "fpfh":
        g.synth.add_fpfh(sc)
    return sc


def run_forced_overflow(g, orc, monkeypatch, name, slack):
    """slack: how far a saturated counter may pass the cap (threads that read it below the cap before it got there)."""
    ft, ct, dof = REDO_CASES[name]
    monkeypatch.setenv("GHICP_CAND_CAP_MAX", str(CAP))
    stats = lockstep(g, orc, route_scene(g, ft, dof), ft, ct, dof, ITERS)
    for a in stats:
        at = (name, a.iteration)
        if is_filter_iteration(ft, ct, a.iteration):
            assert a.exact_fallback & 1, at
            assert CAP <= a.candidates <= (CAP + slack) * (2 if ct == "nnr" else 1), (at, a.candidates)
        else:
            assert a.exact_fallback == 0 and a.candidates == 0, at


def run_partial_overflow(g, orc, monkeypatch):
    """A cap between the candidate counts of the first iterations (pre-pass, loose seeds) and the later ones: redone
    iterations are followed by filter iterations that keep their own result (seeds and have_prev come from the redo).  The
    cap is the largest count of iterations 3+ of an unhooked run, which the hooked run repeats (a redo reproduces the
    filter's result)."""
    sc = route_scene(g, "none", 6)
    reg = g.registration.from_scene(sc, g.FT_NONE, g.CT_NN)
    try:
        counts = [reg.iterate().candidates for _ in range(ITERS)]
    finally:
        reg.close()
    cap = max(counts[3:])
    assert max(counts[:3]) > cap, counts
    monkeypatch.setenv("GHICP_CAND_CAP_MAX", str(cap))
    stats = lockstep(g, orc, sc, "none", "nn", 6, ITERS)
    redone = [bool(a.exact_fallback & 1) for a in stats]
    for a, r in zip(stats, redone):
        assert a.candidates >= cap if r else a.candidates <= cap, (a.iteration, a.candidates, cap)
    assert any(redone[k] and not redone[k + 1] for k in range(len(redone) - 1)), [(a.candidates, r) for a, r in zip(stats, redone)]


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(REDO_CASES))
def test_forced_overflow_redo_equals_all_double_and_oracle(g, orc, monkeypatch, name):
    run_forced_overflow(g, orc, monkeypatch, name, slack=RESIDENT)


@pytest.mark.gpu
def test_iteration_after_a_redo(g, orc, monkeypatch):
    run_partial_overflow(g, orc, monkeypatch)


# ---- c. the NN gate's error band ----------------------------------------------------------------------------------------------
def numpy_fd(bs, bt, bits, V):
    s = np.unpackbits(bs[:V], axis=-1, bitorder="little")[..., :bits].astype(np.float64)
    t = np.unpackbits(bt, axis=-1, bitorder="little")[..., :bits].astype(np.float64)
    return np.min([s[v].sum(1)[:, None] + t.sum(1)[None, :] - 2.0 * (s[v] @ t.T) for v in range(V)], axis=0)


def band_scene(g, ft, N, rel, seed=5):
    """A scene (overlap 1: every other row minimum lies far below the penalty) in which source row N-1, moved along +z,
    has its exact minimum CD at penalty * (1 + rel) in the iteration under test: 0 for Ft = None (penalty = max(CDmean, 1)),
    1 for BSC (penalty = max(CDmean - 2 CDstd, 5)).  The row itself moves the statistics, so the bisection is on
    rowmin(t) / penalty(t) - 1 - rel; bbx_magnitude stays that of the unmoved scene."""
    sc = g.synth.gen_points(N, N, overlap=1.0, extent=(60, 60, 12), noise=0.03, seed=seed)
    it = 0 if ft == "none" else 1
    scale = float(np.float32(0.005 * sc.bbx_magnitude))
    wfd = math.exp(-it / 6.0) if ft == "bsc" else 0.0
    fd = 0.0
    if ft == "bsc":
        g.synth.add_bsc(sc, bits=441, V=4)
        fd = numpy_fd(sc.bsc_s, sc.bsc_t, 441, 4)

    def cd(S):
        d = np.sqrt(((S[:, None, :] - sc.T[None, :, :]) ** 2).sum(-1))
        return (1.0 - wfd) * scale * d + wfd * fd if ft == "bsc" else scale * d

    k = N - 1
    CD = cd(sc.S)
    s1, s2, nm = CD[:k].sum(), (CD[:k] ** 2).sum(), float(N * N)
    p0 = np.array(sc.S[k])
    fdk = fd[k] if ft == "bsc" else 0.0

    def f(t):
        p = p0 + [0.0, 0.0, t]
        row = np.sqrt(((p[None, :] - sc.T) ** 2).sum(-1))
        row = (1.0 - wfd) * scale * row + wfd * fdk if ft == "bsc" else scale * row
        S1, S2 = s1 + row.sum(), s2 + (row ** 2).sum()
        mean = S1 / nm
        pen = max(mean - 2.0 * math.sqrt(max(S2 / nm - mean * mean, 0.0)), 5.0) if ft == "bsc" else max(mean, 1.0)
        return row.min() / pen - 1.0 - rel

    lo, hi = 0.0, 1.0
    assert f(lo) < 0
    while f(hi) <= 0:
        hi *= 2.0
    for _ in range(200):
        mid = 0.5 * (lo + hi)
        if f(mid) <= 0:
            lo = mid
        else:
            hi = mid
    S = np.array(sc.S)
    S[k] = p0 + [0.0, 0.0, hi]
    sc.S = np.asfortranarray(S)
    return sc, it


def band_state(it):
    return (it, 99999.0, 0.0, 0.0, 1.0, 1.0)      # iterations 0-1: the penalty comes from this iteration's CD statistics


# offset from the penalty (relative) -> is the row inside the band (bit 0 of exact_fallback)?
BAND_OFFSETS = [(-1e-9, True), (1e-9, True), (-0.5e-5, True), (0.5e-5, True), (-2e-5, False), (2e-5, False)]


def run_gate_band(g, orc, ft, rel, in_band, N):
    sc, it = band_scene(g, ft, N, rel)
    k = N - 1
    o = oracle_for(orc, sc, ft, "nn", 6)
    o.set_state(*band_state(it))
    c = o.iterate()
    got = o.cd()[k].min() / c.penalty - 1.0
    assert abs(got - rel) <= 0.05 * abs(rel), (got, rel)      # the planted distance, by the oracle's own arithmetic
    kept = k in o.pairs()[0]
    assert kept == (rel < 0)                                    # CD < penalty keeps the pair (strict)

    def row_decision(a, sp, tp):
        assert (k in sp) == kept, (ft, rel)
        assert bool(a.exact_fallback & 1) == in_band, (ft, rel, a.exact_fallback)

    lockstep(g, orc, sc, ft, "nn", 6, 1, state=band_state(it), on_pairs=row_decision)


@pytest.mark.gpu
@pytest.mark.parametrize("ft", ["none", "bsc"])
@pytest.mark.parametrize("rel,in_band", BAND_OFFSETS)
def test_gate_band_redo_keeps_the_oracles_decision(g, orc, ft, rel, in_band):
    run_gate_band(g, orc, ft, rel, in_band, N=1000)


def run_km_band(g, orc, rel, N, eps=0.01):
    """KM (general route, Ft = None, iteration 0) takes no redo: an edge at penalty * (1 +- 1e-9) may flip with the FP32
    statistics; DESIGN promises nnz within 1 of the oracle's count and the energy within n * KM_eps."""
    sc, _ = band_scene(g, "none", N, rel)
    o = oracle_for(orc, sc, "none", "km", 6)
    reg = g.registration.from_scene(sc, g.FT_NONE, g.CT_KM, km_eps=eps)
    try:
        a, c = reg.iterate(), o.iterate()
    finally:
        reg.close()
    nnz = int((o.cd() < c.penalty).sum())
    assert abs(a.nnz - nnz) <= 1, (a.nnz, nnz)
    assert abs(a.km_energy - c.km_energy) <= N * eps + 1e-6 * abs(c.km_energy), (a.km_energy, c.km_energy)
    assert a.exact_fallback == 0


@pytest.mark.gpu
@pytest.mark.parametrize("rel", [-1e-9, 1e-9])
def test_gate_band_km_within_its_promise(g, orc, scratch_cwd, rel):
    run_km_band(g, orc, rel, N=1000)


# ---- d. far outliers -----------------------------------------------------------------------------------------------------------
UTM = (5e5, 4.1e6, 50.0)


def outlier_scene(g, ft, N, M, kind, seed=3):
    """gen_points (a 100 m cloud) with one more target keypoint: 2 km or 40 km from the target centroid, or (kind "utm") both
    clouds moved to UTM-like coordinates, rounded to float32 as a scanner's points are, and a glitch point at the origin."""
    sc = g.synth.gen_points(N, M - 1, overlap=0.9, extent=(100, 100, 20), noise=0.03, seed=seed)
    S, T = np.array(sc.S), np.array(sc.T)
    if kind == "utm":
        S = (S + UTM).astype(np.float32).astype(np.float64)
        T = np.vstack([(T + UTM).astype(np.float32).astype(np.float64), [0.0, 0.0, 0.0]])
    else:
        far = {"2km": 2e3, "40km": 4e4}[kind]
        T = np.vstack([T, (T.mean(axis=0) + [far, 0.0, 0.0]).astype(np.float32)])
    sc.S, sc.T = np.asfortranarray(S), np.asfortranarray(T)
    if ft == "bsc":
        g.synth.add_bsc(sc, bits=441, V=4)
    return sc


def run_far_outlier(g, orc, ft, ct, kind, N, M, iters=5):
    sc = outlier_scene(g, ft, N, M, kind)
    cap = cand_cap(N, M)
    stats = lockstep(g, orc, sc, ft, ct, 6, iters)
    print(f"\n{ft}-{ct} {kind} {N}x{M} (cap {cap}): candidates / exact_fallback per iteration:",
          [(a.candidates, a.exact_fallback) for a in stats])
    for a in stats:
        assert a.candidates >= 0, a.iteration
        if a.candidates >= cap:
            assert a.exact_fallback & 1, a.iteration


OUTLIER_CASES = [("none", "nn", "2km"), ("none", "nnr", "40km"), ("bsc", "nn", "utm"), ("bsc", "nnr", "2km"), ("none", "nn", "utm")]


@pytest.mark.gpu
@pytest.mark.parametrize("ft,ct,kind", OUTLIER_CASES)
def test_far_outlier_pairs_equal_oracle(g, orc, ft, ct, kind):
    run_far_outlier(g, orc, ft, ct, kind, 3000, 3000)


# ---- b. overflow from exact ties ------------------------------------------------------------------------------------------------
def tie_scene(g, ft, n_sites=8, copies=512, N=4096, seed=21):
    """Targets: n_sites non-coplanar sites, each copied `copies` times (shuffled); sources: N noisy points around the sites.
    Every row has >= `copies` exactly tied minima (same point, same descriptor), so a pass pushes >= N * copies candidates."""
    rng = np.random.default_rng(seed)
    sites = (rng.random((n_sites, 3)) * [40.0, 40.0, 10.0]).astype(np.float32).astype(np.float64)
    labels = rng.permutation(np.repeat(np.arange(n_sites), copies))
    src = rng.integers(0, n_sites, N)
    T = sites[labels]
    S = (sites[src] + rng.normal(0.0, 0.3, (N, 3))).astype(np.float32).astype(np.float64)
    ext = (S.max(axis=0) - S.min(axis=0)).astype(np.float32)
    sc = g.synth.Scene(S=np.asfortranarray(S), T=np.asfortranarray(T), bbx_magnitude=float(np.float32(ext.sum())),
                       R_gt=np.eye(3), t_gt=np.zeros(3), n_overlap=0, perm=np.zeros(0, np.int64), meta=dict(seed=seed))
    if ft == "bsc":
        bits = 441
        site_bits = rng.random((n_sites, bits)) < 0.35
        sb = np.stack([site_bits[src] ^ (rng.random((N, bits)) < 0.08) for _ in range(4)])
        sc.bsc_s, sc.bsc_t, sc.bits = g.synth.pack_bits(sb), g.synth.pack_bits(site_bits[labels]), bits
    if ft == "fpfh":
        h = rng.gamma(0.6, 1.0, size=(n_sites, 3, 11))
        h = (100.0 * h / h.sum(axis=2, keepdims=True)).reshape(n_sites, 33)
        sc.fpfh_t = np.ascontiguousarray(h[labels].astype(np.float32))
        sc.fpfh_s = np.ascontiguousarray(np.clip(h[src] + rng.normal(0.0, 2.0, (N, 33)), 0.0, None).astype(np.float32))
    first = np.array([np.flatnonzero(labels == s)[0] for s in range(n_sites)])
    return sc, first[labels]


TIE_CASES = [("none", "nn"), ("none", "nnr"), ("bsc", "nn"), ("bsc", "nnr"), ("fpfh", "nn"), ("fpfh", "nnr")]


def run_ties(g, orc, ft, ct, iters=3, **kw):
    sc, first_copy = tie_scene(g, ft, **kw)

    def first_minimum(a, sp, tp):
        assert np.array_equal(tp, first_copy[tp]), a.iteration      # the smallest index among the tied copies
        if is_filter_iteration(ft, ct, a.iteration):
            assert a.exact_fallback & 1, a.iteration

    lockstep(g, orc, sc, ft, ct, 6, iters, on_pairs=first_minimum)


@pytest.mark.gpu
@pytest.mark.parametrize("ft,ct", TIE_CASES)
def test_tied_copies_overflow_and_keep_the_first_minimum(g, orc, ft, ct):
    run_ties(g, orc, ft, ct)


# ---- e. beyond 2^31 pushes ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_more_than_2_31_candidate_pushes(g):
    """48 000 x 48 000, Ft = None NN, a 100 m cloud at UTM-like coordinates with a glitch target at the origin: the margin
    (~1.4e-3 x the cloud's 4e6 m radius) covers every pair, ~2.3e9 pushes in the main pass.  The counters saturate near the
    cap instead of wrapping to a negative slot."""
    N = M = 48000
    sc = outlier_scene(g, "none", N, M, "utm")
    cap = cand_cap(N, M)
    fast = g.registration.from_scene(sc, g.FT_NONE, g.CT_NN)
    slow = g.registration.from_scene(sc, g.FT_NONE, g.CT_NN, force_exact=True)
    try:
        a, b = fast.iterate(), slow.iterate()
        check_against_all_double(a, b, fast, slow, "48k")
    finally:
        fast.close()
        slow.close()
    print(f"\n48k x 48k UTM + glitch: candidates {a.candidates} (cap {cap}), exact_fallback {a.exact_fallback}, "
          f"ms_stream {a.ms_stream:.1f}, ms_total {a.ms_total:.1f}")
    assert a.exact_fallback & 1
    assert cap <= a.candidates <= cap + RESIDENT


# ---- the same functions on the emulated library (CPU) ---------------------------------------------------------------------------
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
    for k in ("GHICP_CAND_CAP_MAX", "GHICP_FPFH_EXACT", "GHICP_FPFH_MATRIX_FREE", "GHICP_EMU_SCHED"):
        monkeypatch.delenv(k, raising=False)


@pytest.mark.parametrize("name", list(REDO_CASES))
def test_emulated_forced_overflow(ge, orc, monkeypatch, name):
    # one block at a time, and no fiber switch between the counter's read and its increment: the counters stop at the cap
    run_forced_overflow(ge, orc, monkeypatch, name, slack=0)


def test_emulated_iteration_after_a_redo(ge, orc, monkeypatch):
    run_partial_overflow(ge, orc, monkeypatch)


@pytest.mark.parametrize("ft", ["none", "bsc"])
@pytest.mark.parametrize("rel,in_band", BAND_OFFSETS)
def test_emulated_gate_band(ge, orc, ft, rel, in_band):
    run_gate_band(ge, orc, ft, rel, in_band, N=400)


@pytest.mark.parametrize("rel", [-1e-9, 1e-9])
def test_emulated_gate_band_km(ge, orc, scratch_cwd, rel):
    run_km_band(ge, orc, rel, N=150)


@pytest.mark.parametrize("ft,ct,kind", OUTLIER_CASES)
def test_emulated_far_outlier(ge, orc, ft, ct, kind):
    run_far_outlier(ge, orc, ft, ct, kind, 300, 280, iters=3)


@pytest.mark.parametrize("ft,ct", TIE_CASES)
def test_emulated_ties(ge, orc, monkeypatch, ft, ct):
    # 4 sites x 100 copies, 300 sources: >= 30 000 tied pushes per pass, against a cap lowered to 20 000 (at this size the
    # real cap, 96 * 400 + 2^20, is never reached)
    monkeypatch.setenv("GHICP_CAND_CAP_MAX", "20000")
    run_ties(ge, orc, ft, ct, n_sites=4, copies=100, N=300)
