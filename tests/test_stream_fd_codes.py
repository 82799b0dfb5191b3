"""k_stream's decode of the packed BSC feature-distance plane (gh-icp_b200/csrc/ghicp_stream.cu: fd_pair and the two
arithmetic branches of compute_row) over the whole code range 0 ... bits, for every plane width hb.

The descriptors of gh-icp_b200/synth.py give Hamming distances in a narrow band (about 20 ... 330): no code >= 512, and at
<= 511 bits no code >= 256, ever reaches the stream kernel through them.  The scenes here use thermometer descriptors
instead (`fullrange_scene`): keypoint k has ones at the bit positions [0, level_k), then every descriptor goes through one
shared bit permutation and XOR mask, which keep Hamming distances, so FD(i, j) ~ min_v |level_{v,i} - level_j| can be put
anywhere in 0 ... bits.  Target levels sit in the top eighth [bits - bits / 8, bits]; most unmatched source rows sit more than
256 below all of them, so the iteration-0 row minima (CD = FD there) and everything within the filter margin of them carry
high codes; matched source rows are copies of their target with a few flipped bits; planted pairs give the codes 0 and `bits`.
`assert_coverage` checks, from the oracle's plane, that each scene really carries those codes.

  * the generator against numpy Hamming distances, and its coverage, for every `bits` (CPU);
  * both FD builders (wgmma, GHICP_FD_POPC=1) against the oracle on these planes (GPU);
  * stream NN / NNR against the all-double path (force_exact) and the oracle from iterations 0, 1, 2, 3, 58, 59, 60 and 75:
    the fp16-weight branch (X2) up to iteration 58, the scalar-weight branch from 59 on (WFD = e^(-it/6) < 6.2e-5), each
    start with its pre-pass and then a seeded sweep;
  * stream KM (general route with the edge list and with the fill pass, settled route from iteration 2 and across 58 -> 60);
  * lock-step registrations, one per hb;
  * the same test functions at reduced sizes on the emulated library (CPU), which checks the decode, the branch logic and the
    statistics; only the GPU run checks the rounding of sqrt.approx (the emulator takes the exact root)."""
import math

import numpy as np
import pytest

BITS = [255, 256, 441, 511, 512, 672, 1023, 1024, 1500, 2048]   # both sides of every hb boundary, and code 0x800
STARTS = (0, 1, 2, 3, 58, 59, 60, 75)                             # 58 -> 59: the X2 / scalar-weight switch
KM_EPS = 0.01


# ---- full-range descriptors -------------------------------------------------------------------------------------------------
def fullrange_scene(g, N, M, bits, V, seed, extent=(60, 60, 12)):
    """A synth.gen_points scene (overlap 0.4) with thermometer BSC descriptors spanning FD = 0 ... bits (module docstring)."""
    sc = g.synth.gen_points(N, M, overlap=0.4, extent=extent, noise=0.03, seed=seed)
    rng = np.random.default_rng(seed * 7 + bits)
    K = sc.n_overlap
    pos = np.arange(bits)
    W = max(8, bits // 8)
    L = bits - W                                                   # target levels in [L, bits]

    def thermo(levels, flips):
        x = pos < np.asarray(levels)[..., None]
        for idx in np.ndindex(x.shape[:-1]):
            f = flips[idx]
            if f:
                x[idx + (rng.choice(bits, f, replace=False),)] ^= True
        return x

    tb = thermo(L + rng.integers(0, W + 1, M), rng.integers(0, 4, M))
    # unmatched rows: 70 % spread evenly over [0, L - 264] (every row minimum >= 256 where bits allows it), the rest over [0, L]
    n_far = int(round(0.7 * N))
    far = rng.permutation(np.round(np.linspace(0, max(0, L - 264), n_far)).astype(np.int64))
    base = np.concatenate([far, rng.integers(0, L + 1, N - n_far)])[rng.permutation(N)]
    levels = np.clip(base[None, :] - rng.integers(0, 17, (V, N)), 0, bits)
    sb = thermo(levels, rng.integers(0, 4, (V, N)))
    # matched rows: variant 0 is the partner's descriptor with 0 ... 3 flipped bits
    for i in range(K):
        sb[0, i] = tb[sc.perm[i]]
        sb[0, i, rng.choice(bits, rng.integers(0, 4), replace=False)] ^= True
    # planted codes: `bits` on an nc x nc block (source level 0 in every variant, target level bits), 0 at (N - 1, 0)
    nc = max(1, min(N, M) // 32)
    sb[:, :nc] = False
    tb[M - nc:] = True
    sb[0, N - 1] = tb[0]
    perm, mask = rng.permutation(bits), rng.random(bits) < 0.5
    sc.bsc_s = g.synth.pack_bits(sb[..., perm] ^ mask)
    sc.bsc_t = g.synth.pack_bits(tb[..., perm] ^ mask)
    sc.bits = bits
    return sc


def numpy_fd(bs, bt, bits, V):
    """min over the first V variants of the Hamming distances, from unpacked bits (exact in float32: counts <= 2048)."""
    s = np.unpackbits(bs[:V], axis=-1, bitorder="little")[..., :bits].astype(np.float32)
    t = np.unpackbits(bt, axis=-1, bitorder="little")[..., :bits].astype(np.float32)
    d = [s[v].sum(1)[:, None] + t.sum(1)[None, :] - 2.0 * (s[v] @ t.T) for v in range(V)]
    return np.min(d, axis=0).astype(np.float64)


def assert_coverage(fd, bits):
    """The plane carries 0 and `bits`, every value of the high-bit field, and high iteration-0 row minima."""
    codes = fd.astype(np.int64)
    assert codes.min() == 0 and codes.max() == bits
    assert set(np.unique(codes >> 8).tolist()) == set(range(bits // 256 + 1)), "high-bit field values"
    rowmin = codes.min(axis=1)
    if bits > 256:                     # (at <= 256 bits the only code >= 256 is `bits` itself)
        assert (rowmin >= 256).mean() >= 0.25, np.percentile(rowmin, [25, 50, 75])
    if bits >= 512:                    # hb >= 2: row minima with every high-bit value up to 3 bits / 4
        got = set(np.unique(rowmin >> 8).tolist())
        assert set(range((3 * bits // 4 >> 8) + 1)) <= got, sorted(got)


def dof_of(V):
    return 6 if V == 4 else 4


def oracle_for(orc, sc, ct, V, **kw):
    o = orc.Oracle(orc.FT_BSC, ct, dof=dof_of(V), bbx_magnitude=sc.bbx_magnitude, solve_mode=1, **kw)
    o.set_keypoints(sc.S, sc.T)
    o.set_bsc(sc.bsc_s, sc.bsc_t, sc.bits)
    o.build_fd()
    return o


def resync_oracle(o, sc, S):
    o.set_keypoints(S, sc.T)
    o.set_bsc(sc.bsc_s, sc.bsc_t, sc.bits)
    o.build_fd()


def iteration_cd(sc, fd, it):
    """The reference's CD at iteration `it` (WFD = e^(-it/6), scale = 0.005 * bbx as a float)."""
    wfd = math.exp(-it / 6.0)
    scale = float(np.float32(0.005 * sc.bbx_magnitude))
    d = np.sqrt(((sc.S[:, None, :] - sc.T[None, :, :]) ** 2).sum(-1))
    return (1.0 - wfd) * scale * d + wfd * fd, scale, 1.0 - wfd


def start_state(sc, fd, it, quantile_rows=0.5, cells=None):
    """set_state arguments for a start at iteration `it`.  From iteration 2 on the penalty is RMS * scale * WED (FDM = FDstd
    = 0, para1 = para2 = 1): RMS is chosen to put it at the median row minimum of that iteration's CD (or, with `cells`, at
    the cells-th smallest CD: a sparse KM graph)."""
    if it <= 1:
        return (it, 99999.0, 0.0, 0.0, 1.0, 1.0)     # penalty from this iteration's CD statistics
    cd, scale, wed = iteration_cd(sc, fd, it)
    p = np.sort(cd, axis=None)[cells] if cells is not None else np.quantile(cd.min(axis=1), quantile_rows)
    return (it, float(p) / (scale * wed), 0.0, 0.0, 1.0, 1.0)


# ---- the generator ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", BITS)
@pytest.mark.parametrize("V", [4, 2])
def test_generator_covers_the_code_range(g, orc, bits, V):
    sc = fullrange_scene(g, 300, 281, bits, V, seed=bits + V)
    o = oracle_for(orc, sc, orc.CT_NN, V)
    fd = o.fd()
    assert np.array_equal(fd, numpy_fd(sc.bsc_s, sc.bsc_t, bits, V))
    assert fd[sc.S.shape[0] - 1, 0] == 0 and fd[0, sc.T.shape[0] - 1] == bits
    assert_coverage(fd, bits)


# ---- the FD builders ----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("bits", BITS)
@pytest.mark.parametrize("V", [4, 2])
def test_builders_equal_the_oracle_on_full_range_planes(g, orc, monkeypatch, bits, V, N=333, M=530):
    sc = fullrange_scene(g, N, M, bits, V, seed=bits + 3 * V)
    ref = oracle_for(orc, sc, orc.CT_NN, V).fd()
    if N >= 64:
        assert_coverage(ref, bits)
    for popc in (False, True):
        if popc:
            monkeypatch.setenv("GHICP_FD_POPC", "1")
        reg = g.registration.from_scene(sc, g.FT_BSC, g.CT_NN, dof=dof_of(V))
        try:
            assert np.array_equal(reg.fd(), ref), "popc" if popc else "wgmma"
        finally:
            reg.close()
            monkeypatch.delenv("GHICP_FD_POPC", raising=False)


# ---- stream NN / NNR ------------------------------------------------------------------------------------------------------------
# M > 2048, M % 256 != 0: two column CTAs and a partial panel; N % 4 != 0, N > 256: a partial quad and several row blocks
GPU_SHAPES = [(300, 2305), (1030, 500), (257, 255), (5, 3)]


@pytest.mark.gpu
@pytest.mark.parametrize("bits", BITS)
@pytest.mark.parametrize("ct", ["nn", "nnr"])
@pytest.mark.parametrize("N,M", GPU_SHAPES)
def test_stream_nn_nnr_equals_all_double_and_oracle(g, orc, bits, ct, N, M, V=4, starts=STARTS):
    CT = {"nn": g.CT_NN, "nnr": g.CT_NNR}[ct]
    sc = fullrange_scene(g, N, M, bits, V, seed=N + M + bits)
    fast = g.registration.from_scene(sc, g.FT_BSC, CT, dof=dof_of(V))
    slow = g.registration.from_scene(sc, g.FT_BSC, CT, dof=dof_of(V), force_exact=True)
    o = oracle_for(orc, sc, CT, V)
    fd = o.fd()
    if N >= 64:
        assert_coverage(fd, bits)
    n_fallback = 0
    try:
        for it0 in starts:
            state = start_state(sc, fd, it0)
            for r in (fast, slow):
                r.reset()                       # iteration 0, no previous partners: the first iteration runs the pre-pass
                r.set_keypoints(sc.S, sc.T)
                r.set_state(*state)
            resync_oracle(o, sc, sc.S)
            o.set_state(*state)
            for k in range(2):                  # pre-pass + sweep, then the seeded sweep
                a, b, c = fast.iterate(), slow.iterate(), o.iterate()
                at = (it0, k)
                assert a.iteration == b.iteration == c.iteration == it0 + k, at
                sp, tp = fast.pairs()
                esp, etp = slow.pairs()
                osp, otp = o.pairs()
                assert np.array_equal(sp, esp) and np.array_equal(tp, etp), at
                assert np.array_equal(sp, osp) and np.array_equal(tp, otp), at
                assert a.cor == b.cor == c.cor, at
                assert np.array_equal(np.array(a.Rt), np.array(b.Rt)), at
                assert a.cd_mean == pytest.approx(b.cd_mean, rel=2e-6), at
                assert a.cd_std == pytest.approx(b.cd_std, rel=1e-5), at
                # iterations 0-1: penalty = mean - 2 std, whose error is that of the statistics, not a fraction of the
                # difference (a 5 x 3 plane at iteration 1: 12.9038 from terms of ~ 150)
                assert abs(a.penalty - b.penalty) <= 1e-5 * max(abs(b.penalty), b.cd_mean + 2.0 * b.cd_std), at
                assert b.cd_mean == pytest.approx(c.cd_mean, rel=1e-9) and b.penalty == pytest.approx(c.penalty, rel=1e-8), at
                assert a.stream_passes > 0, at
                assert b.exact_fallback == 0, at
                n_fallback += a.exact_fallback
    finally:
        fast.close()
        slow.close()
    assert n_fallback <= 2


# ---- stream KM --------------------------------------------------------------------------------------------------------------------
def _km_lockstep(g, orc, sc, V, state, n_iter, settled_from):
    """Stream KM, force_exact KM and the oracle from `state`, re-synchronised after every iteration on the stream context's
    source and state (eps-optimal matchings are not unique).  Returns the stream iterations' stats."""
    n = max(sc.S.shape[0], sc.T.shape[0])
    fast = g.registration.from_scene(sc, g.FT_BSC, g.CT_KM, dof=dof_of(V))
    slow = g.registration.from_scene(sc, g.FT_BSC, g.CT_KM, dof=dof_of(V), force_exact=True)
    o = oracle_for(orc, sc, orc.CT_KM, V)
    out = []
    try:
        for r in (fast, slow, o):
            r.set_state(*state)
        for k in range(n_iter):
            a, b, c = fast.iterate(), slow.iterate(), o.iterate()
            it = state[0] + k
            assert a.iteration == b.iteration == it, it
            if it >= 2:        # the penalty comes from the state, not from this iteration's FP32 statistics
                assert a.nnz == b.nnz and a.penalty == b.penalty, it
            else:
                assert abs(a.nnz - b.nnz) <= max(2, 1e-4 * b.nnz), it
                assert a.penalty == pytest.approx(b.penalty, rel=1e-5), it
                assert a.cd_mean == pytest.approx(b.cd_mean, rel=2e-6), it
            assert a.penalty == pytest.approx(c.penalty, rel=1e-5), it
            for e in (b.km_energy, c.km_energy):
                assert abs(a.km_energy - e) <= n * KM_EPS + 1e-6 * abs(e), it
            if it >= settled_from:        # the settled route is eligible: last iteration's graph was sparse
                assert 0 <= out[-1].nnz <= 1.5 * n, it
            assert a.stream_passes > 0 and b.exact_fallback == 0, it
            out.append(a)
            S = fast.source()
            nxt = (a.iteration + 1, a.rmse, a.fdm, a.fdstd, a.para1, a.para2)
            slow.set_keypoints(S, sc.T)
            slow.set_state(*nxt)
            resync_oracle(o, sc, S)
            o.set_state(*nxt)
    finally:
        fast.close()
        slow.close()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("bits", [441, 672, 2048])
def test_stream_km_equals_all_double_and_oracle(g, orc, scratch_cwd, monkeypatch, bits, N=300, M=290, V=4):
    # a wide scene: the penalty's floor of 5 is then far below the typical target spacing (a sparse graph from 57 on)
    sc = fullrange_scene(g, N, M, bits, V, seed=bits + 5, extent=(200, 200, 40))
    fd = oracle_for(orc, sc, orc.CT_NN, V).fd()
    n = max(N, M)
    # general route at 0 (fill pass: no edge count yet) and 1 (edge list), settled at 2 and 3
    st = _km_lockstep(g, orc, sc, V, start_state(sc, fd, 0), 4, settled_from=2)
    assert [s.stream_passes for s in st[:2]] == [3, 2]      # statistics + count + fill, then statistics + count (list)
    # the fill pass in both general iterations
    monkeypatch.setenv("GHICP_KM_FILL", "1")
    st = _km_lockstep(g, orc, sc, V, start_state(sc, fd, 0), 2, settled_from=99)
    assert [s.stream_passes for s in st] == [3, 3]
    monkeypatch.delenv("GHICP_KM_FILL")
    # general at 57, settled at 58 (fp16 weight), 59 and 60 (scalar weight)
    _km_lockstep(g, orc, sc, V, start_state(sc, fd, 57, cells=n), 4, settled_from=58)


# ---- lock-step registrations --------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("bits", [441, 672, 2048])
@pytest.mark.parametrize("ct", ["nn", "nnr"])
def test_lockstep_registration_on_full_range_descriptors(g, orc, bits, ct, N=600, M=500, max_it=40):
    CT = {"nn": g.CT_NN, "nnr": g.CT_NNR}[ct]
    sc = fullrange_scene(g, N, M, bits, 4, seed=17 + bits)
    reg = g.registration.from_scene(sc, g.FT_BSC, CT)
    o = oracle_for(orc, sc, CT, 4)
    try:
        for _ in range(max_it):
            a, b = reg.iterate(), o.iterate()
            sp, tp = reg.pairs()
            osp, otp = o.pairs()
            assert np.array_equal(sp, osp) and np.array_equal(tp, otp), a.iteration
            assert a.cor == b.cor
            if a.converged or b.converged:
                break
        assert a.converged == b.converged
    finally:
        reg.close()


# ---- the same functions on the emulated library (CPU) -----------------------------------------------------------------------------
@pytest.fixture()
def ge(g, emu_library_path):
    from conftest import swap_in_library
    real = swap_in_library(g, emu_library_path)
    try:
        yield g
    finally:
        g.capi._lib = real


@pytest.mark.parametrize("bits", BITS)
def test_emulated_builders(ge, orc, monkeypatch, bits):
    for V in (4, 2):
        test_builders_equal_the_oracle_on_full_range_planes(ge, orc, monkeypatch, bits, V, N=37, M=70)


# two column CTAs with a partial panel and a partial quad; several row blocks with a partial quad; a tiny plane.  Each hb, both
# correspondence types and each shape at least once (the emulated stream kernel runs every fiber of a 2048-column CTA).
EMU_CASES = [(441, "nn", 133, 20), (511, "nnr", 133, 20), (672, "nn", 6, 2100), (1023, "nnr", 133, 20), (2048, "nn", 6, 2100),
             (2048, "nnr", 5, 3)]


@pytest.mark.parametrize("bits,ct,N,M", EMU_CASES)
def test_emulated_stream_nn_nnr(ge, orc, bits, ct, N, M):
    test_stream_nn_nnr_equals_all_double_and_oracle(ge, orc, bits, ct, N, M)


@pytest.mark.parametrize("bits", [441, 672, 2048])
def test_emulated_stream_km(ge, orc, scratch_cwd, monkeypatch, bits):
    test_stream_km_equals_all_double_and_oracle(ge, orc, scratch_cwd, monkeypatch, bits, N=80, M=72)


@pytest.mark.parametrize("bits", [441, 672, 2048])
def test_emulated_lockstep_registration(ge, orc, bits):
    test_lockstep_registration_on_full_range_descriptors(ge, orc, bits, "nnr", N=150, M=130, max_it=12)
