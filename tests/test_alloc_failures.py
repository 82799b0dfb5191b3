"""Running out of device memory at any allocation of a stand-alone or pipeline entry point (emulated library, CPU only).

The host emulation shim (tests/harness/cuda_emu) counts live device allocations and can make the k-th allocation from now
fail; tests/harness/emu_library.cpp exports both controls.  Each entry point is called with k = 0, 1, ... failing until a
call gets through.  Every failed call must return GHICP_E_NOMEM with a message that names the entry point, free everything
it allocated, leave the caller's buffers alone where the header promises to write nothing, and leave a handle usable."""
import ctypes as C

import numpy as np
import pytest

E_NOMEM = -2
INF = float("inf")
fpp, ip, dp = C.POINTER(C.c_float), C.POINTER(C.c_int), C.POINTER(C.c_double)


@pytest.fixture(scope="module")
def emu(g, emu_library_path):
    from conftest import swap_in_library
    real = swap_in_library(g, emu_library_path)
    L = g.capi.lib()
    L.ghicp_emu_live_allocations.restype = C.c_longlong
    L.ghicp_emu_fail_allocation.argtypes = [C.c_longlong]
    try:
        yield g, L
    finally:
        g.capi._lib = real


def F(a):
    return a.ctypes.data_as(fpp)


def I(a):
    return a.ctypes.data_as(ip)


def D(a):
    return a.ctypes.data_as(dp)


def sweep(L, who, call, after_failure=None, before=None, count=True):
    """call() -> status.  Fails the k-th device allocation of the call for k = 0, 1, ... and checks each failure; returns
    (k, status) of the first call that got through.  before() (optional) runs ahead of each call, without a failure armed;
    count=False leaves the count of live allocations to after_failure (a call may leave a cache in a handle)."""
    for k in range(1000):
        if before:
            before()
        live = L.ghicp_emu_live_allocations()
        L.ghicp_emu_fail_allocation(k)
        rc = call()
        L.ghicp_emu_fail_allocation(-1)
        if rc >= 0:
            return k, rc
        msg = L.ghicp_last_error(None).decode()
        assert rc == E_NOMEM, (who, k, rc, msg)
        assert msg.startswith(who + ": "), (who, k, msg)
        assert not count or L.ghicp_emu_live_allocations() == live, (who, k, "leaked", L.ghicp_emu_live_allocations() - live)
        if after_failure:
            after_failure(k)
    raise AssertionError(who + ": no call got through")


@pytest.fixture(scope="module")
def clouds(emu):
    g, _ = emu
    T, S, _, _ = g.synth.scan_pair(400, seed=3)
    return np.ascontiguousarray(T, np.float32), np.ascontiguousarray(S, np.float32)


PREP = dict(voxel_size=0.3, neighborhood_radius=1.0, nms_radius=1.5)


def prep_run(g, L, xyz, bsc_radius=0.0):
    p = g.capi.PrepParams(PREP["voxel_size"], PREP["neighborhood_radius"], 0.65, 5, PREP["nms_radius"], bsc_radius, 7, 6)
    pairs = g.bsc_default_pattern(7)
    h = C.c_void_p()
    rc = L.ghicp_prep_run(0, F(xyz), len(xyz), C.byref(p), I(pairs), C.byref(h))
    return rc, h


def test_standalone_stages(emu, clouds):
    g, L = emu
    A, B = clouds
    n = len(A)
    live = L.ghicp_emu_live_allocations()

    idx, cnt = np.zeros(n + 1, np.int32), C.c_int(0)
    k, _ = sweep(L, "voxel_downsample", lambda: L.ghicp_voxel_downsample(0, F(A), n, 0.3, I(idx), C.byref(cnt)))
    assert k > 0 and cnt.value > 0

    kp, nkp = np.zeros(n, np.int32), C.c_int(0)
    sweep(L, "detect_keypoints", lambda: L.ghicp_detect_keypoints(0, F(A), n, 1.0, 0.65, 5, 1.5, I(kp), C.byref(nkp), None, None, None))
    assert nkp.value > 0

    pairs = g.bsc_default_pattern(7)
    feats, nv = np.zeros((4, nkp.value, 56), np.uint8), C.c_int(0)
    sweep(L, "bsc_extract", lambda: L.ghicp_bsc_extract(0, F(A), n, I(kp), nkp.value, 1.0, 7, I(pairs), 6, feats.ctypes.data,
                                                           C.byref(nv), None, None))

    s = np.ascontiguousarray(A[:50].astype(np.float64).T)
    t = np.ascontiguousarray((A[:50] + np.float32([0.1, -0.2, 0.05])).astype(np.float64).T)
    nrm, w, Rt = np.tile([[0.0], [0.0], [1.0]], (1, 50)), np.linspace(0.5, 1.5, 50), np.zeros(16)
    sweep(L, "rigid_fit", lambda: L.ghicp_rigid_fit(0, D(s), D(t), 50, D(Rt)))
    assert abs(Rt[12] - 0.1) < 1e-6
    sweep(L, "rigid_fit_ex", lambda: L.ghicp_rigid_fit_ex(0, 1, D(s), D(t), None, D(w), 50, D(Rt)))
    sweep(L, "rigid_fit_ex", lambda: L.ghicp_rigid_fit_ex(0, 2, D(s), D(t), D(nrm), D(w), 50, D(Rt)))

    fp = np.zeros((n, 33), np.float32)
    sweep(L, "fpfh_extract", lambda: L.ghicp_fpfh_extract(0, F(A), n, None, 0, 10, F(fp), None, None))

    sel = np.arange(0, n, 7, dtype=np.int32)
    fr = np.full((len(sel), 33), 7.0, np.float32)
    untouched = lambda k: np.testing.assert_array_equal(fr, 7.0)   # noqa: E731  ("writes nothing" on failure)
    sweep(L, "fpfh_extract_radius",
          lambda: L.ghicp_fpfh_extract_radius(0, F(A), n, I(sel), len(sel), 0.8, 1.2, F(fr), None, None), untouched)
    assert not np.any(fr == 7.0)

    fs, ft = np.ascontiguousarray(fp[:120]), np.ascontiguousarray(fp[100:220])
    P, Q = np.ascontiguousarray(A[:120]), np.ascontiguousarray(A[100:220])
    par, res = g.capi._sac_params(20, 3, 2, 0.0, 1.0, 7), g.capi.SacResult()
    sweep(L, "sac_ia", lambda: L.ghicp_sac_ia(0, F(P), F(fs), 120, F(Q), F(ft), 120, C.byref(par), C.byref(res)))

    out, d2 = g.capi.OverlapResult(), np.full(n, 7.0, np.float32)
    out.overlap = 12345

    def unwritten(k):
        assert out.overlap == 12345 and np.all(d2 == 7.0)
    sweep(L, "cloud_overlap", lambda: L.ghicp_cloud_overlap(0, F(A), n, F(B), len(B), None, 0.3, INF, 1, C.byref(out), F(d2)),
          unwritten)
    assert out.overlap != 12345
    assert L.ghicp_emu_live_allocations() == live


def test_pipeline_handles(emu, clouds):
    g, L = emu
    A, B = clouds
    live = L.ghicp_emu_live_allocations()
    made = []

    def run():
        rc, h = prep_run(g, L, A, bsc_radius=1.0)
        if rc >= 0:
            made.append(h)
        return rc
    sweep(L, "prep_run", run)
    ha = made.pop()
    rc, hb = prep_run(g, L, B)
    assert rc == 0

    # prep_fpfh: a failed call drops the histograms
    def dropped(k):
        assert L.ghicp_prep_get_fpfh(ha, F(np.zeros((1000, 33), np.float32))) == -1
    sweep(L, "prep_fpfh", lambda: L.ghicp_prep_fpfh(ha, 10, None), dropped)
    assert L.ghicp_prep_fpfh(hb, 10, None) == 0
    nkp = C.c_int(0)
    assert L.ghicp_prep_info(ha, None, C.byref(nkp), None, None, None, None) == 0

    def fpfh(h):
        out = np.zeros((1000, 33), np.float32)
        assert L.ghicp_prep_get_fpfh(h, F(out)) == 0
        return out

    # prep_sac_ia between two handles with histograms
    par, res = g.capi._sac_params(20, 3, 2, 0.0, 1.0, 7), g.capi.SacResult()
    sweep(L, "prep_sac_ia", lambda: L.ghicp_prep_sac_ia(ha, hb, C.byref(par), C.byref(res)))

    # prep_fpfh_radius: a failed call keeps the histograms the handle had
    assert L.ghicp_prep_fpfh_radius(ha, 0.6, 0.9, None, None) == 0
    old = fpfh(ha)

    def kept(k):
        np.testing.assert_array_equal(fpfh(ha), old)
    sweep(L, "prep_fpfh_radius", lambda: L.ghicp_prep_fpfh_radius(ha, 0.8, 1.2, None, None), kept)
    assert not np.array_equal(fpfh(ha), old)

    # prep_overlap: every failure on a fresh target (its grid is built on the first call and then kept, also when the queries
    # fail); the next call gives what a fresh pair of handles gives, and destroying the target frees everything
    want = g.capi.OverlapResult()
    rc, fresh = prep_run(g, L, B)
    assert rc == 0 and L.ghicp_prep_overlap(ha, fresh, None, 0.3, INF, 1, C.byref(want)) == 0
    L.ghicp_prep_destroy(fresh)
    targets = []
    out = g.capi.OverlapResult()

    base = []

    def new_target():
        base.append(L.ghicp_emu_live_allocations())
        rc, t = prep_run(g, L, B)
        assert rc == 0
        targets.append(t)
        out.overlap = 12345

    def call():
        return L.ghicp_prep_overlap(ha, targets[-1], None, 0.3, INF, 1, C.byref(out))

    def recovers(k):
        assert out.overlap == 12345
        again = g.capi.OverlapResult()
        assert L.ghicp_prep_overlap(ha, targets[-1], None, 0.3, INF, 1, C.byref(again)) == 0
        assert (again.overlap, again.n_fit, again.fitness) == (want.overlap, want.n_fit, want.fitness)
        assert L.ghicp_prep_destroy(targets.pop()) == 0
        assert L.ghicp_emu_live_allocations() == base[-1]
    k, _ = sweep(L, "prep_overlap", call, recovers, new_target, count=False)
    assert k > 0 and (out.overlap, out.n_fit, out.fitness) == (want.overlap, want.n_fit, want.fitness)

    for h in targets + [ha, hb]:
        assert L.ghicp_prep_destroy(h) == 0
    assert L.ghicp_emu_live_allocations() == live
