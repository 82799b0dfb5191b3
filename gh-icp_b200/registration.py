"""Python mirror of the reference's registration interface (include/ghicp_reg.h:15-132) over the C ABI.

Same names and argument meaning as the reference: `Energyfunction.init(kps_num, kpt_num, bbx_magnitude)`,
`Keypoints.setCoordinate / setBSCfeature / setFPFHfeature`, `GHRegistration(Kp, Ef, Ft, Ct, radiusNonMax,
weight_adjustment_ratio, weight_adjustment_step, dof_type, estimated_IoU, converge_tran, converge_rot)`,
`ghicp_reg() -> Rt_final`.  Viewer / raw-cloud setters are accepted and ignored (out of scope).
"""
import ctypes as C

import numpy as np

from . import capi
from .capi import CT_KM, CT_NN, CT_NNR, FT_BSC, FT_FPFH, FT_NONE  # noqa: F401


class Energyfunction:
    """include/ghicp_reg.h:15-42 (the N x M matrices live on the device, not here)."""

    def __init__(self):
        self.bbx_magnitude = 0.0
        self.kps_num = self.kpt_num = 0

    def init(self, kps_num, kpt_num, bbx_magnitude):
        self.kps_num, self.kpt_num, self.bbx_magnitude = kps_num, kpt_num, float(bbx_magnitude)
        return self


class Keypoints:
    """include/ghicp_reg.h:44-72."""

    def __init__(self):
        self.kpSXYZ = self.kpTXYZ = None
        self.bscS = self.bscT = None
        self.bits = 0
        self.fpfhS = self.fpfhT = None

    def setCoordinate(self, kps, kpt):
        self.kpSXYZ = np.asfortranarray(kps, dtype=np.float64)
        self.kpTXYZ = np.asfortranarray(kpt, dtype=np.float64)
        self.kps_num, self.kpt_num = self.kpSXYZ.shape[0], self.kpTXYZ.shape[0]
        return self

    def setBSCfeature(self, bsc_S, bsc_T, bits):
        self.bscS = np.ascontiguousarray(bsc_S, dtype=np.uint8)   # (V, N, B)
        self.bscT = np.ascontiguousarray(bsc_T, dtype=np.uint8)   # (M, B)
        self.bits = int(bits)
        return self

    def setFPFHfeature(self, fpfh_S, fpfh_T):
        self.fpfhS = np.ascontiguousarray(fpfh_S, dtype=np.float32)
        self.fpfhT = np.ascontiguousarray(fpfh_T, dtype=np.float32)
        return self


class GHRegistration:
    """include/ghicp_reg.h:74-132 over libghicp_b200.so."""

    def __init__(self, Kp, Ef, Ft, Ct, radiusNonMax=1.0, weight_adjustment_ratio=1.1,
                 weight_adjustment_step=0.1, dof_type=6, estimated_IoU=0.5,
                 converge_tran=0.02, converge_rot=0.02, max_iter=0, device=0, km_eps=0.0, force_exact=False,
                 comm=None, fpfh_matrix_free=0, solver=capi.SOLVER_SVD, target_normals=None):
        self.L = capi.lib()
        cfg = capi.Config()
        cfg.feature_type, cfg.corr_type, cfg.dof = Ft, Ct, dof_type
        cfg.bbx_magnitude = Ef.bbx_magnitude
        cfg.nonmax = radiusNonMax
        cfg.adjust_ratio, cfg.adjust_step = weight_adjustment_ratio, weight_adjustment_step
        cfg.estimated_iou = estimated_IoU
        cfg.converge_t, cfg.converge_r = converge_tran, converge_rot
        cfg.max_iter, cfg.device, cfg.km_eps = max_iter, device, km_eps
        cfg.force_exact = 1 if force_exact else 0
        cfg.fpfh_matrix_free = int(fpfh_matrix_free)   # extension: 1 = never store the N x M FPFH distance plane
        cfg.solver = int(solver)                       # extension: opt-in estimators, 0 = the reference's SVD
        self.ctx = C.c_void_p()
        capi.check(self.L.ghicp_create(C.byref(cfg), C.byref(self.ctx)))
        if comm is not None:  # (unique_id bytes, rank, world): one process per GPU, source rows sharded
            uid, rank, world = comm
            buf = (C.c_char * 128).from_buffer_copy(uid) if world > 1 else None
            capi.check(self.L.ghicp_comm_init(self.ctx, buf, rank, world), self.ctx)
        self.Ft, self.Ct, self.max_iter = Ft, Ct, max_iter
        if isinstance(Kp, tuple):   # (source Prep, target Prep): device-resident pipeline results, no host copy
            src, tgt = Kp
            self.N, self.M = src.n_kp, tgt.n_kp
            capi.check(self.L.ghicp_set_from_prep(self.ctx, src.h, tgt.h), self.ctx)
        else:
            self.N, self.M = Kp.kps_num, Kp.kpt_num
            self.upload(Kp)
        if target_normals is not None:
            self.set_target_normals(target_normals)
        self.history = []

    def upload(self, Kp):
        capi.check(self.L.ghicp_set_keypoints(self.ctx, capi._dp(Kp.kpSXYZ), Kp.kps_num,
                                              capi._dp(Kp.kpTXYZ), Kp.kpt_num), self.ctx)
        if self.Ft == FT_BSC:
            capi.check(self.L.ghicp_set_bsc(self.ctx, Kp.bscS.ctypes.data, Kp.bscS.shape[0],
                                            Kp.bscT.ctypes.data, Kp.bits), self.ctx)
        elif self.Ft == FT_FPFH:
            capi.check(self.L.ghicp_set_fpfh(self.ctx, Kp.fpfhS.ctypes.data, Kp.fpfhT.ctypes.data), self.ctx)

    def set_keypoints(self, kps, kpt):
        """Re-upload coordinates only (same sizes): the host->device leg of an end-to-end step."""
        kps = np.asfortranarray(kps, dtype=np.float64)
        kpt = np.asfortranarray(kpt, dtype=np.float64)
        capi.check(self.L.ghicp_set_keypoints(self.ctx, capi._dp(kps), kps.shape[0], capi._dp(kpt),
                                              kpt.shape[0]), self.ctx)

    def set_target_normals(self, normals):
        """Unit normals of the target keypoints (M, 3): only read by SOLVER_POINT_TO_PLANE."""
        n = np.asfortranarray(normals, dtype=np.float64)
        capi.check(self.L.ghicp_set_target_normals(self.ctx, capi._dp(n)), self.ctx)

    def set_initial_transform(self, Rt):
        """Start the loop from Rt (4x4, source -> target), e.g. a SAC-IA result: the source keypoints are moved on the device
        and Rt_tillnow starts at Rt, so ghicp_reg() and Rt_tillnow() return the whole transform.  Only before iteration 0."""
        Rt = np.asarray(Rt, dtype=np.float64).reshape(4, 4)
        cm = np.ascontiguousarray(Rt.T).reshape(16)   # column-major (Eigen::Matrix4d::data())
        capi.check(self.L.ghicp_set_initial_transform(self.ctx, capi._dp(cm)), self.ctx)

    def set_solver(self, solver):
        capi.check(self.L.ghicp_set_solver(self.ctx, int(solver)), self.ctx)

    def close(self):
        if getattr(self, "ctx", None):
            self.L.ghicp_destroy(self.ctx)
            self.ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # reference no-ops (viewer / raw clouds are out of scope, SURVEY.md §2)
    def set_raw_pointcloud(self, *a):
        pass

    def set_viewer(self, launch_viewer):
        pass

    def build_fd(self):
        capi.check(self.L.ghicp_build_fd(self.ctx), self.ctx)

    def iterate(self):
        st = capi.IterStats()
        capi.check(self.L.ghicp_iterate(self.ctx, C.byref(st)), self.ctx)
        self.history.append(st)
        return st

    def ghicp_reg(self, track_matches=False):
        """Main entrance (src/ghicp_reg.cpp:24-112). Returns (Rt_final 4x4, iterations).

        track_matches=True runs the loop one ghicp_iterate at a time and fills what the reference's KM branch records per
        iteration (src/ghicp_reg.cpp:443-460): `pre`, `rec` (identity pairs among the returned correspondences; see
        gh-icp_b200/cxx/ghicp_reg.h on the penalty-edge part of src/km.cpp:159) and `matchlist` (N x iterations, target index
        or -1).  The per-iteration statistics (`energy`, `rmse`, `rmseafter`, `cor`, `RMS`) are then available as well; the
        default hands the whole loop to ghicp_run and keeps only its result."""
        if not track_matches:
            Rt = np.zeros(16)
            it = C.c_int(0)
            capi.check(self.L.ghicp_run(self.ctx, capi._dp(Rt), C.byref(it)), self.ctx)
            return Rt.reshape(4, 4).T.copy(), it.value
        self.build_fd()
        self.pre, self.rec, cols = [], [], []
        while True:
            st = self.iterate()
            if self.Ct == CT_KM:
                sp, tp = self.pairs()
                exact = int((sp == tp).sum())
                self.pre.append(exact / len(sp) if len(sp) else 0.0)
                self.rec.append(exact / max(self.N, self.M))
                col = np.full(self.N, -1, np.int32)
                col[sp] = tp
                cols.append(col)
            if st.converged or (self.max_iter > 0 and len(self.history) >= self.max_iter):
                break
        self.matchlist = np.stack(cols, axis=1) if cols else np.zeros((self.N, 0), np.int32)
        return self.Rt_tillnow(), len(self.history)

    # public members of the reference's class (include/ghicp_reg.h:138-152), from the iterations run through iterate()
    @property
    def energy(self):
        return [st.km_energy for st in self.history]

    @property
    def rmse(self):
        return [st.rmse for st in self.history]

    @property
    def rmseafter(self):
        return [st.rmse_after for st in self.history]

    @property
    def cor(self):
        return [st.cor for st in self.history]

    @property
    def RMS(self):
        return self.history[-1].rmse if self.history else 99999.0

    def pairs(self, out=None):
        """(SP, TP) of the last iteration.  out = (sp, tp) int32 buffers of >= max(N, M) entries (e.g. capi.pinned_empty):
        views of them are returned, nothing is allocated or copied on the host."""
        cap = max(self.N, self.M)
        if out is None:
            sp = np.zeros(cap, np.int32)
            tp = np.zeros(cap, np.int32)
        else:
            sp, tp = out
            cap = min(cap, sp.shape[0], tp.shape[0])
        n = C.c_int(0)
        capi.check(self.L.ghicp_get_pairs(self.ctx, capi._ip(sp), capi._ip(tp), cap, C.byref(n)), self.ctx)
        k = min(n.value, cap)
        if out is None:
            return sp[:k].copy(), tp[:k].copy()
        return sp[:k], tp[:k]

    def source(self, out=None):
        """Current source keypoints (N, 3), column-major like Eigen::MatrixX3d; out = a buffer of that layout to fill."""
        if out is None:
            out = np.zeros((self.N, 3), dtype=np.float64, order="F")
        capi.check(self.L.ghicp_get_source(self.ctx, capi._dp(out)), self.ctx)
        return out

    def Rt_tillnow(self):
        Rt = np.zeros(16)
        capi.check(self.L.ghicp_get_rt(self.ctx, capi._dp(Rt)), self.ctx)
        return Rt.reshape(4, 4).T.copy()

    def fd(self):
        out = np.zeros((self.N, self.M), dtype=np.float64)
        capi.check(self.L.ghicp_get_fd(self.ctx, capi._dp(out)), self.ctx)
        return out

    def probe_rowmin(self):
        idx = np.zeros(self.N, np.int32)
        cd = np.zeros(self.N, np.float64)
        m, s, p = C.c_double(0), C.c_double(0), C.c_double(0)
        capi.check(self.L.ghicp_probe_rowmin(self.ctx, capi._ip(idx), capi._dp(cd), C.byref(m), C.byref(s),
                                             C.byref(p)), self.ctx)
        return idx, cd, m.value, s.value, p.value

    def set_state(self, iteration, rms, fdm, fdstd, para1, para2):
        capi.check(self.L.ghicp_set_state(self.ctx, iteration, rms, fdm, fdstd, para1, para2), self.ctx)

    def reset(self):
        """Constructor state again (iteration 0, Rt_tillnow = I); descriptors and the FD plane stay."""
        capi.check(self.L.ghicp_reset(self.ctx), self.ctx)
        self.history = []


def from_scene(scene, Ft, Ct, dof=6, **kw):
    """Convenience: build Keypoints/Energyfunction/GHRegistration from a synth.Scene."""
    Kp = Keypoints().setCoordinate(scene.S, scene.T)
    if Ft == FT_BSC:
        Kp.setBSCfeature(scene.bsc_s, scene.bsc_t, scene.bits)
    elif Ft == FT_FPFH:
        Kp.setFPFHfeature(scene.fpfh_s, scene.fpfh_t)
    Ef = Energyfunction().init(Kp.kps_num, Kp.kpt_num, scene.bbx_magnitude)
    return GHRegistration(Kp, Ef, Ft, Ct, dof_type=dof, **kw)
