"""ctypes binding of libghicp_b200.so (include/ghicp_b200.h)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = os.path.join(_HERE, "libghicp_b200.so")

FT_BSC, FT_ROPS, FT_FPFH, FT_NONE = 0, 1, 2, 3   # include/utility.h:51-57
CT_NN, CT_NNR, CT_KM = 0, 1, 2                   # include/utility.h:59-64

GHICP_W_FEW_PAIRS = 1
GHICP_W_SINGULAR = 2   # point-to-plane ICP or GICP: a singular system stopped the loop
# ghicp_solver_type (include/ghicp_b200.h): SVD is the reference's estimator, the others are opt-in extensions
SOLVER_SVD, SOLVER_WEIGHTED_SVD, SOLVER_POINT_TO_PLANE, SOLVER_YAW_4DOF = 0, 1, 2, 3


class GhicpError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__(f"ghicp error {code}: {msg}")
        self.code = code


class Config(C.Structure):
    _fields_ = [("feature_type", C.c_int), ("corr_type", C.c_int), ("dof", C.c_int),
                ("bbx_magnitude", C.c_float), ("nonmax", C.c_float), ("adjust_ratio", C.c_float),
                ("adjust_step", C.c_float), ("estimated_iou", C.c_float), ("converge_t", C.c_float),
                ("converge_r", C.c_float), ("max_iter", C.c_int), ("device", C.c_int),
                ("km_eps", C.c_double), ("verbose", C.c_int), ("force_exact", C.c_int),
                ("fpfh_matrix_free", C.c_int), ("solver", C.c_int), ("reserved", C.c_int * 4)]


class IterStats(C.Structure):
    _fields_ = [("iteration", C.c_int), ("cor", C.c_int), ("converged", C.c_int), ("warnings", C.c_int),
                ("Rt", C.c_double * 16), ("Rt_tillnow", C.c_double * 16),
                ("cd_mean", C.c_double), ("cd_std", C.c_double), ("penalty", C.c_double),
                ("rmse", C.c_double), ("rmse_after", C.c_double), ("fdm", C.c_double), ("fdstd", C.c_double),
                ("iou", C.c_double), ("para1", C.c_double), ("para2", C.c_double), ("km_energy", C.c_double),
                ("ax", C.c_double), ("ay", C.c_double), ("az", C.c_double),
                ("nnz", C.c_longlong), ("km_rounds", C.c_int), ("km_phases", C.c_int), ("gpu_launches", C.c_int), ("exact_fallback", C.c_int),
                ("ms_cost", C.c_float), ("ms_corr", C.c_float), ("ms_solve", C.c_float), ("ms_total", C.c_float),
                ("ms_stream", C.c_float), ("stream_passes", C.c_int), ("candidates", C.c_longlong)]

    def Rt_np(self):
        return np.array(self.Rt).reshape(4, 4).T.copy()

    def Rt_tillnow_np(self):
        return np.array(self.Rt_tillnow).reshape(4, 4).T.copy()


def lib_path():
    return _LIB


def build_library(force=False):
    """Compile gh-icp_b200/csrc for sm_90a in-tree (nvcc cross-compiles without a GPU)."""
    if force or not os.path.exists(_LIB):
        r = subprocess.run(["make", "-C", os.path.join(_HERE, "csrc"), "-j4"], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("building libghicp_b200.so failed:\n" + r.stdout[-4000:] + r.stderr[-4000:])
    return _LIB


_lib = None

EXPORTS = ["ghicp_abi_version", "ghicp_device_count", "ghicp_last_error", "ghicp_create", "ghicp_destroy",
           "ghicp_set_keypoints", "ghicp_set_bsc", "ghicp_set_fpfh", "ghicp_build_fd", "ghicp_iterate",
           "ghicp_run", "ghicp_get_pairs", "ghicp_get_source", "ghicp_get_rt", "ghicp_get_fd",
           "ghicp_probe_rowmin", "ghicp_set_state", "ghicp_reset", "ghicp_km_solve", "ghicp_rigid_fit", "ghicp_rigid_fit_ex",
           "ghicp_set_target_normals", "ghicp_set_solver", "ghicp_voxel_downsample", "ghicp_detect_keypoints",
           "ghicp_bsc_extract", "ghicp_bsc_default_pattern", "ghicp_comm_unique_id", "ghicp_comm_init",
           "ghicp_prep_run", "ghicp_prep_info", "ghicp_prep_get", "ghicp_prep_destroy", "ghicp_set_from_prep",
           "ghicp_host_alloc", "ghicp_host_free", "ghicp_fpfh_extract", "ghicp_prep_fpfh", "ghicp_prep_get_fpfh",
           "ghicp_prep_fpfh_stats", "ghicp_sac_ia", "ghicp_prep_sac_ia", "ghicp_set_initial_transform",
           "ghicp_fpfh_extract_radius", "ghicp_prep_fpfh_radius", "ghicp_cloud_overlap", "ghicp_prep_overlap",
           "ghicp_cloud_icp", "ghicp_prep_icp", "ghicp_sor_filter", "ghicp_prep_run_sor", "ghicp_prep_sor_info"]


def lib():
    """Load libghicp_b200.so. Fails loudly when it is missing: there is no fallback path."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB):
        raise GhicpError(-100, f"{_LIB} is missing: run __graft_entry__.build() (make -C gh-icp_b200/csrc); "
                               "this package has no CPU fallback")
    L = C.CDLL(_LIB)
    dp, ip, vp = C.POINTER(C.c_double), C.POINTER(C.c_int), C.c_void_p
    L.ghicp_abi_version.restype = C.c_int
    L.ghicp_device_count.restype = C.c_int
    L.ghicp_last_error.restype = C.c_char_p
    L.ghicp_last_error.argtypes = [vp]
    L.ghicp_create.argtypes = [C.POINTER(Config), C.POINTER(vp)]
    L.ghicp_destroy.argtypes = [vp]
    L.ghicp_set_keypoints.argtypes = [vp, dp, C.c_int, dp, C.c_int]
    L.ghicp_set_bsc.argtypes = [vp, vp, C.c_int, vp, C.c_int]
    L.ghicp_set_fpfh.argtypes = [vp, vp, vp]
    L.ghicp_build_fd.argtypes = [vp]
    L.ghicp_iterate.argtypes = [vp, C.POINTER(IterStats)]
    L.ghicp_run.argtypes = [vp, dp, ip]
    L.ghicp_get_pairs.argtypes = [vp, ip, ip, C.c_int, ip]
    L.ghicp_get_source.argtypes = [vp, dp]
    L.ghicp_get_rt.argtypes = [vp, dp]
    L.ghicp_get_fd.argtypes = [vp, dp]
    L.ghicp_probe_rowmin.argtypes = [vp, ip, dp, dp, dp, dp]
    L.ghicp_set_state.argtypes = [vp, C.c_int, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double]
    L.ghicp_reset.argtypes = [vp]
    L.ghicp_km_solve.argtypes = [C.c_int, dp, C.c_int, C.c_int, C.c_int, C.c_double, C.c_double, ip, dp, ip]
    L.ghicp_rigid_fit.argtypes = [C.c_int, dp, dp, C.c_int, dp]
    L.ghicp_rigid_fit_ex.argtypes = [C.c_int, C.c_int, dp, dp, dp, dp, C.c_int, dp]
    L.ghicp_set_target_normals.argtypes = [vp, dp]
    L.ghicp_set_solver.argtypes = [vp, C.c_int]
    fpp = C.POINTER(C.c_float)
    L.ghicp_voxel_downsample.argtypes = [C.c_int, fpp, C.c_int, C.c_float, ip, ip]
    L.ghicp_detect_keypoints.argtypes = [C.c_int, fpp, C.c_int, C.c_float, C.c_float, C.c_int, C.c_float, ip, ip, fpp, dp, ip]
    L.ghicp_bsc_extract.argtypes = [C.c_int, fpp, C.c_int, ip, C.c_int, C.c_float, C.c_int, ip, C.c_int, vp, ip, fpp, ip]
    L.ghicp_bsc_default_pattern.argtypes = [C.c_int, ip]
    L.ghicp_prep_run.argtypes = [C.c_int, fpp, C.c_int, C.POINTER(PrepParams), ip, C.POINTER(vp)]
    L.ghicp_prep_info.argtypes = [vp, ip, ip, ip, fpp, fpp, fpp]
    L.ghicp_prep_get.argtypes = [vp, fpp, ip, dp, vp]
    L.ghicp_prep_destroy.argtypes = [vp]
    L.ghicp_set_from_prep.argtypes = [vp, vp, vp]
    L.ghicp_comm_unique_id.argtypes = [vp]
    L.ghicp_comm_init.argtypes = [vp, vp, C.c_int, C.c_int]
    L.ghicp_host_alloc.argtypes = [C.c_size_t, C.POINTER(vp)]
    L.ghicp_host_free.argtypes = [vp]
    L.ghicp_fpfh_extract.argtypes = [C.c_int, fpp, C.c_int, ip, C.c_int, C.c_int, fpp, fpp, ip]
    L.ghicp_prep_fpfh.argtypes = [vp, C.c_int, fpp]
    L.ghicp_prep_get_fpfh.argtypes = [vp, fpp]
    L.ghicp_prep_fpfh_stats.argtypes = [vp, C.POINTER(C.c_longlong), ip, ip, fpp]
    L.ghicp_sac_ia.argtypes = [C.c_int, fpp, fpp, C.c_int, fpp, fpp, C.c_int, C.POINTER(SacParams), C.POINTER(SacResult)]
    L.ghicp_prep_sac_ia.argtypes = [vp, vp, C.POINTER(SacParams), C.POINTER(SacResult)]
    L.ghicp_set_initial_transform.argtypes = [vp, dp]
    L.ghicp_fpfh_extract_radius.argtypes = [C.c_int, fpp, C.c_int, ip, C.c_int, C.c_float, C.c_float, fpp, fpp, ip]
    L.ghicp_prep_fpfh_radius.argtypes = [vp, C.c_float, C.c_float, fpp, C.POINTER(C.c_longlong)]
    L.ghicp_cloud_overlap.argtypes = [C.c_int, fpp, C.c_int, fpp, C.c_int, dp, C.c_float, C.c_double, C.c_int,
                                      C.POINTER(OverlapResult), fpp]
    L.ghicp_prep_overlap.argtypes = [vp, vp, dp, C.c_float, C.c_double, C.c_int, C.POINTER(OverlapResult)]
    L.ghicp_cloud_icp.argtypes = [C.c_int, fpp, C.c_int, fpp, C.c_int, dp, C.POINTER(IcpParams), C.POINTER(IcpResult), fpp, ip, dp]
    L.ghicp_prep_icp.argtypes = [vp, vp, dp, C.POINTER(IcpParams), C.POINTER(IcpResult)]
    L.ghicp_sor_filter.argtypes = [C.c_int, fpp, C.c_int, C.c_int, C.c_double, ip, fpp, C.POINTER(SorResult)]
    L.ghicp_prep_run_sor.argtypes = [C.c_int, fpp, C.c_int, C.POINTER(PrepParams), ip, C.c_int, C.c_double, C.POINTER(vp)]
    L.ghicp_prep_sor_info.argtypes = [vp, C.POINTER(SorResult), ip, fpp]
    _lib = L
    return L


def device_count():
    return lib().ghicp_device_count()


class SacParams(C.Structure):
    """ghicp_sac_params (include/ghicp_b200.h): SAC-IA, DESIGN.md §3.11."""
    _fields_ = [("max_iterations", C.c_int), ("nr_samples", C.c_int), ("k_correspondences", C.c_int),
                ("min_sample_distance", C.c_float), ("corr_dist_threshold", C.c_float), ("reserved", C.c_int),
                ("seed", C.c_ulonglong)]


class SacResult(C.Structure):
    _fields_ = [("Rt", C.c_double * 16), ("error", C.c_double), ("fitness", C.c_double), ("inliers", C.c_int),
                ("best_hypothesis", C.c_int), ("invalid_hypotheses", C.c_int), ("reserved", C.c_int), ("stage_ms", C.c_float * 4)]


def _sac_params(iterations, samples, k, min_sample_distance, threshold, seed):
    return SacParams(int(iterations), int(samples), int(k), float(min_sample_distance), float(threshold), 0, int(seed))


def _sac_out(r):
    Rt = np.array(r.Rt).reshape(4, 4).T.copy()
    ms = list(r.stage_ms)
    return Rt, dict(error=r.error, fitness=r.fitness, inliers=r.inliers, best_hypothesis=r.best_hypothesis,
                    invalid_hypotheses=r.invalid_hypotheses,
                    stage_ms=dict(sample_knn=ms[0], estimate=ms[1], score=ms[2], pick=ms[3], total=float(sum(ms))))


class OverlapResult(C.Structure):
    """ghicp_overlap_result (include/ghicp_b200.h): overlap and fitness on the dense clouds, DESIGN.md §3.12."""
    _fields_ = [("n", C.c_longlong), ("overlap", C.c_longlong), ("n_fit", C.c_longlong), ("cells_visited", C.c_longlong),
                ("candidates", C.c_longlong), ("ratio", C.c_float), ("overlap_rmse", C.c_double), ("fitness", C.c_double),
                ("stage_ms", C.c_float * 3)]


def _overlap_rt(Rt):
    """4x4 row-major numpy transform -> the column-major double[16] of the ABI (None: the identity, passed as NULL)."""
    if Rt is None:
        return None, None
    m = np.ascontiguousarray(np.asarray(Rt, dtype=np.float64).reshape(4, 4).T).reshape(16)
    return m, _dp(m)


def _overlap_out(r):
    ms = list(r.stage_ms)
    return dict(n=r.n, overlap=r.overlap, ratio=r.ratio, overlap_rmse=r.overlap_rmse, n_fit=r.n_fit, fitness=r.fitness,
                cells_visited=r.cells_visited, candidates=r.candidates, stage_ms=dict(grid=ms[0], queries=ms[1], total=ms[2]))


class IcpParams(C.Structure):
    """ghicp_icp_params (include/ghicp_b200.h): point-to-point (metric 0, DESIGN.md §3.13), point-to-plane (metric 1, §3.14)
    or Generalized (metric 2, §3.15) ICP."""
    _fields_ = [("max_iterations", C.c_int), ("reciprocal", C.c_int), ("trim_ratio", C.c_float),
                ("transformation_epsilon", C.c_double), ("fitness_epsilon", C.c_double), ("metric", C.c_int), ("normal_k", C.c_int),
                ("rotation_epsilon", C.c_double)]


class IcpResult(C.Structure):
    _fields_ = [("Rt", C.c_double * 16), ("mse", C.c_double), ("fitness", C.c_double), ("iterations", C.c_int),
                ("converged", C.c_int), ("state", C.c_int), ("cor", C.c_int), ("cells_visited", C.c_longlong),
                ("candidates", C.c_longlong), ("stage_ms", C.c_float * 4)]


ICP_STATES = {1: "ITERATIONS", 2: "TRANSFORM", 3: "ABS_MSE", 4: "REL_MSE", 5: "NO_CORRESPONDENCES", 7: "SINGULAR"}   # ghicp_icp_state
ICP_METRICS = {"point": 0, "plane": 1, "gicp": 2}   # ghicp_icp_params.metric


def _icp_params(max_iterations, reciprocal, trim_ratio, transformation_epsilon, fitness_epsilon, metric="point", normal_k=20,
                rotation_epsilon=1e-6):
    if metric not in ICP_METRICS:
        raise GhicpError(-1, f"icp: metric must be 'point', 'plane' or 'gicp', not {metric!r}")
    return IcpParams(int(max_iterations), int(bool(reciprocal)), float(trim_ratio), float(transformation_epsilon),
                     float(fitness_epsilon), ICP_METRICS[metric], int(normal_k), float(rotation_epsilon))


def _icp_out(r, rc):
    Rt = np.array(r.Rt).reshape(4, 4).T.copy()
    ms = list(r.stage_ms)
    return Rt, dict(iterations=r.iterations, converged=bool(r.converged), state=ICP_STATES.get(r.state, r.state), cor=r.cor,
                    mse=r.mse, fitness=r.fitness, warnings=rc, cells_visited=r.cells_visited, candidates=r.candidates,
                    stage_ms=dict(grid=ms[0], iterations=ms[1], fitness=ms[2], total=ms[3]))


class SorResult(C.Structure):
    """ghicp_sor_result (include/ghicp_b200.h): statistical outlier removal, DESIGN.md §3.16."""
    _fields_ = [("n_finite", C.c_int), ("n_kept", C.c_int), ("k_eff", C.c_int), ("fallbacks", C.c_int), ("mean", C.c_double),
                ("stddev", C.c_double), ("threshold", C.c_double), ("candidates", C.c_longlong), ("stage_ms", C.c_float * 5)]


def _sor_out(r):
    ms = list(r.stage_ms)
    return dict(n_finite=r.n_finite, n_kept=r.n_kept, k_eff=r.k_eff, mean=r.mean, stddev=r.stddev, threshold=r.threshold,
                candidates=r.candidates, fallbacks=r.fallbacks,
                stage_ms=dict(grid=ms[0], distances=ms[1], statistics=ms[2], compaction=ms[3], total=ms[4]))


def _sor_args(sor):
    """None -> (0, 0.0), the ABI's "no filter"; else the (mean_k, std_mul) pair, mean_k in 1..128 and std_mul finite (mean_k 0
    would silently mean "no filter" to the ABI)."""
    if sor is None:
        return 0, 0.0
    mean_k, std_mul = sor
    mean_k, std_mul = int(mean_k), float(std_mul)
    if not 1 <= mean_k <= 128 or not np.isfinite(std_mul):
        raise GhicpError(-1, f"sor: mean_k must be in 1..128 and std_mul finite, not ({mean_k}, {std_mul})")
    return mean_k, std_mul


class PrepParams(C.Structure):
    """ghicp_prep_params (include/ghicp_b200.h): the driver's per-cloud parameters (test/ghicp_main.cpp:89-116)."""
    _fields_ = [("voxel_size", C.c_float), ("neighborhood_radius", C.c_float), ("ratio_max", C.c_float), ("min_pts", C.c_int),
                ("nms_radius", C.c_float), ("bsc_radius", C.c_float), ("bsc_side", C.c_int), ("dof_type", C.c_int)]


class Prep:
    """Device-resident pipeline result of ONE cloud (ghicp_prep_run): voxel filter -> curvature keypoints -> BSC encoder,
    the raw cloud uploaded once, nothing copied back unless asked for.  sor = (mean_k, std_mul) removes statistical outliers
    from the down-sampled cloud between the voxel filter and the keypoints (ghicp_prep_run_sor, see sor_filter); `sor_info`
    then holds the filter's result, with the down-sampled size before it ("n_voxel") and its time ("ms").  sor=None (the
    default) runs no filter and sor_info is None."""

    def __init__(self, xyz, voxel_size, neighborhood_radius, nms_radius, bsc_radius=0.0, dof_type=0, ratio_max=0.65, min_pts=20,
                 side=7, pairs=None, device=0, sor=None):
        xyz = np.ascontiguousarray(xyz, dtype=np.float32)
        self.params = PrepParams(voxel_size, neighborhood_radius, ratio_max, min_pts, nms_radius, bsc_radius, side, dof_type)
        pr = None
        if bsc_radius > 0:
            pr = bsc_default_pattern(side) if pairs is None else np.ascontiguousarray(pairs, dtype=np.int32)
        self.h = C.c_void_p()
        self.side = side
        mean_k, std_mul = _sor_args(sor)
        check(lib().ghicp_prep_run_sor(device, xyz.ctypes.data_as(C.POINTER(C.c_float)), len(xyz), C.byref(self.params),
                                       None if pr is None else _ip(pr), mean_k, std_mul, C.byref(self.h)))
        self.sor_info = None
        if sor is not None:
            r, nv, ms = SorResult(), C.c_int(0), C.c_float(0)
            check(lib().ghicp_prep_sor_info(self.h, C.byref(r), C.byref(nv), C.byref(ms)))
            self.sor_info = dict(_sor_out(r), n_voxel=nv.value, ms=ms.value)
        nd, nk, nv = C.c_int(0), C.c_int(0), C.c_int(0)
        mn, mx, ms = np.zeros(3, np.float32), np.zeros(3, np.float32), np.zeros(5, np.float32)
        fpp = C.POINTER(C.c_float)
        check(lib().ghicp_prep_info(self.h, C.byref(nd), C.byref(nk), C.byref(nv), mn.ctypes.data_as(fpp), mx.ctypes.data_as(fpp),
                                    ms.ctypes.data_as(fpp)))
        self.n_down, self.n_kp, self.V = nd.value, nk.value, nv.value
        self.bbox_min, self.bbox_max = mn, mx
        self.stage_ms = dict(h2d=float(ms[0]), voxel_filter=float(ms[1]), keypoints=float(ms[2]), bsc=float(ms[3]), total=float(ms[4]))

    @property
    def bbx_magnitude(self):
        """getCloudBound of the down-sampled cloud, test/ghicp_main.cpp:91-93 (float32 arithmetic)."""
        e = self.bbox_max - self.bbox_min
        return float(np.float32(e[0] + e[1] + e[2]))

    def down(self):
        out = np.zeros((self.n_down, 3), np.float32)
        check(lib().ghicp_prep_get(self.h, out.ctypes.data_as(C.POINTER(C.c_float)), None, None, None))
        return out

    def keypoints(self):
        """(indices into the down-sampled cloud, coordinates [n_kp][3] float64)."""
        idx = np.zeros(self.n_kp, np.int32)
        soa = np.zeros((3, self.n_kp), np.float64)
        check(lib().ghicp_prep_get(self.h, None, _ip(idx), _dp(soa), None))
        return idx, np.ascontiguousarray(soa.T)

    def bsc(self):
        nbytes = (9 * self.side * self.side + 7) // 8
        out = np.zeros((max(self.V, 1), self.n_kp, nbytes), np.uint8)
        if self.V > 0:
            check(lib().ghicp_prep_get(self.h, None, None, None, out.ctypes.data))
        return out

    def fpfh(self, k=20):
        """FPFHfeature::compute_fpfh_feature + keyfpfh (include/fpfh.hpp:36-115) at the keypoints, on the down-sampled cloud,
        kept on the device (ghicp_prep_fpfh).  Returns the stage times {knn_normals, spfh_fpfh, total} in ms; fpfh_stats then
        holds the k-NN work (candidates per query, exhaustive-scan queries, cell edge)."""
        ms = np.zeros(3, np.float32)
        check(lib().ghicp_prep_fpfh(self.h, k, ms.ctypes.data_as(C.POINTER(C.c_float))))
        cand, q, fb, cell = C.c_longlong(0), C.c_int(0), C.c_int(0), C.c_float(0)
        check(lib().ghicp_prep_fpfh_stats(self.h, C.byref(cand), C.byref(q), C.byref(fb), C.byref(cell)))
        self.fpfh_k = k
        self.fpfh_stats = dict(candidates=cand.value, queries=q.value, candidates_per_query=cand.value / max(q.value, 1),
                               fallbacks=fb.value, cell=cell.value)
        self.fpfh_ms = dict(knn_normals=float(ms[0]), spfh_fpfh=float(ms[1]), total=float(ms[2]))
        return self.fpfh_ms

    def fpfh_radius(self, normal_radius, feature_radius):
        """fpfh() with the radius estimator (ghicp_prep_fpfh_radius; see fpfh_extract_radius): normals over `normal_radius`,
        histograms over `feature_radius`, at the keypoints, kept on the device where fpfh() keeps them.  Returns the stage
        times {lists, normals, spfh_fpfh, total} in ms; fpfh_work then holds {normal_entries, feature_entries, spfh_points}."""
        ms, work = np.zeros(4, np.float32), np.zeros(3, np.int64)
        check(lib().ghicp_prep_fpfh_radius(self.h, normal_radius, feature_radius, ms.ctypes.data_as(C.POINTER(C.c_float)),
                                           work.ctypes.data_as(C.POINTER(C.c_longlong))))
        self.fpfh_radii = (float(normal_radius), float(feature_radius))
        self.fpfh_work = dict(normal_entries=int(work[0]), feature_entries=int(work[1]), spfh_points=int(work[2]))
        self.fpfh_ms = dict(lists=float(ms[0]), normals=float(ms[1]), spfh_fpfh=float(ms[2]), total=float(ms[3]))
        return self.fpfh_ms

    def get_fpfh(self):
        """The histograms of fpfh(): [n_kp][33] float32, rows in keypoint order."""
        out = np.zeros((self.n_kp, 33), np.float32)
        check(lib().ghicp_prep_get_fpfh(self.h, out.ctypes.data_as(C.POINTER(C.c_float))))
        return out

    def sac_ia(self, target, iterations=1000, samples=3, k=6, min_sample_distance=0.0, threshold=100.0, seed=0):
        """SAC-IA from this cloud's keypoints onto `target`'s (both after fpfh()), device to device: see sac_ia."""
        r = SacResult()
        check(lib().ghicp_prep_sac_ia(self.h, target.h, C.byref(_sac_params(iterations, samples, k, min_sample_distance, threshold,
                                                                             seed)), C.byref(r)))
        return _sac_out(r)

    def overlap(self, target, Rt=None, thre_dis=None, max_range=float("inf"), fitness=True):
        """cloud_overlap of this down-sampled cloud, moved by Rt, against `target`'s, device to device (ghicp_prep_overlap).
        `target` keeps its grid for later calls (its stage_ms["grid"] is then 0)."""
        if thre_dis is None:
            raise GhicpError(-1, "overlap: thre_dis is required")
        keep, rp = _overlap_rt(Rt)
        r = OverlapResult()
        check(lib().ghicp_prep_overlap(self.h, target.h, rp, float(thre_dis), float(max_range), int(bool(fitness)), C.byref(r)))
        del keep
        return _overlap_out(r)

    def icp(self, target, guess=None, max_iterations=50, reciprocal=False, trim_ratio=0.0, transformation_epsilon=1e-8,
            fitness_epsilon=1e-5, metric="point", normal_k=20, rotation_epsilon=1e-6):
        """cloud_icp of this down-sampled cloud onto `target`'s, device to device (ghicp_prep_icp).  The target's grid is the one
        overlap() keeps (its stage_ms["grid"] is 0 once either has built it); with metric="plane" the target also keeps its
        normals for that normal_k (stage_ms["grid"] is 0 again on a second call with the same k), with metric="gicp" both
        results keep theirs (one set per result, shared by the metrics and by either role).  Returns (Rt, info) as
        cloud_icp."""
        keep, gp = _overlap_rt(guess)
        r = IcpResult()
        rc = check(lib().ghicp_prep_icp(self.h, target.h, gp, C.byref(_icp_params(max_iterations, reciprocal, trim_ratio,
                                                                                   transformation_epsilon, fitness_epsilon, metric,
                                                                                   normal_k, rotation_epsilon)),
                                        C.byref(r)))
        del keep
        return _icp_out(r, rc)

    def close(self):
        if getattr(self, "h", None):
            lib().ghicp_prep_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def check(rc, ctx=None):
    if rc < 0:
        msg = lib().ghicp_last_error(ctx)
        raise GhicpError(rc, msg.decode() if msg else "")
    return rc


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


def _ip(a):
    return a.ctypes.data_as(C.POINTER(C.c_int))


class _PinnedBlock:
    """Owner of one page-locked allocation (freed when the last numpy view of it is gone)."""

    def __init__(self, nbytes):
        self.ptr = C.c_void_p()
        check(lib().ghicp_host_alloc(max(int(nbytes), 1), C.byref(self.ptr)))
        self.nbytes = int(nbytes)

    def __del__(self):
        try:
            if self.ptr:
                lib().ghicp_host_free(self.ptr)
        except Exception:
            pass


def pinned_empty(shape, dtype=np.float64, order="C"):
    """numpy array in page-locked host memory (ghicp_host_alloc): set_keypoints / pairs(out=) / source(out=) then move it with
    one DMA, no staging copy inside the library."""
    dtype = np.dtype(dtype)
    shape = (shape,) if np.isscalar(shape) else tuple(shape)
    n = int(np.prod(shape)) if shape else 1
    blk = _PinnedBlock(n * dtype.itemsize)
    buf = (C.c_char * max(blk.nbytes, 1)).from_address(blk.ptr.value)
    buf._pinned_owner = blk   # the array's base object keeps the allocation alive; freed with the last view
    return np.frombuffer(buf, dtype=dtype, count=n).reshape(shape, order=order)


def pinned_copy(a, order="F"):
    out = pinned_empty(a.shape, a.dtype, order=order)
    out[...] = a
    return out


def comm_unique_id():
    """128-byte NCCL unique id (rank 0 creates it, the host runtime broadcasts it)."""
    buf = (C.c_char * 128)()
    check(lib().ghicp_comm_unique_id(buf))
    return bytes(buf)


def km_solve(W, sp=None, tp=None, eps=0.01, penalty=1000.0, device=0):
    """Stand-alone Km replacement on a dense weight matrix (include/km.h:38-53)."""
    W = np.ascontiguousarray(W, dtype=np.float64)
    n = W.shape[0]
    sp = n if sp is None else sp
    tp = n if tp is None else tp
    match = np.zeros(n, np.int32)
    e = C.c_double(0)
    r = C.c_int(0)
    check(lib().ghicp_km_solve(device, _dp(W), n, sp, tp, eps, penalty, _ip(match), C.byref(e), C.byref(r)))
    return match, e.value, r.value


def voxel_downsample(xyz, voxel_size, device=0):
    """CFilter::voxelfilter (include/filter.hpp:28-88) on the GPU: indices of the kept points, in output order."""
    xyz = np.ascontiguousarray(xyz, dtype=np.float32)
    out = np.zeros(len(xyz) + 1, np.int32)
    m = C.c_int(0)
    check(lib().ghicp_voxel_downsample(device, xyz.ctypes.data_as(C.POINTER(C.c_float)), len(xyz), voxel_size, _ip(out),
                                       C.byref(m)))
    return out[:m.value].copy()


def sor_filter(xyz, mean_k=50, std_mul=1.0, return_distances=False, device=0):
    """CFilter::SORFilter (include/filter.hpp:90-102; PCL's StatisticalOutlierRemoval) on the GPU, DESIGN.md §3.16: a finite
    point is kept unless its mean distance to its mean_k (1..128) nearest other finite points exceeds mean + std_mul * stddev
    of those distances; non-finite points are never kept.  Returns (kept indices ascending, info: n_finite, n_kept, k_eff,
    mean, stddev, threshold, candidates, fallbacks, stage_ms); + info["distances"] [n] float32 (NaN for non-finite points)
    with return_distances."""
    xyz = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
    n = len(xyz)
    out = np.zeros(max(n, 1), np.int32)
    dist = np.zeros(n, np.float32) if return_distances else None
    r = SorResult()
    fpp = C.POINTER(C.c_float)
    check(lib().ghicp_sor_filter(device, xyz.ctypes.data_as(fpp), n, int(mean_k), float(std_mul), _ip(out),
                                 None if dist is None else dist.ctypes.data_as(fpp), C.byref(r)))
    info = _sor_out(r)
    if dist is not None:
        info["distances"] = dist
    return out[:r.n_kept].copy(), info


def detect_keypoints(xyz, radius, ratio_max=0.65, min_pts=20, nms_radius=None, device=0):
    """CKeypointDetect::keypointDetectionBasedOnCurvature (include/keypoint_detect.hpp:27-51) on the GPU.
    Returns (keypoint indices in the reference's output order, eigenvalues [n][3], curvature [n], neighbour counts)."""
    xyz = np.ascontiguousarray(xyz, dtype=np.float32)
    n = len(xyz)
    kp, m = np.zeros(n, np.int32), C.c_int(0)
    lam, curv, cnt = np.zeros((n, 3), np.float32), np.zeros(n), np.zeros(n, np.int32)
    check(lib().ghicp_detect_keypoints(device, xyz.ctypes.data_as(C.POINTER(C.c_float)), n, radius, ratio_max, min_pts,
                                       nms_radius if nms_radius is not None else radius, _ip(kp), C.byref(m),
                                       lam.ctypes.data_as(C.POINTER(C.c_float)), _dp(curv), _ip(cnt)))
    return kp[:m.value].copy(), lam, curv, cnt


def bsc_default_pattern(side=7):
    """The grid-pair sampling pattern of the reference's BSCEncoder constructor (binary_feature_extraction.hpp:75-103) in a
    fresh process = the sample_pattern.txt its users generate.  [side*side][2] int32; only side 7 is shipped."""
    pairs = np.zeros((side * side, 2), np.int32)
    check(lib().ghicp_bsc_default_pattern(side, _ip(pairs)))
    return pairs


def read_sample_pattern(path, side=7):
    """sample_pattern.txt as the reference reads it (:107-116): side*side lines of two cell indices."""
    vals = np.loadtxt(path, dtype=np.int64).reshape(-1, 2)
    if len(vals) < side * side:
        raise GhicpError(-1, f"{path}: expected {side * side} pairs, found {len(vals)}")
    return np.ascontiguousarray(vals[:side * side], dtype=np.int32)


def bsc_extract(xyz, kp_idx, extract_radius, dof_type=6, side=7, pairs=None, device=0):
    """BSCEncoder::extractBinaryFeatures (include/binary_feature_extraction.hpp:603-676) on the GPU.
    Returns (features [V][nkp][ceil(9 side^2 / 8)] uint8, lrf [nkp][12] float32, status [nkp]); V = 1 / 2 / 4 for
    dof_type 0 / 1..4 / > 4, the layout Keypoints.setBSCfeature / ghicp_set_bsc take (bits = 9 side^2)."""
    xyz = np.ascontiguousarray(xyz, dtype=np.float32)
    kp_idx = np.ascontiguousarray(kp_idx, dtype=np.int32)
    pairs = bsc_default_pattern(side) if pairs is None else np.ascontiguousarray(pairs, dtype=np.int32)
    nkp = len(kp_idx)
    nbytes = (9 * side * side + 7) // 8
    feats = np.zeros((4, nkp, nbytes), np.uint8)
    lrf, status, V = np.zeros((nkp, 12), np.float32), np.zeros(nkp, np.int32), C.c_int(0)
    check(lib().ghicp_bsc_extract(device, xyz.ctypes.data_as(C.POINTER(C.c_float)), len(xyz), _ip(kp_idx), nkp, extract_radius,
                                  side, _ip(pairs), dof_type, feats.ctypes.data, C.byref(V),
                                  lrf.ctypes.data_as(C.POINTER(C.c_float)), _ip(status)))
    # the ABI writes [V][nkp][bytes] contiguously: re-view the first V * nkp * bytes bytes with that shape
    out = feats.reshape(-1)[:V.value * nkp * nbytes].reshape(V.value, nkp, nbytes).copy()
    return out, lrf, status


def fpfh_extract(xyz, idx=None, k=20, device=0):
    """FPFHfeature::compute_fpfh_feature (idx None: every point) / + keyfpfh (idx = keypoint indices) on the GPU,
    include/fpfh.hpp:36-115 with k-NN normals and histograms (DESIGN.md §3.10).
    Returns (fpfh [len(idx) or n][33] float32, normals [n][3] float32, status [n] int32: 1 = NaN normal, n < 3)."""
    xyz = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
    n = len(xyz)
    fpp = C.POINTER(C.c_float)
    ia = None if idx is None else np.ascontiguousarray(idx, dtype=np.int32).reshape(-1)
    m = n if ia is None else len(ia)
    fpfh = np.zeros((m, 33), np.float32)
    normals, status = np.zeros((n, 3), np.float32), np.zeros(n, np.int32)
    check(lib().ghicp_fpfh_extract(device, xyz.ctypes.data_as(fpp), n, None if ia is None else _ip(ia), m, k,
                                   fpfh.ctypes.data_as(fpp), normals.ctypes.data_as(fpp), _ip(status)))
    return fpfh, normals, status


def fpfh_extract_radius(xyz, idx=None, normal_radius=None, feature_radius=None, device=0):
    """CRegistration::compute_fpfh_feature (src/common_reg.cpp:373-389) on the GPU: PCL's NormalEstimation and FPFHEstimation
    with radius searches (DESIGN.md §3.10, "Radius neighbourhoods").  Normals over every point within `normal_radius`,
    histograms over every point within `feature_radius` (strict d2 < r*r in float32).  Returns (fpfh [len(idx) or n][33]
    float32, normals [n][3] float32, status [n] int32: 1 = NaN normal, fewer than 3 points within the radius; 2 = normal not
    needed by the requested histograms, NaN)."""
    if normal_radius is None or feature_radius is None:
        raise GhicpError(-1, "fpfh_extract_radius: normal_radius and feature_radius are required")
    xyz = np.ascontiguousarray(xyz, dtype=np.float32).reshape(-1, 3)
    n = len(xyz)
    fpp = C.POINTER(C.c_float)
    ia = None if idx is None else np.ascontiguousarray(idx, dtype=np.int32).reshape(-1)
    m = n if ia is None else len(ia)
    fpfh = np.zeros((m, 33), np.float32)
    normals, status = np.zeros((n, 3), np.float32), np.zeros(n, np.int32)
    check(lib().ghicp_fpfh_extract_radius(device, xyz.ctypes.data_as(fpp), n, None if ia is None else _ip(ia), m,
                                          float(normal_radius), float(feature_radius), fpfh.ctypes.data_as(fpp),
                                          normals.ctypes.data_as(fpp), _ip(status)))
    return fpfh, normals, status


def sac_ia(src_xyz, src_fpfh, tgt_xyz, tgt_fpfh, iterations=1000, samples=3, k=6, min_sample_distance=0.0, threshold=100.0,
           seed=0, device=0):
    """FPFHfeature::fpfhalign (include/fpfh.hpp:117-133; PCL SampleConsensusInitialAlignment) on the GPU, DESIGN.md §3.11:
    `iterations` hypotheses of `samples` source points, each paired with one of its `k` nearest target histograms, scored by
    the truncated error over all source points with `threshold` on SQUARED distances.  Deterministic for a given `seed`.
    Returns (Rt 4x4 mapping the source onto the target, info: error, fitness, inliers, best_hypothesis, invalid_hypotheses,
    stage_ms)."""
    fpp = C.POINTER(C.c_float)
    P = np.ascontiguousarray(src_xyz, dtype=np.float32).reshape(-1, 3)
    Fs = np.ascontiguousarray(src_fpfh, dtype=np.float32).reshape(-1, 33)
    Q = np.ascontiguousarray(tgt_xyz, dtype=np.float32).reshape(-1, 3)
    Ft = np.ascontiguousarray(tgt_fpfh, dtype=np.float32).reshape(-1, 33)
    if len(P) != len(Fs) or len(Q) != len(Ft):
        raise GhicpError(-1, "sac_ia: one histogram per point expected")
    r = SacResult()
    check(lib().ghicp_sac_ia(device, P.ctypes.data_as(fpp), Fs.ctypes.data_as(fpp), len(P), Q.ctypes.data_as(fpp),
                             Ft.ctypes.data_as(fpp), len(Q), C.byref(_sac_params(iterations, samples, k, min_sample_distance,
                                                                                threshold, seed)), C.byref(r)))
    return _sac_out(r)


def cloud_overlap(A, B, Rt=None, thre_dis=None, max_range=float("inf"), fitness=True, return_d2=False, device=0):
    """Overlap and fitness of cloud A moved by Rt (4x4, None = identity) against cloud B on the GPU, DESIGN.md §3.12:
    overlap = points of A with a B point at d2 < thre_dis^2 (CRegistration::calOverlap, src/common_reg.cpp:294-317), ratio =
    (0.01 + overlap) / n, overlap_rmse over those points; fitness = mean d2 over the points with d2 <= max_range (PCL's
    getFitnessScore; max_range bounds SQUARED distances), DBL_MAX when there are none.  fitness=False is the overlap-only mode
    (n_fit 0, fitness and overlap_rmse NaN).  Returns a dict (+ "d2" [n] float32 with return_d2, fitness mode only)."""
    if thre_dis is None:
        raise GhicpError(-1, "cloud_overlap: thre_dis is required")
    fpp = C.POINTER(C.c_float)
    A = np.ascontiguousarray(A, dtype=np.float32).reshape(-1, 3)
    B = np.ascontiguousarray(B, dtype=np.float32).reshape(-1, 3)
    keep, rp = _overlap_rt(Rt)
    d2 = np.zeros(len(A), np.float32) if return_d2 else None
    r = OverlapResult()
    check(lib().ghicp_cloud_overlap(device, A.ctypes.data_as(fpp), len(A), B.ctypes.data_as(fpp), len(B), rp, float(thre_dis),
                                    float(max_range), int(bool(fitness)), C.byref(r), None if d2 is None else d2.ctypes.data_as(fpp)))
    del keep
    out = _overlap_out(r)
    if d2 is not None:
        out["d2"] = d2
    return out


def cloud_icp(S, T, guess=None, max_iterations=50, reciprocal=False, trim_ratio=0.0, transformation_epsilon=1e-8,
              fitness_epsilon=1e-5, return_moved=False, trace=False, device=0, metric="point", normal_k=20, rotation_epsilon=1e-6):
    """Point-to-point ICP of source S onto target T on the GPU, DESIGN.md §3.13: PCL's IterativeClosestPoint as
    CRegistration::icp_reg configures it (src/common_reg.cpp:44-107), starting from `guess` (4x4, None = identity).
    reciprocal = setUseReciprocalCorrespondences; trim_ratio > 0 adds CorrespondenceRejectorTrimmed with that overlap ratio.
    metric="plane" estimates each step point-to-plane against T's k-NN normals (k = normal_k, 3..32), DESIGN.md §3.14: PCL's
    IterativeClosestPointWithNormals as CRegistration::ptplicp_reg configures it (src/common_reg.cpp:123-199).
    metric="gicp" runs Generalized ICP, DESIGN.md §3.15: PCL's GeneralizedIterativeClosestPoint as CRegistration::gicp_reg
    configures it (src/common_reg.cpp:217-284), with both clouds' k-NN normals as covariances, a Gauss-Newton inner loop, and
    PCL's GICP stop (max_iterations, or no transform entry moved by more than rotation_epsilon / transformation_epsilon);
    fitness_epsilon is not read, and reciprocal / trim_ratio apply as for the other metrics.
    Returns (Rt 4x4 mapping S onto T, info: iterations, converged, state (ITERATIONS, TRANSFORM, ABS_MSE, REL_MSE,
    NO_CORRESPONDENCES or, point-to-plane and GICP only, SINGULAR), cor and mse of the last iteration, fitness = PCL's
    getFitnessScore, warnings (GHICP_W_FEW_PAIRS when fewer than 3 pairs were left, GHICP_W_SINGULAR for a singular system),
    work counters, stage_ms); + "moved" (S moved by Rt) with return_moved, + "cor_trace" / "mse_trace" per iteration with
    trace."""
    fpp = C.POINTER(C.c_float)
    S = np.ascontiguousarray(S, dtype=np.float32).reshape(-1, 3)
    T = np.ascontiguousarray(T, dtype=np.float32).reshape(-1, 3)
    keep, gp = _overlap_rt(guess)
    K = max(int(max_iterations), 1)
    moved = np.zeros_like(S) if return_moved else None
    cor_tr, mse_tr = (np.zeros(K, np.int32), np.zeros(K)) if trace else (None, None)
    r = IcpResult()
    rc = check(lib().ghicp_cloud_icp(device, S.ctypes.data_as(fpp), len(S), T.ctypes.data_as(fpp), len(T), gp,
                                     C.byref(_icp_params(max_iterations, reciprocal, trim_ratio, transformation_epsilon,
                                                         fitness_epsilon, metric, normal_k, rotation_epsilon)), C.byref(r),
                                     None if moved is None else moved.ctypes.data_as(fpp), None if cor_tr is None else _ip(cor_tr),
                                     None if mse_tr is None else _dp(mse_tr)))
    del keep
    Rt, info = _icp_out(r, rc)
    if moved is not None:
        info["moved"] = moved
    if trace:
        info["cor_trace"], info["mse_trace"] = cor_tr[:r.iterations].copy(), mse_tr[:r.iterations].copy()
    return Rt, info


def rigid_fit_ex(S, T, solver=SOLVER_SVD, normals=None, weights=None, device=0):
    """Opt-in estimators (ghicp_solver_type): weighted point-to-point, point-to-plane LLS, yaw-only 4-DoF.
    Returns (Rt 4x4, warning bits)."""
    S = np.asfortranarray(S, dtype=np.float64)
    T = np.asfortranarray(T, dtype=np.float64)
    Nn = None if normals is None else np.asfortranarray(normals, dtype=np.float64)
    W = None if weights is None else np.ascontiguousarray(weights, dtype=np.float64)
    Rt = np.zeros(16)
    rc = check(lib().ghicp_rigid_fit_ex(device, solver, _dp(S), _dp(T), None if Nn is None else _dp(Nn),
                                        None if W is None else _dp(W), S.shape[0], _dp(Rt)))
    return Rt.reshape(4, 4).T.copy(), rc


def rigid_fit(S, T, device=0):
    S = np.asfortranarray(S, dtype=np.float64)
    T = np.asfortranarray(T, dtype=np.float64)
    Rt = np.zeros(16)
    check(lib().ghicp_rigid_fit(device, _dp(S), _dp(T), S.shape[0], _dp(Rt)))
    return Rt.reshape(4, 4).T.copy()
