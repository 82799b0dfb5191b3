/*
 * ghicp_b200.h — C ABI of the B200-native GH-ICP registration inner loop (libghicp_b200.so).
 *
 * Drop-in boundary for the hot path of YuePanEdward/GH-ICP (citations: file:line in the reference):
 * the private stage methods of ghicp::GHRegistration (include/ghicp_reg.h:156-171) and the Km solver
 * (include/km.h:32-61).  POD only — no Eigen / PCL / STL / torch types cross this boundary.
 * Every function returns an int status (0 = ok, <0 = GHICP_E_*, >0 = GHICP_W_* warning bits);
 * nothing throws across the ABI.  One ctx = one host thread at a time; a ctx owns one CUDA device,
 * one stream and all its device memory.
 *
 * Layout conventions
 *   coordinates : Eigen::MatrixX3d::data() layout = column-major N x 3 = SoA x[N], y[N], z[N]
 *                 (include/ghicp_reg.h:47, Keypoints::kpSXYZ / kpTXYZ)
 *   BSC bits    : bit k of a descriptor lives in byte k/8, bit k%8, LSB first
 *                 (include/stereo_binary_feature.h:140-146); B = ceil(bits/8) bytes
 *   FPFH        : float[33] per keypoint (pcl::FPFHSignature33::histogram, include/fpfh.hpp:135)
 *   transforms  : 4x4 column-major doubles = Eigen::Matrix4d::data()
 */
#ifndef GHICP_B200_H_
#define GHICP_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GHICP_ABI_VERSION 2

/* enum values follow include/utility.h:51-64 */
enum ghicp_feature_type { GHICP_FT_BSC = 0, GHICP_FT_ROPS = 1, GHICP_FT_FPFH = 2, GHICP_FT_NONE = 3 };
enum ghicp_corr_type { GHICP_CT_NN = 0, GHICP_CT_NNR = 1, GHICP_CT_KM = 2 };
/* Transform estimation.  The reference loop always runs GHICP_SOLVER_SVD (unweighted point-to-point, PCL
 * TransformationEstimationSVD, src/ghicp_reg.cpp:857-859).  The others are OPT-IN extensions named by
 * BASELINE.json's north_star / configs 3 and 5 (SURVEY.md §8a-9, §8f N4); the reference holds them only as code the
 * loop never calls, so their parity is pinned by restatement + analytic tests only:
 *   WEIGHTED_SVD    per-pair weights w_k >= 0 in the centroids and the cross-covariance (w = 1 reproduces SVD)
 *   POINT_TO_PLANE  linearised point-to-plane least squares, rows [s x n, n], rhs n.(t - s), 6x6 normal equations,
 *                   R = Rz(gamma) Ry(beta) Rx(alpha)  (PCL TransformationEstimationPointToPlaneLLS, the estimator
 *                   behind IterativeClosestPointWithNormals in src/common_reg.cpp:123-199)
 *   YAW_4DOF        Gauss-Newton on (yaw, tx, ty, tz), CRegistration::LLS_4DOF (src/common_reg.cpp:623-775) */
enum ghicp_solver_type {
  GHICP_SOLVER_SVD = 0,
  GHICP_SOLVER_WEIGHTED_SVD = 1,
  GHICP_SOLVER_POINT_TO_PLANE = 2,
  GHICP_SOLVER_YAW_4DOF = 3
};

enum ghicp_status {
  GHICP_OK = 0,
  GHICP_E_ARG = -1,    /* bad argument / call order */
  GHICP_E_NOMEM = -2,  /* device or host allocation failed / workspace budget exceeded */
  GHICP_E_CUDA = -3,   /* CUDA runtime error, see ghicp_last_error */
  GHICP_E_NCCL = -4,   /* NCCL error / NCCL not loadable */
  GHICP_E_NOCONV = -5, /* ghicp_run hit max_iter without converging */
  GHICP_E_NODEV = -6,  /* no CUDA device: the product path has NO CPU fallback */
  GHICP_W_FEW_PAIRS = 1, /* cor < min_cor (include/ghicp_reg.h:36, src/ghicp_reg.cpp:796-797) */
  GHICP_W_SINGULAR = 2   /* point-to-plane ICP or GICP: the normal equations of an iteration were singular (GHICP_ICP_SINGULAR) */
};

/* Constructor arguments of ghicp::GHRegistration (include/ghicp_reg.h:77-81) + Energyfunction::init
 * argument (include/ghicp_reg.h:26) + execution options. Zero-initialise, then fill. */
typedef struct ghicp_config {
  int feature_type;     /* ghicp_feature_type (Ft) */
  int corr_type;        /* ghicp_corr_type (Ct) */
  int dof;              /* dof_type: 6 → 4 BSC source variants, otherwise 2 (src/ghicp_reg.cpp:178-182) */
  float bbx_magnitude;  /* Energyfunction::init(.., bbx_magnitude) → scale = 0.005*bbx (ghicp_reg.h:40) */
  float nonmax;         /* radiusNonMax */
  float adjust_ratio;   /* weight_adjustment_ratio */
  float adjust_step;    /* weight_adjustment_step */
  float estimated_iou;  /* estimated_IoU */
  float converge_t;     /* converge_tran, reference default 0.02 m */
  float converge_r;     /* converge_rot, reference default 0.02 deg */
  int max_iter;         /* 0 = unbounded like the reference's while(!converge) (src/ghicp_reg.cpp:49) */
  int device;           /* CUDA device ordinal */
  double km_eps;        /* 0 → Energyfunction::KM_eps = 0.01 (ghicp_reg.h:38) */
  int verbose;          /* 0 = silent (the reference prints every iteration; we do not by default) */
  int force_exact;      /* 1 = all-double cost kernels only (no FP32 filter); results are identical, slower */
  int fpfh_matrix_free; /* FPFH only: 0 = auto (NN / NNR: matrix-free, no N x M array at all — the sweeps recompute the
                           feature distance and run the FP32-filter + exact-refinement fast path; KM: stored float plane
                           while it fits in 40 % of the free device memory), 1 = always matrix-free, -1 = always store
                           the plane (all-double sweeps).  Correspondences and transforms are identical either way. */
  int solver;           /* ghicp_solver_type used by ghicp_iterate; 0 = the reference's SVD.  POINT_TO_PLANE needs
                           ghicp_set_target_normals.  WEIGHTED_SVD is stand-alone only (ghicp_rigid_fit_ex). */
  int reserved[4];
} ghicp_config;

/* Everything one loop body of GHRegistration::ghicp_reg (src/ghicp_reg.cpp:49-103) reports. */
typedef struct ghicp_iter_stats {
  int iteration;        /* iteration_number this body ran with (starts at 0) */
  int cor;              /* number of correspondences */
  int converged;        /* converge flag after this iteration */
  int warnings;         /* GHICP_W_* bits */
  double Rt[16];        /* this iteration's transform (Rt_temp), column-major */
  double Rt_tillnow[16];/* accumulated transform */
  double cd_mean, cd_std, penalty;          /* calCD_* outputs.  FPFH fast path (stream_passes > 0): cd_mean is the FP32
                                               filter's ESTIMATE — the statistic is heavy-tailed (ED / FD^ex with FD near
                                               0) and no decision depends on it on the iterations that take that path */
  double rmse, rmse_after, fdm, fdstd, iou; /* findcorrespondence* / transformestimation outputs */
  double para1, para2;                      /* after adjustweight */
  double km_energy;                         /* Km::Calenergy equivalent (KM mode) */
  double ax, ay, az;                        /* Euler angles in degrees (src/ghicp_reg.cpp:873-879) */
  /* execution detail */
  long long nnz;        /* KM: candidate edges with CD < penalty */
  int km_rounds;        /* KM: auction bidding rounds (forward + reverse) */
  int km_phases;        /* KM: epsilon-scaling phases */
  int gpu_launches;     /* kernels launched by this call */
  int exact_fallback;   /* bit 0: this iteration re-ran its cost stage with the all-double kernels; bit 1: a settled KM
                           iteration's candidate block overflowed and the iteration re-ran on the general route; bit 2: the
                           redo of bit 0 was taken because the keypoints' scale put the FP32 filter's operands outside the
                           float range its error bound holds in (None / BSC: roughly 1e-5 ... 1e10 units of extent) */
  float ms_cost, ms_corr, ms_solve, ms_total; /* CUDA-event stage times on the ctx stream */
  float ms_stream;      /* CUDA-event time of ONE streaming pass over the FD plane (the dominant kernel) */
  int stream_passes;    /* passes over the FD plane this iteration (1 NN/NNR, +1 seed pass, 2-3 KM) */
  long long candidates; /* NN/NNR: pairs the FP32 filter handed to exact FP64 evaluation.  Once the candidate buffer has
                           overflowed (exact_fallback bit 0) the count stops growing near the buffer's capacity: it is then
                           a lower bound */
} ghicp_iter_stats;

typedef struct ghicp_ctx ghicp_ctx;

int ghicp_abi_version(void);
int ghicp_device_count(void);
const char *ghicp_last_error(const ghicp_ctx *ctx); /* ctx may be NULL: last global error */

/* GHRegistration::GHRegistration (include/ghicp_reg.h:77-117). */
int ghicp_create(const ghicp_config *cfg, ghicp_ctx **out);
int ghicp_destroy(ghicp_ctx *ctx);

/* Keypoints::setCoordinate (include/ghicp_reg.h:54-60). Copies host → device. May be called again
 * with the same N, M to replace the coordinates (e.g. to restart, or to re-upload per iteration). */
int ghicp_set_keypoints(ghicp_ctx *ctx, const double *sxyz, int N, const double *txyz, int M);
/* Keypoints::setBSCfeature (include/ghicp_reg.h:62-66). s_bits [V][N][B], t_bits [M][B]. */
int ghicp_set_bsc(ghicp_ctx *ctx, const uint8_t *s_bits, int V, const uint8_t *t_bits, int bits);
/* Keypoints::setFPFHfeature (include/ghicp_reg.h:68-72). s [N][33], t [M][33]. */
int ghicp_set_fpfh(ghicp_ctx *ctx, const float *s, const float *t);

/* Unit normals of the target keypoints, column-major M x 3 (only read by GHICP_SOLVER_POINT_TO_PLANE; the
 * reference estimates them by k-NN PCA inside PCL, src/common_reg.cpp:149-150 — here the caller supplies them). */
int ghicp_set_target_normals(ghicp_ctx *ctx, const double *nxyz);
/* Change the in-loop estimator of an existing context (same values / rules as ghicp_config.solver). */
int ghicp_set_solver(ghicp_ctx *ctx, int solver);

/* calFD_BSC / calFD_FPFH (src/ghicp_reg.cpp:143-214): one-time feature-distance build. */
int ghicp_build_fd(ghicp_ctx *ctx);

/* One body of while(!converge): calED + calCD_* + findcorrespondence* + transformestimation +
 * adjustweight + Rt_tillnow update (src/ghicp_reg.cpp:49-103, viewer excluded). */
int ghicp_iterate(ghicp_ctx *ctx, ghicp_iter_stats *out);

/* GHRegistration::ghicp_reg (src/ghicp_reg.cpp:24-112): build FD if needed, iterate to convergence. */
int ghicp_run(ghicp_ctx *ctx, double Rt_final[16], int *iterations);

/* Results of the last iteration. */
int ghicp_get_pairs(ghicp_ctx *ctx, int *sp, int *tp, int cap, int *n); /* SP/TP index lists */
int ghicp_get_source(ghicp_ctx *ctx, double *sxyz);                     /* current KP.kpSXYZ */
int ghicp_get_rt(ghicp_ctx *ctx, double Rt_tillnow[16]);
/* Page-locked host memory (cudaMallocHost).  Optional: coordinate / result buffers allocated here (or page-locked by the
 * caller in any other way) are moved by ghicp_set_keypoints / ghicp_get_pairs / ghicp_get_source with one DMA each; pageable
 * buffers go through a staging copy inside the library.  The reference has no counterpart (its matrices live in host RAM). */
int ghicp_host_alloc(size_t bytes, void **out);
int ghicp_host_free(void *p);
/* FD plane as doubles, row-major N x M (Energyfunction::FD). Test/debug: O(N*M) host memory. */
int ghicp_get_fd(ghicp_ctx *ctx, double *fd);
/* Per-source-row argmin of CD for the state *before* the next iterate (NN scan,
 * src/ghicp_reg.cpp:715-733) without advancing the loop. idx[N], cd[N] (either may be NULL). */
int ghicp_probe_rowmin(ghicp_ctx *ctx, int *idx, double *cd, double *cd_mean, double *cd_std,
                       double *penalty);
/* Loop state the reference keeps between iterations (include/ghicp_reg.h:173-202); for resume/tests. */
int ghicp_set_state(ghicp_ctx *ctx, int iteration, double rms, double fdm, double fdstd, double para1,
                    double para2);
/* Back to the state the GHRegistration constructor leaves (include/ghicp_reg.h:77-117: iteration 0, RMS 99999,
 * para1 = para2 = 1, converge = 0, Rt_tillnow = I) without touching the descriptors or the FD plane: a second
 * registration of the same keypoint sets (ghicp_set_keypoints re-uploads the untransformed source). */
int ghicp_reset(ghicp_ctx *ctx);

/* ---- stand-alone stages -------------------------------------------------------------------- */
/* Km(graph, eps, penalty).kmsolve() + output() (include/km.h:38-53, src/km.cpp:40-233) on a dense
 * n x n row-major weight matrix built like src/ghicp_reg.cpp:348-365 (w = -CD if CD < penalty else
 * -penalty).  match[y] = x for kept pairs, -1 for pairs the reference drops (w == -penalty).
 * energy = Km::Calenergy().  Solved on the GPU by epsilon-scaled forward/reverse auction. */
int ghicp_km_solve(int device, const double *W, int n, int sp, int tp, double eps, double penalty,
                   int *match, double *energy, int *rounds);
/* pcl TransformationEstimationSVD::estimateRigidTransformation as called at src/ghicp_reg.cpp:857-866.
 * s, t column-major n x 3 (Spoint / Tpoint). */
int ghicp_rigid_fit(int device, const double *s, const double *t, int n, double Rt[16]);
/* Opt-in estimators (see ghicp_solver_type).  s, t column-major n x 3; tn = target normals, column-major n x 3
 * (POINT_TO_PLANE, else may be NULL); w = n weights or NULL (all ones).  solver = SVD with w == NULL is
 * ghicp_rigid_fit.  YAW_4DOF starts from yaw0 = 0 like a leveled scan pair (src/common_reg.cpp:646 takes the
 * initial guess from the caller). */
int ghicp_rigid_fit_ex(int device, int solver, const double *s, const double *t, const double *tn, const double *w,
                       int n, double Rt[16]);

/* ---- pre-processing on the GPU (SURVEY.md §8f row N1; BASELINE.json configs 4 / 5) ------------------------------
 * The steps of test/ghicp_main.cpp:86-100 that produce the keypoints the loop consumes.  xyz = [n][3] float32 (PCL
 * points are float32).  Where the reference's result is implementation-defined (unstable std::sort) or delegated to PCL,
 * the canonical definitions documented in oracle/ghicp_prep_oracle.cpp apply.
 * Non-finite points (NaN or infinite in any coordinate, as in an organised scan) take no part in any pre-processing entry
 * point: each returns what it returns on the cloud's finite points, indices mapped back to xyz (pcl::removeNaNFromPointCloud,
 * then the reference).  What that means per entry point is stated with it. */
/* CFilter::voxelfilter (include/filter.hpp:28-88): one point per occupied voxel — the one with the smallest index — in
 * ascending voxel-id order, preceded by point 0 (the reference's phantom voxel-0 entries, :52 + :66).  A non-finite point is
 * never emitted; the phantom entry is the first finite point; without a finite point *n_out = 0.  out_idx: capacity n + 1. */
int ghicp_voxel_downsample(int device, const float *xyz, int n, float voxel_size, int *out_idx, int *n_out);
/* CKeypointDetect::keypointDetectionBasedOnCurvature (include/keypoint_detect.hpp:27-51): radius PCA of every point
 * (include/pca.h:133-250), pruneUnstablePoints (:132-147, ratio_max = 0.65 and min_pts = 20 in ghicp_main.cpp:96-97),
 * non-maximum suppression by curvature (:149-191).  kp_idx (capacity n): keypoint indices in the reference's output order
 * (descending curvature).  lam [n][3] (eigenvalues, descending), curvature [n], pt_num [n] may be NULL.  A non-finite point
 * has lam = 0, curvature = 0, pt_num = 0, is nobody's neighbour and is never a keypoint. */
int ghicp_detect_keypoints(int device, const float *xyz, int n, float radius, float ratio_max, int min_pts, float nms_radius,
                           int *kp_idx, int *n_kp, float *lam, double *curvature, int *pt_num);

/* CFilter::SORFilter (include/filter.hpp:90-102): PCL's StatisticalOutlierRemoval on the canonical definition of DESIGN.md
 * §3.16.  Let F be the finite points, n_f = |F|, k_eff = min(mean_k, n_f - 1).  The mean distance d_p of p in F is the mean of
 * sqrt((double)d2) over the k_eff smallest float32 d2 = (dx*dx + dy*dy) + dz*dz from p to the OTHER points of F (duplicates
 * of p count, at 0), summed in double in ascending d2 order, divided by k_eff in double and rounded to float (0 when k_eff = 0).
 * mean = sum d / n_f, stddev = sqrt(sum (d - mean)^2 / (n_f - 1)) (two-pass; 0 when n_f <= 1), threshold = mean + std_mul *
 * stddev in double; p is kept unless (double)d_p > threshold, kept points in ascending index.  Non-finite points are nobody's
 * neighbour, have no distance (NaN in mean_dist) and are never kept (pcl::removeNaNFromPointCloud first; PCL itself would keep
 * NaN rows, with distance 0).  PCL's one-pass variance can go negative (NaN stddev, every point kept) on a cloud whose points
 * all have about the same mean distance; the two-pass form cannot.  Sums are in double in a fixed order: two calls give
 * identical bits.  mean_k in 1..128, std_mul finite (negative allowed, as in PCL); otherwise, for NULL xyz / out_idx / r or
 * n < 0, GHICP_E_ARG.  A cloud without a finite point returns GHICP_OK with nothing kept (mean, stddev, threshold 0). */
typedef struct ghicp_sor_result {
  int n_finite, n_kept, k_eff;
  int fallbacks;                 /* queries whose ring walk gave up and scanned every finite point (far outliers) */
  double mean, stddev, threshold;
  long long candidates;          /* points examined by every query together */
  float stage_ms[5];             /* CUDA events: grid, distances, statistics, compaction, total */
} ghicp_sor_result;
/* xyz [n][3] (host); out_idx (capacity n) receives the kept indices, mean_dist [n] (may be NULL) every point's d_p */
int ghicp_sor_filter(int device, const float *xyz, int n, int mean_k, double std_mul, int *out_idx, float *mean_dist,
                     ghicp_sor_result *r);

/* ---- BSC descriptor encoder on the GPU (SURVEY.md §8f row N2) -----------------------------------------------------
 * BSCEncoder<PointT>::extractBinaryFeatures (include/binary_feature_extraction.hpp:603-676, called at
 * test/ghicp_main.cpp:113-116 with voxel_side_num = 7, extract_radius = the keypoint NMS radius, dof_type 0 for the target
 * and reg_dof for the source): per keypoint the weighted-PCA local frame (:940-1035), the three projected
 * Gaussian-weighted grids (:197-373), the 9 side^2-bit descriptor (:464-565) and its variants (:762-837).
 * xyz [n][3] float32; kp_idx [nkp] indices into xyz; pairs [side^2][2] = the sampling pattern (sample_pattern.txt of the
 * reference, :107-116; ghicp_bsc_default_pattern for side 7).  features = [V][nkp][ceil(9 side^2 / 8)] bytes, V = 1
 * (dof_type 0), 2 (1..4) or 4 (> 4) — the layout ghicp_set_bsc takes.  lrf [nkp][12] (x, y, z axis, origin of variant 0)
 * and status [nkp] (0 ok, 1 = fewer than 3 neighbours or a non-finite keypoint: descriptor zero) may be NULL.  Non-finite
 * points are nobody's neighbour.  voxel_side_num <= 9.
 * Eigenvector signs (Eigen::EigenSolver's are implementation-defined) follow "largest component positive"; see DESIGN.md
 * §3.9 for the float32 accumulation tolerance against the reference. */
int ghicp_bsc_extract(int device, const float *xyz, int n, const int *kp_idx, int nkp, float extract_radius, int voxel_side_num,
                      const int *pairs, int dof_type, unsigned char *features, int *n_variants, float *lrf, int *status);
/* the pattern the reference's constructor generates (:75-103) in a fresh process; pairs [49][2]; voxel_side_num must be 7 */
int ghicp_bsc_default_pattern(int voxel_side_num, int *pairs);

/* ---- device-resident pre-processing pipeline (BASELINE.json configs 4 / 5) --------------------------------------------
 * The reference's driver runs, per cloud, voxel filter -> curvature keypoints -> BSC encoder (test/ghicp_main.cpp:89-116)
 * and hands the keypoint coordinates + descriptors to GHRegistration (:143-151).  ghicp_prep_run uploads the raw cloud ONCE
 * and chains the three stages on the device (each stage = the stand-alone entry point above, same results bit for bit);
 * nothing but the keypoint set ever needs to come back, and ghicp_set_from_prep moves even that device to device.  A cloud
 * with non-finite points gives bit for bit what its finite points give: n_down, the down-sampled cloud, keypoints, the
 * bounding box, BSC and FPFH (the down-sampled cloud holds finite points only).  A cloud without a finite point (or n <= 0)
 * leaves nothing to register: ghicp_prep_run returns GHICP_E_ARG and *out stays NULL.
 * stage_ms [5] = {host->device copy, voxel filter, keypoints, BSC encoder, total} from CUDA events (the total includes the
 * outlier filter of ghicp_prep_run_sor, which ghicp_prep_sor_info times). */
typedef struct ghicp_prep_params {
  float voxel_size;           /* CFilter::voxelfilter resolution (:89-90) */
  float neighborhood_radius;  /* PCA radius (:96) */
  float ratio_max;            /* 0.65 (:96) */
  int min_pts;                /* 20   (:97) */
  float nms_radius;           /* curvature non-maximum suppression radius (:97) */
  float bsc_radius;           /* BSC extract radius (:113-116: the NMS radius); <= 0: no descriptors */
  int bsc_side;               /* 7 */
  int dof_type;               /* BSC variants: 0 -> 1 (target, :115), 1..4 -> 2, > 4 -> 4 (source, :116) */
} ghicp_prep_params;
typedef struct ghicp_prep ghicp_prep;
int ghicp_prep_run(int device, const float *xyz, int n, const ghicp_prep_params *p, const int *bsc_pairs, ghicp_prep **out);
/* ghicp_prep_run with ghicp_sor_filter (mean_k, std_mul) applied to the DOWN-SAMPLED cloud, between the voxel filter and
 * the keypoints: the voxel filter evens a raw scan's range-dependent density first, so that the filter removes isolated
 * returns rather than far-range surface.  The result's down-sampled cloud, bounding box, keypoints and everything derived
 * from them are those of the kept points.  mean_k = 0 runs no filter (= ghicp_prep_run); otherwise mean_k in 1..128 and
 * std_mul finite.  A filter that keeps nothing returns GHICP_E_ARG, as a cloud without a finite point does. */
int ghicp_prep_run_sor(int device, const float *xyz, int n, const ghicp_prep_params *p, const int *bsc_pairs, int mean_k,
                       double std_mul, ghicp_prep **out);
/* the filter's result, the down-sampled cloud's size before it (n_voxel) and its time in ms (CUDA events); any output may
 * be NULL.  GHICP_E_ARG for a result made without the filter. */
int ghicp_prep_sor_info(const ghicp_prep *h, ghicp_sor_result *r, int *n_voxel, float *ms);
int ghicp_prep_info(const ghicp_prep *h, int *n_down, int *n_kp, int *n_variants, float bbox_min[3], float bbox_max[3],
                    float stage_ms[5]);
/* any of the outputs may be NULL: down_xyz [n_down][3], kp_idx [n_kp] (into the down-sampled cloud), kp_xyz [3][n_kp]
 * doubles (Eigen::MatrixX3d layout), bsc_bits [V][n_kp][ceil(9 side^2 / 8)] */
int ghicp_prep_get(const ghicp_prep *h, float *down_xyz, int *kp_idx, double *kp_xyz, unsigned char *bsc_bits);
int ghicp_prep_destroy(ghicp_prep *h);
/* Keypoints::setCoordinate + setBSCfeature / setFPFHfeature (include/ghicp_reg.h:52-72) straight from two pipeline results
 * on the same device: no host copy of coordinates or descriptors.  BSC descriptors are set when the context's feature type
 * is BSC; FPFH histograms when it is FPFH and both results carry them (ghicp_prep_fpfh). */
int ghicp_set_from_prep(ghicp_ctx *ctx, const ghicp_prep *source, const ghicp_prep *target);

/* ---- FPFH estimator on the GPU ---------------------------------------------------------------------------------------
 * FPFHfeature::compute_fpfh_feature + keyfpfh (include/fpfh.hpp:36-115, called at test/ghicp_main.cpp:120-127): PCL
 * NormalEstimation (k-NN, viewpoint 0) and FPFHEstimation (k-NN) on the canonical definition of DESIGN.md §3.10 (exact
 * k-NN in ascending (distance, index) order, smallest-eigenvector normals flipped towards the origin, 3 x 11 bin SPFH, the
 * 1 / d^2 weighted FPFH without the point's own SPFH).  xyz [n][3] float32; idx [nidx] = the points whose histograms are
 * wanted (NULL: every point, nidx ignored); k in 3..32 (the reference uses 20); fpfh [nidx][33].  normals [n][3] (NaN
 * where status = 1, i.e. fewer than 3 finite points in the cloud or a non-finite point) and status [n] may be NULL.
 * Non-finite points are nobody's neighbour (k_eff = min(k, finite points)); their own histogram row is zero.  The histogram at a point depends
 * only on its neighbours, so a subset equals the same rows of the whole-cloud result. */
int ghicp_fpfh_extract(int device, const float *xyz, int n, const int *idx, int nidx, int k, float *fpfh, float *normals,
                       int *status);
/* Histograms at the keypoints of a pipeline result, on its down-sampled cloud, kept on the device (ghicp_set_from_prep
 * moves them into an FPFH context).  stage_ms [3] = {k-NN + normals, SPFH + FPFH, total} from CUDA events; may be NULL. */
int ghicp_prep_fpfh(ghicp_prep *h, int k, float stage_ms[3]);
/* fpfh [n_kp][33] */
int ghicp_prep_get_fpfh(const ghicp_prep *h, float *fpfh);
/* Work of the last ghicp_prep_fpfh: k-NN candidates examined (all queries together), queries, queries that fell back to
 * the exhaustive scan, grid cell edge.  Any output may be NULL. */
int ghicp_prep_fpfh_stats(const ghicp_prep *h, long long *candidates, int *queries, int *fallbacks, float *cell);
/* The same estimator over radius neighbourhoods, as CRegistration::compute_fpfh_feature (src/common_reg.cpp:373-389, PCL
 * setRadiusSearch) computes it (DESIGN.md §3.10, "Radius neighbourhoods"): N_r(p) = every point q with d2(p, q) < r*r (float32,
 * the query and its duplicates included) in ascending (d2, index) order; normals over N_normal_radius (NaN, status 1, with
 * fewer than 3 points), SPFH and FPFH over N_feature_radius.  Arguments and outputs as ghicp_fpfh_extract; with idx given,
 * only what those histograms read is computed and the other normals are NaN with status 2.  A non-finite point is nobody's
 * neighbour and has a NaN normal, status 1 and a zero histogram row.  Radii must be positive and
 * finite (GHICP_E_ARG).  The neighbour lists live in device memory: when they would exceed the budget (half the free device
 * memory at 16 bytes per entry) the call returns GHICP_E_NOMEM, with the entry count in the message, before writing any
 * output. */
int ghicp_fpfh_extract_radius(int device, const float *xyz, int n, const int *idx, int nidx, float normal_radius,
                              float feature_radius, float *fpfh, float *normals, int *status);
/* ghicp_prep_fpfh with the radius estimator: the keypoint histograms of the down-sampled cloud, stored where ghicp_prep_fpfh
 * stores them (ghicp_set_from_prep, ghicp_prep_get_fpfh and ghicp_prep_sac_ia read them unchanged).  stage_ms [4] = {lists,
 * normals, SPFH + FPFH, total}; work [3] = {normal-radius list entries, feature-radius list entries, SPFH points}; both may
 * be NULL. */
int ghicp_prep_fpfh_radius(ghicp_prep *h, float normal_radius, float feature_radius, float stage_ms[4], long long work[3]);

/* ---- SAC-IA coarse alignment on the GPU -------------------------------------------------------------------------------
 * FPFHfeature::fpfhalign (include/fpfh.hpp:117-133: PCL SampleConsensusInitialAlignment, correspondence randomness 6) and
 * CRegistration::Coarsereg_FPFHSAC (src/common_reg.cpp:393-423, randomness 15) on the canonical definition of DESIGN.md
 * §3.11: max_iterations independent hypotheses of nr_samples source points (counter-based SplitMix64 draws from seed), each
 * paired with one of its k_correspondences nearest target histograms, fitted by the float32 Umeyama of the loop and scored by
 * PCL's truncated error over every source point (d2 / thr if d2 <= thr, else 1; thr applies to SQUARED distances) with exact
 * nearest neighbours; the smallest error wins, ties to the smallest hypothesis.  Deterministic: the same inputs and seed give
 * the same result bit for bit.  Zero-initialise ghicp_sac_params and fill it; the defaults of the definition are
 * max_iterations 1000, nr_samples 3 (3..8), k_correspondences 6 (1..32), min_sample_distance 0, corr_dist_threshold 100,
 * seed 0.  Out-of-range parameters return GHICP_E_ARG. */
typedef struct ghicp_sac_params {
  int max_iterations;          /* hypotheses H >= 1 */
  int nr_samples;              /* 3 .. 8 */
  int k_correspondences;       /* 1 .. 32; min(k, n_t) are used */
  float min_sample_distance;   /* >= 0: every two samples of a hypothesis at least this far apart (float32 Euclidean) */
  float corr_dist_threshold;   /* > 0, on squared distances */
  int reserved;
  unsigned long long seed;
} ghicp_sac_params;
typedef struct ghicp_sac_result {
  double Rt[16];               /* column-major; the chosen float32 transform widened (identity when no hypothesis is valid) */
  double error;                /* sum of the truncated error terms (each rounded to a multiple of 2^-32) */
  double fitness;              /* mean squared nearest distance over the source points within the threshold (DBL_MAX: none) */
  int inliers;                 /* source points within the threshold */
  int best_hypothesis;         /* h* (-1: every hypothesis failed to draw its samples) */
  int invalid_hypotheses;      /* hypotheses without nr_samples acceptable samples (3 n_s rejections in a row) */
  int reserved;
  float stage_ms[4];           /* CUDA events: sampling + feature k-NN, estimation, scoring (with the target grid), pick */
} ghicp_sac_result;
/* src_xyz [n_s][3], src_fpfh [n_s][33], tgt_xyz [n_t][3], tgt_fpfh [n_t][33] (host arrays) */
int ghicp_sac_ia(int device, const float *src_xyz, const float *src_fpfh, int n_s, const float *tgt_xyz, const float *tgt_fpfh,
                 int n_t, const ghicp_sac_params *p, ghicp_sac_result *out);
/* keypoint coordinates + keypoint histograms of two pipeline results (ghicp_prep_fpfh on both), device to device */
int ghicp_prep_sac_ia(const ghicp_prep *source, const ghicp_prep *target, const ghicp_sac_params *p, ghicp_sac_result *out);
/* After ghicp_set_keypoints / ghicp_set_from_prep, before iteration 0: move the source keypoints by Rt on the device (the
 * update every iteration applies, src/ghicp_reg.cpp:891-894) and compose Rt into Rt_tillnow, so that ghicp_get_rt and
 * ghicp_run return the whole transform.  GHICP_E_ARG after iteration 0 or without keypoints. */
int ghicp_set_initial_transform(ghicp_ctx *ctx, const double Rt[16]);

/* ---- overlap and fitness of a registration on the dense clouds (DESIGN.md §3.12) ----------------- */
/* Every point a_i of cloud A is moved by Rt (column-major, rounded once to float32; NULL = identity) and its squared distance
 * d2_i to the nearest point of cloud B found (float32, exact wherever d2_i <= max(thre_dis^2, max_range), +inf beyond).
 * overlap = #{d2_i < thre_dis * thre_dis} (CRegistration::calOverlap, src/common_reg.cpp:294-317); fitness = the mean of the
 * finite d2_i <= max_range (PCL's getFitnessScore; max_range is a bound on SQUARED distances, +inf allowed).  Sums are in
 * double in a fixed order: two calls give identical bits.  want_fitness = 0 is the overlap-only mode: each query stops at the
 * first point within thre_dis; n_fit = 0 and overlap_rmse = fitness = NaN.  A point of A whose moved coordinates are not
 * finite (the NaN returns of an organised scan) gets d2 = +inf at once; non-finite points of B are left out of B, as PCL's
 * KdTreeFLANN leaves them out of its tree.  Argument errors (NULL, n <= 0, no finite point in B, thre_dis <= 0 or NaN,
 * max_range < 0 or NaN, a non-finite entry of Rt, d2 without want_fitness, handles on different devices) return GHICP_E_ARG
 * and write nothing; out of memory returns GHICP_E_NOMEM before anything is written. */
typedef struct ghicp_overlap_result {
  long long n, overlap, n_fit, cells_visited, candidates;   /* points of A; work: B-grid cells read, points examined */
  float ratio;            /* (0.01 + overlap) / n, src/common_reg.cpp:312 */
  double overlap_rmse, fitness;
  float stage_ms[3];      /* grid (0 when cached), queries, total */
} ghicp_overlap_result;
/* a_xyz [n_a][3], b_xyz [n_b][3] (host arrays); d2 [n_a] (host, may be NULL) receives d2_i */
int ghicp_cloud_overlap(int device, const float *a_xyz, int n_a, const float *b_xyz, int n_b, const double Rt[16],
                        float thre_dis, double max_range, int want_fitness, ghicp_overlap_result *out, float *d2);
/* the down-sampled clouds of two pipeline results, device to device; the target keeps B's grid until ghicp_prep_destroy,
 * so a second call on the same target does not rebuild it (stage_ms[0] = 0).  Calls on one target from several host threads
 * are serialised on it (the grid is built once); ghicp_prep_destroy must not overlap them. */
int ghicp_prep_overlap(const ghicp_prep *a, const ghicp_prep *b, const double Rt[16], float thre_dis, double max_range,
                       int want_fitness, ghicp_overlap_result *out);

/* ---- point-to-point ICP on the dense clouds (DESIGN.md §3.13) ------------------------------------------------------------
 * CRegistration::icp_reg (src/common_reg.cpp:44-107): PCL's IterativeClosestPoint<PointXYZ, PointXYZ> with
 * DefaultConvergenceCriteria, on the canonical definition of DESIGN.md §3.13.  Every iteration pairs each source point, moved
 * by the transform so far, with its exact nearest target point ((d2, index) order), optionally keeps only reciprocal pairs
 * and then the floor(trim_ratio * pairs) closest ones, fits the float32 Umeyama of the loop to FP64 two-pass moments of the
 * kept pairs, and stops on the first of: max_iterations, a transform within transformation_epsilon of the identity, an
 * absolute (1e-12) or relative (fitness_epsilon) change of the pairs' mean squared distance, or fewer than 3 pairs.  Sums are
 * in double in a fixed order: two calls give identical bits.  Non-finite source and target points take no part.
 * Point-to-plane (metric = 1, DESIGN.md §3.14): CRegistration::ptplicp_reg (src/common_reg.cpp:123-199), PCL's
 * IterativeClosestPointWithNormals with TransformationEstimationPointToPlaneLLS.  The same loop, but each step solves PCL's
 * point-to-plane normal equations (centred on the kept source points' mean, FP64 fixed-order sums) against the target's k-NN
 * normals (PCL NormalEstimation with k = normal_k, viewpoint 0, non-finite normals replaced by (0.577, 0.577, 0.577) as
 * CheckNormals does).  A singular system stops the loop with GHICP_ICP_SINGULAR.
 * Generalized ICP (metric = 2, DESIGN.md §3.15): CRegistration::gicp_reg (src/common_reg.cpp:217-284), PCL's
 * GeneralizedIterativeClosestPoint.  The same pairs, gated at d2 < 1e12 (gicp_reg's corr_dist_threshold 1e6, squared); each
 * point's covariance is I - 0.999 n n^T from the k-NN normals of both clouds (k = normal_k, the source's on the unmoved
 * source), and each iteration minimises PCL's objective sum r^T (R C_s R^T + C_t)^-1 r / c for those pairs by up to 20
 * Gauss-Newton steps (FP64 fixed-order sums, a step that raises the objective is undone) where PCL runs its BFGS.  The loop
 * stops at max_iterations, or when no entry of the transform moved by more than rotation_epsilon (the 3 x 3 block) or
 * transformation_epsilon (the translation) in the iteration (TRANSFORM), PCL's GICP criterion; fitness_epsilon is not read.
 * Gauss-Newton has no damping: when the first step of an iteration raises the objective it is undone, the transform has not
 * moved, and the call reports TRANSFORM (converged = 1) from where that iteration started, which the result alone does not
 * tell apart from a real convergence (a damped or backtracking step is a possible follow-up).
 * A singular system stops it with GHICP_ICP_SINGULAR, the transform as it was at the start of that iteration.  Unlike PCL's
 * GICP, which ignores them, reciprocal and trim_ratio apply (gicp_reg passes them as off). */
enum ghicp_icp_state {   /* PCL's DefaultConvergenceCriteria::ConvergenceState values, then SINGULAR */
  GHICP_ICP_ITERATIONS = 1,
  GHICP_ICP_TRANSFORM = 2,         /* metric 2: also when an iteration's first step was undone (see above) */
  GHICP_ICP_ABS_MSE = 3,
  GHICP_ICP_REL_MSE = 4,
  GHICP_ICP_NO_CORRESPONDENCES = 5,
  GHICP_ICP_SINGULAR = 7           /* metrics 1, 2: 3 or more pairs but no solution (e.g. every normal parallel); F unchanged */
};
typedef struct ghicp_icp_params {
  int max_iterations;              /* >= 1 (icp_reg's max_iter) */
  int reciprocal;                  /* setUseReciprocalCorrespondences */
  float trim_ratio;                /* CorrespondenceRejectorTrimmed::setOverlapRatio, 0 = no rejector, else (0, 1] */
  double transformation_epsilon;   /* >= 0; icp_reg: 1e-8 */
  double fitness_epsilon;          /* >= 0; icp_reg: 1e-5; not read by metric 2 */
  int metric;                      /* 0 = point-to-point (§3.13), 1 = point-to-plane (§3.14), 2 = Generalized ICP (§3.15) */
  int normal_k;                    /* metrics 1, 2: the normals' k, 3..32 (covariance_K); ignored by metric 0 */
  double rotation_epsilon;         /* metric 2: finite, > 0 (gicp_reg: 1e-6); ignored by metrics 0 and 1 */
} ghicp_icp_params;
typedef struct ghicp_icp_result {
  double Rt[16];                   /* column-major: the float32 accumulated transform widened (the guess when no step ran) */
  double mse;                      /* mean squared distance of the last iteration's kept pairs (NaN without a pair) */
  double fitness;                  /* PCL's getFitnessScore: §3.12 fitness of the source moved by Rt, max_range = +inf */
  int iterations, converged, state, cor;          /* state: ghicp_icp_state; cor: the last iteration's kept pairs */
  long long cells_visited, candidates;            /* work of every nearest-neighbour query of every iteration */
  float stage_ms[4];                              /* target grid (+ the target's normals for metric 1, both clouds' for
                                                     metric 2; 0 when all cached), iterations, fitness, total */
} ghicp_icp_result;
/* src_xyz [n_s][3], tgt_xyz [n_t][3] (host arrays); guess column-major (NULL = identity), rounded once to float32; moved [n_s][3]
 * (may be NULL) receives the source moved by Rt (PCL's align output); cor_trace / mse_trace [max_iterations] (may be NULL)
 * receive each iteration's kept pairs and mean squared distance (entries past `iterations` are left as they are).  Fewer than
 * 3 pairs returns GHICP_W_FEW_PAIRS, a singular point-to-plane or GICP system GHICP_W_SINGULAR, each with the result filled
 * in (converged = 0, Rt = the transform so far).  Argument errors (NULL, n <= 0, no finite source or target point,
 * max_iterations < 1, trim_ratio outside [0, 1] or NaN, a negative or NaN epsilon, a non-finite guess, a metric other than
 * 0, 1 or 2, metric 1 or 2 with normal_k outside 3..32, metric 2 without a finite rotation_epsilon > 0, handles on different
 * devices) return GHICP_E_ARG and write nothing; out of memory returns GHICP_E_NOMEM and writes nothing. */
int ghicp_cloud_icp(int device, const float *src_xyz, int n_s, const float *tgt_xyz, int n_t, const double guess[16],
                    const ghicp_icp_params *p, ghicp_icp_result *out, float *moved, int *cor_trace, double *mse_trace);
/* the down-sampled clouds of two pipeline results, device to device; the target's grid is the one ghicp_prep_overlap keeps
 * (built by whichever call comes first, stage_ms[0] = 0 when it already exists).  Metric 1 also keeps the target's normals
 * and their k there, under the same lock: a later call with the same normal_k reuses them, another k replaces them.  Metric
 * 2 keeps both results' normals that way (each result holds one set, whichever metric or role asked for it) and takes both
 * locks together, so that calls on (a, b) and (b, a) from two host threads cannot deadlock; source == target is allowed. */
int ghicp_prep_icp(const ghicp_prep *source, const ghicp_prep *target, const double guess[16], const ghicp_icp_params *p,
                   ghicp_icp_result *out);

/* ---- multi-GPU (one process per GPU; source rows sharded, target replicated) ---------------- */
/* 128-byte NCCL unique id; rank 0 creates it, the host runtime broadcasts it (torch.distributed,
 * MPI, a file ...). No NCCL symbol is touched unless these are called (world == 1 → never). */
int ghicp_comm_unique_id(void *id128);
int ghicp_comm_init(ghicp_ctx *ctx, const void *id128, int rank, int world);

#ifdef __cplusplus
}
#endif
#endif /* GHICP_B200_H_ */
