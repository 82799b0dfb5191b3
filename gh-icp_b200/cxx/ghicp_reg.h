// ghicp_reg.h — ghicp::Energyfunction / Keypoints / GHRegistration with the reference's public
// interface (include/ghicp_reg.h:15-132), implemented over libghicp_b200.so (include/ghicp_b200.h).
// test/ghicp_main.cpp:143-151 compiles against this header unchanged.
//
// Differences from the reference, all deliberate (DESIGN.md §Boundary):
//  * Energyfunction::ED/FD/CD are not materialised on the host (24*N*M bytes in the reference);
//    the cost matrices live on the GPU (FD as u16) or are never stored (ED, CD).
//  * no PCLVisualizer is created (src/ghicp_reg.cpp:26-29 cannot run headless); set_viewer is kept
//    and ignored; set_raw_pointcloud is accepted and ignored (the clouds only fed the viewer).
//  * an optional max_iterations guard (default 0 = unbounded like src/ghicp_reg.cpp:49).
//  * pre / rec (KM mode, src/ghicp_reg.cpp:443-444) count identity pairs among the RETURNED correspondences; the
//    reference's Km::output (src/km.cpp:159) also counts match[i] == i on penalty edges of the padded graph, where the
//    assignment is arbitrary (any perfect matching of the left-overs is optimal), so that part has no defined value.
//  * the CUDA device is chosen per process: GHRegistration::set_default_device(d) or the GHICP_DEVICE environment
//    variable (the reference has no device notion); one process per GPU shards through ghicp_comm_init (INTEGRATION.md).
#ifndef _INCLUDE_GHICP_REG_H_
#define _INCLUDE_GHICP_REG_H_

#include <algorithm>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <iostream>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/ghicp_b200.h"
#include "ghicp_types.h"
#include "km.h"
#include "utility.h"

namespace ghicp {

struct Energyfunction {  // include/ghicp_reg.h:15-42
  std::vector<std::vector<double>> ED, FD, CD;  // intentionally left empty (device-resident)
  int weight_changing_rate;
  double penalty, para1_penalty, para2_penalty, penalty_initial;
  int min_cor;
  double KM_eps;
  float scale;
  float bbx_magnitude_;
  Energyfunction() : weight_changing_rate(6), penalty(0), para1_penalty(1.0), para2_penalty(1.0),
                     penalty_initial(2.0), min_cor(10), KM_eps(0.01), scale(0), bbx_magnitude_(0) {}
  void init(int /*kps_num*/, int /*kpt_num*/, float bbx_magnitude) {
    penalty_initial = 2.0; para1_penalty = 1.0; para2_penalty = 1.0;
    min_cor = 10; weight_changing_rate = 6; KM_eps = 0.01;
    scale = 0.005 * bbx_magnitude;
    bbx_magnitude_ = bbx_magnitude;
  }
};

struct Keypoints {  // include/ghicp_reg.h:44-72
  int kps_num = 0, kpt_num = 0;
  MatrixX3d kpSXYZ, kpTXYZ;
  doubleVectorSBF bscS, bscT;
  fpfhFeaturePtr fpfhS = fpfhFeaturePtr(), fpfhT = fpfhFeaturePtr();
  Keypoints() {}
  void setCoordinate(MatrixX3d &kps, MatrixX3d &kpt) {
    kpSXYZ = kps; kpTXYZ = kpt;
    kps_num = (int)kpSXYZ.rows(); kpt_num = (int)kpTXYZ.rows();
  }
  void setBSCfeature(const doubleVectorSBF &bsc_S, const doubleVectorSBF &bsc_T) { bscS = bsc_S; bscT = bsc_T; }
  void setFPFHfeature(const fpfhFeaturePtr &fpfh_S, const fpfhFeaturePtr &fpfh_T) { fpfhS = fpfh_S; fpfhT = fpfh_T; }
};

class GHRegistration {
 public:
  GHRegistration(Keypoints Kp, Energyfunction Ef, FeatureType Ft, CorrespondenceType Ct, float radiusNonMax,
                 float weight_adjustment_ratio, float weight_adjustment_step, int dof_type, float estimated_IoU,
                 float converge_tran = 0.02, float converge_rot = 0.02, int ite = 0, int ite2 = 0)
      : KP(Kp), EF(Ef), Ft_(Ft), Ct_(Ct) {
    (void)ite; (void)ite2;
    gt_maxdis = radiusNonMax / 3;
    PCFD = 0;
    RMS = 99999;
    Rt_tillnow = Identity4();
    matchlist.resize(KP.kps_num, std::vector<int>(200));   // include/ghicp_reg.h:100
    ghicp_config cfg;
    std::memset(&cfg, 0, sizeof(cfg));
    cfg.feature_type = (int)Ft; cfg.corr_type = (int)Ct; cfg.dof = dof_type;
    cfg.bbx_magnitude = Ef.bbx_magnitude_;
    cfg.nonmax = radiusNonMax; cfg.adjust_ratio = weight_adjustment_ratio; cfg.adjust_step = weight_adjustment_step;
    cfg.estimated_iou = estimated_IoU; cfg.converge_t = converge_tran; cfg.converge_r = converge_rot;
    cfg.max_iter = 0; cfg.device = default_device(); cfg.km_eps = Ef.KM_eps;
    check(ghicp_create(&cfg, &ctx_), "ghicp_create");
    try {   // a constructor that throws runs no destructor: release the context here
      const CommSpec &cs = default_comm();
      if (cs.world > 1) check(ghicp_comm_init(ctx_, cs.id, cs.rank, cs.world), "ghicp_comm_init");   // before the keypoints
      check(ghicp_set_keypoints(ctx_, KP.kpSXYZ.data(), KP.kps_num, KP.kpTXYZ.data(), KP.kpt_num), "ghicp_set_keypoints");
      if (Ft == BSC) upload_bsc();
      if (Ft == FPFH) upload_fpfh();
    } catch (...) {
      ghicp_destroy(ctx_);
      ctx_ = nullptr;
      throw;
    }
  }
  ~GHRegistration() { if (ctx_) ghicp_destroy(ctx_); }
  GHRegistration(const GHRegistration &) = delete;
  GHRegistration &operator=(const GHRegistration &) = delete;

  template <typename CloudPtr>
  void set_raw_pointcloud(const CloudPtr &, const CloudPtr &) {}  // only fed the viewer (ghicp_reg.cpp:97-100)
  void set_viewer(bool launch_viewer) { launch_viewer_ = launch_viewer; }
  void set_max_iterations(int n) { max_iterations_ = n; }
  void set_verbose(bool v) { verbose_ = v; }
  // matchlist / pre / rec (KM mode) need the pair lists on the host every iteration (two int arrays of cor entries);
  // a caller that reads neither can switch that copy off.
  void set_track_matches(bool on) { track_matches_ = on; }
  // Device of the contexts constructed from now on in this process (default: GHICP_DEVICE, else 0).
  static void set_default_device(int d) { default_device() = d; }
  // One process per GPU (extension, INTEGRATION.md §4): the contexts constructed from now on shard the source keypoints over
  // `world` processes.  id128 = the 128 bytes rank 0 got from ghicp_comm_unique_id and the host runtime broadcast.
  // (The sharded path itself is tested through the Python mirror, tests/test_gpu_multi.py; this setter only forwards.)
  static void set_default_comm(const void *id128, int rank, int world) {
    CommSpec &cs = default_comm();
    if (id128) std::memcpy(cs.id, id128, sizeof(cs.id));
    cs.rank = rank; cs.world = world;
  }
  // Extensions (not in the reference's class): opt-in estimators of include/ghicp_b200.h ghicp_solver_type.
  // GHICP_SOLVER_SVD (default) is what src/ghicp_reg.cpp:857-859 always runs.
  void set_solver(int solver) { check(ghicp_set_solver(ctx_, solver), "ghicp_set_solver"); }
  void set_target_normals(MatrixX3d &normals) {  // unit normals of the target keypoints, for POINT_TO_PLANE
    if ((int)normals.rows() != KP.kpt_num) throw std::runtime_error("set_target_normals: one normal per target keypoint");
    check(ghicp_set_target_normals(ctx_, normals.data()), "ghicp_set_target_normals");
  }

  // Extension: start the loop from Rt (e.g. FPFHfeature::fpfhalign's getFinalTransformation), before the first iteration;
  // ghicp_reg then returns the whole transform.
  void set_initial_transform(const Matrix4d &Rt) {
    check(ghicp_set_initial_transform(ctx_, Rt.data()), "ghicp_set_initial_transform");
    check(ghicp_get_rt(ctx_, Rt_tillnow.data()), "ghicp_get_rt");
  }

  // Main entrance (src/ghicp_reg.cpp:24-112)
  bool ghicp_reg(Matrix4d &Rt_final) {
    check(ghicp_build_fd(ctx_), "ghicp_build_fd");
    bool converge = false;
    int it = 0;
    while (!converge) {
      ghicp_iter_stats st;
      check(ghicp_iterate(ctx_, &st), "ghicp_iterate");
      energy.push_back(st.km_energy);
      rmse.push_back(st.rmse);
      rmseafter.push_back(st.rmse_after);
      cor.push_back(st.cor);
      RMS = st.rmse;
      std::memcpy(Rt_tillnow.data(), st.Rt_tillnow, sizeof(double) * 16);
      if (verbose_)
        std::cout << st.iteration << " : " << st.cor << " pairs, RMSE " << st.rmse << " -> " << st.rmse_after
                  << ", penalty " << st.penalty << std::endl;
      if (Ct_ == KM && track_matches_) record_matches(st.iteration);
      converge = st.converged != 0;
      if (max_iterations_ > 0 && ++it >= max_iterations_) break;
    }
    Rt_final = Rt_tillnow;
    return 1;
  }

  // Last iteration's correspondences (Spoint / Tpoint index lists).
  int get_pairs(std::vector<int> &SP, std::vector<int> &TP) {
    int n = 0;
    const int cap = std::max(KP.kps_num, KP.kpt_num);
    SP.assign(cap, 0); TP.assign(cap, 0);
    check(ghicp_get_pairs(ctx_, SP.data(), TP.data(), cap, &n), "ghicp_get_pairs");
    SP.resize(n); TP.resize(n);
    return n;
  }

  double gt_maxdis;
  double PCFD;
  double RMS;
  Matrix4d Rt_tillnow;
  Matrix4d Rt_gt;
  std::vector<std::vector<int>> matchlist;
  std::vector<int> gtmatchlist;
  std::vector<double> energy, rmse, rmseafter, pre, rec;
  std::vector<int> cor;

 private:
  void check(int rc, const char *what) {
    if (rc < 0) throw std::runtime_error(std::string(what) + ": " + ghicp_last_error(ctx_));
  }
  struct CommSpec { char id[128]; int rank = 0, world = 1; };
  static CommSpec &default_comm() { static CommSpec cs; return cs; }
  static int &default_device() {
    static int d = [] { const char *e = std::getenv("GHICP_DEVICE"); return e ? std::atoi(e) : 0; }();
    return d;
  }
  // src/ghicp_reg.cpp:443-460: precision / recall of this iteration's matching against the identity, and column
  // `iteration` of matchlist (target index of every matched source keypoint, -1 for the others).
  void record_matches(int iteration) {
    std::vector<int> SP, TP;
    const int n = get_pairs(SP, TP);
    int exact = 0;
    for (int k = 0; k < n; ++k) exact += SP[k] == TP[k];
    pre.push_back(n > 0 ? 1.0 * exact / n : 0.0);
    rec.push_back(1.0 * exact / std::max(KP.kps_num, KP.kpt_num));
    if (iteration < 0) return;
    for (auto &row : matchlist) {
      if ((int)row.size() <= iteration) row.resize(iteration + 1, 0);   // the reference stops at 200 columns (UB beyond)
      row[iteration] = -1;
    }
    for (int k = 0; k < n; ++k) matchlist[SP[k]][iteration] = TP[k];
  }
  void upload_bsc() {
    int V = 0;   // extractBinaryFeatures always returns four vectors; the variants dof_type did not ask for hold empty features
    while (V < (int)KP.bscS.size() && !KP.bscS[V].empty() && KP.bscS[V][0].size_ > 0) ++V;
    if (V == 0 || KP.bscT.empty() || KP.bscT[0].empty()) throw std::runtime_error("GHRegistration: BSC features not set");
    const unsigned bits = KP.bscT[0][0].size_, B = KP.bscT[0][0].byte_;
    std::vector<uint8_t> s((size_t)V * KP.kps_num * B), t((size_t)KP.kpt_num * B);
    for (int v = 0; v < V; ++v)
      for (int i = 0; i < KP.kps_num; ++i) std::memcpy(&s[((size_t)v * KP.kps_num + i) * B], KP.bscS[v][i].feature_, B);
    for (int j = 0; j < KP.kpt_num; ++j) std::memcpy(&t[(size_t)j * B], KP.bscT[0][j].feature_, B);
    check(ghicp_set_bsc(ctx_, s.data(), V, t.data(), (int)bits), "ghicp_set_bsc");
  }
  void upload_fpfh() {
    if (!KP.fpfhS || !KP.fpfhT) throw std::runtime_error("GHRegistration: FPFH features not set");
    std::vector<float> s((size_t)KP.kps_num * 33), t((size_t)KP.kpt_num * 33);
    for (int i = 0; i < KP.kps_num; ++i) std::memcpy(&s[(size_t)i * 33], KP.fpfhS->points[i].histogram, 33 * sizeof(float));
    for (int j = 0; j < KP.kpt_num; ++j) std::memcpy(&t[(size_t)j * 33], KP.fpfhT->points[j].histogram, 33 * sizeof(float));
    check(ghicp_set_fpfh(ctx_, s.data(), t.data()), "ghicp_set_fpfh");
  }

  Keypoints KP;
  Energyfunction EF;
  FeatureType Ft_;
  CorrespondenceType Ct_;
  ghicp_ctx *ctx_ = nullptr;
  bool launch_viewer_ = false, verbose_ = false, track_matches_ = true;
  int max_iterations_ = 0;
};

}  // namespace ghicp
#endif  // _INCLUDE_GHICP_REG_H_
