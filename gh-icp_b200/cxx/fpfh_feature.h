// fpfh_feature.h — host-side mirror of the reference's FPFHfeature (include/fpfh.hpp:31-115) over libghicp_b200.so: the
// same constructor, compute_fpfh_feature and keyfpfh, so that the driver's FPFH branch (test/ghicp_main.cpp:120-127)
// compiles unchanged on this repo's stand-in types.  The histograms are computed on the GPU by ghicp_fpfh_extract with the
// canonical definition of DESIGN.md §3.10 (k-NN normals and histograms with k = 20, like fpfh.hpp:36-58).  Differences,
// deliberate:
//   * clouds are ghicp::Cloud (cloud_io.h), keypoint indices plain index vectors, fpfhFeaturePtr the non-owning pointer of
//     ghicp_types.h;
//   * the radius argument is kept for source compatibility and unused, as in the reference (its estimators use k-NN);
//   * no CPU path: without a CUDA device compute_fpfh_feature and fpfhalign throw;
//   * fpfhalign (:117-133, PCL SampleConsensusInitialAlignment with correspondence randomness 6) runs ghicp_sac_ia, the
//     deterministic SAC-IA of DESIGN.md §3.11 (1000 hypotheses of 3 samples, threshold 100 on squared distances, seed 0 —
//     set_sac_params changes them), instead of PCL's std::rand()-driven one; it also keeps the transform and the fitness
//     (getFinalTransformation / getFitnessScore of the PCL object the reference discards) and returns true.
// The radius-based compute_fpfh_keypoint is not mirrored (the driver does not call it).
#pragma once
#include <iostream>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/ghicp_b200.h"
#include "ghicp_types.h"
#include "cloud_io.h"
#include "ghicp_types.h"

namespace ghicp {

template <typename PointT = void>
class FPFHfeature {
 public:
  explicit FPFHfeature(double neighbor_radius, int k = 20) : radius(neighbor_radius), k_(k) {
    sac_.max_iterations = 1000; sac_.nr_samples = 3; sac_.k_correspondences = 6;   // setCorrespondenceRandomness(6), :129
    sac_.min_sample_distance = 0.f; sac_.corr_dist_threshold = 100.f; sac_.seed = 0;
  }

  // :36-58 — normals and FPFH of every point of the cloud
  bool compute_fpfh_feature(const Cloud &input_cloud, fpfhFeaturePtr &fpfh) {
    const int n = (int)input_cloud.size();
    if (n <= 0) return false;
    std::vector<float> hist((size_t)n * 33);
    if (ghicp_fpfh_extract(0, input_cloud.xyz.data(), n, nullptr, n, k_, hist.data(), nullptr, nullptr) < 0)
      throw std::runtime_error(std::string("FPFHfeature: ") + ghicp_last_error(nullptr));
    fpfh->points.resize(n);
    for (int i = 0; i < n; ++i)
      for (int b = 0; b < 33; ++b) fpfh->points[i].histogram[b] = hist[(size_t)i * 33 + b];
    return true;
  }

  // :93-115 — the histograms at the keypoints
  bool keyfpfh(const fpfhFeaturePtr &source_fpfh, const fpfhFeaturePtr &target_fpfh, const std::vector<int> &source_indices,
               const std::vector<int> &target_indices, fpfhFeaturePtr &source_keyfpfh, fpfhFeaturePtr &target_keyfpfh) {
    gather(source_fpfh, source_indices, source_keyfpfh);
    gather(target_fpfh, target_indices, target_keyfpfh);
    return true;
  }

  // :117-133 — SAC-IA of the source onto the target from their histograms; reg_sourcecloud = the moved source
  bool fpfhalign(const Cloud &sourcecloud, const Cloud &targetcloud, const fpfhFeaturePtr source_fpfh,
                 const fpfhFeaturePtr target_fpfh, Cloud &reg_sourcecloud) {
    const int ns = (int)sourcecloud.size(), nt = (int)targetcloud.size();
    if ((int)source_fpfh->points.size() != ns || (int)target_fpfh->points.size() != nt)
      throw std::runtime_error("FPFHfeature::fpfhalign: one histogram per point expected");
    std::vector<float> fs((size_t)ns * 33), ft((size_t)nt * 33);
    for (int i = 0; i < ns; ++i) for (int b = 0; b < 33; ++b) fs[(size_t)i * 33 + b] = source_fpfh->points[i].histogram[b];
    for (int i = 0; i < nt; ++i) for (int b = 0; b < 33; ++b) ft[(size_t)i * 33 + b] = target_fpfh->points[i].histogram[b];
    if (ghicp_sac_ia(0, sourcecloud.xyz.data(), fs.data(), ns, targetcloud.xyz.data(), ft.data(), nt, &sac_, &result_) < 0)
      throw std::runtime_error(std::string("FPFHfeature::fpfhalign: ") + ghicp_last_error(nullptr));
    for (int i = 0; i < 16; ++i) final_transformation_.data()[i] = result_.Rt[i];
    // pcl::transformPointCloud with the float32 matrix, as PCL's align() moves the source
    Cloud out;
    const double *m = result_.Rt;
    for (int i = 0; i < ns; ++i) {
      const float x = sourcecloud.xyz[3 * (size_t)i], y = sourcecloud.xyz[3 * (size_t)i + 1], z = sourcecloud.xyz[3 * (size_t)i + 2];
      float o[3];
      for (int r = 0; r < 3; ++r) o[r] = (((float)m[r] * x + (float)m[4 + r] * y) + (float)m[8 + r] * z) + (float)m[12 + r];
      out.push(o[0], o[1], o[2]);
    }
    reg_sourcecloud = out;
    std::cout << "Has converged:" << (result_.best_hypothesis >= 0) << "score" << result_.fitness << std::endl;   // :130
    return true;
  }
  // PCL's getFinalTransformation (column-major 4 x 4) and getFitnessScore of the last fpfhalign
  const Matrix4d &getFinalTransformation() const { return final_transformation_; }
  double getFitnessScore() const { return result_.fitness; }
  const ghicp_sac_result &sac_result() const { return result_; }
  void set_sac_params(const ghicp_sac_params &p) { sac_ = p; }

 private:
  static void gather(const fpfhFeaturePtr &all, const std::vector<int> &idx, fpfhFeaturePtr &out) {
    out->points.resize(idx.size());
    for (size_t i = 0; i < idx.size(); ++i) {
      if (idx[i] < 0 || (size_t)idx[i] >= all->points.size()) throw std::runtime_error("FPFHfeature::keyfpfh: index out of range");
      out->points[i] = all->points[(size_t)idx[i]];
    }
  }
  double radius;
  int k_;
  ghicp_sac_params sac_{};
  ghicp_sac_result result_{};
  Matrix4d final_transformation_ = Identity4();
};

}  // namespace ghicp
