// common_reg.h — host-side mirror of the reference's CRegistration (include/common_reg.h, src/common_reg.cpp) over
// libghicp_b200.so, with the members the library backs:
//   compute_fpfh_feature (src/common_reg.cpp:373-389)  normals over search_radius, FPFH over 2 search_radius on every point
//                                                      (PCL radius searches), on the GPU by ghicp_fpfh_extract_radius with
//                                                      the canonical definition of DESIGN.md §3.10 ("Radius neighbourhoods")
//   Coarsereg_FPFHSAC    (src/common_reg.cpp:393-423)  both clouds' histograms, then SAC-IA with correspondence randomness 15
//                                                      and PCL's other defaults (1000 hypotheses of 3 samples, threshold 100
//                                                      on squared distances), by ghicp_sac_ia (DESIGN.md §3.11, seed 0)
//   calOverlap           (src/common_reg.cpp:294-317)  the share of Cloud1 with a Cloud2 point within thre_dis, by
//                                                      ghicp_cloud_overlap (DESIGN.md §3.12, overlap-only mode)
//   transformcloud       (src/common_reg.cpp:325-350)  the float32 transform of every point, ((m00 x + m01 y) + m02 z) + m03
//   invTransform         (src/common_reg.cpp:358-370)  the reference's "not mathematically" inverse, kept as it is
//   icp_reg              (src/common_reg.cpp:44-107)   PCL's point-to-point IterativeClosestPoint from the identity, with the
//                                                      reciprocal and trimmed options, by ghicp_cloud_icp (DESIGN.md §3.13)
//   ptplicp_reg          (src/common_reg.cpp:123-199)  PCL's IterativeClosestPointWithNormals (point-to-plane LLS) with the same
//                                                      options against the target's k-NN normals, by ghicp_cloud_icp with
//                                                      metric 1 (DESIGN.md §3.14); the source's normals take no part in PCL's
//                                                      estimate and are not computed
//   gicp_reg             (src/common_reg.cpp:217-284)  PCL's GeneralizedIterativeClosestPoint over both clouds' k-NN normals,
//                                                      by ghicp_cloud_icp with metric 2 (DESIGN.md §3.15); the reciprocal and
//                                                      trimmed options do not reach the loop, as in PCL's GICP (:213-215), and
//                                                      use_trimmed_rejector only refuses a low overlap ratio
// Differences, deliberate: clouds are ghicp::Cloud (cloud_io.h) and fpfhFeaturePtr the stand-in of ghicp_types.h; the
// transform is Eigen::Matrix4f when Eigen is on the include path, else the column-major ghicp::Matrix4f; the SAC-IA is the
// deterministic one of DESIGN.md §3.11 instead of PCL's std::rand()-driven one; no CPU path (without a CUDA device both
// members throw).  The fitness of the last Coarsereg_FPFHSAC or icp_reg, which the reference prints, is kept
// (getFitnessScore).  icp_reg, ptplicp_reg and gicp_reg print their lines to std::cout only (the reference also logs them
// through glog; gicp_reg's fitness warning above 5000, a glog warning there, is printed as a line).  ptplicp_reg writes
// TransformedSource and returns true, where the reference aligns into a local cloud (:141, :182) and leaves the caller's
// untouched, and falls off the end of the function without a return value (:199); gicp_reg returns true where the reference
// falls off the end too (:284).
// Not provided: LLS_4DOF / SVD_6DOF and CSTRAN_4DOF / CSTRAN_7DOF.
#pragma once
#include <algorithm>
#include <ctime>
#include <iostream>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/ghicp_b200.h"
#include "cloud_io.h"
#include "ghicp_types.h"

namespace ghicp {

template <typename PointT = void>
class CRegistration {
 public:
  // :373-389 — normals over search_radius, FPFH over 2 search_radius, every point of the cloud
  void compute_fpfh_feature(const Cloud &input_cloud, fpfhFeaturePtr &cloud_fpfh, float search_radius) {
    const int n = (int)input_cloud.size();
    cloud_fpfh->points.resize(n);
    if (n <= 0) return;
    std::vector<float> hist((size_t)n * 33);
    if (ghicp_fpfh_extract_radius(0, input_cloud.xyz.data(), n, nullptr, n, search_radius, 2.0f * search_radius, hist.data(),
                                  nullptr, nullptr) < 0)
      throw std::runtime_error(std::string("CRegistration::compute_fpfh_feature: ") + ghicp_last_error(nullptr));
    for (int i = 0; i < n; ++i)
      for (int b = 0; b < 33; ++b) cloud_fpfh->points[i].histogram[b] = hist[(size_t)i * 33 + b];
  }

  // :393-423 — SAC-IA of SourceCloud onto TargetCloud from their radius histograms; TransformedSource = the moved source
  void Coarsereg_FPFHSAC(const Cloud &SourceCloud, const Cloud &TargetCloud, Cloud &TransformedSource,
                         Matrix4f &transformationS2T, float search_radius) {
#ifdef GHICP_HAVE_PCL
    fpfhFeaturePtr source_fpfh(new pcl::PointCloud<pcl::FPFHSignature33>), target_fpfh(new pcl::PointCloud<pcl::FPFHSignature33>);
#else
    fpfhFeature source_store, target_store;
    fpfhFeaturePtr source_fpfh = &source_store, target_fpfh = &target_store;
#endif
    compute_fpfh_feature(SourceCloud, source_fpfh, search_radius);
    compute_fpfh_feature(TargetCloud, target_fpfh, search_radius);
    const int ns = (int)SourceCloud.size(), nt = (int)TargetCloud.size();
    std::vector<float> fs((size_t)ns * 33), ft((size_t)nt * 33);
    for (int i = 0; i < ns; ++i) for (int b = 0; b < 33; ++b) fs[(size_t)i * 33 + b] = source_fpfh->points[i].histogram[b];
    for (int i = 0; i < nt; ++i) for (int b = 0; b < 33; ++b) ft[(size_t)i * 33 + b] = target_fpfh->points[i].histogram[b];
    ghicp_sac_params p{};
    p.max_iterations = 1000; p.nr_samples = 3; p.k_correspondences = 15;   // setCorrespondenceRandomness(15), :412
    p.min_sample_distance = 0.f; p.corr_dist_threshold = 100.f; p.seed = 0;
    if (ghicp_sac_ia(0, SourceCloud.xyz.data(), fs.data(), ns, TargetCloud.xyz.data(), ft.data(), nt, &p, &result_) < 0)
      throw std::runtime_error(std::string("CRegistration::Coarsereg_FPFHSAC: ") + ghicp_last_error(nullptr));
    for (int i = 0; i < 16; ++i) transformationS2T.data()[i] = (float)result_.Rt[i];
    // pcl::transformPointCloud with the float32 matrix, as PCL's align() moves the source
    Cloud out;
    const float *m = transformationS2T.data();
    for (int i = 0; i < ns; ++i) {
      const float x = SourceCloud.xyz[3 * (size_t)i], y = SourceCloud.xyz[3 * (size_t)i + 1], z = SourceCloud.xyz[3 * (size_t)i + 2];
      float o[3];
      for (int r = 0; r < 3; ++r) o[r] = ((m[r] * x + m[4 + r] * y) + m[8 + r] * z) + m[12 + r];
      out.push(o[0], o[1], o[2]);
    }
    TransformedSource = out;
    fitness_ = result_.fitness;
    std::cout << "The fitness score of this registration is " << result_.fitness << std::endl;   // :419
  }

  // :44-107 — point-to-point ICP of SourceCloud onto TargetCloud from the identity (transformation epsilon 1e-8, fitness
  // epsilon 1e-5); with use_trimmed_rejector the rejector's ratio is calOverlap(SourceCloud, TargetCloud, thre_dis), and the
  // call returns false without registering when that ratio is below min_overlap_for_reg.  TransformedSource = the moved source.
  bool icp_reg(const Cloud &SourceCloud, const Cloud &TargetCloud, Cloud &TransformedSource, Matrix4f &transformationS2T,
               int max_iter, bool use_reciprocal_correspondence, bool use_trimmed_rejector, float thre_dis,
               float min_overlap_for_reg) {
    return run_icp(SourceCloud, TargetCloud, TransformedSource, transformationS2T, max_iter, use_reciprocal_correspondence,
                   use_trimmed_rejector, thre_dis, 0, 0, min_overlap_for_reg);
  }

  // :123-199 — point-to-plane ICP of SourceCloud onto TargetCloud from the identity against TargetCloud's k-NN normals
  // (k = covariance_K, 3..32; transformation epsilon 1e-8, fitness epsilon 1e-5); the trimmed rejector as icp_reg.
  bool ptplicp_reg(const Cloud &SourceCloud, const Cloud &TargetCloud, Cloud &TransformedSource, Matrix4f &transformationS2T,
                   int max_iter, bool use_reciprocal_correspondence, bool use_trimmed_rejector, float thre_dis, int covariance_K,
                   float min_overlap_for_reg) {
    return run_icp(SourceCloud, TargetCloud, TransformedSource, transformationS2T, max_iter, use_reciprocal_correspondence,
                   use_trimmed_rejector, thre_dis, 1, covariance_K, min_overlap_for_reg);
  }

  // :217-284 — Generalized ICP of SourceCloud onto TargetCloud from the identity with both clouds' k-NN normals as
  // covariances (k = covariance_K, 3..32; transformation epsilon 1e-8, rotation epsilon 1e-6).  PCL's GICP ignores the
  // reciprocal option and the rejectors: the loop runs without them, and use_trimmed_rejector only returns false when
  // calOverlap(SourceCloud, TargetCloud, thre_dis) is below min_overlap_for_reg.
  bool gicp_reg(const Cloud &SourceCloud, const Cloud &TargetCloud, Cloud &TransformedSource, Matrix4f &transformationS2T,
                int max_iter, bool use_reciprocal_correspondence, bool use_trimmed_rejector, float thre_dis, int covariance_K,
                float min_overlap_for_reg) {
    (void)use_reciprocal_correspondence;
    return run_icp(SourceCloud, TargetCloud, TransformedSource, transformationS2T, max_iter, false, use_trimmed_rejector,
                   thre_dis, 2, covariance_K, min_overlap_for_reg);
  }

 private:
  // icp_reg (metric 0), ptplicp_reg (metric 1, normal_k) and gicp_reg (metric 2, normal_k; the overlap ratio gates only)
  bool run_icp(const Cloud &SourceCloud, const Cloud &TargetCloud, Cloud &TransformedSource, Matrix4f &transformationS2T,
               int max_iter, bool use_reciprocal_correspondence, bool use_trimmed_rejector, float thre_dis, int metric, int normal_k,
               float min_overlap_for_reg) {
    const char *who = metric == 2 ? "CRegistration::gicp_reg: " : (metric == 1 ? "CRegistration::ptplicp_reg: " : "CRegistration::icp_reg: ");
    const clock_t t0 = clock();
    ghicp_icp_params p{};
    p.max_iterations = max_iter; p.reciprocal = use_reciprocal_correspondence ? 1 : 0;
    p.transformation_epsilon = 1e-8; p.fitness_epsilon = 1e-5;   // :86, :88 (:166, :168; :263)
    p.metric = metric; p.normal_k = normal_k;
    p.rotation_epsilon = 1e-6;                                   // :265, read by metric 2 only
    if (use_trimmed_rejector) {
      const float overlap_ratio = calOverlap(SourceCloud, TargetCloud, thre_dis);
      if (overlap_ratio < min_overlap_for_reg) {
        std::cout << "The overlap ratio is too small. This registration would not be done." << std::endl;
        return false;
      }
      if (metric != 2) p.trim_ratio = std::min(1.0f, overlap_ratio);   // setOverlapRatio clamps to [0, 1]
    }
    const int n = (int)SourceCloud.size();
    std::vector<float> moved(3 * (size_t)n);
    ghicp_icp_result r{};
    if (ghicp_cloud_icp(0, SourceCloud.xyz.data(), n, TargetCloud.xyz.data(), (int)TargetCloud.size(), nullptr, &p, &r, moved.data(),
                        nullptr, nullptr) < 0)
      throw std::runtime_error(std::string(who) + ghicp_last_error(nullptr));
    for (int i = 0; i < 16; ++i) transformationS2T.data()[i] = (float)r.Rt[i];
    TransformedSource.xyz = moved;
    fitness_ = r.fitness;
    icp_result_ = r;
    const clock_t t1 = clock();
    std::cout << (metric == 2 ? "GICP" : (metric == 1 ? "Point-to-Plane ICP" : "Point-to-Point ICP")) << " done in "
              << float(t1 - t0) / CLOCKS_PER_SEC << " s" << std::endl;
    for (int i = 0; i < 4; ++i) {
      for (int j = 0; j < 4; ++j) std::cout << (j ? " " : "") << transformationS2T(i, j);
      std::cout << std::endl;
    }
    std::cout << "The fitness score of this registration is " << fitness_ << std::endl;
    if (metric == 2 && fitness_ > 5000) std::cout << "The fitness score of this registration is a bit too large" << std::endl;
    if (metric != 1) std::cout << "-----------------------------------------------------------------------------" << std::endl;
    return true;
  }

 public:

  // :294-317 — (0.01 + #{points of Cloud1 with a Cloud2 point at d2 < thre_dis^2}) / |Cloud1|, as the reference's float
  float calOverlap(const Cloud &Cloud1, const Cloud &Cloud2, float thre_dis) {
    ghicp_overlap_result r{};
    if (ghicp_cloud_overlap(0, Cloud1.xyz.data(), (int)Cloud1.size(), Cloud2.xyz.data(), (int)Cloud2.size(), nullptr, thre_dis,
                            0.0, 0, &r, nullptr) < 0)
      throw std::runtime_error(std::string("CRegistration::calOverlap: ") + ghicp_last_error(nullptr));
    std::cout << "The estimated approximate overlap ratio of Cloud 1 is " << r.ratio << std::endl;   // the reference logs this line
    return r.ratio;
  }

  // :325-350 — TransformedCloud receives every point moved by the float32 matrix (the reference appends to it)
  void transformcloud(const Cloud &CloudIn, Cloud &TransformedCloud, const Matrix4f &transformation) {
    const Matrix4f &m = transformation;
    for (size_t i = 0; i < CloudIn.size(); ++i) {
      const float x = CloudIn.xyz[3 * i], y = CloudIn.xyz[3 * i + 1], z = CloudIn.xyz[3 * i + 2];
      float o[3];
      for (int r = 0; r < 3; ++r) o[r] = ((m(r, 0) * x + m(r, 1) * y) + m(r, 2) * z) + m(r, 3);
      TransformedCloud.push(o[0], o[1], o[2]);
    }
    std::cout << "Transform done ..." << std::endl;
  }

  // :358-370 — NOT the inverse of a rigid transform: the rotation is transposed but the translation is only negated
  // (-t instead of -R^T t).  Reproduced as the reference has it; it is the inverse only when R is the identity.
  void invTransform(const Matrix4f &transformation, Matrix4f &invtransformation) {
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) invtransformation(i, j) = transformation(j, i);
    for (int i = 0; i < 3; ++i) invtransformation(i, 3) = -transformation(i, 3);
    for (int j = 0; j < 3; ++j) invtransformation(3, j) = 0.f;
    invtransformation(3, 3) = 1.f;
  }

  double getFitnessScore() const { return fitness_; }
  const ghicp_sac_result &sac_result() const { return result_; }
  const ghicp_icp_result &icp_result() const { return icp_result_; }

 private:
  ghicp_sac_result result_{};
  ghicp_icp_result icp_result_{};
  double fitness_ = 0.0;   // of the last Coarsereg_FPFHSAC or icp_reg
};

}  // namespace ghicp
