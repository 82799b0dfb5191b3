// filter.h — host-side mirror of the reference's CFilter (include/filter.hpp) over libghicp_b200.so, with the members the
// library backs:
//   voxelfilter  (:28-88)   one point per occupied voxel, by ghicp_voxel_downsample (the reference's output order and its
//                           phantom first entry included; non-finite points dropped)
//   SORFilter    (:90-102)  PCL's StatisticalOutlierRemoval with MeanK (1..128) and the standard-deviation multiplier, by
//                           ghicp_sor_filter on the canonical definition of DESIGN.md §3.16 (kept points in input order)
// cloud_out as the reference leaves it: voxelfilter appends to it (the reference push_back()s), SORFilter replaces it (PCL's
// filter() overwrites its output).
// Differences, deliberate: clouds are ghicp::Cloud (cloud_io.h); no CPU path (without a CUDA device both members throw).
// Not provided: DisFilter and ActiveObjectFilter (point-wise predicates with no GPU work).
#pragma once
#include <iostream>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "../../include/ghicp_b200.h"
#include "cloud_io.h"

namespace ghicp {

template <typename PointT = void>
class CFilter {
 public:
  bool voxelfilter(const Cloud &cloud_in, Cloud &cloud_out, float voxel_size) {
    const int n = (int)cloud_in.size();
    std::vector<int> idx((size_t)n + 1);
    int m = 0;
    if (ghicp_voxel_downsample(0, cloud_in.xyz.data(), n, voxel_size, idx.data(), &m) < 0)
      throw std::runtime_error(std::string("CFilter::voxelfilter: ") + ghicp_last_error(nullptr));
    Cloud kept;
    gather(cloud_in, idx, m, kept);
    cloud_out.xyz.insert(cloud_out.xyz.end(), kept.xyz.begin(), kept.xyz.end());
    std::cout << "Downsample done (" << cloud_out.size() << " points)" << std::endl;
    return 1;
  }

  // :90-102 — MeanK 50 and std 2.0 in the reference's comment
  bool SORFilter(const Cloud &cloud_in, Cloud &cloud_out, int MeanK, double std) {
    const int n = (int)cloud_in.size();
    std::vector<int> idx(n > 0 ? (size_t)n : 1);
    ghicp_sor_result r{};
    if (ghicp_sor_filter(0, cloud_in.xyz.data(), n, MeanK, std, idx.data(), nullptr, &r) < 0)
      throw std::runtime_error(std::string("CFilter::SORFilter: ") + ghicp_last_error(nullptr));
    gather(cloud_in, idx, r.n_kept, cloud_out);
    return 1;
  }

 private:
  static void gather(const Cloud &in, const std::vector<int> &idx, int m, Cloud &out) {
    Cloud c;
    c.xyz.reserve(3 * (size_t)m);
    for (int j = 0; j < m; ++j) {
      const float *p = in.xyz.data() + 3 * (size_t)idx[j];
      c.push(p[0], p[1], p[2]);
    }
    out = std::move(c);
  }
};

}  // namespace ghicp
