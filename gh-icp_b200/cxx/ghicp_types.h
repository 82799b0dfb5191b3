// ghicp_types.h — matrix / descriptor types at the boundary of the registration classes.
// With Eigen / PCL on the include path (i.e. inside the reference's own build) the reference's types are
// used unchanged; stand-alone (this repo's tests) minimal column-major PODs with the same member
// names stand in, so the same GHRegistration source compiles both ways.
#pragma once
#include <cmath>
#include <cstddef>
#include <cstring>
#include <vector>

#if defined(__has_include)
#if __has_include(<Eigen/Core>) && !defined(GHICP_NO_EIGEN)
#define GHICP_HAVE_EIGEN 1
#include <Eigen/Core>
#endif
#if __has_include(<pcl/point_types.h>) && !defined(GHICP_NO_PCL)
#define GHICP_HAVE_PCL 1
#include <pcl/point_cloud.h>
#include <pcl/point_types.h>
#endif
#endif

namespace ghicp {

#ifdef GHICP_HAVE_EIGEN
using MatrixX3d = Eigen::MatrixX3d;   // include/ghicp_reg.h:47
using Matrix4d = Eigen::Matrix4d;     // include/ghicp_reg.h:132
using Matrix4f = Eigen::Matrix4f;     // include/common_reg.h:120-124
inline Matrix4d Identity4() { return Matrix4d::Identity(); }
#else
// column-major N x 3 doubles: the layout of Eigen::MatrixX3d::data()
struct MatrixX3d {
  std::vector<double> v;
  std::ptrdiff_t n = 0;
  MatrixX3d() {}
  MatrixX3d(std::ptrdiff_t rows_, int) { resize(rows_, 3); }
  void resize(std::ptrdiff_t rows_, int) { n = rows_; v.assign(3 * (size_t)rows_, 0.0); }
  std::ptrdiff_t rows() const { return n; }
  int cols() const { return 3; }
  double &operator()(std::ptrdiff_t i, int j) { return v[(size_t)j * n + i]; }
  double operator()(std::ptrdiff_t i, int j) const { return v[(size_t)j * n + i]; }
  double *data() { return v.data(); }
  const double *data() const { return v.data(); }
};
// column-major 4 x 4 doubles: the layout of Eigen::Matrix4d::data()
struct Matrix4d {
  double v[16];
  double &operator()(int i, int j) { return v[j * 4 + i]; }
  double operator()(int i, int j) const { return v[j * 4 + i]; }
  double *data() { return v; }
  const double *data() const { return v; }
  Matrix4d operator*(const Matrix4d &o) const {
    Matrix4d r;
    for (int c = 0; c < 4; ++c)
      for (int i = 0; i < 4; ++i) {
        double s = 0;
        for (int k = 0; k < 4; ++k) s += (*this)(i, k) * o(k, c);
        r(i, c) = s;
      }
    return r;
  }
};
inline Matrix4d Identity4() {
  Matrix4d m;
  for (int i = 0; i < 16; ++i) m.v[i] = (i % 5 == 0) ? 1.0 : 0.0;
  return m;
}
// column-major 4 x 4 floats: the layout of Eigen::Matrix4f::data()
struct Matrix4f {
  float v[16];
  float &operator()(int i, int j) { return v[j * 4 + i]; }
  float operator()(int i, int j) const { return v[j * 4 + i]; }
  float *data() { return v; }
  const float *data() const { return v; }
};
#endif

// Binary descriptor with the reference's member names (include/stereo_binary_feature.h:25-58).
// Bit k lives in byte k/8, bit k%8, LSB first (:140-146).
struct StereoBinaryFeature {
  std::vector<char> storage_;
  char *feature_ = nullptr;
  unsigned int size_ = 0;  // bits
  unsigned int byte_ = 0;  // bytes
  explicit StereoBinaryFeature(unsigned int size = 0) : size_(size) {
    if (size) {
      byte_ = static_cast<unsigned int>(std::ceil(float(size_) / 8.f));
      storage_.assign(byte_, 0);
      feature_ = storage_.data();
    }
  }
  StereoBinaryFeature(const StereoBinaryFeature &o) : storage_(o.storage_), size_(o.size_), byte_(o.byte_) {
    feature_ = storage_.empty() ? nullptr : storage_.data();
  }
  StereoBinaryFeature &operator=(const StereoBinaryFeature &o) {
    storage_ = o.storage_; size_ = o.size_; byte_ = o.byte_;
    feature_ = storage_.empty() ? nullptr : storage_.data();
    return *this;
  }
  bool getNthBitValue(int n) const { return (feature_[n / 8] & (char)(1 << (n % 8))) != 0; }
  void setNthBitValue(int n) { feature_[n / 8] |= (char)(1 << (n % 8)); }
};
typedef StereoBinaryFeature SBF;
typedef std::vector<SBF> vectorSBF;
typedef std::vector<vectorSBF> doubleVectorSBF;

#ifdef GHICP_HAVE_PCL
typedef pcl::PointCloud<pcl::FPFHSignature33>::Ptr fpfhFeaturePtr;  // include/utility.h:45
#else
struct FPFHSignature33 { float histogram[33]; };
struct fpfhFeature { std::vector<FPFHSignature33> points; };
typedef fpfhFeature *fpfhFeaturePtr;  // non-owning stand-in for the PCL shared pointer
#endif

}  // namespace ghicp
