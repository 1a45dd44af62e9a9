// Minimal stand-in for <opencv2/opencv.hpp> for oracle/ref_input_driver.cpp — TEST INFRASTRUCTURE ONLY (oracle/build_input_ref.sh).
// OpenCV is not installed here. DS/DepthProvider.h, the clamp of PrecomputedDepthProvider::ReadPrecomputed and CvToItm only need
// matrices with rows, cols, type(), size() and at<T>(row, col) over row-major bytes, and a three-byte pixel. Nothing of OpenCV's
// implementation is reproduced.
#pragma once
#include <cassert>
#include <cstddef>
#include <vector>
typedef unsigned char uchar;
#define CV_16SC1 3
#define CV_32FC1 5
namespace cv {
struct Size {
  int width, height;
  Size(int w = 0, int h = 0) : width(w), height(h) {}
  bool operator==(const Size &o) const { return width == o.width && height == o.height; }
};
class Mat {
 public:
  int rows = 0, cols = 0;
  int type_ = 0;                                       // a CV_* code, set by whoever fills the matrix
  std::vector<unsigned char> bytes;
  Mat() {}
  Mat(int r, int c, int elemSize, int type) : rows(r), cols(c), type_(type), bytes((size_t)r * c * elemSize) {}
  int type() const { return type_; }
  Size size() const { return Size(cols, rows); }
  template <typename T> T &at(int r, int c) { return reinterpret_cast<T *>(bytes.data())[(size_t)r * cols + c]; }
  template <typename T> const T &at(int r, int c) const { return reinterpret_cast<const T *>(bytes.data())[(size_t)r * cols + c]; }
};
template <typename T> class Mat_ : public Mat {
 public:
  Mat_() {}
  Mat_(int r, int c) : Mat(r, c, sizeof(T), 0) {}
  Mat_(const Mat &m) : Mat(m) {}
};
typedef Mat_<short> Mat1s;
struct Vec3b { uchar v[3]; uchar &operator[](int i) { return v[i]; } const uchar &operator[](int i) const { return v[i]; } };
typedef Mat_<Vec3b> Mat3b;
}   // namespace cv
