// ref_input_driver.cpp — TEST INFRASTRUCTURE ONLY. Pins oracle/input_oracle.c to the reference's own code.
//
//  * struct StereoCalibration ... class DepthProvider (DS/DepthProvider.h:22-176), with DepthFromStereo and the template
//    DepthFromDisparityMap<float>, and PrecomputedDepthProvider::DepthFromDisparity (DS/PrecomputedDepthProvider.cpp:77-80);
//  * the max-depth clamp block of PrecomputedDepthProvider::ReadPrecomputed (DS/PrecomputedDepthProvider.cpp:52-74);
//  * CvToItm(const cv::Mat3b &, ITMUChar4Image *) (DS/InfiniTamDriver.cpp:81-100).
// oracle/build_input_ref.sh cuts them out of the reference files AT BUILD TIME into oracle/_ref/ (git-ignored; nothing of the reference
// is stored in this repo) and this driver #includes them unmodified. The cut text sees the declarations of its own translation
// unit: DS/Utils.h's standard headers (<cmath> among them, which decides which `abs` DepthProvider.h:125 calls) and OpenCV's
// matrices, here the stand-in under oracle/input_stubs. The declaration of PrecomputedDepthProvider below is ours: the reference's
// header pulls in the whole Input pipeline.
#include <limits>
#include <cmath>
#include <map>
#include <string>
#include <sys/stat.h>
#include <stack>
#include <vector>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <stdexcept>

#include <opencv2/opencv.hpp>                 // stand-in

namespace dynslam {
namespace utils {
std::string Type2Str(int type) { return std::to_string(type); }
std::string Format(const std::string &fmt, ...) {
  char buf[512];
  va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt.c_str(), ap); va_end(ap);
  return std::string(buf);
}
}   // namespace utils

#include "_ref/depthprovider_extract.inc"   // struct StereoCalibration ... class DepthProvider — unmodified reference text

class PrecomputedDepthProvider : public DepthProvider {
 public:
  PrecomputedDepthProvider(bool input_is_depth, float min_depth_m, float max_depth_m)
      : DepthProvider(input_is_depth, min_depth_m, max_depth_m) {}
  void DisparityMapFromStereo(const cv::Mat &, const cv::Mat &, cv::Mat &out_disparity) override { out_disparity = *stored_; }
  float DepthFromDisparity(const float disparity_px, const StereoCalibration &calibration) override;
  const std::string &GetName() const override { return name_; }
  void Clamp(cv::Mat &out) const {
#include "_ref/clamp_extract.inc"           // if (this->input_is_depth_) { ... } — unmodified reference text
  }
  const cv::Mat *stored_ = nullptr;
  std::string name_ = "precomputed";
};

#include "_ref/dfd_extract.inc"             // PrecomputedDepthProvider::DepthFromDisparity — unmodified reference text
}   // namespace dynslam

// after the depth provider, so that nothing ITMLib declares is visible to it
#include "ITMLib/Utils/ITMLibDefines.h"       // Vector2i, Vector4u, ITMUChar4Image (reference, host build)

namespace dynslam {
namespace drivers {
#include "_ref/cvtoitm_extract.inc"         // CvToItm(const cv::Mat3b &, ITMUChar4Image *) — unmodified reference text
}   // namespace drivers
}   // namespace dynslam

static_assert(sizeof(Vector4u) == 4, "vec4u layout");
static char g_err[512];

extern "C" {

const char *ref_input_last_error() { return g_err; }

// Input::ReadNextFrame's DepthFromStereo on a stored float disparity map (DispNet): 0, or -1 with the reference's message
int ref_depth_from_disparity(int16_t *out, const float *disp, int w, int h, float baseline_m, float focal_length_px, float min_depth_m,
                             float max_depth_m) {
  dynslam::PrecomputedDepthProvider p(false, min_depth_m, max_depth_m);
  cv::Mat stored(h, w, sizeof(float), CV_32FC1);
  memcpy(stored.bytes.data(), disp, (size_t)w * h * sizeof(float));
  p.stored_ = &stored;
  cv::Mat1s depth(h, w);
  cv::Mat none;
  try {
    p.DepthFromStereo(none, none, dynslam::StereoCalibration(baseline_m, focal_length_px), depth, 1.0f);
  } catch (const std::runtime_error &ex) {
    snprintf(g_err, sizeof(g_err), "%s", ex.what());
    return -1;
  }
  memcpy(out, depth.bytes.data(), (size_t)w * h * sizeof(int16_t));
  return 0;
}

// ReadPrecomputed's clamp of a stored int16 depth map (ELAS), in place
void ref_clamp_depth_mm(int16_t *depth, int w, int h, float max_depth_m) {
  dynslam::PrecomputedDepthProvider p(true, 0.0f, max_depth_m);
  cv::Mat m(h, w, sizeof(int16_t), CV_16SC1);
  memcpy(m.bytes.data(), depth, (size_t)w * h * sizeof(int16_t));
  p.Clamp(m);
  memcpy(depth, m.bytes.data(), (size_t)w * h * sizeof(int16_t));
}

void ref_bgr_to_rgba(uint8_t *out, const uint8_t *bgr, int w, int h) {
  cv::Mat3b m(h, w);
  memcpy(m.bytes.data(), bgr, (size_t)w * h * 3);
  ITMUChar4Image img(Vector2i(w, h), MEMORYDEVICE_CPU);
  dynslam::drivers::CvToItm(m, &img);
  memcpy(out, img.GetData(MEMORYDEVICE_CPU), (size_t)w * h * 4);
}

}   // extern "C"
