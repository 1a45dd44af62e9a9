/* input_oracle.c — TEST INFRASTRUCTURE ONLY (never linked into, imported or called by dynslam_b200/).
 *
 * Serial C restatement of DynSLAM's per-frame input conversions, the reference for dynslam_b200/csrc/input.cu:
 *   DepthProvider::DepthFromDisparityMap<float>           DS/DepthProvider.h:94-137
 *   PrecomputedDepthProvider::DepthFromDisparity          DS/PrecomputedDepthProvider.cpp:77-80
 *   PrecomputedDepthProvider::ReadPrecomputed's clamp     DS/PrecomputedDepthProvider.cpp:52-74
 *   CvToItm(const cv::Mat3b &, ITMUChar4Image *)          DS/InfiniTamDriver.cpp:81-100
 * Built by __graft_entry__.build() into oracle/libinputoracle.so. No contraction, no fast-math.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

#include "../include/b200fusion.h"

/* ---- DynSLAM's stored stereo input ---------------------------------------------------------------------------------------
 * Pinned bit for bit against the reference's own functions (oracle/ref_input_driver.cpp; tests/test_stereo_input_oracle.py).
 * Where the reference's C++ casts are undefined (a float outside the int32 range, or NaN, converted to int32), the oracle uses
 * x86's result, INT_MIN; the output is 0 then under any convention (see dynslam_b200/csrc/input.cu). */
static int32_t x86_cvtt_i32(double x) { return (x > -2147483649.0 && x < 2147483648.0) ? (int32_t)x : INT32_MIN; }

/* DepthProvider::DepthFromDisparityMap<float> with scale 1 (DepthProvider.h:94-137) around
 * PrecomputedDepthProvider::DepthFromDisparity (PrecomputedDepthProvider.cpp:77-80). The unqualified abs(disp) of :125 is
 * int abs(int) in the reference's translation unit (only <cmath> is visible there): a disparity whose truncation is 0 gives 0.
 * The max-depth check of :113-117 is the caller's (it throws in the reference). */
void oracle_depth_from_disparity(int16_t *out, const float *disp, int n, float baseline_m, float focal_length_px, float min_depth_m,
                                 float max_depth_m) {
  const float kMetersToMillimeters = 1000.0f, scale = 1.0f;
  const int32_t min_depth_mm = x86_cvtt_i32(min_depth_m * kMetersToMillimeters);
  const int32_t max_depth_mm = x86_cvtt_i32(max_depth_m * kMetersToMillimeters);
  for (int i = 0; i < n; i++) {
    const float d = disp[i];
    const float depth_m = focal_length_px * baseline_m / d;
    int32_t depth_mm = x86_cvtt_i32(kMetersToMillimeters * scale * depth_m);
    int32_t idisp = x86_cvtt_i32(d);
    if (idisp == INT32_MIN || abs(idisp) < 1e-5) depth_mm = 0;   /* abs(INT_MIN) is INT_MIN on x86: below 1e-5 */
    if (depth_mm > max_depth_mm || depth_mm < min_depth_mm) depth_mm = 0;
    out[i] = (int16_t)depth_mm;
  }
}

/* PrecomputedDepthProvider::ReadPrecomputed's clamp of a stored int16 depth map (PrecomputedDepthProvider.cpp:52-74), in place */
void oracle_clamp_depth_mm(int16_t *depth, int n, float max_depth_m) {
  const float max_depth_mm_f = max_depth_m * 1000.0f;
  const int16_t max_depth_mm_s = (int16_t)(uint16_t)(uint32_t)x86_cvtt_i32(round(max_depth_mm_f));
  for (int i = 0; i < n; i++) if (depth[i] > max_depth_mm_s) depth[i] = 0;
}

/* CvToItm(const cv::Mat3b &, ITMUChar4Image *) (InfiniTamDriver.cpp:81-100): .b = col[0], .g = col[1], .r = col[2], .a = 255 */
void oracle_bgr_to_rgba(b200_vec4u *out, const uint8_t *bgr, int n) {
  for (int i = 0; i < n; i++) {
    out[i].x = bgr[3 * i + 2]; out[i].y = bgr[3 * i + 1]; out[i].z = bgr[3 * i]; out[i].w = 255;
  }
}
