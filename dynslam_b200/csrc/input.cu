// input.cu — DynSLAM's stored stereo input on the device: the int16 millimetre depth image and the RGBA8 colour image that
// InfiniTamDriver::UpdateView (DS/InfiniTamDriver.h) hands to ITMLib, made in one pass over the frame.
//
// Depth, one of two modes (b200_depth_input.kind):
//   0  DepthProvider::DepthFromDisparityMap<float> with scale 1 (DS/DepthProvider.h:94-137) around
//      PrecomputedDepthProvider::DepthFromDisparity (DS/PrecomputedDepthProvider.cpp:77-80): a DispNet float disparity map;
//   1  the max-depth clamp PrecomputedDepthProvider::ReadPrecomputed applies to a stored int16 depth map (ELAS XML,
//      DS/PrecomputedDepthProvider.cpp:52-74). There is no lower bound in this mode, as in the reference.
// Colour: CvToItm(const cv::Mat3b &, ITMUChar4Image *) (DS/InfiniTamDriver.cpp:81-100): OpenCV's BGR8 into RGBA8, a = 255.
//
// Bit-exact with the reference (oracle/input_oracle.c, pinned to the reference's own functions in
// tests/test_stereo_input_oracle.py). The quotient is IEEE (-prec-div=true) and nothing is contracted (-fmad=false):
// depth_mm = trunc(1000 * ((focal * baseline) / disp)), with focal * baseline formed on the host in binary32.
//
// Two cases where the reference's C++ is not defined, and how the result is kept independent of them:
//   * static_cast<int32_t> of a value outside the int32 range (or NaN) is undefined behaviour; x86 gives INT_MIN, the device
//     conversion saturates. Such a value is never converted here: it is invalid and gives 0, which is also what the reference
//     ends with under either conversion (INT_MIN fails the lower bound or casts to an int16 of 0, a saturated INT_MAX fails
//     the upper bound, which is below 32767). The bounds themselves are converted on the host with x86's convention
//     (b200_engine's depth_input_bounds).
//   * `abs(disp)` at DepthProvider.h:125 is unqualified. In the reference's translation unit, which sees <cmath> through
//     DS/Utils.h, no float overload of `abs` is visible from namespace dynslam, so it is `int abs(int)` of the truncated
//     disparity: every |disp| < 1 (and NaN) gives 0, not only |disp| < 1e-5. That is the behaviour pinned here. Under the
//     float reading the output would be the same whenever 1000 * (focal * baseline) >= max_depth_mm + 1 and
//     min_depth_m >= 0 (a disparity below 1 px then maps beyond the upper bound, or below 0); KITTI has focal * baseline
//     = 387 m*px against a 20 m maximum.
#include "engine.h"

namespace {

constexpr int IN_THREADS = 256;
constexpr int IN_PX = 4;   // pixels per thread: 12 BGR bytes = three 32-bit words, one 16-byte RGBA store

// DepthFromDisparityMap<float>'s loop body (DepthProvider.h:121-134) for scale == 1
DEV int16_t depth_mm_from_disparity(float disp, float fb, int minMm, int maxMm) {
  if (!(fabsf(disp) >= 1.0f)) return 0;                       // abs(disp) < 1e-5 with int abs(int): see the file comment
  const float v = __fmul_rn(1000.0f, __fdiv_rn(fb, disp));    // kMetersToMillimeters * scale * DepthFromDisparity(...)
  if (!(fabsf(v) < 2147483648.0f)) return 0;                  // the int32 cast would be undefined: the reference ends at 0
  const int d = __float2int_rz(v);
  return (d > maxMm || d < minMm) ? (int16_t)0 : (int16_t)d;
}

// ReadPrecomputed's int16 clamp (PrecomputedDepthProvider.cpp:67-70); maxS = (int16_t)round(max_depth_m * 1000.0f)
DEV int16_t depth_mm_clamped(int16_t d, int maxS) { return d > maxS ? (int16_t)0 : d; }

DEV int16_t depth_px(const void *in, int kind, int i, float fb, int minMm, int maxMm) {
  return kind == 0 ? depth_mm_from_disparity(static_cast<const float *>(in)[i], fb, minMm, maxMm)
                   : depth_mm_clamped(static_cast<const int16_t *>(in)[i], maxMm);
}

// one BGR pixel as a b200_vec4u word (r, g, b, a in memory order): .b = col[0], .g = col[1], .r = col[2], .a = 255
DEV unsigned rgba_word(unsigned b, unsigned g, unsigned r) { return r | (g << 8) | (b << 16) | 0xff000000u; }

// IN_PX pixels per thread. VEC: every pointer is 16-byte aligned (bgr: 4-byte), so a full group of four pixels is read and
// written with vector accesses: depth 16 B (disparity) or 8 B (int16) in, 8 B out; colour 12 B in as three words, 16 B out.
// The depth image may be written in place (kind 1), so the depth pointers are not __restrict__.
template <bool VEC>
__global__ void __launch_bounds__(IN_THREADS) k_stereo_input(const void *depthIn, int kind, int nDepth, float fb, int minMm, int maxMm,
                                                             int16_t *depthOut, int16_t *depthCopy, const uint8_t *__restrict__ bgr,
                                                             b200_vec4u *__restrict__ rgba, int nColour) {
  const int p0 = (blockIdx.x * IN_THREADS + threadIdx.x) * IN_PX;
  if (depthOut && p0 < nDepth) {
    int16_t o[IN_PX];
    if (VEC && p0 + IN_PX <= nDepth) {
      if (kind == 0) {
        const float4 v = *reinterpret_cast<const float4 *>(static_cast<const float *>(depthIn) + p0);
        o[0] = depth_mm_from_disparity(v.x, fb, minMm, maxMm); o[1] = depth_mm_from_disparity(v.y, fb, minMm, maxMm);
        o[2] = depth_mm_from_disparity(v.z, fb, minMm, maxMm); o[3] = depth_mm_from_disparity(v.w, fb, minMm, maxMm);
      } else {
        const short4 v = *reinterpret_cast<const short4 *>(static_cast<const int16_t *>(depthIn) + p0);
        o[0] = depth_mm_clamped(v.x, maxMm); o[1] = depth_mm_clamped(v.y, maxMm);
        o[2] = depth_mm_clamped(v.z, maxMm); o[3] = depth_mm_clamped(v.w, maxMm);
      }
      const short4 s = make_short4(o[0], o[1], o[2], o[3]);
      *reinterpret_cast<short4 *>(depthOut + p0) = s;
      if (depthCopy) *reinterpret_cast<short4 *>(depthCopy + p0) = s;
    } else {
      for (int k = 0; k < IN_PX && p0 + k < nDepth; ++k) {
        const int16_t d = depth_px(depthIn, kind, p0 + k, fb, minMm, maxMm);
        depthOut[p0 + k] = d;
        if (depthCopy) depthCopy[p0 + k] = d;
      }
    }
  }
  if (rgba && p0 < nColour) {
    if (VEC && p0 + IN_PX <= nColour) {
      const unsigned *w = reinterpret_cast<const unsigned *>(bgr + (size_t)p0 * 3);
      const unsigned w0 = w[0], w1 = w[1], w2 = w[2];   // bytes B0 G0 R0 B1 | G1 R1 B2 G2 | R2 B3 G3 R3
      uint4 o;
      o.x = __byte_perm(w0, w1, 0x0012) | 0xff000000u;
      o.y = __byte_perm(w0, w1, 0x0345) | 0xff000000u;
      o.z = __byte_perm(w1, w2, 0x0234) | 0xff000000u;
      o.w = __byte_perm(w2, w2, 0x0123) | 0xff000000u;
      *reinterpret_cast<uint4 *>(rgba + p0) = o;
    } else {
      for (int k = 0; k < IN_PX && p0 + k < nColour; ++k) {
        const uint8_t *c = bgr + (size_t)(p0 + k) * 3;
        reinterpret_cast<unsigned *>(rgba)[p0 + k] = rgba_word(c[0], c[1], c[2]);
      }
    }
  }
}

bool aligned(const void *p, uintptr_t a) { return ((uintptr_t)p & (a - 1)) == 0; }

}  // namespace

void launch_stereo_input(b200_engine *e, cudaStream_t st, const void *depthIn, int kind, int nDepth, float fb, int minMm, int maxMm,
                         int16_t *depthOut, int16_t *depthCopy, const uint8_t *bgr, b200_vec4u *rgba, int nColour) {
  if (!depthOut) nDepth = 0;
  if (!rgba) nColour = 0;
  const int n = nDepth > nColour ? nDepth : nColour;
  if (n <= 0) return;
  const bool vec = (!depthOut || (aligned(depthIn, 16) && aligned(depthOut, 16) && (!depthCopy || aligned(depthCopy, 16)))) &&
                   (!rgba || (aligned(bgr, 4) && aligned(rgba, 16)));
  const int threads = (n + IN_PX - 1) / IN_PX, grid = (threads + IN_THREADS - 1) / IN_THREADS;
  trace_begin(e, st, "k_stereo_input");
  if (vec) k_stereo_input<true><<<grid, IN_THREADS, 0, st>>>(depthIn, kind, nDepth, fb, minMm, maxMm, depthOut, depthCopy, bgr, rgba, nColour);
  else k_stereo_input<false><<<grid, IN_THREADS, 0, st>>>(depthIn, kind, nDepth, fb, minMm, maxMm, depthOut, depthCopy, bgr, rgba, nColour);
  trace_end(e, st);
  e->launches++;
}
