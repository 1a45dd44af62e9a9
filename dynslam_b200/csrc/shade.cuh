// shade.cuh — per-pixel shading from the volume for k_shade (vis.cu): the SDF normal, the interpolated colour, the RGBA pixel
// of every RenderImage type but the depth map, and the depth pixel.
#pragma once
#include "raycast_ray.cuh"

DEV float rvs(const b200_voxel *__restrict__ voxels, const b200_hash_entry *__restrict__ table, int nb, int x, int y, int z) {
  IdxCache c; cache_init(c);   // the 4-argument readVoxel builds a fresh cache per read (:222-228)
  return rv_sdf(voxels, table, nb, x, y, z, c);
}

// computeSingleNormalFromSDF — DA/ITMRepresentationAccess.h:336-449
__device__ inline void normal_from_sdf(const b200_voxel *__restrict__ voxels, const b200_hash_entry *__restrict__ table, int nb, float px, float py,
                                float pz, float &rx, float &ry, float &rz) {
  const float fx = floorf(px), fy = floorf(py), fz = floorf(pz);
  const float cx = px - fx, cy = py - fy, cz = pz - fz;
  const int X = (int)fx, Y = (int)fy, Z = (int)fz;
  const float nx = 1.0f - cx, ny = 1.0f - cy, nz = 1.0f - cz;
#define RV(a, b, c) rvs(voxels, table, nb, X + (a), Y + (b), Z + (c))
  const float f0 = RV(0, 0, 0), f1 = RV(1, 0, 0), f2 = RV(0, 1, 0), f3 = RV(1, 1, 0);
  const float b0 = RV(0, 0, 1), b1 = RV(1, 0, 1), b2 = RV(0, 1, 1), b3 = RV(1, 1, 1);
  float t0, t1, t2, t3, p1, p2, v1;
  p1 = f0 * ny * nz + f2 * cy * nz + b0 * ny * cz + b2 * cy * cz;
  t0 = RV(-1, 0, 0); t1 = RV(-1, 1, 0); t2 = RV(-1, 0, 1); t3 = RV(-1, 1, 1);
  p2 = t0 * ny * nz + t1 * cy * nz + t2 * ny * cz + t3 * cy * cz;
  v1 = p1 * cx + p2 * nx;
  p1 = f1 * ny * nz + f3 * cy * nz + b1 * ny * cz + b3 * cy * cz;
  t0 = RV(2, 0, 0); t1 = RV(2, 1, 0); t2 = RV(2, 0, 1); t3 = RV(2, 1, 1);
  p2 = t0 * ny * nz + t1 * cy * nz + t2 * ny * cz + t3 * cy * cz;
  rx = (p1 * nx + p2 * cx - v1) / 32767.0f;
  p1 = f0 * nx * nz + f1 * cx * nz + b0 * nx * cz + b1 * cx * cz;
  t0 = RV(0, -1, 0); t1 = RV(1, -1, 0); t2 = RV(0, -1, 1); t3 = RV(1, -1, 1);
  p2 = t0 * nx * nz + t1 * cx * nz + t2 * nx * cz + t3 * cx * cz;
  v1 = p1 * cy + p2 * ny;
  p1 = f2 * nx * nz + f3 * cx * nz + b2 * nx * cz + b3 * cx * cz;
  t0 = RV(0, 2, 0); t1 = RV(1, 2, 0); t2 = RV(0, 2, 1); t3 = RV(1, 2, 1);
  p2 = t0 * nx * nz + t1 * cx * nz + t2 * nx * cz + t3 * cx * cz;
  ry = (p1 * ny + p2 * cy - v1) / 32767.0f;
  p1 = f0 * nx * ny + f1 * cx * ny + f2 * nx * cy + f3 * cx * cy;
  t0 = RV(0, 0, -1); t1 = RV(1, 0, -1); t2 = RV(0, 1, -1); t3 = RV(1, 1, -1);
  p2 = t0 * nx * ny + t1 * cx * ny + t2 * nx * cy + t3 * cx * cy;
  v1 = p1 * cz + p2 * nz;
  p1 = b0 * nx * ny + b1 * cx * ny + b2 * nx * cy + b3 * cx * cy;
  t0 = RV(0, 0, 2); t1 = RV(1, 0, 2); t2 = RV(0, 1, 2); t3 = RV(1, 1, 2);
  p2 = t0 * nx * ny + t1 * cx * ny + t2 * nx * cy + t3 * cx * cy;
  rz = (p1 * nz + p2 * cz - v1) / 32767.0f;
#undef RV
}

// computeNormalAndAngle<TVoxel,TIndex> — DA/ITMVisualisationEngine.h:196-210
DEV void normal_and_angle_sdf(bool &found, float px, float py, float pz, const b200_voxel *__restrict__ voxels,
                              const b200_hash_entry *__restrict__ table, int nb, float lx, float ly, float lz, float &nx, float &ny,
                              float &nz, float &angle) {
  if (!found) return;
  normal_from_sdf(voxels, table, nb, px, py, pz, nx, ny, nz);
  const float normScale = 1.0f / sqrtf(nx * nx + ny * ny + nz * nz);
  nx *= normScale; ny *= normScale; nz *= normScale;
  angle = nx * lx + ny * ly + nz * lz;
  if (!(angle > 0.0)) found = false;
}

// readFromSDF_color4u_interpolated_noalpha — DA/ITMRepresentationAccess.h:280-318
__device__ inline void color_interp(const b200_voxel *__restrict__ voxels, const b200_hash_entry *__restrict__ table, int nb, float px, float py,
                             float pz, float &r0, float &r1, float &r2) {
  IdxCache c; cache_init(c);
  const float fx = floorf(px), fy = floorf(py), fz = floorf(pz);
  const float cx = px - fx, cy = py - fy, cz = pz - fz;
  const int X = (int)fx, Y = (int)fy, Z = (int)fz;
  r0 = r1 = r2 = 0.0f;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int ox = k & 1, oy = (k >> 1) & 1, oz = k >> 2;
    const int vi = voxel_index(table, nb, X + ox, Y + oy, Z + oz, c);
    float cr = 0.0f, cg = 0.0f, cb = 0.0f;
    if (vi >= 0) {
      const unsigned lo = __ldg(reinterpret_cast<const unsigned *>(voxels + vi)), hi = __ldg(reinterpret_cast<const unsigned *>(voxels + vi) + 1);
      cr = (float)((lo >> 24) & 0xff); cg = (float)(hi & 0xff); cb = (float)((hi >> 8) & 0xff);
    }
    const float wgt = (ox ? cx : (1.0f - cx)) * (oy ? cy : (1.0f - cy)) * (oz ? cz : (1.0f - cz));
    r0 += wgt * cr; r1 += wgt * cg; r2 += wgt * cb;
  }
  r0 = r0 / 255.0f; r1 = r1 / 255.0f; r2 = r2 / 255.0f;
}

DEV uchar4 grey_px(float angle) {   // drawPixelGrey, DA/ITMVisualisationEngine.h:277-281
  const float outRes = (0.8f * angle + 0.2f) * 255.0f;
  const unsigned char g = (unsigned char)outRes;
  return make_uchar4(g, g, g, g);
}

DEV uchar4 draw_colour(const b200_voxel *__restrict__ voxels, const b200_hash_entry *__restrict__ table, int nb, float px, float py, float pz) {
  float c0, c1, c2;
  color_interp(voxels, table, nb, px, py, pz, c0, c1, c2);
  return make_uchar4((unsigned char)(c0 * 255.0f), (unsigned char)(c1 * 255.0f), (unsigned char)(c2 * 255.0f), 255);
}

// drawPixelDepth — DA/ITMVisualisationEngine.h:304-320
DEV float depth_px(bool found, const float4 &pr, const Mat4 &M, float voxelSize) {
  if (!found) return 0.0f;
  const Vec4 pc = m4v4(M, pr.x * voxelSize, pr.y * voxelSize, pr.z * voxelSize, 1.0f);
  return pc.z / pc.w;
}

// The RGBA pixel of one ray point for every type but RENDER_DEPTH_MAP (RenderImage_common's kernels, Vis_CUDA.cu:735-886;
// WeightRenderingParams(1.0, false, maxW, 2), :303-311). `found` is the ray's hit flag; *px is read only by
// RENDER_COLOUR_FROM_NORMAL, which leaves the alpha of a found pixel as it is.
DEV void shade_rgba_px(int type, bool found, const float4 &pr, const b200_voxel *__restrict__ voxels, const b200_hash_entry *__restrict__ table,
                       int nb, float lx, float ly, float lz, int maxW, uchar4 *px) {
  float nx = 0, ny = 0, nz = 0, angle = 0;
  normal_and_angle_sdf(found, pr.x, pr.y, pr.z, voxels, table, nb, lx, ly, lz, nx, ny, nz, angle);
  switch (type) {
  case B200_RENDER_COLOUR_FROM_VOLUME:
    *px = found ? draw_colour(voxels, table, nb, pr.x, pr.y, pr.z) : make_uchar4(0, 0, 0, 255);
    break;
  case B200_RENDER_COLOUR_FROM_NORMAL:
    if (found) {   // drawPixelNormal :283-288 leaves alpha untouched
      uchar4 o = *px;
      o.x = (unsigned char)((0.3f + (-nx + 1.0f) * 0.35f) * 255.0f);
      o.y = (unsigned char)((0.3f + (-ny + 1.0f) * 0.35f) * 255.0f);
      o.z = (unsigned char)((0.3f + (-nz + 1.0f) * 0.35f) * 255.0f);
      *px = o;
    } else *px = make_uchar4(0, 0, 0, 0);
    break;
  case B200_RENDER_COLOUR_FROM_DEPTH_WEIGHT:
    if (found) {   // drawPixelWeight :322-383
      uchar4 dest = draw_colour(voxels, table, nb, pr.x, pr.y, pr.z);
      IdxCache c; cache_init(c);
      const int ix = (int)pr.x, iy = (int)pr.y, iz = (int)pr.z;
      const int vi = voxel_index(table, nb, ix, iy, iz, c);
      const int wd = vi >= 0 ? (int)((__ldg(reinterpret_cast<const unsigned *>(voxels + vi)) >> 16) & 0xff) : 0;
      const unsigned char intensity = (unsigned char)(255.0f * (((float)wd) / maxW));
      const int blockIdx_ = find_block<false>(table, nb, floordiv8(ix), floordiv8(iy), floordiv8(iz));
      uchar4 ov;
      if (blockIdx_ < 0) ov = make_uchar4(255, 255, 255, 255);
      else if (wd <= 2) ov = make_uchar4(255, 0, 0, 255);
      else if (wd == maxW) ov = make_uchar4(0, 0, 255, 255);
      else ov = make_uchar4(intensity, intensity, intensity, 255);
      const float overlayWeight = 1.0f;
      const float a = (float)(1.0 - overlayWeight);
      dest.x = (unsigned char)(((float)dest.x * a) + ((float)ov.x * overlayWeight));
      dest.y = (unsigned char)(((float)dest.y * a) + ((float)ov.y * overlayWeight));
      dest.z = (unsigned char)(((float)dest.z * a) + ((float)ov.z * overlayWeight));
      dest.w = (unsigned char)(((float)dest.w * a) + ((float)ov.w * overlayWeight));
      *px = dest;
    } else *px = make_uchar4(0, 0, 0, 0);
    break;
  default:
    *px = found ? grey_px(angle) : make_uchar4(0, 0, 0, 0);
    break;
  }
}
