// mesh.cu — marching-cubes meshing of the voxel-hashed TSDF for sm_90a (SURVEY.md 8(f) rank 4: the step after the path).
//
// Replaces ITMMeshingEngine_CUDA<TVoxel, ITMVoxelBlockHash>::MeshScene (reference
// Engine/DeviceSpecific/CUDA/ITMMeshingEngine_CUDA.cu:37-81: findAllocatedBlocks :96-114 + meshScene_device :117-169) with the
// per-cell functions of DeviceAgnostic/ITMMeshingEngine.h:120-231 (findPointNeighbors, sdfInterp, buildVertList) and the colour
// read readFromSDF_color4u_interpolated_noalpha (DeviceAgnostic/ITMRepresentationAccess.h:280-318).
//
// The reference's CUDA kernel appends triangles with atomicAdd, so its output order changes from run to run; its CPU twin
// (Engine/DeviceSpecific/CPU/ITMMeshingEngine_CPU.cpp:19-80) is serial: ascending hash-entry index, then z, y, x, then the case
// table's order. That is the canonical order here, reproduced exactly (the OBJ a maintainer writes from it is byte-identical):
//   1. k_mesh_list: ordered compaction of the entries with ptr >= 0 (one chained scan over the table);
//   2. k_mesh_blocks: one CTA pass per allocated block, one thread per cell: case index and triangle count, block-wide exclusive
//      scan in cell order (x + 8y + 64z == the z, y, x loops), chained look-back over the blocks for the global offset, then the
//      triangles are written at their final positions — a single pass over the volume, no counters to read back in between.
// Cap: like the CUDA reference, a triangle whose index reaches noMaxTriangles - 1 is dropped and noTotalTriangles reports what
// was generated (ITMMesh::WriteOBJ refuses a mesh with more than noMaxTriangles).
// Arithmetic: IEEE binary32 in the reference's operation order (the library is built without contraction), so vertices and
// colours are bit-identical to the CPU engine's — tests/test_gpu_mesh.py compares with the oracle, tests/test_oracle_vs_ref.py
// pins the oracle to the reference's ITMMeshingEngine_CPU compiled from its own source.
#include "engine.h"
#include "raycast_ray.cuh"
#include "mc_tables.cuh"

namespace {

struct V3 { float x, y, z; };

// readVoxel(...).sdf as SDF_valueToFloat would return it, and whether the voxel's block exists (DA/ITMRepresentationAccess.h:176-220)
DEV bool corner(const b200_voxel *__restrict__ voxels, const b200_hash_entry *__restrict__ table, int nb, int x, int y, int z, IdxCache &c,
                float &sdf) {
  const int vi = voxel_index(table, nb, x, y, z, c);
  if (vi < 0) return false;
  sdf = (float)__ldg(reinterpret_cast<const short *>(voxels + vi)) / 32767.0f;
  return sdf != 1.0f;
}

// sdfInterp — DA/ITMMeshingEngine.h:176-183
DEV V3 sdf_interp_edge(const V3 &p1, const V3 &p2, float v1, float v2) {
  if (fabsf(0.0f - v1) < 0.00001f) return p1;
  if (fabsf(0.0f - v2) < 0.00001f) return p2;
  if (fabsf(v1 - v2) < 0.00001f) return p1;
  const float t = (0.0f - v1) / (v2 - v1);
  V3 r; r.x = p1.x + t * (p2.x - p1.x); r.y = p1.y + t * (p2.y - p1.y); r.z = p1.z + t * (p2.z - p1.z);
  return r;
}

// findPointNeighbors + the case index of buildVertList (:120-174, :185-231); -1 = no triangles
DEV int cell_case(const b200_voxel *__restrict__ voxels, const b200_hash_entry *__restrict__ table, int nb, int gx, int gy, int gz, float *sdf) {
  IdxCache c; cache_init(c);
  // corner order of the reference: (0,0,0) (1,0,0) (1,1,0) (0,1,0) (0,0,1) (1,0,1) (1,1,1) (0,1,1)
  const int ox[8] = {0, 1, 1, 0, 0, 1, 1, 0}, oy[8] = {0, 0, 1, 1, 0, 0, 1, 1}, oz[8] = {0, 0, 0, 0, 1, 1, 1, 1};
  int cube = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    if (!corner(voxels, table, nb, gx + ox[k], gy + oy[k], gz + oz[k], c, sdf[k])) return -1;
    if (sdf[k] < 0) cube |= 1 << k;
  }
  return MC_EDGE_MASK[cube] == 0 ? -1 : cube;
}

// readFromSDF_color4u_interpolated_noalpha — DA/ITMRepresentationAccess.h:280-318
DEV V3 colour_at(const b200_voxel *__restrict__ voxels, const b200_hash_entry *__restrict__ table, int nb, const V3 &p) {
  IdxCache c; cache_init(c);
  const float fx = floorf(p.x), fy = floorf(p.y), fz = floorf(p.z);
  const float cx = p.x - fx, cy = p.y - fy, cz = p.z - fz;
  const int X = (int)fx, Y = (int)fy, Z = (int)fz;
  float r0 = 0.0f, r1 = 0.0f, r2 = 0.0f;
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
  V3 r; r.x = r0 / 255.0f; r.y = r1 / 255.0f; r.z = r2 / 255.0f;
  return r;
}

// 1. allocated entries in ascending index order
#define ML_EPT 16
#define ML_TILE (256 * ML_EPT)
__global__ void __launch_bounds__(256)
k_mesh_list(const b200_hash_entry *__restrict__ table, int noTotal, int *list, int capacity, unsigned *count, unsigned long long *scanDesc, unsigned gen,
            unsigned *ticket) {
  __shared__ unsigned sm[33];
  __shared__ unsigned tileBase;
  __shared__ int sTile;
  const int noTiles = (noTotal + ML_TILE - 1) / ML_TILE;
  for (int tile = draw_tile(ticket, noTiles, &sTile); tile < noTiles; tile = draw_tile(ticket, noTiles, &sTile)) {
    const int first = tile * ML_TILE + threadIdx.x * ML_EPT;
    unsigned mask = 0;
#pragma unroll
    for (int k = 0; k < ML_EPT; ++k)
      if (first + k < noTotal && __ldg(reinterpret_cast<const int *>(table) + (size_t)(first + k) * 5 + 3) >= 0) mask |= 1u << k;
    unsigned total;
    const unsigned local = block_exclusive_scan(__popc(mask), sm, &total);
    if (threadIdx.x < 32) {
      const unsigned ex = scan_lookback(scanDesc, gen, tile, total);
      if (threadIdx.x == 0) { tileBase = ex; if (tile == noTiles - 1) *count = ex + total; }
    }
    __syncthreads();
    unsigned o = tileBase + local;
    while (mask) {
      const int k = __ffs(mask) - 1;
      mask &= mask - 1;
      if ((int)o < capacity) list[o] = first + k;
      o++;
    }
  }
}

// 2. one allocated block per tile, one cell per thread
__global__ void __launch_bounds__(512)
k_mesh_blocks(const b200_voxel *__restrict__ voxels, const b200_hash_entry *__restrict__ table, int nb, const int *__restrict__ list,
              const unsigned *__restrict__ listCount, int capacity, float factor, b200_triangle *triangles, unsigned noMaxTriangles,
              unsigned *noTotalTriangles, unsigned long long *scanDesc, unsigned gen, unsigned *ticket) {
  __shared__ unsigned sm[33];
  __shared__ unsigned tileBase;
  __shared__ int sTile;
  unsigned n = *listCount;
  if (n > (unsigned)capacity) n = (unsigned)capacity;
  if (n == 0) { if (blockIdx.x == 0 && threadIdx.x == 0) *noTotalTriangles = 0; return; }
  const int x = threadIdx.x & 7, y = (threadIdx.x >> 3) & 7, z = threadIdx.x >> 6;
  for (unsigned tile = draw_tile(ticket, (int)n, &sTile); tile < n; tile = draw_tile(ticket, (int)n, &sTile)) {
    const Entry en = load_entry(table, list[tile]);
    const int gx = en.x * BS + x, gy = en.y * BS + y, gz = en.z * BS + z;
    float sdf[8];
    const int cube = cell_case(voxels, table, nb, gx, gy, gz, sdf);
    unsigned long long tri = cube >= 0 ? MC_TRIANGLES[cube] : ~0ull;
    unsigned cnt = 0;
    for (unsigned long long t = tri; (t & 0xF) != 0xF; t >>= 12) cnt++;
    unsigned total;
    const unsigned local = block_exclusive_scan(cnt, sm, &total);
    if (threadIdx.x < 32) {
      const unsigned ex = scan_lookback(scanDesc, gen, (int)tile, total);
      if (threadIdx.x == 0) { tileBase = ex; if (tile == n - 1) *noTotalTriangles = ex + total; }
    }
    __syncthreads();
    if (cnt) {
      // buildVertList: the cell's corner positions (voxel units) and the interpolated crossing of every edge the case uses
      const int ox[8] = {0, 1, 1, 0, 0, 1, 1, 0}, oy[8] = {0, 0, 1, 1, 0, 0, 1, 1}, oz[8] = {0, 0, 0, 0, 1, 1, 1, 1};
      const int ea[12] = {0, 1, 2, 3, 4, 5, 6, 7, 0, 1, 2, 3}, eb[12] = {1, 2, 3, 0, 5, 6, 7, 4, 4, 5, 6, 7};
      V3 vert[12];
      const unsigned em = MC_EDGE_MASK[cube];
#pragma unroll
      for (int e = 0; e < 12; ++e) {
        if (!(em & (1u << e))) continue;
        V3 p1, p2;
        p1.x = (float)(gx + ox[ea[e]]); p1.y = (float)(gy + oy[ea[e]]); p1.z = (float)(gz + oz[ea[e]]);
        p2.x = (float)(gx + ox[eb[e]]); p2.y = (float)(gy + oy[eb[e]]); p2.z = (float)(gz + oz[eb[e]]);
        vert[e] = sdf_interp_edge(p1, p2, sdf[ea[e]], sdf[eb[e]]);
      }
      unsigned id = tileBase + local;
      for (; (tri & 0xF) != 0xF; tri >>= 12, ++id) {
        if (id >= noMaxTriangles - 1) continue;           // ITMMeshingEngine_CUDA.cu:139
        b200_triangle T;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const V3 p = vert[(tri >> (4 * k)) & 0xF];
          const V3 c = colour_at(voxels, table, nb, p);
          float *pp = k == 0 ? T.p0 : (k == 1 ? T.p1 : T.p2), *cc = k == 0 ? T.c0 : (k == 1 ? T.c1 : T.c2);
          pp[0] = p.x * factor; pp[1] = p.y * factor; pp[2] = p.z * factor;
          cc[0] = c.x; cc[1] = c.y; cc[2] = c.z;
        }
        triangles[id] = T;
      }
    }
  }
}

}  // namespace

void launch_mesh_scene(b200_engine *e, const SceneRef &s, float voxelSize, b200_triangle *triangles, unsigned noMaxTriangles) {
  unsigned *count = &e->d_ctr->noRenderingBlocks, *total = &e->d_ctr->noTotalPoints;   // scratch counters of calls that are never in flight together
  if (!e->d_meshDesc) {     // one chained-scan descriptor per allocated block (the shared descriptor array is sized for table tiles)
    if (cudaMalloc(&e->d_meshDesc, sizeof(unsigned long long) * (size_t)(e->numBlocks + 1)) != cudaSuccess) return;
    cudaMemsetAsync(e->d_meshDesc, 0, sizeof(unsigned long long) * (size_t)(e->numBlocks + 1), e->stream);
  }
  const int listTiles = (s.noTotal + ML_TILE - 1) / ML_TILE;
  k_mesh_list<<<ticket_grid(e, 4, listTiles), 256, 0, e->stream>>>(s.hash, s.noTotal, e->d_delList, s.numBlocks, count, e->d_scanDesc, ++e->scanGen,
                                                                    &e->d_ctr->ticket[TK_MESH_LIST]);
  k_mesh_blocks<<<ticket_grid(e, 2, s.numBlocks), 512, 0, e->stream>>>(s.voxels, s.hash, s.numBuckets, e->d_delList, count, s.numBlocks, voxelSize,
                                                                       triangles, noMaxTriangles, total, e->d_meshDesc, ++e->scanGen,
                                                                       &e->d_ctr->ticket[TK_MESH_BLOCKS]);
  e->launches += 2;
}
