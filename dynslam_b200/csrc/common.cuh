// common.cuh — shared PODs, canonical float arithmetic and device helpers of libb200fusion.
//
// Arithmetic contract: every floating-point expression on the path is evaluated in IEEE binary32
// in exactly the operation order of the reference's DeviceAgnostic code (and therefore of
// oracle/tsdf_oracle.c); the library is compiled with -fmad=false and the default
// -prec-div=true -prec-sqrt=true, so results are bit-identical to the CPU oracle, not merely
// within the 1e-5 tolerance north_star asks for. (The reference's own CUDA build uses
// --use_fast_math, ITMLib/CMakeLists.txt:230, which is why it cannot serve as a bit-exact oracle.)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/b200fusion.h"

#define BS 8
#define BS3 512

#define HD __host__ __device__ __forceinline__
#define DEV __device__ __forceinline__

// ---- OR/MathUtils.h:5-23 -------------------------------------------------------------------
HD float minf_(float a, float b) { return (a < b) ? a : b; }
HD float maxf_(float a, float b) { return (a < b) ? b : a; }
HD int mini_(int a, int b) { return (a < b) ? a : b; }
HD float round_(float x) { return (x < 0) ? (x - 0.5f) : (x + 0.5f); }
HD int clampi_(int x, int a, int b) { int t = (b < x) ? b : x; return (a < t) ? t : a; }

struct Mat4 { float m[16]; };   // m[col*4+row], OR/Matrix.h:23-33
struct Vec4 { float x, y, z, w; };
struct Vec3 { float x, y, z; };

// OR/Matrix.h:115-122
HD Vec4 m4v4(const Mat4 &M, float x, float y, float z, float w) {
  Vec4 r;
  r.x = M.m[0] * x + M.m[4] * y + M.m[8] * z + M.m[12] * w;
  r.y = M.m[1] * x + M.m[5] * y + M.m[9] * z + M.m[13] * w;
  r.z = M.m[2] * x + M.m[6] * y + M.m[10] * z + M.m[14] * w;
  r.w = M.m[3] * x + M.m[7] * y + M.m[11] * z + M.m[15] * w;
  return r;
}

// DA/ITMRepresentationAccess.h:10-12
HD int hash_index(int x, int y, int z, int mask) {
  return (int)((((unsigned)x * 73856093u) ^ ((unsigned)y * 19349669u) ^ ((unsigned)z * 83492791u)) & (unsigned)mask);
}

HD int floordiv8(int p) { return ((p < 0) ? p - BS + 1 : p) / BS; }

// ---- hash entry access: 20-byte AoS, 4-byte aligned -> 32-bit words -------------------------
struct Entry { int x, y, z, offset, ptr; };

DEV Entry load_entry(const b200_hash_entry *table, int idx) {
  const int *p = reinterpret_cast<const int *>(table) + (size_t)idx * 5;
  int w0 = __ldg(p), w1 = __ldg(p + 1);
  Entry e;
  e.x = (short)(w0 & 0xffff); e.y = (short)(w0 >> 16); e.z = (short)(w1 & 0xffff);
  e.offset = __ldg(p + 2); e.ptr = __ldg(p + 3);
  return e;
}
// volatile-free but non-__ldg variant for kernels that also write the table (within one CTA: L1 is written through)
DEV Entry load_entry_rw(const b200_hash_entry *table, int idx) {
  const int *p = reinterpret_cast<const int *>(table) + (size_t)idx * 5;
  int w0 = p[0], w1 = p[1];
  Entry e;
  e.x = (short)(w0 & 0xffff); e.y = (short)(w0 >> 16); e.z = (short)(w1 & 0xffff);
  e.offset = p[2]; e.ptr = p[3];
  return e;
}

// L2 variant for entries OTHER CTAs of the same launch may have written (an L1 line fetched earlier in the launch would be stale)
DEV Entry load_entry_cg(const b200_hash_entry *table, int idx) {
  const int *p = reinterpret_cast<const int *>(table) + (size_t)idx * 5;
  int w0 = __ldcg(p), w1 = __ldcg(p + 1);
  Entry e;
  e.x = (short)(w0 & 0xffff); e.y = (short)(w0 >> 16); e.z = (short)(w1 & 0xffff);
  e.offset = __ldcg(p + 2); e.ptr = __ldcg(p + 3);
  return e;
}
DEV int find_block_cg(const b200_hash_entry *table, int numBuckets, int x, int y, int z, int *ptrOut) {
  int idx = hash_index(x, y, z, numBuckets - 1);
  for (;;) {
    const Entry e = load_entry_cg(table, idx);
    if (e.x == x && e.y == y && e.z == z && e.ptr >= 0) { *ptrOut = e.ptr; return idx; }
    if (e.offset < 1) break;
    idx = numBuckets + e.offset - 1;
  }
  return -1;
}

// findBlock — DA/ITMRepresentationAccess.h:62-85; -1 when absent
template <bool RW>
DEV int find_block(const b200_hash_entry *table, int numBuckets, int x, int y, int z, int *ptrOut = nullptr) {
  int idx = hash_index(x, y, z, numBuckets - 1);
  for (;;) {
    Entry e = RW ? load_entry_rw(table, idx) : load_entry(table, idx);
    if (e.x == x && e.y == y && e.z == z && e.ptr >= 0) { if (ptrOut) *ptrOut = e.ptr; return idx; }
    if (e.offset < 1) break;
    idx = numBuckets + e.offset - 1;
  }
  return -1;
}

// ---- device-resident counters (mirrored to pinned host memory by the engine) ----------------
// tile tickets of the kernels whose CTAs wait on one another (draw_tile), one counter each
enum { TK_SERVE, TK_SERVE_DEFERRED, TK_FREEVIEW, TK_DECAY_RANK, TK_MESH_LIST, TK_MESH_BLOCKS, TK_CK_CLASSIFY, TK_SWAP_LIST,
       TK_FWD_MISSING, TK_POINT_CLOUD, TK_COUNT };
struct DevCounters {
  int lastFreeBlockId;
  int lastFreeExcessListId;
  int noVisibleBlocks;
  int allocBaseVba;        // lastFreeBlockId before this frame's requests
  int allocBaseExl;
  int noRequests;
  int noRequestsExcess;
  int noIntegrated;
  int decayItems;          // number of list items of the decay pass in flight
  int decayDeleted;        // unique blocks deleted by the pass
  int freedLastDecay;
  int decayCand;           // partial decay: items that found their block empty this pass (candidates, unordered)
  unsigned decayCtasDone;  // partial decay: CTAs of the sweep that have finished (the last one commits the pass)
  int droppedSnapshots;    // decay: snapshots found overwritten in the ring when their turn came (swept as empty)
  unsigned noRenderingBlocks;
  unsigned visCtasDone;    // k_serve_list: CTAs that have finished (the last one applies the rendering-block cap if needed)
  unsigned depthCtasDone;  // k_expected_depths: the same for the stand-alone CreateExpectedDepths
  unsigned ticket[TK_COUNT];   // next tile to hand out, per kernel (draw_tile; reset by each launch's last draw)
  unsigned tilesRanked;    // k_serve_list, CTA-owned tiles: tiles that have published their request counts
  unsigned tilesWithExcess, tilesExcessServed;   // ... of which have excess-list requests / have served them (excess-part tiles list only after all have)
  unsigned tilesServed;    // k_serve_list, ticketed tiles: tiles that have ranked and served their requests
  unsigned tilesListed;    // both forms: tiles that have written their part of the visible list (the per-entry phase starts when all have)
  int anyExcessRequest;    // set by the marking kernel when it files an excess-list request; cleared by k_serve_list's last CTA
  int noNeededEntries;     // swapping
  unsigned noTotalPoints;
  int noFwdMissing;
  long long ringHead;      // device-side bump cursor of the decay ring (items)
  long long totalDecayed;  // GetDecayedBlockCount, Reco_CUDA.cu:563-566
  long long totalIntegrated; // cumulative blocks integrated (never reset; bench reads deltas)
  int integCursor;         // k_integrate_v3: next visible-list item to hand out (dynamic distribution over the persistent grid)
  int integDone;           // k_integrate_v3: CTAs that have stopped claiming; the last one zeroes both for the next launch
  long long decayReplays;  // partial decay, cumulative: flagged blocks whose reset stores k_decay_commit replayed after the rays
};

// ---- tile hand-out for kernels whose CTAs wait on one another --------------------------------
// A CTA that waits on another CTA (a chained scan's look-back, a device-wide counter) waits only on work that a running CTA has
// already claimed. Tiles are therefore drawn from a ticket counter, never owned by blockIdx: tile t is claimed only after tiles
// 0 .. t-1 have been, each by a CTA that is running and that waits, in turn, only on lower tiles, so the grid need not be
// resident all at once (other engines' kernels on the same GPU, or a grid larger than the GPU holds: b200_diag_set_grid_scale).
// Every CTA draws until it gets a ticket past the last tile, so each CTA draws exactly one such ticket and draw
// noTiles + gridDim.x - 1 is the launch's last: the CTA that makes it resets the counter for the next launch. Called by every
// thread of the CTA, after the kernel's pdl_wait(); all CTAs pass the same noTiles. Returns the tile (>= noTiles: none left).
DEV int draw_tile(unsigned *ticket, int noTiles, int *slot /* __shared__ */) {
  __syncthreads();                     // every thread has read the previous draw
  if (threadIdx.x == 0) {
    const unsigned t = atomicAdd(ticket, 1u);
    if (t == (unsigned)noTiles + gridDim.x - 1) *ticket = 0;
    *slot = (int)t;
  }
  __syncthreads();
  return *slot;
}

// ---- chained-scan (decoupled look-back) for ordered compaction --------------------------------
// Tiles come from draw_tile, so every predecessor tile is owned by a CTA that is running.
// Descriptor: [63:34] generation (30 bit) | [33:32] status (1 = aggregate, 2 = inclusive prefix) |
// [31:0] value. A fresh generation per launch makes resets unnecessary.
DEV unsigned long long scan_pack(unsigned gen, unsigned status, unsigned value) {
  return ((unsigned long long)(gen & 0x3fffffffu) << 34) | ((unsigned long long)status << 32) | value;
}

// Called by all threads of warp 0 of the CTA. Returns the exclusive prefix of tile `tile`
// (valid in all lanes of warp 0).
DEV unsigned scan_lookback(unsigned long long *desc, unsigned gen, int tile, unsigned aggregate) {
  const int lane = threadIdx.x & 31;
  volatile unsigned long long *vdesc = desc;
  if (tile == 0) {
    if (lane == 0) { vdesc[0] = scan_pack(gen, 2, aggregate); }
    return 0;
  }
  if (lane == 0) { vdesc[tile] = scan_pack(gen, 1, aggregate); }
  unsigned exclusive = 0;
  int look = tile - 1;
  for (;;) {
    int t = look - lane;
    unsigned long long d = 0;
    unsigned status = 0;
    if (t >= 0) {
      d = vdesc[t];
      if ((unsigned)(d >> 34) == (gen & 0x3fffffffu)) status = (unsigned)(d >> 32) & 3u;
    } else status = 3; // out of range: treat as "prefix 0" sentinel
    // every tile between this one and the nearest published inclusive prefix must be published
    const unsigned validMask = __ballot_sync(0xffffffffu, status != 0);
    const unsigned prefixMask = __ballot_sync(0xffffffffu, status >= 2);
    const int firstPrefix = prefixMask ? (__ffs(prefixMask) - 1) : 32;
    const unsigned need = (firstPrefix >= 32) ? 0xffffffffu : ((1u << firstPrefix) - 1u);
    if ((validMask & need) != need) continue;   // spin (volatile re-read)
    unsigned v = (lane <= firstPrefix && t >= 0) ? (unsigned)(d & 0xffffffffu) : 0u;
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    exclusive += v;
    if (prefixMask) break;
    look -= 32;
  }
  if (lane == 0) { __threadfence(); vdesc[tile] = scan_pack(gen, 2, exclusive + aggregate); }
  return exclusive;
}

// block-wide exclusive scan of one unsigned per thread; returns exclusive prefix, *total = block sum.
// smem must hold 33 unsigned.
DEV unsigned block_exclusive_scan(unsigned v, unsigned *smem, unsigned *total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = (blockDim.x + 31) >> 5;
  unsigned inc = v;
  for (int o = 1; o < 32; o <<= 1) { unsigned n = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += n; }
  if (lane == 31) smem[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    unsigned w = (lane < nwarps) ? smem[lane] : 0;
    unsigned winc = w;
    for (int o = 1; o < 32; o <<= 1) { unsigned n = __shfl_up_sync(0xffffffffu, winc, o); if (lane >= o) winc += n; }
    smem[lane] = winc - w;
    if (lane == 31) smem[32] = winc;
  }
  __syncthreads();
  unsigned res = smem[warp] + inc - v;
  *total = smem[32];
  __syncthreads();
  return res;
}

// 128-bit streaming accesses for voxel payloads (8 B voxels -> 2 per access)
DEV uint4 ld_stream(const uint4 *p) {
  uint4 r;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
  return r;
}
DEV void st_stream(uint4 *p, uint4 v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// Programmatic dependent launch (Hopper griddepcontrol). The rules every kernel of the fused frame's chain keeps are written at
// launch_chained (engine.h). In a grid launched without the programmatic attribute both instructions are no-ops.
DEV void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
DEV void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

DEV unsigned long long global_timer() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }

// Span of one launch in %globaltimer nanoseconds (b200_set_timing modes 2 and 4): span[0] = ~(earliest stamp at a CTA's entry,
// taken after its pdl_wait), span[1] = latest stamp at a warp's exit. The complement lets one zero-filled slot take both as
// atomicMax. span == nullptr: nothing is stamped. Constructed by thread 0 of a CTA for the entry; destroyed by every thread,
// lane 0 of each warp stamps when its warp leaves the scope (early returns included).
struct SpanStamp {
  unsigned long long *span;
  DEV explicit SpanStamp(unsigned long long *s) : span(s) {
    if (span && threadIdx.x == 0) atomicMax(span, ~global_timer());
  }
  DEV ~SpanStamp() {
    if (span && (threadIdx.x & 31) == 0) atomicMax(span + 1, global_timer());
  }
};

// positive-float atomic min/max through the order-preserving int view (all values here are > 0)
DEV void atomic_min_posf(float *a, float v) { atomicMin(reinterpret_cast<int *>(a), __float_as_int(v)); }
DEV void atomic_max_posf(float *a, float v) { atomicMax(reinterpret_cast<int *>(a), __float_as_int(v)); }

// ------------------------------------------------------------------------------------------------
// visibility test (DA/ITMSceneReconstructionEngine.h:315-397): alloc.cu's sweeps and FindVisibleBlocks (vis.cu)
// ------------------------------------------------------------------------------------------------
DEV bool point_visible(const Mat4 &M, const float *proj, float x, float y, float z, int w, int h) {
  Vec4 b = m4v4(M, x, y, z, 1.0f);
  if (b.z < 1e-10f) return false;
  float u = proj[0] * b.x / b.z + proj[2];
  float v = proj[1] * b.y / b.z + proj[3];
  return (u >= 0 && u < w && v >= 0 && v < h);
}

// checkBlockVisibility<false>: corner order and the incremental +=/-= updates are part of the arithmetic contract
__device__ inline bool block_visible(int bx, int by, int bz, const Mat4 &M, const float *proj, float voxelSize, int w, int h) {
  const float factor = (float)BS * voxelSize;
  float x = (float)bx * factor, y = (float)by * factor, z = (float)bz * factor;
  if (point_visible(M, proj, x, y, z, w, h)) return true;
  z += factor; if (point_visible(M, proj, x, y, z, w, h)) return true;
  y += factor; if (point_visible(M, proj, x, y, z, w, h)) return true;
  x += factor; if (point_visible(M, proj, x, y, z, w, h)) return true;
  z -= factor; if (point_visible(M, proj, x, y, z, w, h)) return true;
  y -= factor; if (point_visible(M, proj, x, y, z, w, h)) return true;
  x -= factor; y += factor; if (point_visible(M, proj, x, y, z, w, h)) return true;
  x += factor; y -= factor; z += factor; if (point_visible(M, proj, x, y, z, w, h)) return true;
  return false;
}

// ------------------------------------------------------------------------------------------------
// expected depths: block projection shared by vis.cu (k_expected_depths) and alloc.cu (k_serve_list)
// ------------------------------------------------------------------------------------------------
// ProjectSingleBlock — DA/ITMVisualisationEngine.h:29-71
DEV bool project_single_block(int bx, int by, int bz, const Mat4 &pose, const float *intr, int w, int h, float voxelSize,
                              int &ulx, int &uly, int &lrx, int &lry, float &zmin, float &zmax) {
  ulx = w / B200_MINMAX_SUBSAMPLE; uly = h / B200_MINMAX_SUBSAMPLE;
  lrx = -1; lry = -1;
  zmin = B200_FAR_AWAY; zmax = B200_VERY_CLOSE;
#pragma unroll
  for (int corner = 0; corner < 8; ++corner) {
    const short tx = (short)(bx + ((corner & 1) ? 1 : 0)), ty = (short)(by + ((corner & 2) ? 1 : 0)), tz = (short)(bz + ((corner & 4) ? 1 : 0));
    Vec4 q = m4v4(pose, (float)tx * (float)BS * voxelSize, (float)ty * (float)BS * voxelSize, (float)tz * (float)BS * voxelSize, 1.0f);
    if (q.z < 1e-6) continue;
    const float px = (intr[0] * q.x / q.z + intr[2]) / B200_MINMAX_SUBSAMPLE;
    const float py = (intr[1] * q.y / q.z + intr[3]) / B200_MINMAX_SUBSAMPLE;
    if (ulx > floorf(px)) ulx = (int)floorf(px);
    if (lrx < ceilf(px)) lrx = (int)ceilf(px);
    if (uly > floorf(py)) uly = (int)floorf(py);
    if (lry < ceilf(py)) lry = (int)ceilf(py);
    if (zmin > q.z) zmin = q.z;
    if (zmax < q.z) zmax = q.z;
  }
  if (ulx < 0) ulx = 0;
  if (uly < 0) uly = 0;
  if (lrx >= w) lrx = w - 1;
  if (lry >= h) lry = h - 1;
  if (ulx > lrx) return false;
  if (uly > lry) return false;
  if (zmin < B200_VERY_CLOSE) zmin = B200_VERY_CLOSE;
  if (zmax < B200_VERY_CLOSE) return false;
  return true;
}


// ProjectSingleBlock for an 8-lane group: lane (lane & 7) projects corner (lane & 7) of block (ex, ey, ez), the min / max over the
// corners are taken with shuffles (min and max do not depend on the order; NaNs are skipped by fminf / fmaxf exactly as the
// serial comparisons skip them), then every lane applies the function's bookkeeping. All 32 lanes of the warp must call it;
// `have` (group-uniform) says whether the group has a block at all. Returns whether the block is drawn (all 8 lanes agree).
DEV bool project_block_group(bool have, int ex, int ey, int ez, const Mat4 &M, const float *proj, int rw, int rh, float voxelSize,
                             int &ulx, int &uly, int &lrx, int &lry, float &zl, float &zh) {
  const int sub = threadIdx.x & 7;
  float fxl = 3.0e38f, fxh = -3.0e38f, fyl = 3.0e38f, fyh = -3.0e38f;
  zl = B200_FAR_AWAY; zh = B200_VERY_CLOSE;
  if (have) {
    const short tx = (short)(ex + (sub & 1)), ty = (short)(ey + ((sub >> 1) & 1)), tz = (short)(ez + (sub >> 2));
    const Vec4 q = m4v4(M, (float)tx * (float)BS * voxelSize, (float)ty * (float)BS * voxelSize, (float)tz * (float)BS * voxelSize, 1.0f);
    if (!(q.z < 1e-6)) {
      const float px = (proj[0] * q.x / q.z + proj[2]) / B200_MINMAX_SUBSAMPLE;
      const float py = (proj[1] * q.y / q.z + proj[3]) / B200_MINMAX_SUBSAMPLE;
      fxl = floorf(px); fxh = ceilf(px); fyl = floorf(py); fyh = ceilf(py);
      zl = fminf(zl, q.z); zh = fmaxf(zh, q.z);
    }
  }
#pragma unroll
  for (int d = 1; d < 8; d <<= 1) {
    fxl = fminf(fxl, __shfl_xor_sync(0xffffffffu, fxl, d)); fxh = fmaxf(fxh, __shfl_xor_sync(0xffffffffu, fxh, d));
    fyl = fminf(fyl, __shfl_xor_sync(0xffffffffu, fyl, d)); fyh = fmaxf(fyh, __shfl_xor_sync(0xffffffffu, fyh, d));
    zl = fminf(zl, __shfl_xor_sync(0xffffffffu, zl, d)); zh = fmaxf(zh, __shfl_xor_sync(0xffffffffu, zh, d));
  }
  // the function's bookkeeping on the reduced values (ulx starts at w/8, lrx at -1; then the clamps and the early outs)
  ulx = rw / B200_MINMAX_SUBSAMPLE; uly = rh / B200_MINMAX_SUBSAMPLE; lrx = -1; lry = -1;
  if ((float)ulx > fxl) ulx = (int)fxl;
  if ((float)lrx < fxh) lrx = (int)fxh;
  if ((float)uly > fyl) uly = (int)fyl;
  if ((float)lry < fyh) lry = (int)fyh;
  if (ulx < 0) ulx = 0;
  if (uly < 0) uly = 0;
  if (lrx >= rw) lrx = rw - 1;
  if (lry >= rh) lry = rh - 1;
  bool draw = have && !(ulx > lrx) && !(uly > lry);
  if (zl < B200_VERY_CLOSE) zl = B200_VERY_CLOSE;
  if (zh < B200_VERY_CLOSE) draw = false;
  return draw;
}

// rasterises [ax..bx] x [ay..by] into the expected-depth image: by the 8 lanes of a group (no divisions) ...
DEV void raster_box_group(float2 *minmax, int rw, int ax, int ay, int bx, int by, float zn, float zx) {
  const int sub = threadIdx.x & 7, bw = bx - ax + 1;
  int xx = ax + sub, yy = ay;
  while (xx > bx) { xx -= bw; ++yy; }
  while (yy <= by) {
    float2 *pxl = &minmax[xx + yy * rw];
    atomic_min_posf(&pxl->x, zn); atomic_max_posf(&pxl->y, zx);
    xx += 8;
    while (xx > bx) { xx -= bw; ++yy; }
  }
}
// ... or by one warp
DEV void raster_box_warp(float2 *minmax, int rw, int ax, int ay, int bx, int by, float zn, float zx) {
  const int lane = threadIdx.x & 31;
  const int bw = bx - ax + 1;
  if (bw <= 32) {
    const int rpi = 32 / bw, inv = (65536 + bw - 1) / bw;          // warp-uniform; rows per iteration, magic number of lane / bw
    const int r = (lane * inv) >> 16, c = lane - r * bw;
    for (int y0 = ay; y0 <= by; y0 += rpi) {
      const int yy = y0 + r;
      if (r < rpi && yy <= by) { float2 *px = &minmax[(ax + c) + yy * rw]; atomic_min_posf(&px->x, zn); atomic_max_posf(&px->y, zx); }
    }
  } else {
    for (int yy = ay; yy <= by; ++yy)
      for (int xx = ax + lane; xx <= bx; xx += 32) { float2 *px = &minmax[xx + yy * rw]; atomic_min_posf(&px->x, zn); atomic_max_posf(&px->y, zx); }
  }
}

// one visible block's 1/8-resolution bounding box + depth range (an undrawn block has ulx > lrx)
struct __align__(16) BlockRec { short ulx, uly, lrx, lry; float zmin, zmax; };

DEV unsigned rendering_tiles(int ulx, int uly, int lrx, int lry) {   // CreateRenderingBlocks' count, DA/ITMVisualisationEngine.h:73-91
  const int rx = (int)ceilf((float)(lrx - ulx + 1) / 16), ry = (int)ceilf((float)(lry - uly + 1) / 16);
  return (unsigned)(rx * ry);
}
