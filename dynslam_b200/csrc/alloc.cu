// alloc.cu — ResetScene and AllocateSceneFromDepth for sm_90a.
//
// Replaces (reference, src/InfiniTAM/InfiniTAM/ITMLib/Engine/DeviceSpecific/CUDA/
// ITMSceneReconstructionEngine_CUDA.cu): memsetKernel/fillArrayKernel (:145-172), setToType3
// (:776-810), buildHashAllocAndVisibleType_device (:752-773 -> DeviceAgnostic/
// ITMSceneReconstructionEngine.h:176-313), allocateVoxelBlocksList_device (:812-905),
// buildVisibleList_device (:924-999) and the host-side visible-list snapshot (:302-317).
//
// Design (not a port): the reference resolves races with a 4 MiB lock array that is memset every
// frame, lets contended pixels skip ray steps, and hands out VBA slots with atomicSub, so its
// result differs run to run. Here every stage is deterministic and equal to the serial oracle:
//  * a request is a 64-bit atomicMax of (frame | pixel | step): the LAST pixel in raster order wins
//    the bucket, exactly as in the serial loop; the winner's block position is recomputed from
//    (pixel, step) when the request is served, so no 12 MB blockCoords array is written;
//  * requested entries are recorded in a 1-bit-per-entry bitmap; one prefix over the bitmap words
//    gives every request its rank in ascending entry order => slot = allocationList[lastFree - rank];
//  * the visible list is an ordered compaction (decoupled look-back scan over 32-entry/thread tiles
//    of the visibility bytes, 128-bit loads), not an atomicAdd of per-CTA group offsets;
//  * all counters stay on the device; nothing here synchronises with the host;
//  * the whole call is TWO launches (k_mark_prepare, k_serve_list) whose latency chains were what the frame paid for:
//    round 1 ran four (prepare, mark, serve, list: 11 + 19 + 15 + 26 us for ~50 new blocks and ~4.7 k listed ones).
#include "engine.h"

// ------------------------------------------------------------------------------------------------
// ResetScene
// ------------------------------------------------------------------------------------------------
__global__ void k_reset(uint4 *voxels16, size_t nVox16, int *allocList, int numBlocks, int *hashWords, size_t nHashWords,
                        int *excessList, int excessSize, DevCounters *ctr) {
  const size_t tid = blockIdx.x * (size_t)blockDim.x + threadIdx.x, nth = (size_t)gridDim.x * blockDim.x;
  // two voxels {sdf 32767, everything else 0} per 16 bytes
  const uint4 v = make_uint4(0x00007fffu, 0u, 0x00007fffu, 0u);
  for (size_t i = tid; i < nVox16; i += nth) st_stream(voxels16 + i, v);
  for (size_t i = tid; i < (size_t)numBlocks; i += nth) allocList[i] = (int)i;
  // entry = {pos 0, pad 0, offset 0, ptr -2, allocatedTime 0}: word 3 of every 5 is -2
  for (size_t i = tid; i < nHashWords; i += nth) hashWords[i] = ((i % 5) == 3) ? -2 : 0;
  for (size_t i = tid; i < (size_t)excessSize; i += nth) excessList[i] = (int)i;
  if (tid == 0) { ctr->lastFreeBlockId = numBlocks - 1; ctr->lastFreeExcessListId = excessSize - 1; ctr->totalDecayed = 0; }
}

void launch_reset(b200_engine *e, const SceneRef &s) {
  size_t nVox16 = (size_t)s.numBlocks * BS3 / 2;
  k_reset<<<e->smCount * 8, 256, 0, e->stream>>>((uint4 *)s.voxels, nVox16, s.allocationList, s.numBlocks, (int *)s.hash,
                                                (size_t)s.noTotal * 5, s.excessList, s.excessSize, e->d_ctr);
  e->launches++;
}

// ------------------------------------------------------------------------------------------------
// visibility test (DA/ITMSceneReconstructionEngine.h:315-397)
// ------------------------------------------------------------------------------------------------
DEV bool point_visible(const Mat4 &M, const float *proj, float x, float y, float z, int w, int h) {
  Vec4 b = m4v4(M, x, y, z, 1.0f);
  if (b.z < 1e-10f) return false;
  float u = proj[0] * b.x / b.z + proj[2];
  float v = proj[1] * b.y / b.z + proj[3];
  return (u >= 0 && u < w && v >= 0 && v < h);
}

// checkBlockVisibility<false>: corner order and the incremental +=/-= updates are part of the arithmetic contract
__device__ bool block_visible(int bx, int by, int bz, const Mat4 &M, const float *proj, float voxelSize, int w, int h) {
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

// Transient visibility codes, only alive between the two kernels of ONE allocate call: the reference marks every
// previously visible block 3 (setToType3) and re-tests the survivors' frustum visibility inside the full-table sweep.
// Here the re-test is done eagerly, one previously visible block per thread, and its verdict is parked in the byte; the
// sweep then only decodes it.
#define VT_PREV_VISIBLE 5   // was 3, frustum test passed  -> ends as 3 unless re-observed (1)
#define VT_PREV_HIDDEN 4    // was 3, frustum test failed  -> ends as 0 unless re-observed (1)

// ------------------------------------------------------------------------------------------------
// ray set-up shared by the marking kernel and by the request server (which replays one ray)
// ------------------------------------------------------------------------------------------------
struct Ray { float px, py, pz, dx, dy, dz; int noSteps; };

DEV bool make_ray(Ray &r, int x, int y, float d, const FrameGeom &g, float invfx, float invfy, float oneOverVoxelSize) {
  if (d <= 0 || (d - g.mu) < 0 || (d - g.mu) < g.vfmin || (d + g.mu) > g.vfmax) return false;
  float pz = d;
  float px = pz * (((float)x - g.proj_d[2]) * invfx);
  float py = pz * (((float)y - g.proj_d[3]) * invfy);
  float norm = sqrtf(px * px + py * py + pz * pz);
  Vec4 a = m4v4(g.invM_d, px * (1.0f - g.mu / norm), py * (1.0f - g.mu / norm), pz * (1.0f - g.mu / norm), 1.0f);
  float sx = a.x * oneOverVoxelSize, sy = a.y * oneOverVoxelSize, sz = a.z * oneOverVoxelSize;
  Vec4 b = m4v4(g.invM_d, px * (1.0f + g.mu / norm), py * (1.0f + g.mu / norm), pz * (1.0f + g.mu / norm), 1.0f);
  float ex = b.x * oneOverVoxelSize, ey = b.y * oneOverVoxelSize, ez = b.z * oneOverVoxelSize;
  float dx = ex - sx, dy = ey - sy, dz = ez - sz;
  norm = sqrtf(dx * dx + dy * dy + dz * dz);
  int noSteps = (int)ceilf(2.0f * norm);
  float den = (float)(noSteps - 1);
  r.px = sx; r.py = sy; r.pz = sz;
  r.dx = dx / den; r.dy = dy / den; r.dz = dz / den;
  r.noSteps = noSteps;
  return true;
}

#define KEY_PIXEL_BITS 24
#define KEY_STEP_BITS 16
DEV unsigned long long make_key(unsigned frameTag, unsigned pixel, unsigned step) {
  return ((unsigned long long)(frameTag & 0xffffffu) << (KEY_PIXEL_BITS + KEY_STEP_BITS)) |
         ((unsigned long long)pixel << KEY_STEP_BITS) | step;
}

// set a bit of a device-wide bitmap; the bit is read through L2 first (an L1 copy could stay stale for the whole launch
// and make every warp of the SM repeat the atomic), so in the steady state — the bit already set by an earlier warp —
// no atomic is issued at all
DEV void bitmap_set(unsigned *bits, int idx) {
  const unsigned bit = 1u << (idx & 31);
  if (!(__ldcg(bits + (idx >> 5)) & bit)) atomicOr(bits + (idx >> 5), bit);
}

// ------------------------------------------------------------------------------------------------
// kernel 1 of AllocateSceneFromDepth: marking (buildHashAllocAndVisibleTypePP) and, in the same launch on a few extra CTAs,
// everything that only depends on the PREVIOUS frame's list: setToType3 by position lookup with the eager frustum re-test,
// and the initialisation of the expected-depth image of the fused frame.
//
// The two parts do not touch the same state, so they need no ordering between them:
//  * marking reads the table and records what it saw on the side — `markBytes` (entry observed this frame, i.e. the
//    reference's entriesVisibleType = 1 / 2; plain idempotent byte stores: a bitmap would need an atomic per probe, measured
//    3x slower) and the request bitmaps `reqBits` / `req2Bits` + the 64-bit request key (rare) — and never writes the
//    visibility bytes;
//  * the prepare part writes the transient codes VT_PREV_* into the bytes of the previously visible entries.
// k_serve_list merges both (an entry observed this frame ends as 1 / 2 whatever its byte says) and clears the bitmaps it
// consumed, so nothing has to be reset at the start of a frame.
//
// Marking: one warp covers an 8x4 pixel tile (neighbouring rays probe the same buckets, so the 20-byte entry loads of a
// warp collapse to a few L1/L2 transactions). The ray's steps are independent probes: four bucket heads are fetched at a time
// before any of them is looked at, so a pixel pays two dependent table latencies instead of eight.
// ------------------------------------------------------------------------------------------------
#define MARK_BATCH 4
__global__ void __launch_bounds__(256)
k_mark_prepare(const float *__restrict__ depth, const b200_hash_entry *__restrict__ table, int numBuckets,
               const b200_vec3i *__restrict__ prevList, uint8_t *visType, DevCounters *ctr, unsigned long long *reqKey, unsigned *reqBits,
               unsigned *req2Bits, uint8_t *markBytes, const __grid_constant__ FrameGeom g, unsigned frameTag, int capacity, int prepCtas,
               float2 *minmax, int mw, int mh, unsigned tilesXMagic) {
  if ((int)blockIdx.x < prepCtas) {
    // ---- prepare part ----
    const int tid = blockIdx.x * blockDim.x + threadIdx.x, nth = prepCtas * blockDim.x;
    if (minmax) {
      // fused frame: k_serve_list rasterises every listed block's box into the expected-depth image with atomic min / max,
      // so the WHOLE image starts from (FAR_AWAY, VERY_CLOSE) here (Vis_CUDA.cu:204)
      if (tid == 0) ctr->noRenderingBlocks = 0;
      const int cells = mw * mh;
      if ((reinterpret_cast<uintptr_t>(minmax) & 15) == 0) {
        const float4 v2 = make_float4(B200_FAR_AWAY, B200_VERY_CLOSE, B200_FAR_AWAY, B200_VERY_CLOSE);
        float4 *m4 = reinterpret_cast<float4 *>(minmax);
        for (int i = tid; i < cells / 2; i += nth) m4[i] = v2;
        if ((cells & 1) && tid == 0) minmax[cells - 1] = make_float2(B200_FAR_AWAY, B200_VERY_CLOSE);
      } else {
        for (int i = tid; i < cells; i += nth) minmax[i] = make_float2(B200_FAR_AWAY, B200_VERY_CLOSE);
      }
    }
    int n = ctr->noVisibleBlocks;
    if (n > capacity) n = capacity;
    for (int i = tid; i < n; i += nth) {
      const b200_vec3i p = prevList[i];
      const int idx = find_block<false>(table, numBuckets, p.x, p.y, p.z);
      if (idx >= 0) visType[idx] = block_visible(p.x, p.y, p.z, g.M_d, g.proj_d, g.voxelSize, g.w, g.h) ? VT_PREV_VISIBLE : VT_PREV_HIDDEN;
    }
    return;
  }
  // ---- marking part ----
  const int tilesX = (g.w + 7) >> 3, tilesY = (g.h + 3) >> 2;
  const int warpGlobal = (((int)blockIdx.x - prepCtas) * blockDim.x + threadIdx.x) >> 5;
  if (warpGlobal >= tilesX * tilesY) return;
  const int lane = threadIdx.x & 31;
  const int tileY = (int)__umulhi((unsigned)warpGlobal, tilesXMagic);      // warpGlobal / tilesX (magic = ceil(2^32 / tilesX), exact for these sizes)
  const int x = (warpGlobal - tileY * tilesX) * 8 + (lane & 7), y = tileY * 4 + (lane >> 3);
  if (x >= g.w || y >= g.h) return;
  const float invfx = 1.0f / g.proj_d[0], invfy = 1.0f / g.proj_d[1];
  const float oneOverVoxelSize = 1.0f / (g.voxelSize * BS);
  Ray r;
  if (!make_ray(r, x, y, __ldg(depth + x + y * g.w), g, invfx, invfy, oneOverVoxelSize)) return;
  const unsigned pixel = (unsigned)(x + y * g.w);
  float px = r.px, py = r.py, pz = r.pz;
  int lastX = 0x7fffffff, lastY = 0, lastZ = 0;   // block of the previous step
  for (int i0 = 0; i0 < r.noSteps; i0 += MARK_BATCH) {
    int bx[MARK_BATCH], by[MARK_BATCH], bz[MARK_BATCH], hidx[MARK_BATCH];
    bool fresh[MARK_BATCH];
    Entry head[MARK_BATCH];
#pragma unroll
    for (int j = 0; j < MARK_BATCH; ++j) {
      fresh[j] = false;
      if (i0 + j < r.noSteps) {      // (a ray has two or three steps at the default band: the rest of the batch costs nothing)
        // (short)(int)floorf(p): cvt.rmi is floor and conversion in one instruction, same value
        bx[j] = (short)__float2int_rd(px); by[j] = (short)__float2int_rd(py); bz[j] = (short)__float2int_rd(pz);
        // A step is half a block long, so about every other step lands in the block of the step before: probing it again
        // would find (or request) the same entry — same mark, same request up to the step number in its key, which only
        // breaks ties between requests of the SAME pixel for the SAME block. Skipped.
        fresh[j] = !(bx[j] == lastX && by[j] == lastY && bz[j] == lastZ);
        lastX = bx[j]; lastY = by[j]; lastZ = bz[j];
        if (fresh[j]) { hidx[j] = hash_index(bx[j], by[j], bz[j], numBuckets - 1); head[j] = load_entry(table, hidx[j]); }
        px += r.dx; py += r.dy; pz += r.dz;     // the reference's own accumulation (DA/ITMSceneReconstructionEngine.h:311)
      }
    }
#pragma unroll
    for (int j = 0; j < MARK_BATCH; ++j) {
      if (!fresh[j]) continue;
      Entry he = head[j];
      int hashIdx = hidx[j];
      bool isFound = (he.x == bx[j] && he.y == by[j] && he.z == bz[j] && he.ptr >= -1);
      bool isExcess = false;
      if (!isFound && he.ptr >= -1) {
        while (he.offset >= 1) {
          hashIdx = numBuckets + he.offset - 1;
          he = load_entry(table, hashIdx);
          if (he.x == bx[j] && he.y == by[j] && he.z == bz[j] && he.ptr >= -1) { isFound = true; break; }
        }
        isExcess = true;
      }
      if (isFound) {
        markBytes[hashIdx] = 1;               // entriesVisibleType = 1 (2 when swapped out: k_serve_list reads the entry's ptr)
      } else {
        // Neighbouring rays miss the same block at the same step: the lanes of the warp that request the same entry elect
        // the one with the largest key (lane order == raster order inside the 8x4 tile, the step is warp-uniform) and only
        // that lane issues the atomics.
        const unsigned peers = __match_any_sync(__activemask(), hashIdx);
        if (lane == 31 - __clz(peers)) {
          atomicMax(&reqKey[hashIdx], make_key(frameTag, pixel, (unsigned)(i0 + j)));
          bitmap_set(reqBits, hashIdx);
          if (isExcess) { bitmap_set(req2Bits, hashIdx); ctr->anyExcessRequest = 1; }   // k_serve_list: tiles of the excess part must wait for the service
          else markBytes[hashIdx] = 1;          // a requested ordered entry is visible (type 1) whether or not it gets a block
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// Chained scans of kernel 2. Same descriptor format as scan_lookback (common.cuh), two differences in the walk:
//  * the look-back window is 256 tiles — eight descriptors per lane, all eight loads in flight at once — so a table of up to
//    2 M entries (256 tiles of 8192) is summed in ONE memory round trip instead of one per 32 tiles;
//  * a tile that does not need its own prefix (no request of its own: the usual case, a frame adds a few dozen blocks) only
//    publishes its aggregate and moves on; the tiles that do need one walk over plain aggregates, however far back.
// NDESC descriptor arrays are walked together (the request ranks need the prefix of all requests AND of the excess ones).
// ------------------------------------------------------------------------------------------------
#define LB_WIN 8   // descriptors per lane and step
// publish this tile's aggregates (tile 0: they are its inclusive prefixes). Called by warp 0 of the CTA.
template <int NDESC>
DEV void lookback_publish(unsigned long long *const *desc, unsigned gen, int tile, const unsigned *agg) {
  if ((threadIdx.x & 31) == 0)
    for (int d = 0; d < NDESC; ++d) ((volatile unsigned long long *)desc[d])[tile] = scan_pack(gen, tile == 0 ? 2 : 1, agg[d]);
}
// exclusive prefixes of `tile` (its aggregates must have been published); publishes its inclusive prefixes. Warp 0 of the CTA.
template <int NDESC>
DEV void lookback_walk(unsigned long long *const *desc, unsigned gen, int tile, const unsigned *agg, unsigned *ex) {
  const int lane = threadIdx.x & 31;
  const unsigned g30 = gen & 0x3fffffffu;
#pragma unroll
  for (int d = 0; d < NDESC; ++d) ex[d] = 0;
  if (tile == 0) return;
  int look = tile - 1;          // nearest tile not yet accounted for
  for (;;) {
    // window: tiles look, look-1, ..., look-255; lane l holds look - (l + 32 j), j = 0..7
    unsigned long long v[NDESC][LB_WIN];
#pragma unroll
    for (int j = 0; j < LB_WIN; ++j) {
      const int t = look - (lane + 32 * j);
#pragma unroll
      for (int d = 0; d < NDESC; ++d) v[d][j] = (t >= 0) ? ((volatile unsigned long long *)desc[d])[t] : 0ull;
    }
    // status of a tile = the weaker of its descriptors' (they are published one after the other)
    bool retry = false, done = false;
    unsigned sum[NDESC];
#pragma unroll
    for (int d = 0; d < NDESC; ++d) sum[d] = 0;
#pragma unroll
    for (int j = 0; j < LB_WIN; ++j) {
      const int t = look - (lane + 32 * j);
      unsigned st = 3;              // beyond tile 0: nothing to add, ends the walk
      if (t >= 0) {
        bool mixed = false;
        st = 2;
#pragma unroll
        for (int d = 0; d < NDESC; ++d) {
          const unsigned sd = ((unsigned)(v[d][j] >> 34) == g30) ? ((unsigned)(v[d][j] >> 32) & 3u) : 0u;
          if (d > 0 && sd != st && sd != 0 && st != 0) mixed = true;      // caught between its two publications
          st = sd < st ? sd : st;
        }
        if (mixed) st = 0;          // re-read: an aggregate must not be mixed with a prefix
      }
      const unsigned validMask = __ballot_sync(0xffffffffu, st != 0);
      const unsigned prefixMask = __ballot_sync(0xffffffffu, st >= 2);
      const int firstPrefix = prefixMask ? (__ffs(prefixMask) - 1) : 32;
      const unsigned need = (firstPrefix >= 32) ? 0xffffffffu : ((1u << firstPrefix) - 1u);
      if (!done && !retry) {
        if ((validMask & need) != need) retry = true;       // a tile in front of the nearest prefix has not published yet
        else {
          if (lane <= firstPrefix && t >= 0) {
#pragma unroll
            for (int d = 0; d < NDESC; ++d) sum[d] += (unsigned)(v[d][j] & 0xffffffffu);
          }
          if (prefixMask) done = true;
        }
      }
    }
    if (retry) continue;            // spin: re-read the window (volatile)
#pragma unroll
    for (int d = 0; d < NDESC; ++d) {
      unsigned a = sum[d];
      for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
      ex[d] += a;
    }
    if (done) break;
    look -= 32 * LB_WIN;
  }
  if (lane == 0) {
    __threadfence();
    for (int d = 0; d < NDESC; ++d) ((volatile unsigned long long *)desc[d])[tile] = scan_pack(gen, 2, ex[d] + agg[d]);
  }
}

// the frustum re-test of a type-3 byte the prepare pass did not produce (decay moved it, Reco_CUDA.cu:1109) — rare, kept out of line
static __device__ __noinline__ bool stale_three_visible(const b200_hash_entry *table, int idx, const FrameGeom *g) {
  const Entry en = load_entry(table, idx);
  return block_visible(en.x, en.y, en.z, g->M_d, g->proj_d, g->voxelSize, g->w, g->h);
}

// 4-bit mask of the non-zero bytes of a word
DEV unsigned nz_bytes(unsigned w) { return ((__vcmpne4(w, 0u) & 0x80808080u) * 0x00204081u) >> 28; }

// ------------------------------------------------------------------------------------------------
// kernel 2 of AllocateSceneFromDepth: request service (allocateVoxelBlocksList) + visible list (buildVisibleList) in one
// persistent launch. A tile is 8192 consecutive entries: one word of each request bitmap and 32 mark / visibility bytes per
// thread.
//
// Phase A, per tile: rank the requests in ascending entry order (block scan + chained look-back over both request bitmaps
// at once) and serve them:  vbaIdx = lastFree - rank(all requests),  exlIdx = lastFreeExcess - rank(excess requests)
// (every request decrements the counters, served or not — Reco_CUDA.cu:833, :857-858); the winning pixel's ray is replayed
// up to its step to recover the block position. The bitmaps are cleared as they are read.
// Phase B, per tile: final visibility byte of every entry (observed this frame -> 1 / 2, else the decoded previous state),
// ordered compaction of the entries with type > 0 (block scan + look-back), and per listed entry: list item, decay-ring
// snapshot (Reco_CUDA.cu:302-317 without the per-frame cudaMalloc), resolved VBA pointer, and — in the fused frame, where
// CreateExpectedDepths renders from this very pose — ProjectSingleBlock and the rasterisation of the block's 1/8-resolution
// box into the expected-depth image with atomic min / max on the (positive) float bit patterns. The listed entries of a
// tile are dealt round-robin to its eight warps.
// A new excess-list entry lies in another tile than the request that creates it: tiles of the excess part of the table
// start phase B only when every tile has finished phase A (device-wide counter; the grid is persistent and co-resident, and
// a CTA finishes phase A of ALL its tiles before it starts phase B of any).
// ------------------------------------------------------------------------------------------------
#define AL_EPT 32
#define AL_TILE (256 * AL_EPT)   // 8192 entries = 256 bitmap words per tile
#define AL_BIG 64                // boxes of more than 512 live cells are rasterised by the whole CTA (at most AL_BIG per tile pass)

#define AL_GROUP_BOX 64          // live cells up to which the entry's 8-lane group rasterises the box

__global__ void __launch_bounds__(256, 2)
k_serve_list(const float *__restrict__ depth, b200_hash_entry *table, int numBuckets, int noTotal, uint8_t *visType,
             const unsigned long long *__restrict__ reqKey, unsigned *reqBits, unsigned *req2Bits, uint8_t *markBytes,
             const int *__restrict__ allocList, const int *__restrict__ excessList, DevCounters *ctr, const __grid_constant__ FrameGeom g,
             int currentFrame, int onlyVisible, unsigned long long *descA, unsigned long long *descB, unsigned long long *descC,
             unsigned gen, b200_vec3i *visiblePos, int *visiblePtr, int capacity, b200_vec3i *ring, long long ringCap, long long *snapStart,
             int *snapCount, int slot, BlockRec *recs, float2 *minmax, int rw, int rh, unsigned maxRB, unsigned long long *dbg) {
  __shared__ unsigned sm[33];
  __shared__ unsigned tileBase, tileBase2;
  __shared__ BlockRec bigRecs[AL_BIG];
  __shared__ int bigCount;
  // measurement hook (b200_diag_read_debug): CTAs 0, 1/3, 2/3 and the last one stamp %globaltimer at their phase boundaries
  const int dbgSlot = !dbg ? -1 : (blockIdx.x == 0 ? 0 : (blockIdx.x == gridDim.x / 3 ? 1 : (blockIdx.x == 2 * gridDim.x / 3 ? 2 : (blockIdx.x == gridDim.x - 1 ? 3 : -1))));
#define K2_TILE_STAMP(k, tile) do { if (dbg && threadIdx.x == 0 && (tile) < 1024) { unsigned long long t_; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_)); dbg[64 + (k) * 1024 + (tile)] = t_; } } while (0)
#define K2_SUB(j, cond) do { if (dbgSlot >= 0 && threadIdx.x == 0 && (cond)) { unsigned long long t_; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_)); dbg[32 + dbgSlot * 8 + (j)] = t_; } } while (0)
#define K2_STAMP(i) do { if (dbgSlot >= 0 && threadIdx.x == 0) { unsigned long long t_; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_)); dbg[dbgSlot * 8 + (i)] = t_; } } while (0)
  K2_STAMP(0);
  const int noWords = noTotal >> 5;
  const int noTiles = (noTotal + AL_TILE - 1) / AL_TILE;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  // One pass (every tile: requests, then its list) when each CTA owns a single tile — the usual case: 192 tiles for the
  // default table — so that a tile's list count is published before anybody serves a request and nobody waits on a serving
  // tile. Two passes (all requests first) when CTAs own several tiles: a tile of the excess part may have to wait for every
  // tile's requests, including those this very CTA still has to serve.
  const bool twoPass = noTiles > (int)gridDim.x;
  // the marking kernel says whether ANY excess-list request was filed this frame: only then can a tile of the excess part
  // receive an entry (and a visibility mark) from another tile's service, and has to wait for all of them
  const bool anyExcess = !onlyVisible && *(volatile int *)&ctr->anyExcessRequest != 0;
  const int baseVba = ctr->lastFreeBlockId, baseExl = ctr->lastFreeExcessListId;   // only the last tile updates them
  const float invfx = 1.0f / g.proj_d[0], invfy = 1.0f / g.proj_d[1];
  const float oneOverVoxelSize = 1.0f / (g.voxelSize * BS);
  const long long ringStart = ctr->ringHead;   // advanced by the last tile only, at its very end
  const int liveX = (rw - 1) / B200_MINMAX_SUBSAMPLE, liveY = (rh - 1) / B200_MINMAX_SUBSAMPLE;   // last live cell of the expected-depth image
  unsigned long long *const dAB[2] = {descA, descB};
  unsigned long long *const dC[1] = {descC};
  unsigned myTiles = 0;   // rendering tiles of the blocks this thread projected (fused frame only)

  const long long ringBase = ringStart % ringCap;   // one 64-bit division per thread instead of one per listed entry
  const int grp = warp * 4 + (lane >> 3), sub = lane & 7;   // hit phase: an 8-lane group per listed entry, one lane per block corner
  for (int pass = 0; pass < (twoPass ? 2 : 1); ++pass) {
    const bool doReq = !twoPass || pass == 0, doList = !twoPass || pass == 1;
    for (int tile = blockIdx.x; tile < noTiles; tile += gridDim.x) {
      const int first = tile * AL_TILE + threadIdx.x * AL_EPT;
      const int w = tile * 256 + threadIdx.x;
      const bool last = (tile == noTiles - 1);
      const bool deferList = anyExcess && ((tile + 1) * AL_TILE > numBuckets);   // its new children arrive from other tiles' service
      K2_TILE_STAMP(0, tile);
      // ---- every load of the tile is issued up front: request words, the first request's key, visibility and mark bytes ----
      unsigned rq = 0, rq2 = 0, localPacked = 0, total = 0, total2 = 0;
      unsigned long long key0 = 0ull;
      uint4 raw[2], mb[2];
      raw[0] = raw[1] = mb[0] = mb[1] = make_uint4(0u, 0u, 0u, 0u);
      if (w < noWords) {
        if (doReq) { rq = reqBits[w]; rq2 = req2Bits[w]; }
        if (doList) {
          raw[0] = __ldcg(reinterpret_cast<const uint4 *>(visType + first));          // noTotal is a multiple of 32
          raw[1] = __ldcg(reinterpret_cast<const uint4 *>(visType + first + 16));
          mb[0] = __ldcg(reinterpret_cast<const uint4 *>(markBytes + first));         // written by the marking kernel and by other tiles' service: L2
          mb[1] = __ldcg(reinterpret_cast<const uint4 *>(markBytes + first + 16));
        }
      }
      // ---- requests: rank (published at once), serve later ----
      if (doReq) {
        if (w < noWords) {
          if (rq) reqBits[w] = 0u;                 // consumed: clean for the next frame
          if (rq2) req2Bits[w] = 0u;
        }
        if (onlyVisible) { rq = 0u; rq2 = 0u; }     // onlyUpdateVisibleList: the marking ran, nothing is allocated (Reco_CUDA.cu:254-262)
        if (rq) key0 = reqKey[w * 32 + __ffs(rq) - 1];
        unsigned totalPacked;
        localPacked = block_exclusive_scan(__popc(rq) | (__popc(rq2) << 16), sm, &totalPacked);   // <= 8192 each: no carry
        total = totalPacked & 0xffffu; total2 = totalPacked >> 16;
        if (threadIdx.x < 32) { const unsigned agg[2] = {total, total2}; lookback_publish<2>(dAB, gen, tile, agg); }
        if (threadIdx.x == 0) {
          if (total2) atomicAdd(&ctr->tilesWithExcess, 1u);
          __threadfence();
          atomicAdd(&ctr->tilesRanked, 1u);         // after the count above: tilesRanked == noTiles makes tilesWithExcess final
        }
      }
      // ---- list, first half: visibility bytes -> mask of listed entries, count published ----
      unsigned mask = 0, mk = 0, local = 0, totalC = 0;
      auto decode = [&](const bool marksOnly, const bool clearMarks) {
        // Byte-parallel (four entries per 32-bit operation, no loop over the interesting bytes): the excess part of the table
        // is dense — every listed excess entry of a KITTI frame sits in the last tile, a dozen per thread — and a per-byte
        // loop there was the longest chain of the launch.
        if (w < noWords) {
#pragma unroll
          for (int q = 0; q < 2; ++q) {
            const unsigned mw[4] = {mb[q].x, mb[q].y, mb[q].z, mb[q].w};
            unsigned xv[4] = {raw[q].x, raw[q].y, raw[q].z, raw[q].w};
            if ((mw[0] | mw[1] | mw[2] | mw[3]) && clearMarks) *reinterpret_cast<uint4 *>(markBytes + first + q * 16) = make_uint4(0u, 0u, 0u, 0u);   // consumed
            bool dirty = false;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
              const unsigned markM = __vcmpne4(mw[j], 0u);      // 0xff where the entry was observed this frame
              const unsigned x = xv[j];
              unsigned nv;
              if (marksOnly) nv = (x & ~markM) | (markM & 0x01010101u);
              else {
                const unsigned pvM = __vcmpeq4(x, VT_PREV_VISIBLE * 0x01010101u) & ~markM, phM = __vcmpeq4(x, VT_PREV_HIDDEN * 0x01010101u) & ~markM;
                // observed -> 1 (2 = swapped out is patched where the entry is read); previous list: re-tested visible -> 3, hidden -> 0
                nv = (x & ~(markM | pvM | phM)) | (markM & 0x01010101u) | (pvM & 0x03030303u);
                unsigned st = __vcmpeq4(x, 0x03030303u) & ~markM & 0x80808080u;      // a 3 the prepare pass did not re-test (list overflow): rare
                while (st) {
                  const int byte = (__ffs(st) - 1) >> 3;
                  st &= st - 1;
                  if (!stale_three_visible(table, first + q * 16 + j * 4 + byte, &g)) nv &= ~(0xffu << (byte * 8));
                }
              }
              if (nv != x) { dirty = true; xv[j] = nv; }
              mask |= nz_bytes(nv) << (q * 16 + j * 4);
              mk |= nz_bytes(mw[j]) << (q * 16 + j * 4);
            }
            if (dirty) {
              raw[q] = make_uint4(xv[0], xv[1], xv[2], xv[3]);
              *reinterpret_cast<uint4 *>(visType + first + q * 16) = raw[q];
            }
          }
        }
      };
      auto count_and_publish = [&]() {
        local = block_exclusive_scan(__popc(mask), sm, &totalC);
        if (threadIdx.x < 32) { const unsigned agg[1] = {totalC}; lookback_publish<1>(dC, gen, tile, agg); }
        K2_TILE_STAMP(1, tile);
        if (dbg && threadIdx.x == 0 && tile < 1024) dbg[64 + 3 * 1024 + tile] = totalC;
      };
      K2_STAMP(1);
      // The list count of a tile never depends on the tile's OWN service (the marking kernel already marked the ordered entries
      // it requested; children land in the excess part), so it is published before anybody serves anything: no tile of the
      // ordered part ever waits for a serving tile. (A tile that still waits for other tiles' child marks leaves the mark bytes
      // alone in this early pass: clearing a 16-byte group here could wipe a mark another tile is writing into it right now.)
      if (doList) { decode(false, !deferList); if (!deferList) count_and_publish(); }
      K2_STAMP(2);
      // ---- requests, second half: ranks of this tile's requests (and the grand totals on the last tile), service ----
      if (doReq) {
        const bool needRank = (total != 0) || last;
        if (needRank && threadIdx.x < 32) {
          const unsigned agg[2] = {total, total2};
          unsigned ex[2];
          lookback_walk<2>(dAB, gen, tile, agg, ex);
          if (threadIdx.x == 0) { tileBase = ex[0]; tileBase2 = ex[1]; }
        }
        __syncthreads();
        if (needRank) {
          unsigned rank = tileBase + (localPacked & 0xffffu), rank2 = tileBase2 + (localPacked >> 16);
          const unsigned grand = tileBase + total, grand2 = tileBase2 + total2;
          bool firstReq = true;
          while (rq) {
            const int b = __ffs(rq) - 1;
            rq &= rq - 1;
            const int targetIdx = w * 32 + b;
            const bool isExcess = (rq2 >> b) & 1u;
            const int vbaIdx = baseVba - (int)rank;
            const int exlIdx = baseExl - (int)rank2;
            rank++;
            if (isExcess) rank2++;
            const unsigned long long key = firstReq ? key0 : reqKey[targetIdx];
            firstReq = false;
            if (vbaIdx < 0 || (isExcess && exlIdx < 0)) continue;   // exhausted: the counters still go negative
            const unsigned step = (unsigned)(key & ((1u << KEY_STEP_BITS) - 1));
            const unsigned pixel = (unsigned)((key >> KEY_STEP_BITS) & ((1u << KEY_PIXEL_BITS) - 1));
            const int x = pixel % g.w, y = pixel / g.w;
            Ray r;
            make_ray(r, x, y, __ldg(depth + pixel), g, invfx, invfy, oneOverVoxelSize);
            float px = r.px, py = r.py, pz = r.pz;
            for (unsigned i = 0; i < step; ++i) { px += r.dx; py += r.dy; pz += r.dz; }
            const int bx = (short)(int)floorf(px), by = (short)(int)floorf(py), bz = (short)(int)floorf(pz);
            int *ew;
            if (!isExcess) {
              ew = reinterpret_cast<int *>(table) + (size_t)targetIdx * 5;
            } else {
              const int exlOffset = excessList[exlIdx];
              reinterpret_cast<int *>(table)[(size_t)targetIdx * 5 + 2] = exlOffset + 1;   // connect to child
              ew = reinterpret_cast<int *>(table) + (size_t)(numBuckets + exlOffset) * 5;
              markBytes[numBuckets + exlOffset] = 1;                                       // child visible (:875)
            }
            ew[0] = (int)(((unsigned)bx & 0xffffu) | ((unsigned)by << 16));
            ew[1] = (bz & 0xffff);
            ew[2] = 0;
            ew[3] = allocList[vbaIdx];
            ew[4] = currentFrame;
          }
          if (last && threadIdx.x == 0) {
            ctr->allocBaseVba = baseVba; ctr->allocBaseExl = baseExl;
            ctr->noRequests = (int)grand; ctr->noRequestsExcess = (int)grand2;
            ctr->lastFreeBlockId = baseVba - (int)grand;
            ctr->lastFreeExcessListId = baseExl - (int)grand2;
          }
        }
        __syncthreads();             // the hit phase below reads entries this tile's service wrote
        if (total2 != 0 && threadIdx.x == 0) {
          __threadfence();                              // this tile's new child entries and their marks are visible device-wide ...
          atomicAdd(&ctr->tilesExcessServed, 1u);       // ... before it counts as served
        }
      }
      K2_STAMP(3);
      K2_TILE_STAMP(4, tile);
      if (!doList) continue;
      // ---- list, late part of the first half: a tile of the excess part in a frame with excess requests ----
      if (deferList) {
        // everything but this frame's new children is decoded already; wait until every tile with excess requests has
        // served them (their number is final once all tiles have published their counts), then pick up the new marks
        if (threadIdx.x == 0) {
          while (*(volatile unsigned *)&ctr->tilesRanked < (unsigned)noTiles) { }
          const unsigned need = *(volatile unsigned *)&ctr->tilesWithExcess;
          while (*(volatile unsigned *)&ctr->tilesExcessServed < need) { }
          __threadfence();
        }
        __syncthreads();
        if (w < noWords) {
          mb[0] = __ldcg(reinterpret_cast<const uint4 *>(markBytes + first));
          mb[1] = __ldcg(reinterpret_cast<const uint4 *>(markBytes + first + 16));
        }
        decode(true, true);
        count_and_publish();
      }
      // ---- list, second half: global offset; the listed entries go to their places in the list ----
      if (threadIdx.x < 32) {
        unsigned ex[1] = {0};
        if (totalC != 0 || last) { const unsigned agg[1] = {totalC}; lookback_walk<1>(dC, gen, tile, agg, ex); }
        if (threadIdx.x == 0) tileBase = ex[0];
        K2_TILE_STAMP(2, tile);
      }
      __syncthreads();
      K2_STAMP(4);
      {
        // the ptr list doubles as the hand-over: entry index | bit 31 (observed this frame) now, the block's ptr after the
        // entry has been read (below, by whichever CTA gets the item)
        long long o = (long long)tileBase + local;
        while (mask) {
          const int k = __ffs(mask) - 1;
          mask &= mask - 1;
          if (o < capacity) reinterpret_cast<unsigned *>(visiblePtr)[o] = (unsigned)(first + k) | (((mk >> k) & 1u) << 31);
          ++o;
        }
      }
      if (last && threadIdx.x == 0) {
        const int n = (int)(tileBase + totalC);
        ctr->noVisibleBlocks = n;
        ctr->noIntegrated = 0;            // IntegrateIntoScene of this frame counts from zero (no separate memset)
        const int kept = n < capacity ? n : capacity;
        // (a snapshot that wraps onto older live ones simply overwrites them: decay.cu recognises an overwritten snapshot by
        // ringHead - snapStart > ringCap when its turn comes and sweeps nothing — the oldest snapshots are dropped, never an error)
        publish_snapshot(ctr, snapStart, snapCount, slot, ringStart, kept);
      }
      __syncthreads();
      if (threadIdx.x == 0) {
        __threadfence();                         // this tile's items (and, on the last tile, the total) are visible device-wide ...
        atomicAdd(&ctr->tilesListed, 1u);        // ... before the tile counts as listed
      }
      K2_STAMP(5);
    }
  }
  // ---------------- the listed entries, dealt evenly over the grid ----------------
  // Entries are not spread evenly over the tiles (every excess-list entry lives in the last tile or two, which are also the
  // last to know their offset), so the per-entry work — read the entry, write the list items, project the block, rasterise
  // its box — is done on the finished list: item i goes to 8-lane group i % 32 of CTA (i / 32) % gridDim. Lane 0 of the group
  // writes the list items, each lane projects one corner of the block (ProjectSingleBlock's loop body; the min/max over the
  // corners by shuffles — min and max do not depend on the order), the group rasterises the box.
  if (threadIdx.x == 0) {
    bigCount = 0;
    while (*(volatile unsigned *)&ctr->tilesListed < (unsigned)noTiles) { }
    __threadfence();
  }
  __syncthreads();
  K2_STAMP(6);
  {
    int nList = *(volatile int *)&ctr->noVisibleBlocks;
    if (nList > capacity) nList = capacity;
    for (int i0 = blockIdx.x * 32; i0 < nList; i0 += gridDim.x * 32) {
      const int item = i0 + grp;
      bool have = false;       // group-uniform: the entry is listed and its box is wanted
      int ex = 0, ey = 0, ez = 0;
      if (item < nList) {
        const unsigned hv = __ldcg(reinterpret_cast<const unsigned *>(visiblePtr) + item);
        const int idx = (int)(hv & 0x7fffffffu);
        const Entry en = load_entry_cg(table, idx);       // the 8 lanes read the same words: one transaction (L2: another CTA may have written the entry)
        int ptr = en.ptr;
        if (ptr < 0) { if (find_block_cg(table, numBuckets, en.x, en.y, en.z, &ptr) < 0) ptr = -1; }   // stale entry: what findBlock(pos) would hit
        __syncwarp(0xffu << (lane & 24));                 // every lane of the group has read the hand-over word before lane 0 replaces it
        if (sub == 0) {
          if (en.ptr == -1 && (hv >> 31)) visType[idx] = 2;   // observed while swapped out (DA/ITMSceneReconstructionEngine.h:261, :281)
          b200_vec3i p; p.x = en.x; p.y = en.y; p.z = en.z;
          visiblePos[item] = p;
          long long rp = ringBase + item;                 // item < capacity <= ringCap
          if (rp >= ringCap) rp -= ringCap;
          ring[rp] = p;
          visiblePtr[item] = ptr;
          if (recs && ptr < 0) { BlockRec e0; e0.ulx = 1; e0.uly = 1; e0.lrx = 0; e0.lry = 0; e0.zmin = 0; e0.zmax = 0; recs[item] = e0; }
        }
        have = recs != nullptr && ptr >= 0;
        ex = en.x; ey = en.y; ez = en.z;
      }
      K2_SUB(0, i0 == blockIdx.x * 32);
      if (recs) {
        // fused frame: the block's 1/8-resolution box (ProjectSingleBlock, DA/ITMVisualisationEngine.h:29-71). All blocks are
        // assumed drawn; if the tile total breaks MAX_RENDERING_BLOCKS (never at KITTI sizes) the last CTA re-applies the
        // ordered rule and rebuilds the image.
        int ulx, uly, lrx, lry; float zl, zh;
        const bool draw = project_block_group(have, ex, ey, ez, g.M_d, g.proj_d, rw, rh, g.voxelSize, ulx, uly, lrx, lry, zl, zh);
        if (have && sub == 0) {
          BlockRec r; r.ulx = 1; r.uly = 1; r.lrx = 0; r.lry = 0; r.zmin = 0; r.zmax = 0;
          if (draw) {
            r.ulx = (short)ulx; r.uly = (short)uly; r.lrx = (short)lrx; r.lry = (short)lry; r.zmin = zl; r.zmax = zh;
            myTiles += rendering_tiles(ulx, uly, lrx, lry);
          }
          recs[item] = r;
        }
        K2_SUB(1, i0 == blockIdx.x * 32);
        // rasterise the part of the box inside the live 1/8-resolution corner — the only cells the raycast reads. (The
        // reference clamps boxes to the FULL-resolution bounds, DA/ITMVisualisationEngine.h:57-60: the cells outside the corner
        // are brought up to date from the records when the host can next see the image, engine.cu.) Up to 64 cells: the
        // group's 8 lanes; more: the whole warp, one box at a time; hundreds (a block next to the camera): the whole CTA.
        const bool live = draw && ulx <= liveX && uly <= liveY;
        const int bxx = min(lrx, liveX), byy = min(lry, liveY);
        const int bw = bxx - ulx + 1, cells = live ? bw * (byy - uly + 1) : 0;
        if (cells > 0 && cells <= AL_GROUP_BOX) raster_box_group(minmax, rw, ulx, uly, bxx, byy, zl, zh);
        K2_SUB(2, i0 == blockIdx.x * 32);
        unsigned todo = __ballot_sync(0xffffffffu, sub == 0 && cells > AL_GROUP_BOX);
        while (todo) {
          const int src = __ffs(todo) - 1;
          todo &= todo - 1;
          const int ax = __shfl_sync(0xffffffffu, ulx, src), ay = __shfl_sync(0xffffffffu, uly, src);
          const int cx = __shfl_sync(0xffffffffu, bxx, src), cy = __shfl_sync(0xffffffffu, byy, src);
          const float zn = __shfl_sync(0xffffffffu, zl, src), zx = __shfl_sync(0xffffffffu, zh, src);
          if ((cx - ax + 1) * (cy - ay + 1) > 512) {
            int slotBig = -1;
            if (lane == 0) slotBig = atomicAdd(&bigCount, 1);
            slotBig = __shfl_sync(0xffffffffu, slotBig, 0);
            if (slotBig < AL_BIG) {
              if (lane == 0) { BlockRec b; b.ulx = (short)ax; b.uly = (short)ay; b.lrx = (short)cx; b.lry = (short)cy; b.zmin = zn; b.zmax = zx; bigRecs[slotBig] = b; }
              continue;
            }
          }
          raster_box_warp(minmax, rw, ax, ay, cx, cy, zn, zx);
        }
        K2_SUB(3, i0 == blockIdx.x * 32);
      }
    }
    __syncthreads();
    K2_SUB(4, true);
    if (recs) {     // the big boxes this CTA met: every thread takes cells
      const int nb = bigCount < AL_BIG ? bigCount : AL_BIG;
      for (int b = 0; b < nb; ++b) {
        const BlockRec br = bigRecs[b];
        const int bw = br.lrx - br.ulx + 1, cnt = bw * (br.lry - br.uly + 1);
        for (int k = threadIdx.x; k < cnt; k += blockDim.x) {
          float2 *px = &minmax[(br.ulx + k % bw) + (br.uly + k / bw) * rw];
          atomic_min_posf(&px->x, br.zmin); atomic_max_posf(&px->y, br.zmax);
        }
      }
    }
  }
  // ---------------- tail: the CTA that finishes last resets the per-launch counters and owns the cap rule ----------------
  if (recs) {
    for (int o = 16; o > 0; o >>= 1) myTiles += __shfl_xor_sync(0xffffffffu, myTiles, o);
    if (lane == 0 && myTiles) atomicAdd(&ctr->noRenderingBlocks, myTiles);
  }
  __shared__ bool lastCta;
  __threadfence();
  __syncthreads();
  K2_STAMP(7);
  if (threadIdx.x == 0) lastCta = (atomicAdd(&ctr->visCtasDone, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!lastCta) return;
  if (threadIdx.x == 0) { ctr->visCtasDone = 0; ctr->tilesRanked = 0; ctr->tilesWithExcess = 0; ctr->tilesExcessServed = 0; ctr->tilesListed = 0; ctr->anyExcessRequest = 0; }
  __threadfence();
  if (!recs) return;
  // The last CTA knows the tile total. In the (pathological) case that it breaks MAX_RENDERING_BLOCKS it re-applies the
  // reference's ordered rule (Vis_CUDA.cu:609: a block is dropped when the running tile count would pass the cap), serially
  // over the list, on the records, and REBUILDS the live corner from the surviving records — every other CTA has finished,
  // so its atomics are all in.
  if (*(volatile unsigned *)&ctr->noRenderingBlocks <= maxRB) return;
  int n = *(volatile int *)&ctr->noVisibleBlocks; if (n > capacity) n = capacity;
  for (int c = threadIdx.x; c < (liveX + 1) * (liveY + 1); c += blockDim.x)
    minmax[(c % (liveX + 1)) + (c / (liveX + 1)) * rw] = make_float2(B200_FAR_AWAY, B200_VERY_CLOSE);
  __syncthreads();
  unsigned running = 0;
  for (int base = 0; base < n; base += blockDim.x) {
    const int item = base + threadIdx.x;
    unsigned required = 0;
    BlockRec r; r.ulx = 1; r.uly = 1; r.lrx = 0; r.lry = 0; r.zmin = 0; r.zmax = 0;
    if (item < n) {
      const uint4 q = __ldcg(reinterpret_cast<const uint4 *>(recs) + item);     // written by other CTAs: L2
      r.ulx = (short)(q.x & 0xffff); r.uly = (short)(q.x >> 16); r.lrx = (short)(q.y & 0xffff); r.lry = (short)(q.y >> 16);
      r.zmin = __uint_as_float(q.z); r.zmax = __uint_as_float(q.w);
      if (r.ulx <= r.lrx) required = rendering_tiles(r.ulx, r.uly, r.lrx, r.lry);
    }
    unsigned total;
    const unsigned local = running + block_exclusive_scan(required, sm, &total);
    bool draw = required > 0;
    if (item < n && required > 0 && local + required > maxRB) {
      r.ulx = 1; r.uly = 1; r.lrx = 0; r.lry = 0; r.zmin = 0; r.zmax = 0;
      recs[item] = r;
      draw = false;
    }
    running += total;
    unsigned todo = __ballot_sync(0xffffffffu, draw && r.ulx <= liveX && r.uly <= liveY);
    while (todo) {
      const int src = __ffs(todo) - 1;
      todo &= todo - 1;
      const int ax = __shfl_sync(0xffffffffu, (int)r.ulx, src), ay = __shfl_sync(0xffffffffu, (int)r.uly, src);
      const int bxx = min(__shfl_sync(0xffffffffu, (int)r.lrx, src), liveX), byy = min(__shfl_sync(0xffffffffu, (int)r.lry, src), liveY);
      const float zn = __shfl_sync(0xffffffffu, r.zmin, src), zx = __shfl_sync(0xffffffffu, r.zmax, src);
      raster_box_warp(minmax, rw, ax, ay, bxx, byy, zn, zx);
    }
  }
}

// free-view visible list (FindVisibleBlocks, Vis_CUDA.cu:151-180, :536-569): every entry with ptr >= 0
// that passes the frustum test, ascending entry order; the visibility bytes are not touched.
#define FV_EPT 16
#define FV_TILE (256 * FV_EPT)
__global__ void __launch_bounds__(256, 4)
k_freeview_list(const b200_hash_entry *__restrict__ table, int noTotal, b200_vec3i *visiblePos, int capacity, DevCounters *ctr,
                unsigned long long *scanDesc, unsigned gen, Mat4 M, float p0, float p1, float p2, float p3, float voxelSize, int w, int h) {
  __shared__ unsigned sm[33];
  __shared__ unsigned tileBase;
  const float proj[4] = {p0, p1, p2, p3};
  const int noTiles = (noTotal + FV_TILE - 1) / FV_TILE;
  for (int tile = blockIdx.x; tile < noTiles; tile += gridDim.x) {
    // strided assignment inside the tile keeps the 20-byte entry reads of a warp adjacent
    unsigned mask = 0;
    for (int k = 0; k < FV_EPT; ++k) {
      const int idx = tile * FV_TILE + k * 256 + threadIdx.x;
      if (idx < noTotal) {
        Entry en = load_entry(table, idx);
        if (en.ptr >= 0 && block_visible(en.x, en.y, en.z, M, proj, voxelSize, w, h)) mask |= 1u << k;
      }
    }
    // order inside the tile must be ascending entry index: rank = sum over k' < k of count(k') + rank within row k
    unsigned total = 0;
    unsigned offs[FV_EPT];
#pragma unroll
    for (int k = 0; k < FV_EPT; ++k) {
      unsigned rowTotal;
      const unsigned r = block_exclusive_scan((mask >> k) & 1u, sm, &rowTotal);
      offs[k] = total + r;
      total += rowTotal;
    }
    if (threadIdx.x < 32) {
      const unsigned ex = scan_lookback(scanDesc, gen, tile, total);
      if (threadIdx.x == 0) { tileBase = ex; if (tile == noTiles - 1) ctr->noVisibleBlocks = (int)(ex + total); }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < FV_EPT; ++k) if ((mask >> k) & 1u) {
      const int idx = tile * FV_TILE + k * 256 + threadIdx.x;
      const Entry en = load_entry(table, idx);
      const unsigned o = tileBase + offs[k];
      if ((int)o < capacity) { b200_vec3i p; p.x = en.x; p.y = en.y; p.z = en.z; visiblePos[o] = p; }
    }
    __syncthreads();
  }
}

void launch_allocate(b200_engine *e, const SceneRef &s, const FrameGeom &g, const float *depth, bool onlyVisible, int frameIdx,
                     int snapSlot, b200_vec2f *minmaxFused, int mw, int mh) {
  cudaStream_t st = e->stream;
  const unsigned frameTag = (unsigned)(frameIdx + 1) & 0xffffffu;
  if (frameTag == 0) cudaMemsetAsync(e->d_reqKey, 0, sizeof(unsigned long long) * (size_t)s.noTotal, st);
  const int tiles = ((g.w + 7) / 8) * ((g.h + 3) / 4);
  const int prepCtas = e->smCount;      // previous list (one block per thread) + expected-depth image initialisation
  trace_begin(e, st, "k_mark_prepare");
  k_mark_prepare<<<prepCtas + (tiles + 7) / 8, 256, 0, st>>>(depth, s.hash, s.numBuckets, s.visiblePos, s.visType, e->d_ctr, e->d_reqKey,
                                                            e->d_reqBits, e->d_req2Bits, e->d_markBytes, g, frameTag, s.numBlocks, prepCtas,
                                                            (float2 *)minmaxFused, mw, mh,
                                                            (unsigned)((0x100000000ull + (unsigned)((g.w + 7) / 8) - 1) / (unsigned)((g.w + 7) / 8)));
  trace_end(e, st);
  const int noTiles = (s.noTotal + AL_TILE - 1) / AL_TILE;
  const unsigned gen = ++e->scanGen;
  const int third = e->scanDescCap / 3;
  trace_begin(e, st, "k_serve_list");
  k_serve_list<<<persistent_grid(e, 2, noTiles), 256, 0, st>>>(depth, s.hash, s.numBuckets, s.noTotal, s.visType, e->d_reqKey, e->d_reqBits,
                                                              e->d_req2Bits, e->d_markBytes, s.allocationList, s.excessList, e->d_ctr, g,
                                                              frameIdx, onlyVisible ? 1 : 0, e->d_scanDesc, e->d_scanDesc + third,
                                                              e->d_scanDesc + 2 * third, gen, s.visiblePos, e->d_visiblePtr, s.numBlocks,
                                                              e->d_ring, e->ringCap, e->d_snapStart, e->d_snapCount, snapSlot,
                                                              minmaxFused ? (BlockRec *)e->d_blockRecs : nullptr, (float2 *)minmaxFused, mw, mh,
                                                              (unsigned)e->maxRenderingBlocks, e->traceOn ? e->d_dbg : nullptr);
  trace_end(e, st);
  e->launches += 2;
}

void launch_find_visible(b200_engine *e, const SceneRef &s, const Mat4 &M, const float proj[4], int w, int h, float voxelSize) {
  const int noTiles = (s.noTotal + FV_TILE - 1) / FV_TILE;
  k_freeview_list<<<persistent_grid(e, 4, noTiles), 256, 0, e->stream>>>(s.hash, s.noTotal, s.visiblePos, s.numBlocks, e->d_ctr,
                                                                        e->d_scanDesc, ++e->scanGen, M, proj[0], proj[1], proj[2], proj[3],
                                                                        voxelSize, w, h);
  e->launches++;
}
