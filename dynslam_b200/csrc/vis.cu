// vis.cu — ITMVisualisationEngine for sm_90a: visible list, expected depths, hierarchical raycast, shading, ICP maps,
// forward render, point cloud.
//
// Replaces (reference ITMVisualisationEngine_CUDA.cu): buildVisibleList_device (:151-180, :536-569), memsetKernel +
// projectAndSplitBlocks_device + fillBlocks_device (:194-240, :572-637), genericRaycast_device (:672-684) with castRay
// (DeviceAgnostic/ITMVisualisationEngine.h:93-179), the five render*_device kernels (:735-886), renderICP_device (:716-724),
// forwardProject/findMissingPoints/genericRaycastMissingPoints/renderForward (:639-733) and renderPointCloud_device (:820-871).
//
// Differences in shape: no materialised RenderingBlock list and no blocking copy of its length —
// each visible block rasterises its own bounding box into the 1/8-resolution min/max image with
// native integer atomics on the (positive) float bit patterns, and the MAX_RENDERING_BLOCKS rule is
// applied on the device by the CTA that finishes last, only when the tile total breaks it; rays are
// traced by 8x4-pixel warps so that a warp's rays walk the same voxel blocks; the voxel reads fetch
// the 2-byte sdf only.
#include "engine.h"
#include "decay_sweep.cuh"
#include "raycast_ray.cuh"
#include "shade.cuh"
#include <cstdlib>

// ------------------------------------------------------------------------------------------------
// visible list
// ------------------------------------------------------------------------------------------------
// FindVisibleBlocks: every entry with ptr >= 0 that passes the frustum test, ascending entry order; the visibility bytes are
// not touched. *count receives the number found, not capped by the list's capacity (the reference's count is not either).
// Tiles come from the caller's ticket (draw_tile, common.cuh).
__global__ void __launch_bounds__(256, 4)
k_freeview_list(const b200_hash_entry *__restrict__ table, int noTotal, b200_vec3i *visiblePos, int capacity, int *count,
                unsigned *ticket, unsigned long long *scanDesc, unsigned gen, Mat4 M, float p0, float p1, float p2, float p3,
                float voxelSize, int w, int h) {
  __shared__ unsigned sm[33];
  __shared__ unsigned tileBase;
  __shared__ int sTile;
  const float proj[4] = {p0, p1, p2, p3};
  const int noTiles = (noTotal + FV_TILE - 1) / FV_TILE;
  for (int tile = draw_tile(ticket, noTiles, &sTile); tile < noTiles; tile = draw_tile(ticket, noTiles, &sTile)) {
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
      if (threadIdx.x == 0) { tileBase = ex; if (tile == noTiles - 1) *count = (int)(ex + total); }
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < FV_EPT; ++k) if ((mask >> k) & 1u) {
      const int idx = tile * FV_TILE + k * 256 + threadIdx.x;
      const Entry en = load_entry(table, idx);
      const unsigned o = tileBase + offs[k];
      if ((int)o < capacity) { b200_vec3i p; p.x = en.x; p.y = en.y; p.z = en.z; visiblePos[o] = p; }
    }
  }
}

void launch_find_visible(b200_engine *e, const SceneRef &s, const Mat4 &M, const float proj[4], int w, int h, float voxelSize,
                         int *count, unsigned *ticket, unsigned long long *scanDesc, unsigned gen) {
  const int noTiles = (s.noTotal + FV_TILE - 1) / FV_TILE;
  trace_begin(e, e->stream, "k_freeview_list");
  k_freeview_list<<<ticket_grid(e, 4, noTiles), 256, 0, e->stream>>>(s.hash, s.noTotal, s.visiblePos, s.numBlocks, count, ticket,
                                                                        scanDesc, gen, M, proj[0], proj[1], proj[2], proj[3], voxelSize,
                                                                        w, h);
  trace_end(e, e->stream);
  e->launches++;
}

// ------------------------------------------------------------------------------------------------
// expected depths
// ------------------------------------------------------------------------------------------------
// ProjectSingleBlock (DA/ITMVisualisationEngine.h:29-71), its 8-lane form, the box rasterisers and the 16-byte block record
// live in common.cuh: the visible-list pass of the fused frame (alloc.cu) uses them too.
__global__ void k_minmax_reset(float2 *minmax, int n, unsigned *tiles) {
  if (blockIdx.x == 0 && threadIdx.x == 0) *tiles = 0;
  const float2 v = make_float2(B200_FAR_AWAY, B200_VERY_CLOSE);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) minmax[i] = v;
}

// CreateExpectedDepths over a visible list, into the image k_minmax_reset has reset. Every listed block goes to an 8-lane
// group (a corner per lane, project_block_group); its box — clamped to the FULL-resolution bounds, as the reference does — is
// rasterised with atomic min / max: by the group up to 64 cells, by the warp up to 512, by the whole CTA beyond (the boxes of
// blocks that leave the frustum on the right or at the bottom spill over up to 10^5 cells of the part of the image nothing
// reads). The rendering tiles of the drawn boxes are summed into *tiles.
// The MAX_RENDERING_BLOCKS rule (Vis_CUDA.cu:609: a block is dropped when the running tile count in list order would pass the
// cap) depends on the order, so every box is drawn first; the CTA that finishes last (*done counts them and is reset by it)
// knows the total, and only if that breaks the cap (never at KITTI sizes) does it reset the image and walk the list in order,
// re-projecting every block and drawing the ones the rule keeps. Every other CTA has finished, so their atomics are all in.
#define XD_BIG 64
__global__ void __launch_bounds__(256)
k_expected_depths(const b200_hash_entry *__restrict__ table, int numBuckets, const b200_vec3i *__restrict__ visiblePos,
                  const int *__restrict__ visiblePtr, int capacity, const int *count, unsigned *tiles, unsigned *done, Mat4 M, float p0,
                  float p1, float p2, float p3, int w, int h, float voxelSize, float2 *minmax, unsigned maxRB) {
  __shared__ BlockRec bigRecs[XD_BIG];
  __shared__ int bigCount;
  __shared__ unsigned sm[33];
  __shared__ bool lastCta;
  const float intr[4] = {p0, p1, p2, p3};
  const int lane = threadIdx.x & 31, grp = threadIdx.x >> 3, sub = threadIdx.x & 7;
  if (threadIdx.x == 0) bigCount = 0;
  __syncthreads();
  int n = *count;
  if (n > capacity) n = capacity;
  // the box of list item `item` for the calling 8-lane group (all 32 lanes call it); false: not drawn
  auto item_box = [&](int item, int &ulx, int &uly, int &lrx, int &lry, float &zl, float &zh) {
    bool have = false;
    int ex = 0, ey = 0, ez = 0;
    if (item < n) {
      const b200_vec3i p = visiblePos[item];
      ex = p.x; ey = p.y; ez = p.z;
      have = visiblePtr ? (__ldg(visiblePtr + item) >= 0) : (find_block<false>(table, numBuckets, p.x, p.y, p.z) >= 0);
    }
    return project_block_group(have, ex, ey, ez, M, intr, w, h, voxelSize, ulx, uly, lrx, lry, zl, zh);
  };
  unsigned myTiles = 0;
  for (int i0 = blockIdx.x * 32; i0 < n; i0 += gridDim.x * 32) {
    int ulx, uly, lrx, lry; float zl, zh;
    const bool draw = item_box(i0 + grp, ulx, uly, lrx, lry, zl, zh);
    if (draw && sub == 0) myTiles += rendering_tiles(ulx, uly, lrx, lry);
    const int cells = draw ? (lrx - ulx + 1) * (lry - uly + 1) : 0;
    if (cells > 0 && cells <= 64) raster_box_group(minmax, w, ulx, uly, lrx, lry, zl, zh);
    unsigned todo = __ballot_sync(0xffffffffu, sub == 0 && cells > 64);
    while (todo) {
      const int src = __ffs(todo) - 1;
      todo &= todo - 1;
      const int ax = __shfl_sync(0xffffffffu, ulx, src), ay = __shfl_sync(0xffffffffu, uly, src);
      const int cx = __shfl_sync(0xffffffffu, lrx, src), cy = __shfl_sync(0xffffffffu, lry, src);
      const float zn = __shfl_sync(0xffffffffu, zl, src), zx = __shfl_sync(0xffffffffu, zh, src);
      if ((cx - ax + 1) * (cy - ay + 1) > 512) {
        int slotBig = -1;
        if (lane == 0) slotBig = atomicAdd(&bigCount, 1);
        slotBig = __shfl_sync(0xffffffffu, slotBig, 0);
        if (slotBig < XD_BIG) {
          if (lane == 0) { BlockRec b; b.ulx = (short)ax; b.uly = (short)ay; b.lrx = (short)cx; b.lry = (short)cy; b.zmin = zn; b.zmax = zx; bigRecs[slotBig] = b; }
          continue;
        }
      }
      raster_box_warp(minmax, w, ax, ay, cx, cy, zn, zx);
    }
  }
  for (int o = 16; o > 0; o >>= 1) myTiles += __shfl_xor_sync(0xffffffffu, myTiles, o);
  if (lane == 0 && myTiles) atomicAdd(tiles, myTiles);
  __syncthreads();
  const int nb = bigCount < XD_BIG ? bigCount : XD_BIG;
  for (int b = 0; b < nb; ++b) {
    const BlockRec br = bigRecs[b];
    const int bw = br.lrx - br.ulx + 1, bh = br.lry - br.uly + 1;
    // rows of the box over the warps, columns over the lanes: no division per cell
    for (int yy = br.uly + (int)(threadIdx.x >> 5); yy < br.uly + bh; yy += (int)(blockDim.x >> 5))
      for (int xx = br.ulx + lane; xx < br.ulx + bw; xx += 32) {
        float2 *px = &minmax[xx + yy * w];
        atomic_min_posf(&px->x, br.zmin); atomic_max_posf(&px->y, br.zmax);
      }
  }
  // ---------------- tail: the CTA that finishes last owns the cap rule ----------------
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) lastCta = (atomicAdd(done, 1u) == gridDim.x - 1);
  __syncthreads();
  if (!lastCta) return;
  if (threadIdx.x == 0) *done = 0;
  if (*(volatile unsigned *)tiles <= maxRB) return;
  for (int i = threadIdx.x; i < w * h; i += blockDim.x) minmax[i] = make_float2(B200_FAR_AWAY, B200_VERY_CLOSE);
  __syncthreads();
  unsigned running = 0;
  for (int base = 0; base < n; base += 32) {     // 32 items per round, in list order over the groups
    int ulx, uly, lrx, lry; float zl, zh;
    const bool draw = item_box(base + grp, ulx, uly, lrx, lry, zl, zh);
    const unsigned required = (draw && sub == 0) ? rendering_tiles(ulx, uly, lrx, lry) : 0u;
    unsigned total;
    const unsigned before = running + block_exclusive_scan(required, sm, &total);
    running += total;
    unsigned todo = __ballot_sync(0xffffffffu, required > 0 && before + required <= maxRB);   // :609
    while (todo) {
      const int src = __ffs(todo) - 1;
      todo &= todo - 1;
      const int ax = __shfl_sync(0xffffffffu, ulx, src), ay = __shfl_sync(0xffffffffu, uly, src);
      const int bx = __shfl_sync(0xffffffffu, lrx, src), by = __shfl_sync(0xffffffffu, lry, src);
      const float zn = __shfl_sync(0xffffffffu, zl, src), zx = __shfl_sync(0xffffffffu, zh, src);
      raster_box_warp(minmax, w, ax, ay, bx, by, zn, zx);
    }
  }
}

// reset + list pass; *count is the list's length as the sweep that built it counted it
void launch_expected_depths(b200_engine *e, const SceneRef &s, const Mat4 &M, const float proj[4], int w, int h, float voxelSize,
                            b200_vec2f *minmax, const int *count, unsigned *tiles, unsigned *done) {
  k_minmax_reset<<<e->smCount * 4, 256, 0, e->stream>>>((float2 *)minmax, w * h, tiles);
  const int groupsOf32 = (s.numBlocks + 31) / 32;
  trace_begin(e, e->stream, "k_expected_depths");
  k_expected_depths<<<persistent_grid(e, 4, groupsOf32), 256, 0, e->stream>>>(s.hash, s.numBuckets, s.visiblePos, fresh_ptr_list(e, s),
                                                                              s.numBlocks, count, tiles, done, M, proj[0], proj[1], proj[2],
                                                                              proj[3], w, h, voxelSize, (float2 *)minmax,
                                                                              (unsigned)e->maxRenderingBlocks);
  trace_end(e, e->stream);
  e->launches += 2;
}

// The cells of the fused frame's expected-depth image outside the live 1/8-resolution corner. k_serve_list (alloc.cu) wrote the
// block records, cap rule included, and rasterised the live corner; the rest of the boxes is read by nothing in the frame (a
// block next to the camera can cover 10^5 of those cells), so it is drawn from the records when the host can next see the
// image (b200_sync, engine.cu): one record per thread, the boxes that reach outside the corner one at a time per warp.
#define DEAD_THREADS 128   // small CTAs: they must fit beside the integrate kernel's CTAs (register file)
__global__ void __launch_bounds__(DEAD_THREADS)
k_dead_cells(const BlockRec *__restrict__ recs, const DevCounters *ctr, int capacity, int w, int h, float2 *minmax) {
  const int liveX = (w - 1) / B200_MINMAX_SUBSAMPLE, liveY = (h - 1) / B200_MINMAX_SUBSAMPLE;   // last live cell
  const int lane = threadIdx.x & 31;
  int n = ctr->noVisibleBlocks;
  if (n > capacity) n = capacity;
  const int noTiles = (n + DEAD_THREADS - 1) / DEAD_THREADS;
  for (int tile = blockIdx.x; tile < noTiles; tile += gridDim.x) {
    const int item = tile * DEAD_THREADS + threadIdx.x;
    int ulx = 0, uly = 0, lrx = -1, lry = -1; float zmin = 0, zmax = 0;
    if (item < n) {
      const uint4 q = __ldg(reinterpret_cast<const uint4 *>(recs) + item);
      ulx = (short)(q.x & 0xffff); uly = (short)(q.x >> 16); lrx = (short)(q.y & 0xffff); lry = (short)(q.y >> 16);
      zmin = __uint_as_float(q.z); zmax = __uint_as_float(q.w);
    }
    unsigned todo = __ballot_sync(0xffffffffu, ulx <= lrx && (lrx > liveX || lry > liveY));
    while (todo) {
      const int src = __ffs(todo) - 1;
      todo &= todo - 1;
      const int ax = __shfl_sync(0xffffffffu, ulx, src), ay = __shfl_sync(0xffffffffu, uly, src);
      const int bx = __shfl_sync(0xffffffffu, lrx, src), by = __shfl_sync(0xffffffffu, lry, src);
      const float zn = __shfl_sync(0xffffffffu, zmin, src), zx = __shfl_sync(0xffffffffu, zmax, src);
      const int bw = bx - ax + 1, cnt = bw * (by - ay + 1);
      for (int k = lane; k < cnt; k += 32) {
        const int yy = ay + k / bw, xx = ax + k % bw;
        if (xx > liveX || yy > liveY) { float2 *px = &minmax[xx + yy * w]; atomic_min_posf(&px->x, zn); atomic_max_posf(&px->y, zx); }
      }
    }
  }
}

void launch_expected_depths_dead(b200_engine *e, const SceneRef &s, int w, int h, b200_vec2f *minmax) {
  const int noTiles = (s.numBlocks + DEAD_THREADS - 1) / DEAD_THREADS;
  trace_begin(e, e->stream, "k_dead_cells");
  k_dead_cells<<<persistent_grid(e, 2, noTiles), DEAD_THREADS, 0, e->stream>>>((const BlockRec *)e->d_blockRecs, e->d_ctr, s.numBlocks, w, h,
                                                                              (float2 *)minmax);
  trace_end(e, e->stream);
  e->launches++;
}

// GenericRaycast — Vis_CUDA.cu:242-265, :672-684. One ray per thread, 8x4-pixel warps (a warp's rays walk the same
// voxel blocks). The march is bound by the chain of dependent L2 reads per step, not by lane utilisation — a ray-refill
// variant (fewer, longer-lived warps) was slower, so the kernel keeps
// the maximum number of independent rays in flight and shortens the chain per step instead (see cast_ray).
// 64-thread CTAs: rays finish at very different times, small CTAs hand their SM slots back sooner.
#define RC_THREADS 64
template <bool useNbr>
__global__ void __launch_bounds__(RC_THREADS)
k_raycast(float4 *out, const b200_voxel *__restrict__ voxels, const b200_hash_entry *__restrict__ table, int nb, int w, int h, Mat4 invM,
          float fx, float fy, float cxp, float cyp, float voxelSize, float mu, const float2 *__restrict__ minmax, int twLog2, int centreRow,
          int tilesX, int tilesY, unsigned tilesXMagic, unsigned long long *span, DecaySweep sweep, int sweepCtas) {
  if ((int)blockIdx.x < sweepCtas) {
    // CTAs [0, sweepCtas): a partial Decay's sweep (decay_sweep.cuh), which reads what the rays read and writes only decay
    // scratch (launch_chained's rules). Dispatched first, they take SM slots while the first waves of rays are issue-bound.
    pdl_wait();
    pdl_trigger();
    SpanStamp stamp(sweep.span);
    decay_sweep<0>(sweep, (blockIdx.x * RC_THREADS + threadIdx.x) >> 5, sweepCtas * (RC_THREADS / 32));
    return;
  }
  // warp tile: (1 << twLog2) x (32 >> twLog2) pixels
  const int tw = 1 << twLog2, th = 32 >> twLog2;
  const int warpGlobal = ((blockIdx.x - sweepCtas) * blockDim.x + threadIdx.x) >> 5;
  if (warpGlobal >= tilesX * tilesY) return;
  const int lane = threadIdx.x & 31;
  const int rowLinear = (int)__umulhi((unsigned)warpGlobal, tilesXMagic);      // warpGlobal / tilesX (magic = ceil(2^32 / tilesX))
  int tileRow = rowLinear;
  if (centreRow >= 0) {
    // dispatch order = tile rows sorted by distance from `centreRow` (c, c+1, c-1, c+2, ...): the rows around the horizon
    // hold the rays that skim the ground inside its truncation band for hundreds of steps; started first, they overlap
    // the rest of the image instead of forming the kernel's tail. Every pixel is still written exactly once.
    const int c = centreRow, up = tilesY - 1 - c, down = c, m = up < down ? up : down, k = tileRow;
    if (k <= 2 * m) { const int off = (k + 1) >> 1; tileRow = (k & 1) ? c + off : c - off; }
    else { const int rest = k - 2 * m; tileRow = (up > down) ? c + m + rest : c - m - rest; }
  }
  const int x = (warpGlobal - rowLinear * tilesX) * tw + (lane & (tw - 1)), y = tileRow * th + (lane >> twLog2);
  if (x >= w || y >= h) return;
  const int locId2 = (int)floorf((float)x / B200_MINMAX_SUBSAMPLE) + (int)floorf((float)y / B200_MINMAX_SUBSAMPLE) * w;
  // In the fused frame the expected-depth image was last written by the list kernel, two launches back (launch_chained's rules):
  // it is read before the wait for the integrate kernel, which writes only voxels.
  const float2 mm = __ldg(minmax + locId2);
  pdl_wait();
  pdl_trigger();
  SpanStamp stamp(span);
  float4 o;
  if (useNbr) {
    __shared__ int nbr[8][RC_THREADS];     // per thread: the 2x2x2 block neighbourhood of the ray's current block (raycast_ray.cuh)
    cast_ray_nbr(o, x, y, voxels, table, nb, invM, 1.0f / fx, 1.0f / fy, cxp, cyp, 1.0f / voxelSize, mu, mm, &nbr[0][threadIdx.x], RC_THREADS);
  } else {
    cast_ray(o, x, y, voxels, table, nb, invM, 1.0f / fx, 1.0f / fy, cxp, cyp, 1.0f / voxelSize, mu, mm);
  }
  out[x + y * w] = o;
}

void launch_raycast(b200_engine *e, const SceneRef &s, const Mat4 &invM, const float proj[4], int w, int h, float voxelSize, float mu,
                    const b200_vec2f *minmax, b200_vec4f *out, bool fused, const DecaySweep *sweep) {
  const int twLog2 = e->rcTileLog2;   // warp tile (1 << twLog2) x (32 >> twLog2) pixels; 3: 8x4 (default)
  const int tw = 1 << twLog2, th = 32 >> twLog2;
  const int tiles = ((w + tw - 1) / tw) * ((h + th - 1) / th);
  const int warpsPerCta = RC_THREADS / 32;
  int centreRow = -1;
  if (e->rcOrder == 1) {   // principal-point row first (level camera: the horizon); 0 = plain row-major
    const int tilesY = (h + th - 1) / th;
    centreRow = (int)(proj[3] / (float)th);
    if (centreRow < 0) centreRow = 0;
    if (centreRow > tilesY - 1) centreRow = tilesY - 1;
  }
  const int tilesXh = (w + tw - 1) / tw, tilesYh = (h + th - 1) / th;
  const unsigned magic = (unsigned)((0x100000000ull + (unsigned)tilesXh - 1) / (unsigned)tilesXh);
  const int impl = e->rcImpl;   // 1: neighbourhood cache (default); 0: per-lane one-entry cache (cross-check)
  // The sweep's CTAs loop over the snapshot's items (a visible list, a few thousand blocks): 4 CTAs (8 warps) per SM, beside
  // the 25 raycast CTAs an SM holds.
  const int sweepCtas = sweep ? e->smCount * 4 : 0;
  trace_begin(e, e->stream, "k_raycast");
  launch_chained(fused, impl ? k_raycast<true> : k_raycast<false>, sweepCtas + (tiles + warpsPerCta - 1) / warpsPerCta, RC_THREADS, 0,
                 e->stream, (float4 *)out, s.voxels, s.hash, s.numBuckets, w, h, invM, proj[0], proj[1], proj[2], proj[3], voxelSize, mu,
                 (const float2 *)minmax, twLog2, centreRow, tilesXh, tilesYh, magic, fused ? span_slot(e, SPAN_RAYCAST) : nullptr,
                 sweep ? *sweep : DecaySweep{}, sweepCtas);
  trace_end(e, e->stream);
  e->launches++;
}

// ------------------------------------------------------------------------------------------------
// shading from the volume
// ------------------------------------------------------------------------------------------------
// RenderImage_common kernels — Vis_CUDA.cu:735-886; the per-pixel functions are in shade.cuh. Two outputs, either may be null:
// the RGBA pixel of `type` and the depth pixel (drawPixelDepth), so that the free-view preview gets both from one read of the
// ray point.
__global__ void __launch_bounds__(256)
k_shade(const float4 *__restrict__ rays, const b200_voxel *__restrict__ voxels, const b200_hash_entry *__restrict__ table, int nb, int w, int h,
        Mat4 M, float lx, float ly, float lz, float voxelSize, int maxW, uchar4 *outChar, float *outDepth, int type) {
  const int tilesX = (w + 7) >> 3, tilesY = (h + 3) >> 2;
  const int warpGlobal = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (warpGlobal >= tilesX * tilesY) return;
  const int lane = threadIdx.x & 31;
  const int x = (warpGlobal % tilesX) * 8 + (lane & 7), y = (warpGlobal / tilesX) * 4 + (lane >> 3);
  if (x >= w || y >= h) return;
  const int locId = x + y * w;
  const float4 pr = rays[locId];
  const bool found = pr.w > 0;
  if (outDepth) outDepth[locId] = depth_px(found, pr, M, voxelSize);
  if (outChar) shade_rgba_px(type, found, pr, voxels, table, nb, lx, ly, lz, maxW, &outChar[locId]);
}

// either output may be null; `type` is the RGBA type outChar is shaded with
void launch_shade(b200_engine *e, const SceneRef &s, const Mat4 &M, const Mat4 &invM, int w, int h, float voxelSize, int maxW,
                  const b200_vec4f *rays, b200_vec4u *outChar, float *outDepth, int type) {
  const int tiles = ((w + 7) / 8) * ((h + 3) / 4);
  trace_begin(e, e->stream, "k_shade");
  k_shade<<<(tiles + 7) / 8, 256, 0, e->stream>>>((const float4 *)rays, s.voxels, s.hash, s.numBuckets, w, h, M, -invM.m[8], -invM.m[9],
                                                 -invM.m[10], voxelSize, maxW, (uchar4 *)outChar, outDepth, type);
  trace_end(e, e->stream);
  e->launches++;
}

// ------------------------------------------------------------------------------------------------
// image-space normals: processPixelICP<true> / processPixelForwardRender<true>
// ------------------------------------------------------------------------------------------------
// computeNormalAndAngle<useSmoothing=true> — DA/ITMVisualisationEngine.h:212-275
DEV void normal_and_angle_img(bool &found, int x, int y, const float4 *__restrict__ pr, float lx, float ly, float lz, float voxelSize,
                              int w, int h, float &nx, float &ny, float &nz, float &angle) {
  if (!found) return;
  if (y <= 2 || y >= h - 3 || x <= 2 || x >= w - 3) { found = false; return; }
  float4 xp1 = pr[(x + 2) + y * w], yp1 = pr[x + (y + 2) * w], xm1 = pr[(x - 2) + y * w], ym1 = pr[x + (y - 2) * w];
  float dxx = 0, dxy = 0, dxz = 0, dyx = 0, dyy = 0, dyz = 0;
  bool doPlus1 = false;
  if (xp1.w <= 0 || yp1.w <= 0 || xm1.w <= 0 || ym1.w <= 0) doPlus1 = true;
  else {
    dxx = xp1.x - xm1.x; dxy = xp1.y - xm1.y; dxz = xp1.z - xm1.z;
    dyx = yp1.x - ym1.x; dyy = yp1.y - ym1.y; dyz = yp1.z - ym1.z;
    const float length_diff = maxf_(dxx * dxx + dxy * dxy + dxz * dxz, dyx * dyx + dyy * dyy + dyz * dyz);
    if (length_diff * voxelSize * voxelSize > (0.15f * 0.15f)) doPlus1 = true;
  }
  if (doPlus1) {
    xp1 = pr[(x + 1) + y * w]; yp1 = pr[x + (y + 1) * w]; xm1 = pr[(x - 1) + y * w]; ym1 = pr[x + (y - 1) * w];
    dxx = xp1.x - xm1.x; dxy = xp1.y - xm1.y; dxz = xp1.z - xm1.z;
    dyx = yp1.x - ym1.x; dyy = yp1.y - ym1.y; dyz = yp1.z - ym1.z;
    if (xp1.w <= 0 || yp1.w <= 0 || xm1.w <= 0 || ym1.w <= 0) { found = false; return; }
  }
  nx = -(dxy * dyz - dxz * dyy);
  ny = -(dxz * dyx - dxx * dyz);
  nz = -(dxx * dyy - dxy * dyx);
  const float normScale = 1.0f / sqrtf(nx * nx + ny * ny + nz * nz);
  nx *= normScale; ny *= normScale; nz *= normScale;
  angle = nx * lx + ny * ly + nz * lz;
  if (!(angle > 0.0)) found = false;
}

__global__ void __launch_bounds__(256)
k_icp(const float4 *__restrict__ rays, int w, int h, float voxelSize, float lx, float ly, float lz, uchar4 *outImg, float4 *points,
      float4 *normals, unsigned long long *span) {
  SpanStamp stamp(span);
  const int x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= w || y >= h) return;
  const int locId = x + y * w;
  const float4 p = rays[locId];
  bool found = p.w > 0.0f;
  float nx = 0, ny = 0, nz = 0, angle = 0;
  normal_and_angle_img(found, x, y, rays, lx, ly, lz, voxelSize, w, h, nx, ny, nz, angle);
  if (found) {
    outImg[locId] = grey_px(angle);
    if (points) { points[locId] = make_float4(p.x * voxelSize, p.y * voxelSize, p.z * voxelSize, 1.0f); normals[locId] = make_float4(nx, ny, nz, 0.0f); }
  } else {
    outImg[locId] = make_uchar4(0, 0, 0, 0);
    if (points) { points[locId] = make_float4(0.0f, 0.0f, 0.0f, -1.0f); normals[locId] = make_float4(0.0f, 0.0f, 0.0f, -1.0f); }
  }
}

void launch_icp(b200_engine *e, const Mat4 &invM, int w, int h, float voxelSize, const b200_vec4f *rays, b200_vec4u *outImg,
                b200_vec4f *points, b200_vec4f *normals, bool fused) {
  dim3 grid((w + 31) / 32, (h + 7) / 8);
  trace_begin(e, e->stream, "k_icp");
  k_icp<<<grid, 256, 0, e->stream>>>((const float4 *)rays, w, h, voxelSize, -invM.m[8], -invM.m[9], -invM.m[10], (uchar4 *)outImg,
                                     (float4 *)points, (float4 *)normals, fused ? span_slot(e, SPAN_ICP) : nullptr);
  trace_end(e, e->stream);
  e->launches++;
}

// ------------------------------------------------------------------------------------------------
// forward render (approximate raycast path; dead under DynSLAM settings, kept for the interface)
// Canonical order (oracle): raster order; the forward splat keeps the LAST source pixel that lands
// on a target pixel -> atomicMax on the source index, then a gather.
// ------------------------------------------------------------------------------------------------
__global__ void k_fwd_splat(const float4 *__restrict__ rays, int w, int h, Mat4 M, float p0, float p1, float p2, float p3, float voxelSize,
                            int *winner) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= w * h) return;
  const float4 px = rays[i];
  // forwardProjectPixel(pixel * voxelSize, ...) — DA/ITMVisualisationEngine.h:181-194
  Vec4 q = m4v4(M, px.x * voxelSize, px.y * voxelSize, px.z * voxelSize, 1.0f);
  const float ix = p0 * q.x / q.z + p2, iy = p1 * q.y / q.z + p3;
  if ((ix < 0) || (ix > w - 1) || (iy < 0) || (iy > h - 1)) return;
  atomicMax(&winner[(int)(ix + 0.5f) + (int)(iy + 0.5f) * w], i);
}

#define FWD_TILE 1024
__global__ void __launch_bounds__(256)
k_fwd_gather_missing(const float4 *__restrict__ rays, const int *__restrict__ winner, float4 *fwd, const float *__restrict__ depth,
                     const float2 *__restrict__ minmax, int w, int h, int *missing, DevCounters *ctr, unsigned long long *scanDesc,
                     unsigned gen) {
  __shared__ unsigned sm[33];
  __shared__ unsigned tileBase;
  __shared__ int sTile;
  const int n = w * h, noTiles = (n + FWD_TILE - 1) / FWD_TILE;
  unsigned *ticket = &ctr->ticket[TK_FWD_MISSING];
  for (int tile = draw_tile(ticket, noTiles, &sTile); tile < noTiles; tile = draw_tile(ticket, noTiles, &sTile)) {
    unsigned mask = 0;
    const int first = tile * FWD_TILE + threadIdx.x * 4;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int locId = first + k;
      if (locId >= n) continue;
      const int src = winner[locId];
      const float4 fp = src >= 0 ? rays[src] : make_float4(0, 0, 0, 0);
      fwd[locId] = fp;
      const int y = locId / w, x = locId - y * w;
      const int locId2 = (int)floorf((float)x / B200_MINMAX_SUBSAMPLE) + (int)floorf((float)y / B200_MINMAX_SUBSAMPLE) * w;
      const float2 mm = minmax[locId2];
      const float d = depth[locId];
      if ((fp.w <= 0) && ((fp.x == 0 && fp.y == 0 && fp.z == 0) || (d > 0)) && (mm.x < mm.y)) mask |= 1u << k;
    }
    unsigned total;
    unsigned local = block_exclusive_scan(__popc(mask), sm, &total);
    if (threadIdx.x < 32) {
      unsigned ex = scan_lookback(scanDesc, gen, tile, total);
      if (threadIdx.x == 0) { tileBase = ex; if (tile == noTiles - 1) ctr->noFwdMissing = (int)(ex + total); }
    }
    __syncthreads();
    unsigned o = tileBase + local;
#pragma unroll
    for (int k = 0; k < 4; ++k) if (mask & (1u << k)) missing[o++] = first + k;
  }
}

__global__ void k_fwd_raycast_missing(float4 *fwd, const int *__restrict__ missing, const DevCounters *ctr, const b200_voxel *__restrict__ voxels,
                                      const b200_hash_entry *__restrict__ table, int nb, int w, Mat4 invM, float fx, float fy, float cxp,
                                      float cyp, float voxelSize, float mu, const float2 *__restrict__ minmax) {
  const int n = ctr->noFwdMissing;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    const int locId = missing[i];
    const int y = locId / w, x = locId - y * w;
    const int locId2 = (int)floorf((float)x / B200_MINMAX_SUBSAMPLE) + (int)floorf((float)y / B200_MINMAX_SUBSAMPLE) * w;
    float4 o;
    cast_ray(o, x, y, voxels, table, nb, invM, 1.0f / fx, 1.0f / fy, cxp, cyp, 1.0f / voxelSize, mu, minmax[locId2]);
    fwd[locId] = o;
  }
}

void launch_forward_render(b200_engine *e, const SceneRef &s, const FrameGeom &g, const float *depth, const b200_vec2f *minmax,
                           const b200_vec4f *rays, b200_vec4f *fwd, int *missing, b200_vec4u *outImg) {
  cudaStream_t st = e->stream;
  const int n = g.w * g.h;
  int *winner = reinterpret_cast<int *>(e->d_tileCounts);   // per target pixel: last source pixel landing on it
  cudaMemsetAsync(winner, 0xff, sizeof(int) * (size_t)n, st);   // -1 = none
  k_fwd_splat<<<(n + 255) / 256, 256, 0, st>>>((const float4 *)rays, g.w, g.h, g.M_d, g.proj_d[0], g.proj_d[1], g.proj_d[2], g.proj_d[3],
                                              g.voxelSize, winner);
  const int noTiles = (n + FWD_TILE - 1) / FWD_TILE;
  k_fwd_gather_missing<<<ticket_grid(e, 4, noTiles), 256, 0, st>>>((const float4 *)rays, winner, (float4 *)fwd, depth,
                                                                      (const float2 *)minmax, g.w, g.h, missing, e->d_ctr, e->d_scanDesc,
                                                                      ++e->scanGen);
  k_fwd_raycast_missing<<<e->smCount * 4, 128, 0, st>>>((float4 *)fwd, missing, e->d_ctr, s.voxels, s.hash, s.numBuckets, g.w, g.invM_d,
                                                       g.proj_d[0], g.proj_d[1], g.proj_d[2], g.proj_d[3], g.voxelSize, g.mu,
                                                       (const float2 *)minmax);
  dim3 grid((g.w + 31) / 32, (g.h + 7) / 8);
  trace_begin(e, st, "k_icp");
  k_icp<<<grid, 256, 0, st>>>((const float4 *)fwd, g.w, g.h, g.voxelSize, -g.invM_d.m[8], -g.invM_d.m[9], -g.invM_d.m[10], (uchar4 *)outImg,
                              nullptr, nullptr, nullptr);
  trace_end(e, st);
  e->launches += 4;
}

// ------------------------------------------------------------------------------------------------
// point cloud for the colour tracker (dead under DynSLAM settings, kept for the interface);
// canonical order of the compacted cloud: raster order
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
k_point_cloud(const float4 *__restrict__ rays, const b200_voxel *__restrict__ voxels, const b200_hash_entry *__restrict__ table, int nb, int w,
              int h, float lx, float ly, float lz, float voxelSize, int skipPoints, uchar4 *outImg, float4 *locations, float4 *colours,
              DevCounters *ctr, unsigned long long *scanDesc, unsigned gen) {
  __shared__ unsigned sm[33];
  __shared__ unsigned tileBase;
  __shared__ int sTile;
  const int n = w * h, noTiles = (n + 255) / 256;
  unsigned *ticket = &ctr->ticket[TK_POINT_CLOUD];
  for (int tile = draw_tile(ticket, noTiles, &sTile); tile < noTiles; tile = draw_tile(ticket, noTiles, &sTile)) {
    const int locId = tile * 256 + threadIdx.x;
    bool found = false; float4 pr = make_float4(0, 0, 0, 0);
    if (locId < n) {
      const int y = locId / w, x = locId - y * w;
      pr = rays[locId];
      found = pr.w > 0;
      float nx = 0, ny = 0, nz = 0, angle = 0;
      normal_and_angle_sdf(found, pr.x, pr.y, pr.z, voxels, table, nb, lx, ly, lz, nx, ny, nz, angle);
      outImg[locId] = found ? grey_px(angle) : make_uchar4(0, 0, 0, 0);
      if (skipPoints && ((x % 2 == 0) || (y % 2 == 0))) found = false;
    }
    unsigned total;
    unsigned local = block_exclusive_scan(found ? 1u : 0u, sm, &total);
    if (threadIdx.x < 32) {
      unsigned ex = scan_lookback(scanDesc, gen, tile, total);
      if (threadIdx.x == 0) { tileBase = ex; if (tile == noTiles - 1) ctr->noTotalPoints = ex + total; }
    }
    __syncthreads();
    if (found) {
      const unsigned o = tileBase + local;
      float c0, c1, c2;
      color_interp(voxels, table, nb, pr.x, pr.y, pr.z, c0, c1, c2);
      float4 tmp = make_float4(c0, c1, c2, 1.0f);
      tmp.x /= tmp.w; tmp.y /= tmp.w; tmp.z /= tmp.w;
      colours[o] = tmp;
      locations[o] = make_float4(pr.x * voxelSize, pr.y * voxelSize, pr.z * voxelSize, 1.0f);
    }
  }
}

void launch_point_cloud(b200_engine *e, const SceneRef &s, const Mat4 &invM, int w, int h, float voxelSize, int skipPoints,
                        const b200_vec4f *rays, b200_vec4u *outImg, b200_vec4f *locations, b200_vec4f *colours) {
  const int noTiles = (w * h + 255) / 256;
  k_point_cloud<<<ticket_grid(e, 2, noTiles), 256, 0, e->stream>>>((const float4 *)rays, s.voxels, s.hash, s.numBuckets, w, h,
                                                                      -invM.m[8], -invM.m[9], -invM.m[10], voxelSize, skipPoints,
                                                                      (uchar4 *)outImg, (float4 *)locations, (float4 *)colours, e->d_ctr,
                                                                      e->d_scanDesc, ++e->scanGen);
  e->launches++;
}
