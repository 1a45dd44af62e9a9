// preview.cu — the free-view preview: FindVisibleBlocks + CreateExpectedDepths + RenderImage(type) + RenderImage(DEPTH_MAP)
// from one pose as ONE enqueue (b200_render_view_async), its pipelined hand-over to the host (b200_render_view_submit /
// _wait) and the device-side ordering between engines that compositing several volumes' previews needs
// (b200_engine_wait_engine).
//
// Replaces, for this use, the reference's stop-and-go shape (ITMMainEngine::GetImage for the FREECAMERA types,
// ITMMainEngine.cpp:231-278, called twice per volume by DynSLAM: once for the RGBA image, once more for the depth): four
// launches, no host synchronisation, one raycast shaded two ways.
//
//   k_preview_init    resets the expected-depth image and the preview's own counters
//   k_preview_sweep   sweeps the hash table once: ordered visible list, every listed block's box rasterised into the image, the
//                     MAX_RENDERING_BLOCKS rule decided per block from the list-order prefix of the rendering-tile counts
//   k_raycast         vis.cu, unchanged
//   k_preview_shade   reads every ray point once, writes the RGBA pixel and the depth pixel
//
// Nothing here touches the volume's counters (DevCounters), the block records or the scan descriptors of the fused frame: the
// preview has a counter block, descriptors and staging of its own, so it can be enqueued between asynchronous frames.
#include "engine.h"
#include "shade.cuh"

#include <cstdio>
#include <cstring>

struct PreviewCounters {
  int noVisible;         // blocks the sweep listed (not capped by the list's capacity, as FindVisibleBlocks' count is not)
  unsigned noTiles;      // rendering tiles of the listed blocks (CreateExpectedDepths' noTotalBlocks before the cap)
  unsigned ticket;       // next table tile to hand out
  unsigned pad;
};

struct PreviewScratch {
  PreviewCounters *d_ctr;
  int *h_count;                          // pinned: noVisible, noTiles as b200_render_view_sync reads them back
  unsigned long long *d_descN, *d_descT; // chained-scan descriptors of the list positions / the rendering-tile prefix
  unsigned gen;
  const void *lastList;                  // the visible list of the render state the counters describe
  cudaEvent_t evOut;                     // b200_engine_wait_engine: "everything enqueued on this engine's stream so far"
  // host hand-over: two slots, a copy stream of its own (a host frame's image download never queues in front of a preview)
  cudaStream_t d2h;
  cudaEvent_t evRender[2], evD2H[2];
  b200_vec4u *d_char[2]; float *d_depth[2];
  size_t pixels; bool busy[2];
};

#define CK(call)                                                                                   \
  do {                                                                                             \
    cudaError_t _e = (call);                                                                       \
    if (_e != cudaSuccess) {                                                                       \
      snprintf(e->err, sizeof(e->err), "%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e)); \
      return B200_ERR_CUDA;                                                                        \
    }                                                                                              \
  } while (0)

// ------------------------------------------------------------------------------------------------
// kernels
// ------------------------------------------------------------------------------------------------
__global__ void k_preview_init(float2 *minmax, int n, PreviewCounters *ctr) {
  if (blockIdx.x == 0 && threadIdx.x == 0) { ctr->noVisible = 0; ctr->noTiles = 0; ctr->ticket = 0; }
  const float2 v = make_float2(B200_FAR_AWAY, B200_VERY_CLOSE);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) minmax[i] = v;
}

// One pass over the hash table. Per tile of PV_TILE entries: (A) frustum-test the allocated entries and compact the visible
// ones, ascending entry order, into shared memory; their place in the list comes from a chained scan over the tiles. (B) Project
// them (ProjectSingleBlock) and sum their rendering tiles; a second chained scan gives the tile's list-order prefix of that
// count, which is what the MAX_RENDERING_BLOCKS rule is stated on (Vis_CUDA.cu:609): a block is drawn when prefix + own <= cap.
// (C) Write the list and rasterise the drawn boxes, clamped to the full-resolution bounds as the reference clamps them, with
// atomic min / max (order-free, so the image has the bytes of the ordered form). The blocks are sparse among the entries (a few
// thousand in 1.5 M), so projecting them in (B) and again in (C) costs less than keeping 16-byte records of a whole tile.
//
// Tiles are handed out through a ticket, not by blockIdx: a tile then only ever waits for tiles whose CTAs are already running,
// so the look-back cannot stall when the grid is not co-resident — two engines' sweeps sharing the GPU, which is exactly how
// several volumes' previews are rendered.
#define PV_EPT 16
#define PV_TILE (256 * PV_EPT)
#define PV_BIG 32          // boxes of more than 512 cells are rasterised by the whole CTA (at most PV_BIG per 256 blocks, the rest by their warp)
__global__ void __launch_bounds__(256, 4)
k_preview_sweep(const b200_hash_entry *__restrict__ table, int noTotal, b200_vec3i *visiblePos, int capacity, PreviewCounters *ctr,
                unsigned long long *descN, unsigned long long *descT, unsigned gen, Mat4 M, float p0, float p1, float p2, float p3,
                float voxelSize, int w, int h, float2 *minmax, unsigned maxRB) {
  __shared__ unsigned sm[33];
  __shared__ short4 sPos[PV_TILE];
  __shared__ BlockRec sBig[PV_BIG];
  __shared__ int sBigCount, sTile;
  __shared__ unsigned sBaseN, sBaseT;
  const float proj[4] = {p0, p1, p2, p3};
  const int noTiles = (noTotal + PV_TILE - 1) / PV_TILE;
  const int lane = threadIdx.x & 31;
  if (threadIdx.x == 0) sBigCount = 0;
  for (;;) {
    if (threadIdx.x == 0) sTile = (int)atomicAdd(&ctr->ticket, 1u);
    __syncthreads();
    const int tile = sTile;
    if (tile >= noTiles) break;
    // (A) strided assignment inside the tile keeps the 20-byte entry reads of a warp adjacent; list order is ascending entry
    // index: rank = sum over k' < k of count(k') + rank within row k
    unsigned mask = 0;
#pragma unroll 4
    for (int k = 0; k < PV_EPT; ++k) {
      const int idx = tile * PV_TILE + k * 256 + threadIdx.x;
      if (idx < noTotal) {
        const Entry en = load_entry(table, idx);
        if (en.ptr >= 0 && block_visible(en.x, en.y, en.z, M, proj, voxelSize, w, h)) mask |= 1u << k;
      }
    }
    unsigned total = 0;
    for (int k = 0; k < PV_EPT; ++k) {
      unsigned rowTotal;
      const unsigned r = block_exclusive_scan((mask >> k) & 1u, sm, &rowTotal);
      if ((mask >> k) & 1u) {
        const Entry en = load_entry(table, tile * PV_TILE + k * 256 + threadIdx.x);
        sPos[total + r] = make_short4((short)en.x, (short)en.y, (short)en.z, 0);
      }
      total += rowTotal;
    }
    if (threadIdx.x < 32) {
      const unsigned ex = scan_lookback(descN, gen, tile, total);
      if (threadIdx.x == 0) { sBaseN = ex; if (tile == noTiles - 1) ctr->noVisible = (int)(ex + total); }
    }
    __syncthreads();
    // what lies beyond the list's capacity is counted (as FindVisibleBlocks counts it) but neither listed nor drawn
    const unsigned baseN = sBaseN;
    const unsigned cnt = baseN >= (unsigned)capacity ? 0u : min(total, (unsigned)capacity - baseN);
    // (B)
    unsigned myTiles = 0;
    for (unsigned i = threadIdx.x; i < cnt; i += 256) {
      const short4 p = sPos[i];
      int ulx, uly, lrx, lry; float zl, zh;
      if (project_single_block(p.x, p.y, p.z, M, proj, w, h, voxelSize, ulx, uly, lrx, lry, zl, zh)) myTiles += rendering_tiles(ulx, uly, lrx, lry);
    }
    unsigned tileTiles;
    block_exclusive_scan(myTiles, sm, &tileTiles);
    if (threadIdx.x < 32) {
      const unsigned ex = scan_lookback(descT, gen, tile, tileTiles);
      if (threadIdx.x == 0) { sBaseT = ex; if (tile == noTiles - 1) ctr->noTiles = ex + tileTiles; }
    }
    __syncthreads();
    // (C)
    unsigned running = sBaseT;
    for (unsigned i0 = 0; i0 < cnt; i0 += 256) {
      const unsigned i = i0 + threadIdx.x;
      int ulx = 0, uly = 0, lrx = -1, lry = -1; float zl = 0, zh = 0;
      unsigned required = 0;
      if (i < cnt) {
        const short4 p = sPos[i];
        b200_vec3i q; q.x = p.x; q.y = p.y; q.z = p.z;
        visiblePos[baseN + i] = q;
        if (project_single_block(p.x, p.y, p.z, M, proj, w, h, voxelSize, ulx, uly, lrx, lry, zl, zh)) required = rendering_tiles(ulx, uly, lrx, lry);
      }
      unsigned chunkTiles;
      const unsigned before = running + block_exclusive_scan(required, sm, &chunkTiles);
      running += chunkTiles;
      const bool draw = required > 0 && before + required <= maxRB;   // :609
      unsigned todo = __ballot_sync(0xffffffffu, draw);
      while (todo) {
        const int src = __ffs(todo) - 1;
        todo &= todo - 1;
        const int ax = __shfl_sync(0xffffffffu, ulx, src), ay = __shfl_sync(0xffffffffu, uly, src);
        const int bx = __shfl_sync(0xffffffffu, lrx, src), by = __shfl_sync(0xffffffffu, lry, src);
        const float zn = __shfl_sync(0xffffffffu, zl, src), zx = __shfl_sync(0xffffffffu, zh, src);
        if ((bx - ax + 1) * (by - ay + 1) > 512) {
          int slot = -1;
          if (lane == 0) slot = atomicAdd(&sBigCount, 1);
          slot = __shfl_sync(0xffffffffu, slot, 0);
          if (slot < PV_BIG) {
            if (lane == 0) { BlockRec b; b.ulx = (short)ax; b.uly = (short)ay; b.lrx = (short)bx; b.lry = (short)by; b.zmin = zn; b.zmax = zx; sBig[slot] = b; }
            continue;
          }
        }
        raster_box_warp(minmax, w, ax, ay, bx, by, zn, zx);
      }
      __syncthreads();
      const int nBig = sBigCount < PV_BIG ? sBigCount : PV_BIG;
      for (int b = 0; b < nBig; ++b) {
        const BlockRec br = sBig[b];
        // rows of the box over the warps, columns over the lanes: no division per cell
        for (int yy = br.uly + (int)(threadIdx.x >> 5); yy <= br.lry; yy += 8)
          for (int xx = br.ulx + lane; xx <= br.lrx; xx += 32) {
            float2 *px = &minmax[xx + yy * w];
            atomic_min_posf(&px->x, br.zmin); atomic_max_posf(&px->y, br.zmax);
          }
      }
      __syncthreads();
      if (threadIdx.x == 0) sBigCount = 0;
    }
  }
}

// RenderImage's shading pass with two outputs: the RGBA pixel of `type` and the depth pixel (drawPixelDepth) from one read of
// the ray point. Either output may be null.
__global__ void __launch_bounds__(256)
k_preview_shade(const float4 *__restrict__ rays, const b200_voxel *__restrict__ voxels, const b200_hash_entry *__restrict__ table, int nb, int w,
                int h, Mat4 M, float lx, float ly, float lz, float voxelSize, int maxW, uchar4 *outChar, float *outDepth, int type) {
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

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static Mat4 to_mat(const float *m) { Mat4 r; memcpy(r.m, m, sizeof(r.m)); return r; }

static b200_status ensure_scratch(b200_engine *e) {
  if (e->pv) return B200_OK;
  PreviewScratch *p = new PreviewScratch();
  memset(p, 0, sizeof(*p));
  e->pv = p;                 // from here on preview_release frees whatever a failed step leaves behind
  const size_t noTiles = ((size_t)e->noTotal + PV_TILE - 1) / PV_TILE;
  CK(cudaMalloc(&p->d_ctr, sizeof(PreviewCounters)));
  CK(cudaMemset(p->d_ctr, 0, sizeof(PreviewCounters)));
  CK(cudaMallocHost(&p->h_count, 2 * sizeof(int)));
  CK(cudaMalloc(&p->d_descN, 2 * noTiles * sizeof(unsigned long long)));
  CK(cudaMemset(p->d_descN, 0, 2 * noTiles * sizeof(unsigned long long)));
  p->d_descT = p->d_descN + noTiles;
  CK(cudaEventCreateWithFlags(&p->evOut, cudaEventDisableTiming));
  return B200_OK;
}

void preview_release(b200_engine *e) {
  PreviewScratch *p = e->pv;
  if (!p) return;
  if (p->d2h) cudaStreamSynchronize(p->d2h);
  cudaFree(p->d_ctr); cudaFreeHost(p->h_count); cudaFree(p->d_descN);
  if (p->evOut) cudaEventDestroy(p->evOut);
  for (int i = 0; i < 2; ++i) {
    cudaFree(p->d_char[i]); cudaFree(p->d_depth[i]);
    if (p->evRender[i]) cudaEventDestroy(p->evRender[i]);
    if (p->evD2H[i]) cudaEventDestroy(p->evD2H[i]);
  }
  if (p->d2h) cudaStreamDestroy(p->d2h);
  delete p;
  e->pv = nullptr;
}

// every rejection of b200_render_view_async / _submit, before anything is allocated or enqueued
static b200_status check_view(b200_engine *e, const b200_scene *s, const b200_render_state *rs, const b200_camera *cam, int type,
                              const void *outChar, const void *outDepth) {
  b200_status st = check_scene(e, s); if (st) return st;
  if (!rs || !cam || !rs->d_visibleBlockPositions || !rs->d_minmax || !rs->d_raycastResult) {
    snprintf(e->err, sizeof(e->err), "render_view: render state, one of its buffers or the camera missing"); return B200_ERR_INVALID;
  }
  if (rs->img_w <= 0 || rs->img_h <= 0 || (long long)rs->img_w * rs->img_h >= (1ll << 31) / 4) {
    snprintf(e->err, sizeof(e->err), "render_view: render state size %dx%d", rs->img_w, rs->img_h); return B200_ERR_INVALID;
  }
  if (!outChar && !outDepth) { snprintf(e->err, sizeof(e->err), "render_view: both outputs are NULL"); return B200_ERR_INVALID; }
  if (type < B200_RENDER_SHADED_GREYSCALE || type >= B200_RENDER_DEPTH_MAP) {
    snprintf(e->err, sizeof(e->err), "render_view: type %d is not an RGBA render type (the depth map is the second output)", type);
    return B200_ERR_INVALID;
  }
  if (e->ptrListFor == (const void *)rs->d_visibleBlockPositions || (e->deadPending && e->deadMinmax == rs->d_minmax)) {
    snprintf(e->err, sizeof(e->err), "render_view: rs is the live render state of the volume being fused; use a free-view render state");
    return B200_ERR_INVALID;
  }
  return B200_OK;
}

static b200_status enqueue_view(b200_engine *e, const b200_scene *s, b200_render_state *rs, const b200_camera *cam, int type,
                                b200_vec4u *d_outChar, float *d_outDepth) {
  CK(cudaSetDevice(e->device));
  b200_status st = ensure_scratch(e); if (st) return st;
  PreviewScratch *p = e->pv;
  const SceneRef r = scene_ref(s, rs);
  const Mat4 M = to_mat(cam->M), invM = to_mat(cam->invM);
  const int w = rs->img_w, h = rs->img_h;
  k_preview_init<<<e->smCount * 4, 256, 0, e->stream>>>((float2 *)rs->d_minmax, w * h, p->d_ctr);
  const int noTiles = (r.noTotal + PV_TILE - 1) / PV_TILE;
  trace_begin(e, e->stream, "k_preview_sweep");
  k_preview_sweep<<<persistent_grid(e, 4, noTiles), 256, 0, e->stream>>>(r.hash, r.noTotal, r.visiblePos, r.numBlocks, p->d_ctr, p->d_descN,
                                                                        p->d_descT, ++p->gen, M, cam->proj[0], cam->proj[1], cam->proj[2],
                                                                        cam->proj[3], s->voxelSize, w, h, (float2 *)rs->d_minmax,
                                                                        (unsigned)e->maxRenderingBlocks);
  trace_end(e, e->stream);
  e->launches += 2;
  launch_raycast(e, r, invM, cam->proj, w, h, s->voxelSize, s->mu, rs->d_minmax, rs->d_raycastResult);
  const int tiles = ((w + 7) / 8) * ((h + 3) / 4);
  trace_begin(e, e->stream, "k_preview_shade");
  k_preview_shade<<<(tiles + 7) / 8, 256, 0, e->stream>>>((const float4 *)rs->d_raycastResult, r.voxels, r.hash, r.numBuckets, w, h, M, -invM.m[8],
                                                         -invM.m[9], -invM.m[10], s->voxelSize, s->maxW, (uchar4 *)d_outChar, d_outDepth, type);
  trace_end(e, e->stream);
  e->launches++;
  p->lastList = rs->d_visibleBlockPositions;
  CK(cudaGetLastError());
  return B200_OK;
}

static b200_status ensure_slots(b200_engine *e, size_t pixels) {
  b200_status st = ensure_scratch(e); if (st) return st;
  PreviewScratch *p = e->pv;
  if (!p->d2h) {
    CK(cudaStreamCreateWithFlags(&p->d2h, cudaStreamNonBlocking));
    for (int i = 0; i < 2; ++i) {
      CK(cudaEventCreateWithFlags(&p->evRender[i], cudaEventDisableTiming));
      CK(cudaEventCreateWithFlags(&p->evD2H[i], cudaEventDisableTiming));
    }
  }
  if (p->pixels >= pixels) return B200_OK;
  if (p->busy[0] || p->busy[1]) {
    snprintf(e->err, sizeof(e->err), "render_view_submit: a larger image needs both slots waited for first"); return B200_ERR_INVALID;
  }
  CK(cudaStreamSynchronize(e->stream));     // a waited-for slot's kernels are done; this covers staging a plain _async caller never sees
  for (int i = 0; i < 2; ++i) {
    cudaFree(p->d_char[i]); cudaFree(p->d_depth[i]); p->d_char[i] = nullptr; p->d_depth[i] = nullptr;
  }
  p->pixels = 0;
  for (int i = 0; i < 2; ++i) {
    CK(cudaMalloc(&p->d_char[i], pixels * sizeof(b200_vec4u)));
    CK(cudaMalloc(&p->d_depth[i], pixels * sizeof(float)));
  }
  p->pixels = pixels;
  return B200_OK;
}

// marks "everything enqueued on e's stream so far" in e's own event
static b200_status record_out(b200_engine *e) {
  CK(cudaSetDevice(e->device));
  b200_status st = ensure_scratch(e); if (st) return st;
  CK(cudaEventRecord(e->pv->evOut, e->stream));
  return B200_OK;
}

extern "C" {

b200_status b200_render_view_async(b200_engine *e, const b200_scene *scene, b200_render_state *rs, const b200_camera *cam,
                                   b200_render_type type, b200_vec4u *d_outChar, float *d_outDepth) {
  if (!e) return B200_ERR_INVALID;
  b200_status st = check_view(e, scene, rs, cam, (int)type, d_outChar, d_outDepth); if (st) return st;
  return enqueue_view(e, scene, rs, cam, (int)type, d_outChar, d_outDepth);
}

b200_status b200_render_view_sync(b200_engine *e, b200_render_state *rs) {
  if (!e) return B200_ERR_INVALID;
  if (!rs || !e->pv || e->pv->lastList != (const void *)rs->d_visibleBlockPositions) {
    snprintf(e->err, sizeof(e->err), "render_view_sync: rs is not the render state of this engine's latest free-view render");
    return B200_ERR_INVALID;
  }
  CK(cudaSetDevice(e->device));
  CK(cudaMemcpyAsync(e->pv->h_count, e->pv->d_ctr, 2 * sizeof(int), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  CK(cudaGetLastError());
  rs->noVisibleBlocks = e->pv->h_count[0];
  return B200_OK;
}

b200_status b200_render_view_submit(b200_engine *e, const b200_scene *scene, b200_render_state *rs, const b200_camera *cam,
                                    b200_render_type type, b200_vec4u *h_outChar, float *h_outDepth, int slot) {
  if (!e) return B200_ERR_INVALID;
  if (slot < 0 || slot > 1) { snprintf(e->err, sizeof(e->err), "slot must be 0 or 1"); return B200_ERR_INVALID; }
  b200_status st = check_view(e, scene, rs, cam, (int)type, h_outChar, h_outDepth); if (st) return st;
  if (e->pv && e->pv->busy[slot]) { snprintf(e->err, sizeof(e->err), "slot %d resubmitted before b200_render_view_wait", slot); return B200_ERR_INVALID; }
  CK(cudaSetDevice(e->device));
  const size_t px = (size_t)rs->img_w * rs->img_h;
  st = ensure_slots(e, px); if (st) return st;
  PreviewScratch *p = e->pv;
  b200_vec4u *dc = h_outChar ? p->d_char[slot] : nullptr;
  float *dd = h_outDepth ? p->d_depth[slot] : nullptr;
  // RENDER_COLOUR_FROM_NORMAL keeps the alpha of found pixels: over the engine's staging that is 0, the alpha of a fresh image
  if (dc && type == B200_RENDER_COLOUR_FROM_NORMAL) CK(cudaMemsetAsync(dc, 0, px * sizeof(b200_vec4u), e->stream));
  st = enqueue_view(e, scene, rs, cam, (int)type, dc, dd); if (st) return st;
  CK(cudaEventRecord(p->evRender[slot], e->stream));
  CK(cudaStreamWaitEvent(p->d2h, p->evRender[slot], 0));
  trace_begin(e, p->d2h, "d2h_preview");
  if (dc) CK(cudaMemcpyAsync(h_outChar, dc, px * sizeof(b200_vec4u), cudaMemcpyDeviceToHost, p->d2h));
  if (dd) CK(cudaMemcpyAsync(h_outDepth, dd, px * sizeof(float), cudaMemcpyDeviceToHost, p->d2h));
  trace_end(e, p->d2h);
  CK(cudaEventRecord(p->evD2H[slot], p->d2h));
  p->busy[slot] = true;
  return B200_OK;
}

b200_status b200_render_view_wait(b200_engine *e, int slot) {
  if (!e) return B200_ERR_INVALID;
  if (slot < 0 || slot > 1) { snprintf(e->err, sizeof(e->err), "slot must be 0 or 1"); return B200_ERR_INVALID; }
  if (!e->pv || !e->pv->busy[slot]) return B200_OK;   // nothing in flight on this slot
  CK(cudaEventSynchronize(e->pv->evD2H[slot]));
  e->pv->busy[slot] = false;
  return B200_OK;
}

b200_status b200_engine_wait_engine(b200_engine *e, b200_engine *producer) {
  if (!e) return B200_ERR_INVALID;
  if (!producer) { snprintf(e->err, sizeof(e->err), "wait_engine: producer missing"); return B200_ERR_INVALID; }
  if (producer == e || producer->stream == e->stream) return B200_OK;   // one stream: already ordered
  const b200_status st = record_out(producer);
  if (st) { snprintf(e->err, sizeof(e->err), "wait_engine: producer: %.400s", producer->err); return st; }
  CK(cudaSetDevice(e->device));
  CK(cudaStreamWaitEvent(e->stream, producer->pv->evOut, 0));
  return B200_OK;
}

}  // extern "C"
