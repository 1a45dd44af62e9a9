// preview.cu — the free-view preview: FindVisibleBlocks + CreateExpectedDepths + RenderImage(type) + RenderImage(DEPTH_MAP)
// from one pose as ONE enqueue (b200_render_view_async), its pipelined hand-over to the host (b200_render_view_submit /
// _wait) and the device-side ordering between engines that compositing several volumes' previews needs
// (b200_engine_wait_engine).
//
// Replaces, for this use, the reference's stop-and-go shape (ITMMainEngine::GetImage for the FREECAMERA types,
// ITMMainEngine.cpp:231-278, called twice per volume by DynSLAM: once for the RGBA image, once more for the depth): the
// stand-alone calls' kernels (vis.cu) enqueued back to back — k_freeview_list, k_minmax_reset, k_expected_depths (the
// MAX_RENDERING_BLOCKS rule decided on the device), k_raycast, and k_shade writing both images from one read of the ray
// point — five launches, no host synchronisation, one raycast shaded two ways. This file is the host side only.
//
// Nothing here touches the volume's counters (DevCounters), the block records or the scan descriptors of the fused frame: the
// preview has a counter block, descriptors and staging of its own, so it can be enqueued between asynchronous frames.
#include "engine.h"

#include <cstdio>
#include <cstring>

struct PreviewCounters {
  int noVisible;         // blocks the sweep listed (not capped by the list's capacity, as FindVisibleBlocks' count is not)
  unsigned noTiles;      // rendering tiles of the listed blocks (CreateExpectedDepths' noTotalBlocks before the cap)
  unsigned ticket;       // k_freeview_list: next table tile to hand out
  unsigned ctasDone;     // k_expected_depths: CTAs that have finished
};

struct PreviewScratch {
  PreviewCounters *d_ctr;
  int *h_count;                          // pinned: noVisible, noTiles as b200_render_view_sync reads them back
  unsigned long long *d_desc;            // chained-scan descriptors of the list sweep
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
// host side
// ------------------------------------------------------------------------------------------------
static Mat4 to_mat(const float *m) { Mat4 r; memcpy(r.m, m, sizeof(r.m)); return r; }

static b200_status ensure_scratch(b200_engine *e) {
  if (e->pv) return B200_OK;
  PreviewScratch *p = new PreviewScratch();
  memset(p, 0, sizeof(*p));
  e->pv = p;                 // from here on preview_release frees whatever a failed step leaves behind
  const size_t noTiles = ((size_t)e->noTotal + FV_TILE - 1) / FV_TILE;
  CK(cudaMalloc(&p->d_ctr, sizeof(PreviewCounters)));
  CK(cudaMemset(p->d_ctr, 0, sizeof(PreviewCounters)));
  CK(cudaMallocHost(&p->h_count, 2 * sizeof(int)));
  CK(cudaMalloc(&p->d_desc, noTiles * sizeof(unsigned long long)));
  CK(cudaMemset(p->d_desc, 0, noTiles * sizeof(unsigned long long)));
  CK(cudaEventCreateWithFlags(&p->evOut, cudaEventDisableTiming));
  return B200_OK;
}

void preview_release(b200_engine *e) {
  PreviewScratch *p = e->pv;
  if (!p) return;
  if (p->d2h) cudaStreamSynchronize(p->d2h);
  cudaFree(p->d_ctr); cudaFreeHost(p->h_count); cudaFree(p->d_desc);
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

bool preview_slot_busy(const b200_engine *e) { return e->pv && (e->pv->busy[0] || e->pv->busy[1]); }

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
  PreviewCounters *c = p->d_ctr;
  launch_find_visible(e, r, M, cam->proj, w, h, s->voxelSize, &c->noVisible, &c->ticket, p->d_desc, ++p->gen);
  launch_expected_depths(e, r, M, cam->proj, w, h, s->voxelSize, rs->d_minmax, &c->noVisible, &c->noTiles, &c->ctasDone);
  launch_raycast(e, r, invM, cam->proj, w, h, s->voxelSize, s->mu, rs->d_minmax, rs->d_raycastResult);
  launch_shade(e, r, M, invM, w, h, s->voxelSize, s->maxW, rs->d_raycastResult, d_outChar, d_outDepth, type);
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
