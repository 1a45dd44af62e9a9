// engine.cu — the extern "C" boundary of libb200fusion (include/b200fusion.h) and the host-side
// sequencing of one volume's engine.
//
// Mirrors the host bodies of the reference engines (ITMSceneReconstructionEngine_CUDA.cu:115-566,
// ITMVisualisationEngine_CUDA.cu:109-533, ITMSwappingEngine_CUDA.cu:20-216) with one structural
// change: the reference blocks on the host four times per frame to move 4-12 byte counters, and
// allocates/frees device memory every frame for the decay snapshot. Here the counters live in a
// device struct that kernels update and read; the synchronous entry points (the ones the ITMLib
// shim calls, which must return with host-visible counters valid) do exactly one asynchronous
// upload, the launches, one asynchronous download and one stream synchronise; the fused
// b200_process_frame_async path does none of that until b200_sync().
#include "engine.h"
#include "../../include/b200fusion_diag.h"

#include <cstdio>
#include <cstdlib>
#include <cstring>

#define CK(call)                                                                                   \
  do {                                                                                             \
    cudaError_t _e = (call);                                                                       \
    if (_e != cudaSuccess) {                                                                       \
      snprintf(e->err, sizeof(e->err), "%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(_e)); \
      return B200_ERR_CUDA;                                                                        \
    }                                                                                              \
  } while (0)

static Mat4 to_mat(const float *m) { Mat4 r; memcpy(r.m, m, sizeof(r.m)); return r; }

// lhs * rhs for column-major 4x4 (m[col*4+row]), accumulated over k in ascending order from 0.0f like the reference's
// operator* (OR/Matrix.h:102-108) so that CreatePointCloud's invM * calib keeps its bits
static void mat_mul(const float *lhs, const float *rhs, float *out) {
  float r[16];
  for (int c = 0; c < 4; ++c) for (int row = 0; row < 4; ++row) {
    float acc = 0.0f;
    for (int k = 0; k < 4; ++k) acc += lhs[k * 4 + row] * rhs[c * 4 + k];
    r[c * 4 + row] = acc;
  }
  memcpy(out, r, sizeof(r));
}

static SceneRef scene_ref(const b200_scene *s, const b200_render_state *rs) {
  SceneRef r;
  r.voxels = s->d_voxels; r.allocationList = s->d_allocationList; r.hash = s->d_hash; r.excessList = s->d_excessList;
  r.swapStates = s->d_swapStates;
  r.numBlocks = s->numBlocks; r.numBuckets = s->numBuckets; r.excessSize = s->excessSize; r.noTotal = s->numBuckets + s->excessSize;
  r.visiblePos = rs ? rs->d_visibleBlockPositions : nullptr;
  r.visType = rs ? rs->d_entriesVisibleType : nullptr;
  return r;
}

static FrameGeom frame_geom(const b200_scene *s, const b200_view *v) {
  FrameGeom g;
  g.M_d = to_mat(v->M_d); g.invM_d = to_mat(v->invM_d); g.M_rgb = to_mat(v->M_rgb);
  memcpy(g.proj_d, v->proj_d, sizeof(g.proj_d)); memcpy(g.proj_rgb, v->proj_rgb, sizeof(g.proj_rgb));
  g.w = v->depth_w; g.h = v->depth_h; g.rgb_w = v->rgb_w; g.rgb_h = v->rgb_h;
  g.voxelSize = s->voxelSize; g.mu = s->mu; g.maxW = s->maxW; g.vfmin = s->viewFrustum_min; g.vfmax = s->viewFrustum_max;
  g.depthWeighting = v->depthWeighting; g.stopMaxW = s->stopIntegratingAtMaxW; g.approx = !v->requiresFullRendering;
  { volatile float a = -1.0f, b = s->mu; g.negOneOverMu = a / b; }
  g.sameRgbCam = (memcmp(v->M_rgb, v->M_d, sizeof(v->M_d)) == 0 && memcmp(v->proj_rgb, v->proj_d, sizeof(v->proj_d)) == 0 &&
                  v->rgb_w == v->depth_w && v->rgb_h == v->depth_h) ? 1 : 0;
  return g;
}

static b200_status check_scene(b200_engine *e, const b200_scene *s) {
  if (!s || s->numBlocks > e->numBlocks || s->numBuckets != e->numBuckets || s->excessSize != e->excessSize ||
      (s->numBuckets & (s->numBuckets - 1))) {
    snprintf(e->err, sizeof(e->err), "scene sizes do not match the engine configuration");
    return B200_ERR_INVALID;
  }
  return B200_OK;
}

// host -> device counters (only the three the host owns); device -> host (everything)
static b200_status upload(b200_engine *e, const b200_scene *s, const b200_render_state *rs) {
  // Frames enqueued by the asynchronous entry points since the last b200_sync() have moved the device counters on: the
  // host copies are stale then and must not be written over them (the call's own download refreshes the host fields).
  if (!e->hostAuthoritative) return B200_OK;
  int *in = reinterpret_cast<int *>(e->h_ctr + 1);   // second pinned struct = upload staging
  in[0] = s->lastFreeBlockId; in[1] = s->lastFreeExcessListId; in[2] = rs ? rs->noVisibleBlocks : 0;
  CK(cudaMemcpyAsync(e->d_ctr, in, rs ? 3 * sizeof(int) : 2 * sizeof(int), cudaMemcpyHostToDevice, e->stream));
  return B200_OK;
}

static b200_status download_sync(b200_engine *e, b200_scene *s, b200_render_state *rs) {
  CK(cudaMemcpyAsync(e->h_ctr, e->d_ctr, sizeof(DevCounters), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  CK(cudaGetLastError());
  if (s) { s->lastFreeBlockId = e->h_ctr->lastFreeBlockId; s->lastFreeExcessListId = e->h_ctr->lastFreeExcessListId; }
  if (rs) { rs->noVisibleBlocks = e->h_ctr->noVisibleBlocks; }
  e->totalDecayed = e->h_ctr->totalDecayed;
  e->lastNoIntegrated = e->h_ctr->noIntegrated;
  e->hostAuthoritative = true;
  return B200_OK;
}

extern "C" {

static b200_status engine_create_body(const b200_engine_config *cfg, b200_engine *e);
static void read_switches(b200_engine *e);

static thread_local char g_createErr[512] = "";

b200_status b200_engine_create(const b200_engine_config *cfg, b200_engine **out) {
  if (out) *out = nullptr;
  if (!cfg || !out) { snprintf(g_createErr, sizeof(g_createErr), "null configuration or output pointer"); return B200_ERR_INVALID; }
  b200_engine *e = new b200_engine();
  memset(e, 0, sizeof(*e));
  const b200_status st = engine_create_body(cfg, e);
  if (st != B200_OK) {          // nothing stays allocated after a failed create; the reason survives in b200_last_error(NULL)
    snprintf(g_createErr, sizeof(g_createErr), "%s", e->err);
    b200_engine_destroy(e);
    return st;
  }
  *out = e;
  return B200_OK;
}

static b200_status engine_create_body(const b200_engine_config *cfg, b200_engine *e) {
  e->maxRenderingBlocks = B200_MAX_RENDERING_BLOCKS;
  e->device = cfg->device;
  e->numBlocks = cfg->numBlocks; e->numBuckets = cfg->numBuckets; e->excessSize = cfg->excessSize;
  e->noTotal = cfg->numBuckets + cfg->excessSize; e->img_w = cfg->img_w; e->img_h = cfg->img_h;
  if (cfg->numBlocks <= 0 || cfg->numBuckets <= 0 || (cfg->numBuckets & (cfg->numBuckets - 1)) || cfg->excessSize < 0 ||
      (long long)cfg->img_w * cfg->img_h >= (1ll << 24) || (e->noTotal % 32) != 0) {
    snprintf(e->err, sizeof(e->err), "invalid engine configuration");
    return B200_ERR_INVALID;
  }
  CK(cudaSetDevice(e->device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, e->device));
  e->smCount = prop.multiProcessorCount;
  if (prop.major != 9 || prop.minor != 0) {     // sm_90a code runs on compute capability 9.0 only
    snprintf(e->err, sizeof(e->err), "libb200fusion is built for sm_90a; device %d is sm_%d%d", e->device, prop.major, prop.minor);
    return B200_ERR_UNSUPPORTED;
  }
  if (cfg->stream) { e->stream = (cudaStream_t)cfg->stream; e->ownStream = false; }
  else { CK(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking)); e->ownStream = true; }
  CK(cudaMalloc(&e->d_ctr, sizeof(DevCounters)));
  CK(cudaMemset(e->d_ctr, 0, sizeof(DevCounters)));
  CK(cudaMallocHost(&e->h_ctr, 2 * sizeof(DevCounters)));
  memset(e->h_ctr, 0, 2 * sizeof(DevCounters));
  e->noWords = e->noTotal / 32;
  CK(cudaMalloc(&e->d_reqKey, sizeof(unsigned long long) * (size_t)e->noTotal));
  CK(cudaMemset(e->d_reqKey, 0, sizeof(unsigned long long) * (size_t)e->noTotal));
  CK(cudaMalloc(&e->d_reqBits, sizeof(unsigned) * (size_t)e->noWords * 2));
  e->d_req2Bits = e->d_reqBits + e->noWords;
  CK(cudaMemset(e->d_reqBits, 0, sizeof(unsigned) * (size_t)e->noWords * 2));   // kept clean by k_serve_list from here on
  CK(cudaMalloc(&e->d_dbg, B200_DBG_WORDS * sizeof(unsigned long long)));
  CK(cudaMemset(e->d_dbg, 0, B200_DBG_WORDS * sizeof(unsigned long long)));
  CK(cudaMalloc(&e->d_markBytes, (size_t)e->noTotal));
  CK(cudaMemset(e->d_markBytes, 0, (size_t)e->noTotal));
  long long px = (long long)e->img_w * e->img_h;
  long long maxTiles = (e->noTotal + 255) / 256 + (px + 255) / 256 + e->numBlocks / 256 + 1024;
  e->scanDescCap = (int)maxTiles;
  CK(cudaMalloc(&e->d_scanDesc, sizeof(unsigned long long) * (size_t)e->scanDescCap));
  CK(cudaMemset(e->d_scanDesc, 0, sizeof(unsigned long long) * (size_t)e->scanDescCap));
  e->ringCap = cfg->decayRingItems > 0 ? cfg->decayRingItems : 24ll * e->numBlocks;
  if (e->ringCap < e->numBlocks) e->ringCap = e->numBlocks;   // one frame's list (at most numBlocks items) always fits: k_serve_list wraps with one subtraction
  CK(cudaMalloc(&e->d_ring, sizeof(b200_vec3i) * (size_t)e->ringCap));
  CK(cudaMalloc(&e->d_snapCount, sizeof(int) * SNAP_SLOTS));
  CK(cudaMalloc(&e->d_snapStart, sizeof(long long) * SNAP_SLOTS));
  CK(cudaMemset(e->d_snapCount, 0, sizeof(int) * SNAP_SLOTS));
  CK(cudaMemset(e->d_snapStart, 0, sizeof(long long) * SNAP_SLOTS));
  CK(cudaMalloc(&e->d_delTag, sizeof(unsigned long long) * (size_t)e->numBlocks));
  CK(cudaMemset(e->d_delTag, 0, sizeof(unsigned long long) * (size_t)e->numBlocks));
  CK(cudaMalloc(&e->d_visiblePtr, sizeof(int) * (size_t)e->numBlocks));
  CK(cudaMalloc(&e->d_itemPtr, sizeof(int) * (size_t)e->numBlocks));
  CK(cudaMalloc(&e->d_delList, sizeof(int) * (size_t)e->numBlocks));
  CK(cudaMalloc(&e->d_candList, sizeof(int) * DECAY_CAND_CAP));
  CK(cudaMalloc(&e->d_isLeader, (size_t)e->numBlocks));
  CK(cudaMalloc(&e->d_allocatedPos, sizeof(short4) * (size_t)e->numBlocks));
  CK(cudaMalloc(&e->d_blockRecs, 16 * (size_t)e->numBlocks));
  CK(cudaMalloc(&e->d_tileCounts, sizeof(unsigned) * (size_t)(px > 0 ? px : 1)));
  for (int i = 0; i < 8; ++i) CK(cudaEventCreate(&e->ev[i]));
  if (!getenv("B200_NO_OVERLAP")) {
    CK(cudaStreamCreateWithFlags(&e->sideStream, cudaStreamNonBlocking));
    CK(cudaEventCreateWithFlags(&e->evFork, cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&e->evJoin, cudaEventDisableTiming));
  }
  e->hostAuthoritative = true;
  read_switches(e);
  integrate_init_device(e);     // per-device tables and function attributes of integrate.cu (one engine per GPU is the multi-GPU unit)
  CK(cudaGetLastError());
  return B200_OK;
}

// The run-time switches (README) are read once per engine, here: an engine keeps the values it was created with, and an
// engine created after a variable was set or removed gets the new value (nothing is remembered per process).
static void read_switches(b200_engine *e) {
  const char *v;
  // default: V4 (packed-pair arithmetic, integrate.cu); B200_INTEGRATE_IMPL = v3 | tma | ldg select the earlier bit-exact variants,
  // fast = V4 in tolerance mode (TSDF within 1 LSB of the 16-bit code, everything else bit-exact)
  v = getenv("B200_INTEGRATE_IMPL");
  e->integrateImpl = !v ? 3 : (v[0] == 'l' ? 0 : (v[0] == 't' ? 1 : (v[0] == 'f' ? 4 : ((v[0] == 'v' && v[1] == '3') ? 2 : 3))));
  v = getenv("B200_V4_PPL"); e->pplV4 = (v && (atoi(v) == 1 || atoi(v) == 2)) ? atoi(v) : 0;
  v = getenv("B200_V4_TAIL"); e->v4TailFloor = (v && atoi(v) >= 1 && atoi(v) <= 6) ? atoi(v) : 3;
  v = getenv("B200_V3_PREFETCH"); e->v3Prefetch = v ? atoi(v) != 0 : true;
  v = getenv("B200_V3_CTAS"); e->ctasV3 = (v && (atoi(v) == 2 || atoi(v) == 4)) ? atoi(v) : 3;   // 3: 72 registers per thread; 4 = 56, 2 = 96
  v = getenv("B200_INTEGRATE_REGS"); e->regsTma = (v && atoi(v) == 56) ? 56 : 48;
  v = getenv("B200_INTEGRATE_CTAS"); e->ctasTma = v ? atoi(v) : 0;   // an upper bound; integrate_init_device sets the count
  v = getenv("B200_RC_TILE"); e->rcTileLog2 = v ? atoi(v) : 3; if (e->rcTileLog2 < 0 || e->rcTileLog2 > 5) e->rcTileLog2 = 3;
  v = getenv("B200_RC_ORDER"); e->rcOrder = v ? atoi(v) : 1;
  v = getenv("B200_RC_IMPL"); e->rcImpl = (v && v[0] == 'o') ? 0 : 1;
  v = getenv("B200_GRAPH"); e->useGraph = (v && atoi(v) != 0) ? 1 : 0;
  e->lastIntegrateKernel = -1; e->lastIntegrateGrid = 0;
}

void b200_engine_destroy(b200_engine *e) {
  if (!e) return;
  cudaSetDevice(e->device);
  if (e->stream) cudaStreamSynchronize(e->stream);
  cudaFree(e->d_ctr); cudaFreeHost(e->h_ctr); cudaFree(e->d_reqKey); cudaFree(e->d_reqBits); cudaFree(e->d_markBytes); cudaFree(e->d_dbg); cudaFree(e->d_meshDesc); cudaFree(e->d_evalCounters); cudaFreeHost(e->h_evalCounters); cudaFree(e->d_scanDesc);
  cudaFree(e->d_ring); cudaFree(e->d_snapCount); cudaFree(e->d_snapStart); cudaFree(e->d_delTag); cudaFree(e->d_itemPtr); cudaFree(e->d_visiblePtr);
  cudaFree(e->d_viewScratch); cudaFree(e->d_delList); cudaFree(e->d_candList); cudaFree(e->d_isLeader); cudaFree(e->d_allocatedPos); cudaFree(e->d_tileCounts); cudaFree(e->d_blockRecs);
  for (int i = 0; i < 8; ++i) if (e->ev[i]) cudaEventDestroy(e->ev[i]);
  if (e->copyStream) {
    cudaStreamSynchronize(e->copyStream);
    for (int i = 0; i < 2; ++i) { cudaFree(e->d_stageDepth[i]); cudaFree(e->d_stageRgb[i]); cudaFree(e->d_stageOut[i]); cudaFree(e->d_stageRaw[i]);
      if (e->evH2D[i]) cudaEventDestroy(e->evH2D[i]); if (e->evCompute[i]) cudaEventDestroy(e->evCompute[i]); if (e->evD2H[i]) cudaEventDestroy(e->evD2H[i]); }
    cudaStreamDestroy(e->copyStream);
    if (e->d2hStream) { cudaStreamSynchronize(e->d2hStream); cudaStreamDestroy(e->d2hStream); }
    if (e->evMid) cudaEventDestroy(e->evMid);
  }
  if (e->frameGraph) cudaGraphExecDestroy(e->frameGraph);
  if (e->sideStream) { cudaStreamSynchronize(e->sideStream); if (e->evFork) cudaEventDestroy(e->evFork); if (e->evJoin) cudaEventDestroy(e->evJoin); cudaStreamDestroy(e->sideStream); }
  if (e->evRing) { for (int i = 0; i < e->evRingCap * 2; ++i) cudaEventDestroy(e->evRing[i]); free(e->evRing); }
  if (e->traceEv) { for (int i = 0; i < e->traceCap * 2; ++i) cudaEventDestroy(e->traceEv[i]); free(e->traceEv); free(e->traceName); }
  cudaGetLastError();
  if (e->ownStream && e->stream) cudaStreamDestroy(e->stream);
  delete e;
}

const char *b200_last_error(const b200_engine *e) { return e ? e->err : g_createErr; }
void *b200_engine_stream(b200_engine *e) { return (void *)e->stream; }
int32_t b200_frame_index(const b200_engine *e) { return e->frameIdx; }
size_t b200_decayed_block_count(const b200_engine *e) { return (size_t)e->totalDecayed; }
void b200_set_timing(b200_engine *e, int mode) {
  e->timing = mode != 0;
  e->evRingCount = 0;
  if (mode >= 2 && !e->evRing) {
    e->evRingCap = 8192;
    e->evRing = (cudaEvent_t *)calloc((size_t)e->evRingCap * 2, sizeof(cudaEvent_t));
    for (int i = 0; i < e->evRingCap * 2; ++i) cudaEventCreate(&e->evRing[i]);
  }
  e->timingMode = mode;
  e->traceOn = mode == 3;
  e->traceCount = 0;
  if (mode == 3 && !e->traceEv) {
    e->traceCap = 4096;
    e->traceEv = (cudaEvent_t *)calloc((size_t)e->traceCap * 2, sizeof(cudaEvent_t));
    e->traceName = (const char **)calloc((size_t)e->traceCap, sizeof(char *));
    for (int i = 0; i < e->traceCap * 2; ++i) cudaEventCreate(&e->traceEv[i]);
  }
}

// Text dump of the launch trace: one line per launch, "name start_us end_us" relative to the first launch's begin event.
int b200_get_trace(b200_engine *e, char *out, int cap) {
  if (!e->traceEv || e->traceCount == 0 || cap <= 0) { if (cap > 0) out[0] = 0; return 0; }
  cudaSetDevice(e->device);
  cudaDeviceSynchronize();
  int n = 0;
  for (int i = 0; i < e->traceCount; ++i) {
    float a = 0, b = 0;
    cudaEventElapsedTime(&a, e->traceEv[0], e->traceEv[2 * i]);
    cudaEventElapsedTime(&b, e->traceEv[0], e->traceEv[2 * i + 1]);
    int w = snprintf(out + n, (size_t)(cap - n), "%s %.2f %.2f\n", e->traceName[i], a * 1000.0f, b * 1000.0f);
    if (w < 0 || w >= cap - n) break;
    n += w;
  }
  e->traceCount = 0;
  return n;
}

void b200_diag_set_max_rendering_blocks(b200_engine *e, int n) { e->maxRenderingBlocks = n > 0 ? n : B200_MAX_RENDERING_BLOCKS; }

void b200_diag_last_integrate(const b200_engine *e, int *kernel, int *grid) {
  if (kernel) *kernel = e->lastIntegrateKernel;
  if (grid) *grid = e->lastIntegrateGrid;
}

int b200_diag_read_debug(b200_engine *e, unsigned long long *out, int n) {
  if (!e || !out || n <= 0) return 0;
  if (n > B200_DBG_WORDS) n = B200_DBG_WORDS;
  cudaSetDevice(e->device);
  cudaDeviceSynchronize();
  return cudaMemcpy(out, e->d_dbg, sizeof(unsigned long long) * (size_t)n, cudaMemcpyDeviceToHost) == cudaSuccess ? n : 0;
}

// ---- ITMSceneReconstructionEngine ---------------------------------------------------------------

b200_status b200_reset_scene(b200_engine *e, b200_scene *s) {
  b200_status st = check_scene(e, s); if (st) return st;
  CK(cudaSetDevice(e->device));
  e->totalDecayed = 0;
  e->qHead += e->qSize; e->qSize = 0;          // clear the decay queue; frameIdx is NOT reset (Reco_CUDA.cu:150-155)
  e->deadPending = false;
  e->tableVersion++;
  launch_reset(e, scene_ref(s, nullptr));
  return download_sync(e, s, nullptr);
}

// Host half of a decay-queue push: the slot the next snapshot goes to, now counted in the queue. The reference's queue of
// visible-list copies is unbounded (Reco_CUDA.cu:302-317); this one has SNAP_SLOTS frame slots and a ring of list items.
// When Decay() is never called (--voxel_decay=false) or min_decay_age is very large, the OLDEST snapshot is dropped to make
// room — never an error (the ring's item overflow is handled the same way on the device: decay.cu recognises an overwritten
// snapshot by its start position and sweeps nothing).
static int push_snapshot_slot(b200_engine *e) {
  if (e->qSize >= SNAP_SLOTS - 1) { e->qHead++; e->qSize--; e->droppedSnapshots++; }
  const int slot = (e->qHead + e->qSize) % SNAP_SLOTS;
  e->qSize++;
  return slot;
}

static b200_status enqueue_allocate(b200_engine *e, b200_scene *s, b200_render_state *rs, const b200_view *v, int onlyVisible,
                                    bool fuseDeadInit = false) {
  if (v->depth_w != e->img_w || v->depth_h != e->img_h) {
    snprintf(e->err, sizeof(e->err), "view size %dx%d differs from engine %dx%d", v->depth_w, v->depth_h, e->img_w, e->img_h);
    return B200_ERR_INVALID;
  }
  const int slot = push_snapshot_slot(e);
  e->tableVersion++;
  launch_allocate(e, scene_ref(s, rs), frame_geom(s, v), v->d_depth, onlyVisible != 0, e->frameIdx, slot,
                  fuseDeadInit ? rs->d_minmax : nullptr, rs->img_w, rs->img_h);
  e->ptrListFor = rs->d_visibleBlockPositions; e->ptrListVersion = e->tableVersion;
  e->frameIdx++;
  return B200_OK;
}

b200_status b200_diag_push_decay_snapshot(b200_engine *e, const b200_vec3i *d_positions, int n) {
  if (n < 0 || n > e->numBlocks || (n > 0 && !d_positions)) {
    snprintf(e->err, sizeof(e->err), "a decay snapshot holds 0 to numBlocks (%d) positions, got %d", e->numBlocks, n);
    return B200_ERR_INVALID;
  }
  CK(cudaSetDevice(e->device));
  launch_push_snapshot(e, d_positions, n, push_snapshot_slot(e));
  CK(cudaStreamSynchronize(e->stream));
  CK(cudaGetLastError());
  return B200_OK;
}

void b200_diag_set_frame_index(b200_engine *e, int32_t f) { e->frameIdx = f; }

b200_status b200_allocate_from_depth(b200_engine *e, b200_scene *s, b200_render_state *rs, const b200_view *v, int onlyVisible) {
  b200_status st = check_scene(e, s); if (st) return st;
  CK(cudaSetDevice(e->device));
  st = upload(e, s, rs); if (st) return st;
  st = enqueue_allocate(e, s, rs, v, onlyVisible); if (st) return st;
  st = download_sync(e, s, rs); if (st) return st;
  if (s->lastFreeBlockId < 0) { snprintf(e->err, sizeof(e->err), "out of space in the voxel block array"); return B200_ERR_VBA_FULL; }
  if (s->lastFreeExcessListId < 0) { snprintf(e->err, sizeof(e->err), "out of slots in the hash table excess list"); return B200_ERR_EXCESS_FULL; }
  return B200_OK;
}

b200_status b200_integrate(b200_engine *e, b200_scene *s, b200_render_state *rs, const b200_view *v) {
  b200_status st = check_scene(e, s); if (st) return st;
  CK(cudaSetDevice(e->device));
  if (rs->noVisibleBlocks == 0) return B200_OK;   // Reco_CUDA.cu:372-378
  st = upload(e, s, rs); if (st) return st;
  CK(cudaMemsetAsync(&e->d_ctr->noIntegrated, 0, sizeof(int), e->stream));
  launch_integrate(e, scene_ref(s, rs), frame_geom(s, v), v->d_depth, v->d_rgb);
  return download_sync(e, s, rs);
}

static void enqueue_decay(b200_engine *e, b200_scene *s, b200_render_state *rs, int maxWeight, int minAge, int forceAll) {
  SceneRef r = scene_ref(s, rs);
  e->tableVersion++;
  if (forceAll) launch_decay_full(e, r, minAge, maxWeight, e->frameIdx);
  else if ((long)e->qSize > minAge) {
    const int slot = e->qHead % SNAP_SLOTS;
    e->qHead++; e->qSize--;
    launch_decay_partial(e, r, slot, minAge, maxWeight, e->frameIdx);
  }
}

b200_status b200_decay(b200_engine *e, b200_scene *s, b200_render_state *rs, int maxWeight, int minAge, int forceAll) {
  b200_status st = check_scene(e, s); if (st) return st;
  CK(cudaSetDevice(e->device));
  st = upload(e, s, rs); if (st) return st;
  enqueue_decay(e, s, rs, maxWeight, minAge, forceAll);
  return download_sync(e, s, rs);
}

// ---- ITMVisualisationEngine ---------------------------------------------------------------------

b200_status b200_find_visible_blocks(b200_engine *e, const b200_scene *s, b200_render_state *rs, const b200_camera *cam) {
  b200_status st = check_scene(e, s); if (st) return st;
  CK(cudaSetDevice(e->device));
  st = upload(e, s, rs); if (st) return st;
  if (e->ptrListFor == (const void *)rs->d_visibleBlockPositions) e->ptrListFor = nullptr;   // list rebuilt without ptrs
  launch_find_visible(e, scene_ref(s, rs), to_mat(cam->M), cam->proj, rs->img_w, rs->img_h, s->voxelSize);
  return download_sync(e, nullptr, rs);
}

b200_status b200_expected_depths(b200_engine *e, const b200_scene *s, b200_render_state *rs, const b200_camera *cam) {
  b200_status st = check_scene(e, s); if (st) return st;
  CK(cudaSetDevice(e->device));
  st = upload(e, s, rs); if (st) return st;
  e->deadPending = false;      // the whole image is rebuilt here
  // one pass with atomics; it counts the rendering tiles, and only if they break MAX_RENDERING_BLOCKS (whose rule depends on the
  // list order) the ordered two-kernel form rebuilds the image
  launch_expected_depths_fast(e, scene_ref(s, rs), to_mat(cam->M), cam->proj, rs->img_w, rs->img_h, s->voxelSize, rs->d_minmax);
  st = download_sync(e, nullptr, nullptr); if (st) return st;
  if (e->h_ctr->noRenderingBlocks <= (unsigned)e->maxRenderingBlocks) return B200_OK;
  launch_expected_depths(e, scene_ref(s, rs), to_mat(cam->M), cam->proj, rs->img_w, rs->img_h, s->voxelSize, rs->d_minmax);
  return download_sync(e, nullptr, nullptr);
}

b200_status b200_find_surface(b200_engine *e, const b200_scene *s, b200_render_state *rs, const b200_camera *cam) {
  b200_status st = check_scene(e, s); if (st) return st;
  CK(cudaSetDevice(e->device));
  launch_raycast(e, scene_ref(s, rs), to_mat(cam->invM), cam->proj, rs->img_w, rs->img_h, s->voxelSize, s->mu, rs->d_minmax,
                 rs->d_raycastResult);
  CK(cudaStreamSynchronize(e->stream));
  CK(cudaGetLastError());
  return B200_OK;
}

b200_status b200_render_image(b200_engine *e, const b200_scene *s, b200_render_state *rs, const b200_camera *cam, b200_vec4u *d_outChar,
                              float *d_outFloat, int out_w, int out_h, b200_render_type type) {
  b200_status st = check_scene(e, s); if (st) return st;
  CK(cudaSetDevice(e->device));
  SceneRef r = scene_ref(s, rs);
  launch_raycast(e, r, to_mat(cam->invM), cam->proj, out_w, out_h, s->voxelSize, s->mu, rs->d_minmax, rs->d_raycastResult);
  launch_shade(e, r, to_mat(cam->M), to_mat(cam->invM), out_w, out_h, s->voxelSize, s->maxW, rs->d_raycastResult, d_outChar, d_outFloat,
               (int)type);
  CK(cudaStreamSynchronize(e->stream));
  CK(cudaGetLastError());
  return B200_OK;
}

b200_status b200_icp_maps(b200_engine *e, const b200_scene *s, b200_render_state *rs, const b200_view *v, b200_vec4f *d_points,
                          b200_vec4f *d_normals) {
  b200_status st = check_scene(e, s); if (st) return st;
  CK(cudaSetDevice(e->device));
  Mat4 invM = to_mat(v->invM_d);
  launch_raycast(e, scene_ref(s, rs), invM, v->proj_d, rs->img_w, rs->img_h, s->voxelSize, s->mu, rs->d_minmax, rs->d_raycastResult);
  launch_icp(e, invM, rs->img_w, rs->img_h, s->voxelSize, rs->d_raycastResult, rs->d_raycastImage, d_points, d_normals);
  CK(cudaStreamSynchronize(e->stream));
  CK(cudaGetLastError());
  return B200_OK;
}

b200_status b200_forward_render(b200_engine *e, const b200_scene *s, b200_render_state *rs, const b200_view *v) {
  b200_status st = check_scene(e, s); if (st) return st;
  CK(cudaSetDevice(e->device));
  if (!rs->d_forwardProjection || !rs->d_fwdProjMissingPoints) { snprintf(e->err, sizeof(e->err), "forward buffers missing"); return B200_ERR_INVALID; }
  launch_forward_render(e, scene_ref(s, rs), frame_geom(s, v), v->d_depth, rs->d_minmax, rs->d_raycastResult, rs->d_forwardProjection,
                        rs->d_fwdProjMissingPoints, rs->d_raycastImage);
  st = download_sync(e, nullptr, nullptr);
  rs->noFwdProjMissingPoints = e->h_ctr->noFwdMissing;
  return st;
}

b200_status b200_point_cloud(b200_engine *e, const b200_scene *s, b200_render_state *rs, const b200_view *v, const float *calib,
                             int skipPoints, b200_vec4f *d_locations, b200_vec4f *d_colours, uint32_t *noTotalPoints) {
  b200_status st = check_scene(e, s); if (st) return st;
  CK(cudaSetDevice(e->device));
  float invMf[16];
  mat_mul(v->invM_d, calib, invMf);
  Mat4 invM = to_mat(invMf);
  SceneRef r = scene_ref(s, rs);
  launch_raycast(e, r, invM, v->proj_rgb, rs->img_w, rs->img_h, s->voxelSize, s->mu, rs->d_minmax, rs->d_raycastResult);
  launch_point_cloud(e, r, invM, rs->img_w, rs->img_h, s->voxelSize, skipPoints, rs->d_raycastResult, rs->d_raycastImage, d_locations,
                     d_colours);
  st = download_sync(e, nullptr, nullptr);
  if (noTotalPoints) *noTotalPoints = e->h_ctr->noTotalPoints;
  return st;
}

// ---- ITMMeshingEngine (mesh.cu) --------------------------------------------------------------------
b200_status b200_mesh_scene(b200_engine *e, const b200_scene *s, b200_triangle *d_triangles, uint32_t noMaxTriangles, uint32_t *noTotalTriangles) {
  b200_status st = check_scene(e, s); if (st) return st;
  if (!d_triangles || noMaxTriangles < 2 || !noTotalTriangles) { snprintf(e->err, sizeof(e->err), "mesh_scene: bad arguments"); return B200_ERR_INVALID; }
  CK(cudaSetDevice(e->device));
  launch_mesh_scene(e, scene_ref(s, nullptr), s->voxelSize, d_triangles, noMaxTriangles);
  CK(cudaGetLastError());
  st = download_sync(e, nullptr, nullptr); if (st) return st;
  *noTotalTriangles = e->h_ctr->noTotalPoints;
  return B200_OK;
}

// ---- evaluation consumer (Evaluation::EvaluateDepth) -----------------------------------------------

b200_status b200_evaluate_depth(b200_engine *e, const b200_eval_params *params, const float *d_lidar, int n, const float *d_rendered_depth,
                                const int16_t *d_input_depth_mm, const uint8_t *d_association, const b200_eval_callback *callbacks,
                                int n_callbacks, b200_eval_result *out_static, b200_eval_result *out_dynamic, b200_eval_summary *summary) {
  if (!e) return B200_ERR_INVALID;
  if (!params || !d_rendered_depth || !d_input_depth_mm || !callbacks || !out_static || !summary || n < 0 || (n > 0 && !d_lidar) ||
      n_callbacks < 1 || n_callbacks > B200_EVAL_MAX_CALLBACKS || params->frame_width <= 0 || params->frame_height <= 0) {
    snprintf(e->err, sizeof(e->err), "evaluate_depth: bad arguments (1..%d callbacks)", B200_EVAL_MAX_CALLBACKS);
    return B200_ERR_INVALID;
  }
  if (((uintptr_t)d_lidar & 15) != 0) { snprintf(e->err, sizeof(e->err), "evaluate_depth: the point array must be 16-byte aligned"); return B200_ERR_INVALID; }
  CK(cudaSetDevice(e->device));
  const int maxWords = eval_counter_words(B200_EVAL_MAX_CALLBACKS);
  if (!e->d_evalCounters) {
    CK(cudaMalloc(&e->d_evalCounters, sizeof(unsigned long long) * (size_t)maxWords));
    CK(cudaMallocHost(&e->h_evalCounters, sizeof(unsigned long long) * (size_t)maxWords));
  }
  launch_evaluate_depth(e, params, callbacks, n_callbacks, out_dynamic ? 1 : 0, d_lidar, n, d_rendered_depth, d_input_depth_mm, d_association,
                        e->d_evalCounters);
  const int words = eval_counter_words(n_callbacks);
  CK(cudaMemcpyAsync(e->h_evalCounters, e->d_evalCounters, sizeof(unsigned long long) * (size_t)words, cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream)); CK(cudaGetLastError());
  const unsigned long long *h = e->h_evalCounters;
  for (int cls = 0; cls < 2; ++cls) {
    b200_eval_result *out = cls ? out_dynamic : out_static;
    if (!out) continue;
    for (int c = 0; c < n_callbacks; ++c) {
      const unsigned long long *q = h + (size_t)(cls * n_callbacks + c) * 9;
      out[c].measurement_count = (int64_t)q[0];
      out[c].rendered.missing = (int64_t)q[1]; out[c].rendered.error = (int64_t)q[2]; out[c].rendered.correct = (int64_t)q[3]; out[c].rendered.missing_separate = (int64_t)q[4];
      out[c].input.missing = (int64_t)q[5]; out[c].input.error = (int64_t)q[6]; out[c].input.correct = (int64_t)q[7]; out[c].input.missing_separate = (int64_t)q[8];
    }
  }
  const unsigned long long *sq = h + (size_t)2 * n_callbacks * 9;
  summary->valid_lidar_points = (int64_t)sq[0]; summary->epi_errors = (int64_t)sq[1];
  summary->negative_disparities = (int64_t)sq[2]; summary->skipped_lidar_points = (int64_t)sq[3];
  if (sq[2]) { snprintf(e->err, sizeof(e->err), "Negative disparity in ground truth."); return B200_ERR_NEGATIVE_DISPARITY; }
  return B200_OK;
}

// ---- ITMSwappingEngine ---------------------------------------------------------------------------

b200_status b200_swap_list_in(b200_engine *e, b200_scene *s, b200_transfer_buffers *tb, int *noNeeded) {
  b200_status st = check_scene(e, s); if (st) return st;
  if (!s->d_swapStates) { snprintf(e->err, sizeof(e->err), "scene has no swap states"); return B200_ERR_INVALID; }
  CK(cudaSetDevice(e->device));
  launch_swap_list_in(e, scene_ref(s, nullptr), tb->d_neededEntryIDs);
  st = download_sync(e, nullptr, nullptr);
  *noNeeded = e->h_ctr->noNeededEntries;
  return st;
}

b200_status b200_swap_integrate_in(b200_engine *e, b200_scene *s, b200_transfer_buffers *tb, int noNeeded) {
  b200_status st = check_scene(e, s); if (st) return st;
  CK(cudaSetDevice(e->device));
  launch_swap_integrate_in(e, scene_ref(s, nullptr), tb->d_syncedVoxelBlocks, tb->d_neededEntryIDs, noNeeded, s->maxW);
  CK(cudaStreamSynchronize(e->stream));
  CK(cudaGetLastError());
  return B200_OK;
}

b200_status b200_swap_out(b200_engine *e, b200_scene *s, b200_render_state *rs, b200_transfer_buffers *tb, int *noNeeded) {
  b200_status st = check_scene(e, s); if (st) return st;
  if (!s->d_swapStates) { snprintf(e->err, sizeof(e->err), "scene has no swap states"); return B200_ERR_INVALID; }
  CK(cudaSetDevice(e->device));
  st = upload(e, s, rs); if (st) return st;
  SceneRef r = scene_ref(s, rs);
  launch_swap_list_out(e, r, tb->d_neededEntryIDs);
  st = download_sync(e, nullptr, nullptr); if (st) return st;   // the count sizes the next grid, as in the reference (:161)
  const int n = e->h_ctr->noNeededEntries;
  *noNeeded = n;
  if (n > 0) {
    e->tableVersion++;
    launch_swap_move_out(e, r, tb->d_syncedVoxelBlocks, tb->d_hasSyncedData, tb->d_neededEntryIDs, n);
    st = download_sync(e, s, nullptr);
  }
  return st;
}

// ---- fused fast path -----------------------------------------------------------------------------

static b200_status frame_enqueue(b200_engine *e, b200_scene *s, b200_render_state *rs, const b200_view *v, b200_vec4f *d_points,
                                 b200_vec4f *d_normals, const b200_frame_opts *opts);

b200_status b200_process_frame_async(b200_engine *e, b200_scene *s, b200_render_state *rs, const b200_view *v, b200_vec4f *d_points,
                                     b200_vec4f *d_normals, const b200_frame_opts *opts) {
  b200_status st = check_scene(e, s); if (st) return st;
  CK(cudaSetDevice(e->device));
  if (e->hostAuthoritative) { st = upload(e, s, rs); if (st) return st; e->hostAuthoritative = false; }
  if (!e->useGraph || e->timing || e->traceOn || !e->graphWarm) {   // (events recorded inside a capture cannot be synchronised on)   // the first frame also runs one-time initialisation: never captured
    e->graphWarm = true;
    return frame_enqueue(e, s, rs, v, d_points, d_normals, opts);
  }
  // Graph mode: the frame's ~11 launches (two streams, two fork/joins) are captured and replayed as ONE graph launch; the
  // executable graph is updated in place every frame (same topology, new kernel arguments), re-instantiated if that fails.
  cudaGraph_t graph = nullptr;
  CK(cudaStreamBeginCapture(e->stream, cudaStreamCaptureModeThreadLocal));
  st = frame_enqueue(e, s, rs, v, d_points, d_normals, opts);
  cudaError_t ce = cudaStreamEndCapture(e->stream, &graph);
  if (st) { if (graph) cudaGraphDestroy(graph); return st; }
  CK(ce);
  if (e->frameGraph) {
    cudaGraphExecUpdateResultInfo info;
    if (cudaGraphExecUpdate(e->frameGraph, graph, &info) != cudaSuccess) { cudaGetLastError(); cudaGraphExecDestroy(e->frameGraph); e->frameGraph = nullptr; }
  }
  if (!e->frameGraph) CK(cudaGraphInstantiate(&e->frameGraph, graph, 0));
  CK(cudaGraphDestroy(graph));
  CK(cudaGraphLaunch(e->frameGraph, e->stream));
  return B200_OK;
}

static b200_status frame_enqueue(b200_engine *e, b200_scene *s, b200_render_state *rs, const b200_view *v, b200_vec4f *d_points,
                                 b200_vec4f *d_normals, const b200_frame_opts *opts) {
  b200_status st;
  if (e->timing) CK(cudaEventRecord(e->ev[0], e->stream));
  const bool doRay = (!opts || opts->doRaycast);
  st = enqueue_allocate(e, s, rs, v, 0, doRay); if (st) return st;
  if (e->timing) CK(cudaEventRecord(e->ev[1], e->stream));
  SceneRef r = scene_ref(s, rs);
  FrameGeom g = frame_geom(s, v);
  const bool ring = e->timingMode >= 2 && e->evRingCount < e->evRingCap;
  if (ring) CK(cudaEventRecord(e->evRing[2 * e->evRingCount], e->stream));
  // The expected-depth image of the live 1/8-resolution corner was rasterised by the allocation's list pass (alloc.cu),
  // MAX_RENDERING_BLOCKS rule included. Fork: what is left — the cells outside the corner, which nothing in the frame reads —
  // runs on the side stream underneath the integrate kernel.
  cudaStream_t mainStream = e->stream;
  const bool overlap = doRay && e->sideStream != nullptr;
  if (doRay) {
    // The cells of the expected-depth image OUTSIDE the live corner (the reference clamps block boxes to the full-resolution
    // bounds, so blocks along the right and bottom image borders smear over thousands of them: ~10^6 atomics, 38 us measured)
    // are read by nothing on the device. They are brought up to date when the host can next look at the image — b200_sync() —
    // from the block records of the latest frame, instead of every frame.
    e->deadPending = true; e->deadScene = r; e->deadM = g.M_d; memcpy(e->deadProj, g.proj_d, sizeof(e->deadProj));
    e->deadW = rs->img_w; e->deadH = rs->img_h; e->deadVoxelSize = s->voxelSize; e->deadMinmax = rs->d_minmax;
  }
  launch_integrate(e, r, g, v->d_depth, v->d_rgb);
  if (e->evMid && !e->useGraph) { CK(cudaEventRecord(e->evMid, e->stream)); e->midValid = true; }
  if (ring) { CK(cudaEventRecord(e->evRing[2 * e->evRingCount + 1], e->stream)); e->evRingCount++; }
  if (e->timing) CK(cudaEventRecord(e->ev[2], e->stream));
  if (doRay) {
    if (e->timing) CK(cudaEventRecord(e->ev[3], e->stream));
    launch_raycast(e, r, g.invM_d, g.proj_d, rs->img_w, rs->img_h, s->voxelSize, s->mu, rs->d_minmax, rs->d_raycastResult);
    // optional colour render for compositing: reads voxel colours, so it has to run before this frame's decay resets any
    if (opts && opts->d_colourRender)
      launch_shade(e, r, g.M_d, g.invM_d, rs->img_w, rs->img_h, s->voxelSize, s->maxW, rs->d_raycastResult, opts->d_colourRender, nullptr,
                   B200_RENDER_COLOUR_FROM_VOLUME);
    if (overlap) {   // the ICP-map pass (image space) runs beside the decay sweep (voxel space)
      CK(cudaEventRecord(e->evFork, mainStream));
      CK(cudaStreamWaitEvent(e->sideStream, e->evFork, 0));
      e->stream = e->sideStream;
      launch_icp(e, g.invM_d, rs->img_w, rs->img_h, s->voxelSize, rs->d_raycastResult, rs->d_raycastImage, d_points, d_normals);
      if (opts && opts->d_depthRender)   // depth render: ray points and the pose only, nothing of the volume — also beside the decay
        launch_shade(e, r, g.M_d, g.invM_d, rs->img_w, rs->img_h, s->voxelSize, s->maxW, rs->d_raycastResult, nullptr, opts->d_depthRender,
                     B200_RENDER_DEPTH_MAP);
      e->stream = mainStream;
      CK(cudaEventRecord(e->evJoin, e->sideStream));
    } else {
      launch_icp(e, g.invM_d, rs->img_w, rs->img_h, s->voxelSize, rs->d_raycastResult, rs->d_raycastImage, d_points, d_normals);
      if (opts && opts->d_depthRender)
        launch_shade(e, r, g.M_d, g.invM_d, rs->img_w, rs->img_h, s->voxelSize, s->maxW, rs->d_raycastResult, nullptr, opts->d_depthRender,
                     B200_RENDER_DEPTH_MAP);
    }
  } else if (e->timing) CK(cudaEventRecord(e->ev[3], e->stream));
  if (e->timing) CK(cudaEventRecord(e->ev[4], e->stream));
  if (opts && opts->doDecay) enqueue_decay(e, s, rs, opts->decayMaxWeight, opts->decayMinAge, 0);
  if (overlap) CK(cudaStreamWaitEvent(mainStream, e->evJoin, 0));   // join: the frame is complete on the main stream
  if (e->timing) CK(cudaEventRecord(e->ev[5], e->stream));
  return B200_OK;
}

b200_status b200_sync(b200_engine *e, b200_scene *s, b200_render_state *rs) {
  CK(cudaSetDevice(e->device));
  if (e->deadPending) {      // see frame_enqueue: the part of the expected-depth image nothing on the device reads
    launch_expected_depths_dead(e, e->deadScene, e->deadM, e->deadProj, e->deadW, e->deadH, e->deadVoxelSize, e->deadMinmax);
    e->deadPending = false;
  }
  b200_status st = download_sync(e, s, rs); if (st) return st;
  if (s && s->lastFreeBlockId < 0) { snprintf(e->err, sizeof(e->err), "out of space in the voxel block array"); return B200_ERR_VBA_FULL; }
  if (s && s->lastFreeExcessListId < 0) { snprintf(e->err, sizeof(e->err), "out of slots in the hash table excess list"); return B200_ERR_EXCESS_FULL; }
  return B200_OK;
}

b200_status b200_process_frame_host(b200_engine *e, b200_scene *s, b200_render_state *rs, b200_view *v, const float *h_depth,
                                    const b200_vec4u *h_rgb, float *d_depth_stage, b200_vec4u *d_rgb_stage, b200_vec4f *d_points,
                                    b200_vec4f *d_normals, const b200_frame_opts *opts, b200_vec4u *h_outImage) {
  CK(cudaSetDevice(e->device));
  const size_t nd = (size_t)v->depth_w * v->depth_h, nc = (size_t)v->rgb_w * v->rgb_h;
  CK(cudaMemcpyAsync(d_depth_stage, h_depth, nd * sizeof(float), cudaMemcpyHostToDevice, e->stream));
  CK(cudaMemcpyAsync(d_rgb_stage, h_rgb, nc * sizeof(b200_vec4u), cudaMemcpyHostToDevice, e->stream));
  v->d_depth = d_depth_stage; v->d_rgb = d_rgb_stage;
  b200_status st = b200_process_frame_async(e, s, rs, v, d_points, d_normals, opts); if (st) return st;
  if (h_outImage) CK(cudaMemcpyAsync(h_outImage, rs->d_raycastImage, (size_t)rs->img_w * rs->img_h * sizeof(b200_vec4u), cudaMemcpyDeviceToHost, e->stream));
  return b200_sync(e, s, rs);
}

static b200_status ensure_pipeline(b200_engine *e, size_t pixels) {
  if (e->copyStream && e->stagePixels >= pixels) return B200_OK;
  if (!e->copyStream) {
    CK(cudaStreamCreateWithFlags(&e->copyStream, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&e->d2hStream, cudaStreamNonBlocking));
    CK(cudaEventCreateWithFlags(&e->evMid, cudaEventDisableTiming));
    for (int i = 0; i < 2; ++i) {
      CK(cudaEventCreateWithFlags(&e->evH2D[i], cudaEventDisableTiming));
      CK(cudaEventCreateWithFlags(&e->evCompute[i], cudaEventDisableTiming));
      CK(cudaEventCreateWithFlags(&e->evD2H[i], cudaEventDisableTiming));
    }
  }
  for (int i = 0; i < 2; ++i) {
    cudaFree(e->d_stageDepth[i]); cudaFree(e->d_stageRgb[i]); cudaFree(e->d_stageOut[i]); cudaFree(e->d_stageRaw[i]);
    CK(cudaMalloc(&e->d_stageDepth[i], pixels * sizeof(float)));
    CK(cudaMalloc(&e->d_stageRaw[i], pixels * sizeof(int16_t)));
    CK(cudaMalloc(&e->d_stageRgb[i], pixels * sizeof(b200_vec4u)));
    CK(cudaMalloc(&e->d_stageOut[i], pixels * sizeof(b200_vec4u)));
    e->slotBusy[i] = false;
  }
  e->stagePixels = pixels;
  return B200_OK;
}

// ---- view builder (view.cu) -------------------------------------------------------------------------
static b200_status check_image(b200_engine *e, const void *a, const void *b, int w, int h) {
  if (!a || !b || w < 5 || h < 5) { snprintf(e->err, sizeof(e->err), "view builder: null image or image smaller than 5x5"); return B200_ERR_INVALID; }
  return B200_OK;
}

b200_status b200_convert_disparity_to_depth(b200_engine *e, float *d_out, const int16_t *d_in, int w, int h, float p0, float p1,
                                            float fx_depth) {
  b200_status st = check_image(e, d_out, d_in, w, h); if (st) return st;
  CK(cudaSetDevice(e->device));
  launch_view_convert(e, d_in, d_out, w, h, 0, p0, p1, fx_depth);
  CK(cudaStreamSynchronize(e->stream)); CK(cudaGetLastError());
  return B200_OK;
}

b200_status b200_convert_depth_affine_to_float(b200_engine *e, float *d_out, const int16_t *d_in, int w, int h, float p0, float p1) {
  b200_status st = check_image(e, d_out, d_in, w, h); if (st) return st;
  CK(cudaSetDevice(e->device));
  launch_view_convert(e, d_in, d_out, w, h, 1, p0, p1, 0.0f);
  CK(cudaStreamSynchronize(e->stream)); CK(cudaGetLastError());
  return B200_OK;
}

b200_status b200_depth_filtering(b200_engine *e, float *d_out, const float *d_in, int w, int h) {
  b200_status st = check_image(e, d_out, d_in, w, h); if (st) return st;
  if (d_out == d_in) { snprintf(e->err, sizeof(e->err), "DepthFiltering cannot run in place"); return B200_ERR_INVALID; }
  CK(cudaSetDevice(e->device));
  launch_view_filter_pass(e, d_in, d_out, w, h);
  CK(cudaStreamSynchronize(e->stream)); CK(cudaGetLastError());
  return B200_OK;
}

b200_status b200_compute_normal_and_weights(b200_engine *e, b200_vec4f *d_normal, float *d_sigmaZ, const float *d_depth, int w, int h,
                                            const float intrinsic[4]) {
  b200_status st = check_image(e, d_normal, d_depth, w, h); if (st) return st;
  if (!d_sigmaZ) { snprintf(e->err, sizeof(e->err), "sigmaZ image missing"); return B200_ERR_INVALID; }
  CK(cudaSetDevice(e->device));
  launch_view_normals(e, d_depth, d_normal, d_sigmaZ, w, h, intrinsic);
  CK(cudaStreamSynchronize(e->stream)); CK(cudaGetLastError());
  return B200_OK;
}

b200_status b200_update_view_async(b200_engine *e, const int16_t *d_rawDepth, int w, int h, const b200_view_calib *c, float *d_depth,
                                   b200_vec4f *d_depthNormal, float *d_depthUncertainty) {
  b200_status st = check_image(e, d_depth, d_rawDepth, w, h); if (st) return st;
  if (c->trafoType != 0 && c->trafoType != 1) { snprintf(e->err, sizeof(e->err), "unknown disparity calibration type %d", c->trafoType); return B200_ERR_INVALID; }
  if (c->modelSensorNoise && (!d_depthNormal || !d_depthUncertainty)) { snprintf(e->err, sizeof(e->err), "modelSensorNoise needs depthNormal and depthUncertainty"); return B200_ERR_INVALID; }
  CK(cudaSetDevice(e->device));
  if (c->useBilateralFilter && e->viewScratchPixels < (size_t)w * h) {
    CK(cudaStreamSynchronize(e->stream));
    cudaFree(e->d_viewScratch);
    CK(cudaMalloc(&e->d_viewScratch, (size_t)w * h * sizeof(float)));
    e->viewScratchPixels = (size_t)w * h;
  }
  launch_update_view(e, d_rawDepth, d_depth, e->d_viewScratch, w, h, c->trafoType, c->params[0], c->params[1], c->fx_depth,
                     c->useBilateralFilter != 0);
  if (c->modelSensorNoise) launch_view_normals(e, d_depth, d_depthNormal, d_depthUncertainty, w, h, c->intrinsics_d);
  return B200_OK;
}

b200_status b200_update_view(b200_engine *e, const int16_t *d_rawDepth, int w, int h, const b200_view_calib *c, float *d_depth,
                             b200_vec4f *d_depthNormal, float *d_depthUncertainty) {
  b200_status st = b200_update_view_async(e, d_rawDepth, w, h, c, d_depth, d_depthNormal, d_depthUncertainty); if (st) return st;
  CK(cudaStreamSynchronize(e->stream)); CK(cudaGetLastError());
  return B200_OK;
}

// ---- instance frame splitting and compositing (frames.cu) -------------------------------------------------
b200_status b200_process_silhouettes_async(b200_engine *e, b200_vec4u *d_rgb, float *d_depth, int w, int h, const b200_silhouette_op *ops,
                                           int n) {
  if (!d_rgb || !d_depth || w <= 0 || h <= 0 || n < 0 || (n > 0 && !ops)) { snprintf(e->err, sizeof(e->err), "process_silhouettes: bad arguments"); return B200_ERR_INVALID; }
  for (int k = 0; k < n; ++k) {
    const b200_silhouette_op &o = ops[k];
    if (o.action < 0 || o.action > 2) { snprintf(e->err, sizeof(e->err), "op %d: unknown action %d", k, o.action); return B200_ERR_INVALID; }
    if (o.action == 2 && (!o.d_dest_rgb || !o.d_dest_depth || !o.copy_mask.d_data)) { snprintf(e->err, sizeof(e->err), "op %d: instance frame or copy mask missing", k); return B200_ERR_INVALID; }
    if (o.action != 0 && !o.delete_mask.d_data) { snprintf(e->err, sizeof(e->err), "op %d: delete mask missing", k); return B200_ERR_INVALID; }
  }
  CK(cudaSetDevice(e->device));
  if (n > 0) launch_process_silhouettes(e, d_rgb, d_depth, w, h, ops, n);
  return B200_OK;
}

b200_status b200_process_silhouettes(b200_engine *e, b200_vec4u *d_rgb, float *d_depth, int w, int h, const b200_silhouette_op *ops, int n) {
  b200_status st = b200_process_silhouettes_async(e, d_rgb, d_depth, w, h, ops, n); if (st) return st;
  CK(cudaStreamSynchronize(e->stream)); CK(cudaGetLastError());
  return B200_OK;
}

b200_status b200_composite_depth(b200_engine *e, float *d_target, const float *d_source, int n) {
  if (!d_target || !d_source || n <= 0) { snprintf(e->err, sizeof(e->err), "composite_depth: bad arguments"); return B200_ERR_INVALID; }
  CK(cudaSetDevice(e->device));
  launch_composite_depth(e, d_target, d_source, n);
  CK(cudaStreamSynchronize(e->stream)); CK(cudaGetLastError());
  return B200_OK;
}

b200_status b200_composite_instances(b200_engine *e, b200_vec4u *d_out_color, float *d_out_depth, int n, const b200_instance_layer *layers,
                                     int n_layers, float dim_factor, float tint_strength) {
  if (!d_out_color || !d_out_depth || n <= 0 || n_layers < 0 || (n_layers > 0 && !layers)) { snprintf(e->err, sizeof(e->err), "composite_instances: bad arguments"); return B200_ERR_INVALID; }
  for (int k = 0; k < n_layers; ++k)
    if (!layers[k].d_color || !layers[k].d_depth) { snprintf(e->err, sizeof(e->err), "layer %d: image missing", k); return B200_ERR_INVALID; }
  CK(cudaSetDevice(e->device));
  launch_composite_layers(e, d_out_color, d_out_depth, n, layers, n_layers, dim_factor >= 0.0f, dim_factor, tint_strength);
  CK(cudaStreamSynchronize(e->stream)); CK(cudaGetLastError());
  return B200_OK;
}

b200_status b200_composite_color(b200_engine *e, b200_vec4u *d_target_color, float *d_target_depth, const b200_vec4u *d_instance_color,
                                 const float *d_instance_depth, int n, const int32_t tint[4], float tint_strength) {
  b200_instance_layer l{};
  l.d_color = d_instance_color; l.d_depth = d_instance_depth;
  for (int k = 0; k < 4; ++k) l.tint[k] = tint ? tint[k] : 0;
  return b200_composite_instances(e, d_target_color, d_target_depth, n, &l, 1, -1.0f, tint_strength);
}

// ---- pipelined host frames ----------------------------------------------------------------------------
static b200_status host_frame_submit(b200_engine *e, b200_scene *s, b200_render_state *rs, b200_view *v, const float *h_depth,
                                     const int16_t *h_raw, const b200_view_calib *calib, const b200_vec4u *h_rgb, b200_vec4f *d_points,
                                     b200_vec4f *d_normals, const b200_frame_opts *opts, b200_vec4u *h_outImage, int slot) {
  if (slot < 0 || slot > 1) { snprintf(e->err, sizeof(e->err), "slot must be 0 or 1"); return B200_ERR_INVALID; }
  CK(cudaSetDevice(e->device));
  const size_t nd = (size_t)v->depth_w * v->depth_h, nc = (size_t)v->rgb_w * v->rgb_h, no = (size_t)rs->img_w * rs->img_h;
  size_t px = nd > nc ? nd : nc; if (no > px) px = no;
  b200_status st = ensure_pipeline(e, px); if (st) return st;
  if (e->slotBusy[slot]) { snprintf(e->err, sizeof(e->err), "slot %d resubmitted before b200_host_frame_wait", slot); return B200_ERR_INVALID; }
  // H2D on the copy stream (the slot's previous frame was waited for, so its staging buffers are free)
  // The upload of frame f+1 is held back until frame f's allocation chain and integration are through: its DMA traffic slows
  // the latency-bound scan kernels of the allocation stage down by 2x when they overlap; under the raycast it is free.
  if (e->midValid) CK(cudaStreamWaitEvent(e->copyStream, e->evMid, 0));
  trace_begin(e, e->copyStream, "h2d_frame");
  if (h_raw) CK(cudaMemcpyAsync(e->d_stageRaw[slot], h_raw, nd * sizeof(int16_t), cudaMemcpyHostToDevice, e->copyStream));
  else CK(cudaMemcpyAsync(e->d_stageDepth[slot], h_depth, nd * sizeof(float), cudaMemcpyHostToDevice, e->copyStream));
  CK(cudaMemcpyAsync(e->d_stageRgb[slot], h_rgb, nc * sizeof(b200_vec4u), cudaMemcpyHostToDevice, e->copyStream));
  trace_end(e, e->copyStream);
  CK(cudaEventRecord(e->evH2D[slot], e->copyStream));
  // the frame on the compute stream
  CK(cudaStreamWaitEvent(e->stream, e->evH2D[slot], 0));
  if (h_raw) {
    st = b200_update_view_async(e, e->d_stageRaw[slot], v->depth_w, v->depth_h, calib, e->d_stageDepth[slot], nullptr, nullptr);
    if (st) return st;
  }
  v->d_depth = e->d_stageDepth[slot]; v->d_rgb = e->d_stageRgb[slot];
  st = b200_process_frame_async(e, s, rs, v, d_points, d_normals, opts); if (st) return st;
  if (h_outImage) {
    trace_begin(e, e->stream, "d2d_image");
    CK(cudaMemcpyAsync(e->d_stageOut[slot], rs->d_raycastImage, no * sizeof(b200_vec4u), cudaMemcpyDeviceToDevice, e->stream));
    trace_end(e, e->stream);
    CK(cudaEventRecord(e->evCompute[slot], e->stream));
    CK(cudaStreamWaitEvent(e->d2hStream, e->evCompute[slot], 0));
    trace_begin(e, e->d2hStream, "d2h_image");
    CK(cudaMemcpyAsync(h_outImage, e->d_stageOut[slot], no * sizeof(b200_vec4u), cudaMemcpyDeviceToHost, e->d2hStream));
    trace_end(e, e->d2hStream);
    CK(cudaEventRecord(e->evD2H[slot], e->d2hStream));
  } else {
    CK(cudaEventRecord(e->evD2H[slot], e->stream));
  }
  e->slotBusy[slot] = true;
  return B200_OK;
}

b200_status b200_host_frame_submit(b200_engine *e, b200_scene *s, b200_render_state *rs, b200_view *v, const float *h_depth,
                                   const b200_vec4u *h_rgb, b200_vec4f *d_points, b200_vec4f *d_normals, const b200_frame_opts *opts,
                                   b200_vec4u *h_outImage, int slot) {
  return host_frame_submit(e, s, rs, v, h_depth, nullptr, nullptr, h_rgb, d_points, d_normals, opts, h_outImage, slot);
}

b200_status b200_host_frame_submit_raw(b200_engine *e, b200_scene *s, b200_render_state *rs, b200_view *v, const int16_t *h_rawDepth,
                                       const b200_vec4u *h_rgb, const b200_view_calib *calib, b200_vec4f *d_points, b200_vec4f *d_normals,
                                       const b200_frame_opts *opts, b200_vec4u *h_outImage, int slot) {
  if (!h_rawDepth || !calib) { snprintf(e->err, sizeof(e->err), "raw depth / calibration missing"); return B200_ERR_INVALID; }
  if (calib->modelSensorNoise) { snprintf(e->err, sizeof(e->err), "modelSensorNoise is not available on the pipelined path; call b200_update_view"); return B200_ERR_INVALID; }
  return host_frame_submit(e, s, rs, v, nullptr, h_rawDepth, calib, h_rgb, d_points, d_normals, opts, h_outImage, slot);
}

b200_status b200_host_frame_wait(b200_engine *e, int slot) {
  if (slot < 0 || slot > 1) { snprintf(e->err, sizeof(e->err), "slot must be 0 or 1"); return B200_ERR_INVALID; }
  if (!e->copyStream || !e->slotBusy[slot]) return B200_OK;   // nothing in flight on this slot
  CK(cudaEventSynchronize(e->evD2H[slot]));
  e->slotBusy[slot] = false;
  return B200_OK;
}

b200_status b200_get_stats(b200_engine *e, b200_frame_stats *out) {
  memset(out, 0, sizeof(*out));
  out->launches = e->launches;
  out->noVisibleBlocks = e->h_ctr->noVisibleBlocks;
  out->noIntegratedBlocks = e->h_ctr->noIntegrated;
  out->totalIntegratedBlocks = e->h_ctr->totalIntegrated;
  out->droppedSnapshots = e->droppedSnapshots + e->h_ctr->droppedSnapshots;
  if (e->timingMode >= 2 && e->evRingCount > 0) {
    CK(cudaEventSynchronize(e->evRing[2 * e->evRingCount - 1]));
    float sum = 0;
    for (int i = 0; i < e->evRingCount; ++i) { float ms = 0; cudaEventElapsedTime(&ms, e->evRing[2 * i], e->evRing[2 * i + 1]); sum += ms; }
    out->ring_ms_integrate = sum; out->ring_count = e->evRingCount;
  }
  if (e->timing && e->timingMode != 0 && e->frameIdx > 0) {
    CK(cudaEventSynchronize(e->ev[5]));
    cudaEventElapsedTime(&out->ms_allocate, e->ev[0], e->ev[1]);
    cudaEventElapsedTime(&out->ms_integrate, e->ev[1], e->ev[2]);
    cudaEventElapsedTime(&out->ms_expected, e->ev[2], e->ev[3]);
    cudaEventElapsedTime(&out->ms_raycast, e->ev[3], e->ev[4]);
    cudaEventElapsedTime(&out->ms_decay, e->ev[4], e->ev[5]);
    cudaEventElapsedTime(&out->ms_total, e->ev[0], e->ev[5]);
  }
  return B200_OK;
}

}  // extern "C"
