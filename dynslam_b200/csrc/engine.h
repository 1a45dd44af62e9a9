// engine.h — internal: engine state and kernel launchers shared by the .cu files of libb200fusion.
#pragma once
#include "common.cuh"

struct FrameGeom {          // per-call constants handed to kernels by value
  Mat4 M_d, invM_d, M_rgb;
  float proj_d[4], proj_rgb[4];
  int w, h, rgb_w, rgb_h;
  float voxelSize, mu;
  int maxW;
  float vfmin, vfmax;
  int depthWeighting, stopMaxW, approx;
  float negOneOverMu;       // -1.0f / mu, the quotient of every rejected voxel (eta == -1)
  int sameRgbCam;           // M_rgb, proj_rgb, image size bitwise equal to the depth camera's: ix,iy are shared
};

struct SceneRef {           // raw device views of the caller-owned scene / render-state buffers
  b200_voxel *voxels;
  int *allocationList;
  b200_hash_entry *hash;
  int *excessList;
  uint8_t *swapStates;
  int numBlocks, numBuckets, excessSize, noTotal;
  b200_vec3i *visiblePos;
  uint8_t *visType;
};

struct DecaySnap { long long start; int frameIdx; int hostCountKnown; };

#define B200_DBG_WORDS (64 + 5 * 1024)   // 4 CTAs x 8 phase stamps, then per tile (first 1024): start, list count published, list offset known
struct b200_engine {
  int device;
  cudaStream_t stream;
  bool ownStream;
  int numBlocks, numBuckets, excessSize, noTotal, img_w, img_h;
  int smCount;
  // device scratch
  DevCounters *d_ctr;
  DevCounters *h_ctr;                 // pinned mirror
  unsigned long long *d_reqKey;       // per entry: frameTag | pixel | step of the winning request
  unsigned *d_reqBits, *d_req2Bits;   // request bitmaps (all / excess-type), noTotal/32 words
  uint8_t *d_markBytes;               // per entry: observed by this frame's marking (entriesVisibleType 1 / 2), consumed and cleared by k_serve_list
  int noWords;
  unsigned long long *d_scanDesc;     // chained-scan tile descriptors
  int scanDescCap;
  unsigned scanGen;
  // decay
  b200_vec3i *d_ring;                 // snapshot ring (items)
  long long ringCap;
  int *d_snapCount;                   // device-side count per ring slot (slot = frame % SNAP_SLOTS)
  long long *d_snapStart;
  int qHead, qSize;                   // host view of the queue (slots qHead .. qHead+qSize-1)
  long long droppedSnapshots;         // snapshots dropped on the host side because the queue was SNAP_SLOTS deep
  unsigned long long *d_delTag;       // per VBA block: gen | ~itemIndex of the deleting item
  int *d_visiblePtr;                  // VBA ptr of every item of the list built by the last allocate (or -1)
  const void *ptrListFor;             // the visible list buffer d_visiblePtr describes
  unsigned long long tableVersion, ptrListVersion;   // d_visiblePtr is valid while they are equal
  int *d_itemPtr;                     // per decay item: VBA ptr (or -1)
  unsigned *d_itemFlag;               // per decay item: 1 = deletes its block
  int *d_delList;                     // compacted deleting items (list order)
  int *d_candList;                    // DECAY_CAND_CAP unordered candidates of the partial pass (decay.cu)
  uint8_t *d_isLeader;
  short4 *d_allocatedPos;             // full decay: pos per VBA slot (w = valid)
  unsigned decayGen;
  int frameIdx;
  long long totalDecayed;
  // vis
  unsigned *d_tileCounts;
  void *d_blockRecs;                  // expected depths: per visible block {bbox, z-range}, 16 B
  // timing / stats
  bool timing;
  cudaEvent_t ev[8];
  // pipelined host frames: copy stream, two staging slots
  cudaStream_t sideStream;            // fused frame: small launches overlapped with the big ones
  cudaEvent_t evFork, evJoin;
  cudaStream_t copyStream;     // H2D of the next frame's depth + RGB
  cudaStream_t d2hStream;      // D2H of the previous frame's image (own stream so it never holds up the next upload)
  float *d_stageDepth[2]; b200_vec4u *d_stageRgb[2]; b200_vec4u *d_stageOut[2]; int16_t *d_stageRaw[2];
  cudaEvent_t evH2D[2], evCompute[2], evD2H[2];
  bool slotBusy[2]; size_t stagePixels;
  int maxRenderingBlocks;                           // MAX_RENDERING_BLOCKS; b200_diag_set_max_rendering_blocks lowers it (tests)
  int useGraph; bool graphWarm; cudaGraphExec_t frameGraph;
  cudaEvent_t evMid; bool midValid;                 // "allocation + integration of the last frame are done" (pipelined uploads wait for it)         // B200_GRAPH=1: the fused frame is captured and replayed as a CUDA graph
  float *d_viewScratch; size_t viewScratchPixels;   // plays view->depth inside UpdateView (view.cu)
  cudaEvent_t *evRing;                // timing mode 2: event pairs around every integrate launch
  int evRingCap, evRingCount, timingMode;
  // timing mode 3: an event pair around every kernel launch (launch trace, b200_get_trace)
  bool traceOn; int traceCount, traceCap; cudaEvent_t *traceEv; const char **traceName;
  // expected-depth cells outside the live corner of the latest fused frame: rasterised lazily at b200_sync()
  bool deadPending; SceneRef deadScene; Mat4 deadM; float deadProj[4]; int deadW, deadH; float deadVoxelSize; b200_vec2f *deadMinmax;
  unsigned long long *d_evalCounters, *h_evalCounters;   // evaluation consumer: counters (device) and their pinned mirror, allocated on first use
  unsigned long long *d_meshDesc;     // meshing: chained-scan descriptors, one per VBA block (allocated on first use)
  unsigned long long *d_dbg;          // timestamps written by instrumented kernels while the launch trace is on (b200_diag_read_debug)
  long long launches;
  int lastNoIntegrated;
  int integrateImpl;                  // 0 = LDG variant, 1 = TMA bulk-copy variant (env B200_INTEGRATE_IMPL=ldg|tma)
  // run-time switches, read from the environment when the engine is created (defaults when unset; README)
  int pplV4;                          // B200_V4_PPL=1|2 forces V4's two- / four-voxels-per-lane form; 0: by list length
  int v4TailFloor;                    // B200_V4_TAIL=1..6: blocks a V4 CTA keeps in flight when the list runs out (3)
  bool v3Prefetch;                    // B200_V3_PREFETCH=0 turns off the L2 prefetch of the images in V3 / V4
  int ctasV3;                         // B200_V3_CTAS=2|3|4: resident V3 CTAs per SM (3)
  int regsTma;                        // B200_INTEGRATE_REGS=56: the 56-register TMA build (48)
  int ctasTma;                        // TMA CTAs per SM: occupancy, at most 4, lowered by B200_INTEGRATE_CTAS
  int rcTileLog2, rcOrder, rcImpl;    // B200_RC_TILE=0..5 (3: 8x4), B200_RC_ORDER=0|1 (1), B200_RC_IMPL=old (1: neighbourhood cache)
  int lastIntegrateKernel, lastIntegrateGrid;   // what the last launch_integrate ran (b200_diag_last_integrate)
  bool hostAuthoritative;            // host copies of the counters are newer than the device ones
  char err[512];
};

#define SNAP_SLOTS 4096

// Device half of a decay-queue push (Reco_CUDA.cu:302-316): the `kept` positions written to the ring from ringStart on
// become snapshot `slot`, and the ring's cursor moves past them. Allocation's list pass and b200_diag_push_decay_snapshot
// both publish through here; the host half is push_snapshot_slot (engine.cu).
DEV void publish_snapshot(DevCounters *ctr, long long *snapStart, int *snapCount, int slot, long long ringStart, int kept) {
  snapStart[slot] = ringStart;
  snapCount[slot] = kept;
  ctr->ringHead = ringStart + kept;
}
void launch_push_snapshot(b200_engine *e, const b200_vec3i *positions, int n, int snapSlot);

// launchers (each enqueues on e->stream and bumps e->launches)
void launch_reset(b200_engine *e, const SceneRef &s);
void launch_allocate(b200_engine *e, const SceneRef &s, const FrameGeom &g, const float *depth, bool onlyVisible,
                     int frameIdx, int snapSlot, b200_vec2f *minmaxDead, int mw, int mh);
void launch_integrate(b200_engine *e, const SceneRef &s, const FrameGeom &g, const float *depth, const b200_vec4u *rgb);
void integrate_init_device(b200_engine *e);   // per-device: division table upload, dynamic shared-memory attributes
static inline const int *fresh_ptr_list(const b200_engine *e, const SceneRef &s) {
  return (e->ptrListFor == (const void *)s.visiblePos && e->ptrListVersion == e->tableVersion) ? e->d_visiblePtr : nullptr;
}
void launch_decay_partial(b200_engine *e, const SceneRef &s, int snapSlot, int minAge, int maxWeight, int frameIdx);
void launch_decay_full(b200_engine *e, const SceneRef &s, int minAge, int maxWeight, int frameIdx);
void launch_find_visible(b200_engine *e, const SceneRef &s, const Mat4 &M, const float proj[4], int w, int h, float voxelSize);
void launch_expected_depths(b200_engine *e, const SceneRef &s, const Mat4 &M, const float proj[4], int w, int h,
                            float voxelSize, b200_vec2f *minmax, bool deadInitDone = false, bool recsReady = false);
void launch_expected_depths_fast(b200_engine *e, const SceneRef &s, const Mat4 &M, const float proj[4], int w, int h, float voxelSize,
                                 b200_vec2f *minmax);
void launch_expected_depths_dead(b200_engine *e, const SceneRef &s, const Mat4 &M, const float proj[4], int w, int h, float voxelSize,
                                 b200_vec2f *minmax);
void launch_raycast(b200_engine *e, const SceneRef &s, const Mat4 &invM, const float proj[4], int w, int h, float voxelSize,
                    float mu, const b200_vec2f *minmax, b200_vec4f *out);
void launch_shade(b200_engine *e, const SceneRef &s, const Mat4 &M, const Mat4 &invM, int w, int h, float voxelSize, int maxW,
                  const b200_vec4f *rays, b200_vec4u *outChar, float *outFloat, int type);
void launch_icp(b200_engine *e, const Mat4 &invM, int w, int h, float voxelSize, const b200_vec4f *rays, b200_vec4u *outImg,
                b200_vec4f *points, b200_vec4f *normals);
void launch_forward_render(b200_engine *e, const SceneRef &s, const FrameGeom &g, const float *depth, const b200_vec2f *minmax,
                           const b200_vec4f *rays, b200_vec4f *fwd, int *missing, b200_vec4u *outImg);
void launch_point_cloud(b200_engine *e, const SceneRef &s, const Mat4 &invM, int w, int h, float voxelSize, int skipPoints,
                        const b200_vec4f *rays, b200_vec4u *outImg, b200_vec4f *locations, b200_vec4f *colours);
int eval_counter_words(int nCallbacks);
void launch_evaluate_depth(b200_engine *e, const b200_eval_params *p, const b200_eval_callback *cb, int nCallbacks, int hasDynamic,
                           const float *lidar, int n, const float *rendered, const int16_t *inputMm, const uint8_t *association,
                           unsigned long long *counters);
void launch_mesh_scene(b200_engine *e, const SceneRef &s, float voxelSize, b200_triangle *triangles, unsigned noMaxTriangles);
void launch_swap_list_in(b200_engine *e, const SceneRef &s, int *needed);
void launch_swap_integrate_in(b200_engine *e, const SceneRef &s, const b200_voxel *synced, const int *needed, int n, int maxW);
void launch_swap_list_out(b200_engine *e, const SceneRef &s, int *needed);
void launch_swap_move_out(b200_engine *e, const SceneRef &s, b200_voxel *synced, uint8_t *hasSynced, const int *needed, int n);

void launch_view_convert(b200_engine *e, const int16_t *raw, float *out, int w, int h, int type, float p0, float p1, float fx);
void launch_view_filter_pass(b200_engine *e, const float *in, float *out, int w, int h);
void launch_update_view(b200_engine *e, const int16_t *raw, float *out, float *scratch, int w, int h, int type, float p0, float p1,
                        float fx, bool filter);
void launch_view_normals(b200_engine *e, const float *depth, b200_vec4f *normal, float *sigmaZ, int w, int h, const float intr[4]);

void launch_process_silhouettes(b200_engine *e, b200_vec4u *rgb, float *depth, int w, int h, const b200_silhouette_op *ops, int n);
void launch_composite_depth(b200_engine *e, float *target, const float *source, int n);
void launch_composite_layers(b200_engine *e, b200_vec4u *tcol, float *tdep, int n, const b200_instance_layer *layers, int nLayers,
                             bool dim, float dimFactor, float tintStrength, cudaStream_t other = nullptr, const b200_vec4u *bgcol = nullptr,
                             const float *bgdep = nullptr);

// Launch trace (timing mode 3): TRACED(e, stream, "kernel", launch-statement) brackets the launch with two events.
static inline void trace_begin(b200_engine *e, cudaStream_t st, const char *name) {
  if (!e->traceOn || e->traceCount >= e->traceCap) return;
  e->traceName[e->traceCount] = name;
  cudaEventRecord(e->traceEv[2 * e->traceCount], st);
}
static inline void trace_end(b200_engine *e, cudaStream_t st) {
  if (!e->traceOn || e->traceCount >= e->traceCap) return;
  cudaEventRecord(e->traceEv[2 * e->traceCount + 1], st);
  e->traceCount++;
}
#define TRACED(e, st, name, ...) do { trace_begin(e, st, name); __VA_ARGS__; trace_end(e, st); } while (0)

#define DECAY_CAND_CAP 1024

static inline int persistent_grid(const b200_engine *e, int ctasPerSm, long long workItems) {
  long long g = (long long)e->smCount * ctasPerSm;
  if (workItems < g) g = workItems;
  return (int)(g < 1 ? 1 : g);
}
