// engine.h — internal: engine state and kernel launchers shared by the .cu files of libb200fusion.
#pragma once
#include "common.cuh"

#include <utility>

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
  int *d_resetPtr;                    // per partial-decay item: VBA ptr of its block when the sweep found voxels to reset (or -1)
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
  uint8_t *d_stageBgr[2];      // BGR8 colour of a stereo-input frame (b200_host_frame_submit_stereo), 3 B/px
  cudaEvent_t evH2D[2], evCompute[2], evD2H[2];
  bool slotBusy[2]; size_t stagePixels;
  int maxRenderingBlocks;                           // MAX_RENDERING_BLOCKS; b200_diag_set_max_rendering_blocks lowers it (tests)
  int gridScale;                                    // ticket_grid's factor, 1; b200_diag_set_grid_scale raises it (tests)
  bool registered;                                  // counted among the device's live engines (device_shared, engine.cu)
  int useGraph; bool graphWarm; cudaGraphExec_t frameGraph;
  cudaEvent_t evMid; bool midValid;                 // "allocation + integration of the last frame are done" (pipelined uploads wait for it)         // B200_GRAPH=1: the fused frame is captured and replayed as a CUDA graph
  float *d_viewScratch; size_t viewScratchPixels;   // plays view->depth inside UpdateView (view.cu)
  unsigned long long *d_spans;        // timing modes 2 to 4: %globaltimer spans of the chain's kernels, per fused frame (span_slot)
  int spanCount, timingMode;          // fused frames stamped since the mode was set
  // timing mode 3: an event pair around every kernel launch (launch trace, b200_get_trace)
  bool traceOn; int traceCount, traceCap; cudaEvent_t *traceEv; const char **traceName;
  // expected-depth cells outside the live corner of the latest fused frame: rasterised lazily at b200_sync()
  bool deadPending; SceneRef deadScene; int deadW, deadH; b200_vec2f *deadMinmax;
  unsigned long long *d_evalCounters, *h_evalCounters;   // evaluation consumer: counters (device) and their pinned mirror, allocated on first use
  unsigned long long *d_meshDesc;     // meshing: chained-scan descriptors, one per VBA block (allocated on first use)
  unsigned long long *d_dbg;          // timestamps written by instrumented kernels while the launch trace is on (b200_diag_read_debug)
  long long launches;
  int lastNoIntegrated;
  int integrateImpl;                  // 1 = TMA kernel, 2 = V3, 3 = V4, 4 = V4 in tolerance mode (env B200_INTEGRATE_IMPL=tma|v3|v4|fast)
  // run-time switches, read from the environment when the engine is created (defaults when unset; README)
  int pplV4;                          // B200_V4_PPL=1|2 forces V4's two- / four-voxels-per-lane form; 0: by list length
  int v4TailFloor;                    // B200_V4_TAIL=1..6: blocks a V4 CTA keeps in flight when the list runs out (3)
  bool v3Prefetch;                    // B200_V3_PREFETCH=0 turns off the L2 prefetch of the images in V3 / V4
  int ctasV3;                         // B200_V3_CTAS=2|3|4: resident V3 CTAs per SM (3)
  int ctasTma;                        // TMA CTAs per SM: occupancy of k_integrate_tma48, at most 4
  int rcTileLog2, rcOrder, rcImpl;    // B200_RC_TILE=0..5 (3: 8x4), B200_RC_ORDER=0|1 (1), B200_RC_IMPL=old (1: neighbourhood cache)
  int lastIntegrateKernel, lastIntegrateGrid;   // what the last launch_integrate ran (b200_diag_last_integrate)
  bool hostAuthoritative;            // host copies of the counters are newer than the device ones
  struct CheckpointScratch *ck;      // checkpoint.cu: staging, bounce buffers and the kept classification (allocated on first use)
  struct PreviewScratch *pv;         // preview.cu: the free-view preview's own counters, scan descriptors and hand-over slots (allocated on first use)
  char err[512];
};

// engine.cu helpers shared with checkpoint.cu
SceneRef scene_ref(const b200_scene *s, const b200_render_state *rs);
b200_status check_scene(b200_engine *e, const b200_scene *s);
b200_status download_sync(b200_engine *e, b200_scene *s, b200_render_state *rs);
extern "C" int push_snapshot_slot(b200_engine *e);   // (defined inside engine.cu's extern "C" block)
void checkpoint_release(b200_engine *e);
void preview_release(b200_engine *e);
bool preview_slot_busy(const b200_engine *e);   // a b200_render_view_submit slot not yet waited for

#define SNAP_SLOTS 4096

// Device half of a decay-queue push (Reco_CUDA.cu:302-316): the `kept` positions written to the ring from ringStart on
// become snapshot `slot`, and the ring's cursor moves past them. Allocation's list pass, b200_diag_push_decay_snapshot and
// b200_checkpoint_load all publish through here; the host half is push_snapshot_slot (engine.cu).
DEV void publish_snapshot(DevCounters *ctr, long long *snapStart, int *snapCount, int slot, long long ringStart, int kept) {
  snapStart[slot] = ringStart;
  snapCount[slot] = kept;
  ctr->ringHead = ringStart + kept;
}
// n == -1 pushes a snapshot the ring has already overwritten: its Decay sweeps nothing and counts it as dropped
void launch_push_snapshot(b200_engine *e, const b200_vec3i *positions, int n, int snapSlot);

// launchers (each enqueues on e->stream and bumps e->launches)
void launch_reset(b200_engine *e, const SceneRef &s);
void launch_allocate(b200_engine *e, const SceneRef &s, const FrameGeom &g, const float *depth, bool onlyVisible,
                     int frameIdx, int snapSlot, b200_vec2f *minmaxDead, int mw, int mh, bool fused = false);
// fused = true: a launch of the fused frame's chain (launch_chained), stamped in timing modes 2 and 4
void launch_integrate(b200_engine *e, const SceneRef &s, const FrameGeom &g, const float *depth, const b200_vec4u *rgb, bool fused = false);
void integrate_init_device(b200_engine *e);   // per-device: division table upload, dynamic shared-memory attributes
static inline const int *fresh_ptr_list(const b200_engine *e, const SceneRef &s) {
  return (e->ptrListFor == (const void *)s.visiblePos && e->ptrListVersion == e->tableVersion) ? e->d_visiblePtr : nullptr;
}
// Arguments of a decay sweep (decay_sweep.cuh). Partial decay: items = ring snapshot `slot`; full decay: VBA slots.
struct DecaySweep {
  b200_voxel *voxels;
  const b200_hash_entry *table;
  int numBuckets, numBlocks;
  const b200_vec3i *ring;
  long long ringCap;
  const long long *snapStart;
  const int *snapCount;
  int slot;
  const short4 *allocatedPos;
  int minAge, maxWeight, currentFrame;
  unsigned gen;
  unsigned long long *delTag;
  int *itemPtr, *resetPtr, *candList;
  DevCounters *ctr;
  unsigned long long *span;           // SpanStamp of the sweep (fused frame, timing modes 3 and 4), or nullptr
};
// A partial Decay of snapshot `snapSlot`, in two parts: the sweep (read and decide) and k_decay_commit (the reset stores and the
// commit). decay_sweep_args takes the pass's generation; launch_decay_partial launches the sweep as a grid of its own unless
// it already rode in the raycast's grid (swept = true: launch_raycast with the same arguments), then k_decay_commit.
DecaySweep decay_sweep_args(b200_engine *e, const SceneRef &s, int snapSlot, int minAge, int maxWeight, int frameIdx, bool fused = false);
void launch_decay_partial(b200_engine *e, const SceneRef &s, const DecaySweep &d, bool swept, bool fused = false);
void launch_decay_full(b200_engine *e, const SceneRef &s, int minAge, int maxWeight, int frameIdx);
// FindVisibleBlocks into s.visiblePos; the count, the tile ticket and the scan descriptors (FV_TILE entries per tile) are the
// caller's, so that the free-view preview keeps its own
#define FV_EPT 16
#define FV_TILE (256 * FV_EPT)
void launch_find_visible(b200_engine *e, const SceneRef &s, const Mat4 &M, const float proj[4], int w, int h, float voxelSize,
                         int *count, unsigned *ticket, unsigned long long *scanDesc, unsigned gen);
// CreateExpectedDepths over the first *count items of s.visiblePos; *tiles receives the rendering-tile total, *done is the
// pass's self-resetting CTA counter
void launch_expected_depths(b200_engine *e, const SceneRef &s, const Mat4 &M, const float proj[4], int w, int h, float voxelSize,
                            b200_vec2f *minmax, const int *count, unsigned *tiles, unsigned *done);
// the fused frame's expected-depth cells outside the live corner, from the block records of its allocation
void launch_expected_depths_dead(b200_engine *e, const SceneRef &s, int w, int h, b200_vec2f *minmax);
// sweep != nullptr: the raycast's grid also runs that partial Decay's sweep, on CTAs of its own ahead of the ray tiles
void launch_raycast(b200_engine *e, const SceneRef &s, const Mat4 &invM, const float proj[4], int w, int h, float voxelSize,
                    float mu, const b200_vec2f *minmax, b200_vec4f *out, bool fused = false, const DecaySweep *sweep = nullptr);
void launch_shade(b200_engine *e, const SceneRef &s, const Mat4 &M, const Mat4 &invM, int w, int h, float voxelSize, int maxW,
                  const b200_vec4f *rays, b200_vec4u *outChar, float *outDepth, int type);
// fused = true: the fused frame's ICP pass, stamped in timing modes 3 and 4 (SPAN_ICP)
void launch_icp(b200_engine *e, const Mat4 &invM, int w, int h, float voxelSize, const b200_vec4f *rays, b200_vec4u *outImg,
                b200_vec4f *points, b200_vec4f *normals, bool fused = false);
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
// input.cu: int16 mm depth from a disparity map (kind 0) or a clamped int16 depth map (kind 1), and BGR8 -> RGBA8, on stream st.
// depthOut / rgba may be null (that half is skipped); depthCopy (may be null) receives a second copy of the depth.
void launch_stereo_input(b200_engine *e, cudaStream_t st, const void *depthIn, int kind, int nDepth, float fb, int minMm, int maxMm,
                         int16_t *depthOut, int16_t *depthCopy, const uint8_t *bgr, b200_vec4u *rgba, int nColour);

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

// Launch of a kernel of the fused frame's main-stream chain k_mark_prepare -> k_serve_list -> k_integrate_v4 -> k_raycast ->
// k_decay_commit. With chained = true the launch carries programmatic stream serialisation: its CTAs may become resident and
// run the code before their pdl_wait() while the previous kernel of the stream drains. Rules kept by every kernel of the chain:
//  * a kernel calls pdl_trigger() only after its own pdl_wait() has returned. By induction, when a kernel runs its pre-wait code,
//    everything two or more launches back has completed and its memory is visible;
//  * pre-wait code reads only data whose last writer is at least two launches back, or that the caller wrote before the
//    frame's first launch (k_mark_prepare, launched with chained = false, waits for everything enqueued before it);
//  * pre-wait code writes only scratch that the previous kernel neither reads nor writes;
//  * no stream operation (event record, copy, memset) sits between two chained launches: it would serialise them again.
// The partial Decay's sweep runs on CTAs of k_raycast's grid, after the same wait. The rays read the voxels and the hash table
// and write only the ray points, so the sweep may read the ring, the table and the voxels, and write only decay scratch that
// nothing else in the grid touches: the delTag claims, itemPtr, resetPtr, the candidate list and the decay counters. The reset
// stores and the table edits wait for k_decay_commit, launched after everything in the frame that reads the voxels.
// Stand-alone entry points launch with chained = false; pdl_wait() is then a no-op and the kernels are unchanged.
template <typename... KArgs, typename... Args>
static inline void launch_chained(bool chained, void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                                  Args &&...args) {
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cfg.attrs = attr; cfg.numAttrs = chained ? 1 : 0;
  cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

// %globaltimer spans of the chain's kernels (b200_set_timing modes 2 to 4): one record of SPAN_KERNELS SpanStamp slots per fused
// frame, SPAN_FRAMES records, zero-filled whenever the mode is set. Mode 2 stamps the integrate kernel only.
// SPAN_RAYCAST: the ray CTAs only; SPAN_COMMIT: the commit in CTA 0 of k_decay_commit (rank, elect, unlink, counters); SPAN_ICP: k_icp on the side stream
enum { SPAN_MARK, SPAN_SERVE, SPAN_INTEGRATE, SPAN_RAYCAST, SPAN_SWEEP, SPAN_DECAY, SPAN_COMMIT, SPAN_ICP, SPAN_KERNELS };
#define SPAN_FRAMES 8192
// the slot of kernel k in the record of the fused frame being enqueued, or nullptr when that kernel is not stamped
static inline unsigned long long *span_slot(const b200_engine *e, int k) {
  if (e->timingMode < 2 || !e->d_spans || e->spanCount >= SPAN_FRAMES || (e->timingMode == 2 && k != SPAN_INTEGRATE)) return nullptr;
  return e->d_spans + ((size_t)e->spanCount * SPAN_KERNELS + k) * 2;
}

#define DECAY_CAND_CAP 1024

static inline int persistent_grid(const b200_engine *e, int ctasPerSm, long long workItems) {
  long long g = (long long)e->smCount * ctasPerSm;
  if (workItems < g) g = workItems;
  return (int)(g < 1 ? 1 : g);
}
// grid of a kernel that hands out its tiles with draw_tile: persistent_grid, or with b200_diag_set_grid_scale's factor k > 1,
// k times the whole GPU's worth of CTAs whatever the number of tiles (ctasPerSm >= 1 and k >= 8 are at least the 2048 threads an
// SM holds for CTAs of 256 threads or more, so most CTAs start only after others have retired)
static inline int ticket_grid(const b200_engine *e, int ctasPerSm, long long workItems) {
  return e->gridScale > 1 ? e->smCount * ctasPerSm * e->gridScale : persistent_grid(e, ctasPerSm, workItems);
}
// another engine is live on this engine's device (engine.cu counts them); k_serve_list then hands out its tiles by ticket
bool device_shared(const b200_engine *e);
