/*
 * b200fusion.h — C-ABI of the voxel-hashed TSDF fusion / raycast engine (built for sm_90a).
 *
 * This is the drop-in boundary behind DynSLAM's ITMLib engine interfaces. Every entry point
 * below replaces one virtual of the reference (paths relative to
 * src/InfiniTAM/InfiniTAM/ITMLib/ in AndreiBarsan/DynSLAM):
 *
 *   ITMSceneReconstructionEngine<TVoxel,ITMVoxelBlockHash>   Engine/ITMSceneReconstructionEngine.h:33-78
 *   IITMVisualisationEngine / ITMVisualisationEngine          Engine/ITMVisualisationEngine.h:19-127
 *   ITMSwappingEngine<TVoxel,ITMVoxelBlockHash>               Engine/ITMSwappingEngine.h:22-31
 *
 * Plain pointers and sizes only; all pointers named d_* are CUDA device pointers owned by the
 * caller (exactly the buffers ITMScene / ITMRenderState_VH / ITMView already own), the engine
 * handle owns only its scratch. Byte layouts are those of the reference:
 *   ITMHashEntry   20 B  Utils/ITMLibDefines.h:69-84
 *   ITMVoxel_s_rgb  8 B  Utils/ITMLibDefines.h:138-169 (one 8x8x8 block = 4096 B)
 *   Matrix4f       m[col*4+row]  ORUtils/Matrix.h:23-33
 *
 * Error convention (reference: ORcudaSafeCall exits, logic errors throw std::runtime_error,
 * Reco_CUDA.cu:348-357): every function returns a b200_status; b200_last_error() gives text.
 * The C++ shim (dynslam_b200/itm_shim) maps the codes back onto throw / exit.
 */
#ifndef B200FUSION_H
#define B200FUSION_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200_SDF_BLOCK_SIZE 8
#define B200_SDF_BLOCK_SIZE3 512
#define B200_MAX_RENDERING_BLOCKS (65536 * 4) /* DeviceAgnostic/ITMVisualisationEngine.h:25 */
#define B200_MINMAX_SUBSAMPLE 8               /* DeviceAgnostic/ITMVisualisationEngine.h:27 */
#define B200_FAR_AWAY 999999.9f
#define B200_VERY_CLOSE 0.05f
#define B200_TRANSFER_BLOCK_NUM 0x1000        /* Utils/ITMLibDefines.h:39 */

typedef enum {
  B200_OK = 0,
  B200_ERR_CUDA = 1,          /* reference: ORcudaSafeCall -> exit(-1) */
  B200_ERR_VBA_FULL = 2,      /* reference: throw runtime_error, Reco_CUDA.cu:348-351 */
  B200_ERR_EXCESS_FULL = 3,   /* reference: throw runtime_error, Reco_CUDA.cu:353-357 */
  B200_ERR_INVALID = 4,
  B200_ERR_DECAY_RING_FULL = 5, /* no longer returned: a full decay queue drops its oldest snapshots (see b200_engine_config) */
  B200_ERR_UNSUPPORTED = 6,
  B200_ERR_NEGATIVE_DISPARITY = 7  /* reference: throw runtime_error("Negative disparity in ground truth."), Evaluation.cpp:273-275 */
} b200_status;

/* ---- byte-exact mirrors of the reference PODs ---------------------------------------- */

typedef struct {            /* ITMHashEntry */
  int16_t pos[3];
  int16_t _pad;
  int32_t offset;           /* 1-based index into the excess part, <1 = end of chain */
  int32_t ptr;              /* >=0 VBA block id, -1 swapped out, <-1 free */
  int32_t allocatedTime;
} b200_hash_entry;

typedef struct {            /* ITMVoxel_s_rgb */
  int16_t sdf;              /* tsdf * 32767 */
  uint8_t w_depth;
  uint8_t clr[3];
  uint8_t w_color;
  uint8_t _pad;
} b200_voxel;

typedef struct { int32_t x, y, z; } b200_vec3i;   /* Vector3i, visible-list item */
typedef struct { float x, y; } b200_vec2f;        /* Vector2f, min/max image pixel */
typedef struct { float x, y, z, w; } b200_vec4f;  /* Vector4f */
typedef struct { uint8_t x, y, z, w; } b200_vec4u;/* Vector4u, RGBA8 */

/* ---- scene (ITMScene = ITMVoxelBlockHash + ITMLocalVBA + ITMSceneParams) --------------- */

typedef struct {
  b200_voxel *d_voxels;          /* localVBA.GetVoxelBlocks(): numBlocks*512 voxels */
  int32_t *d_allocationList;     /* localVBA.GetAllocationList(): numBlocks ints */
  b200_hash_entry *d_hash;       /* index.GetEntries(): numBuckets+excessSize entries */
  int32_t *d_excessList;         /* index.GetExcessAllocationList(): excessSize ints */
  uint8_t *d_swapStates;         /* globalCache->GetSwapStates(true) or NULL (swapping off) */
  int32_t numBlocks;             /* sdfLocalBlockNum */
  int32_t numBuckets;            /* SDF_BUCKET_NUM, power of two */
  int32_t excessSize;            /* SDF_EXCESS_LIST_SIZE */
  /* host-visible counters, valid on return of every synchronous call (SURVEY 8b) */
  int32_t lastFreeBlockId;       /* localVBA.lastFreeBlockId */
  int32_t lastFreeExcessListId;  /* index.lastFreeExcessListId */
  /* ITMSceneParams (Objects/ITMSceneParams.h:14-71) */
  float voxelSize, mu;
  int32_t maxW;
  float viewFrustum_min, viewFrustum_max;
  int32_t stopIntegratingAtMaxW;
  int32_t useSwapping;
} b200_scene;

/* ---- render state (ITMRenderState_VH + base) ------------------------------------------ */

typedef struct {
  b200_vec3i *d_visibleBlockPositions; /* GetVisibleBlockPositions(): numBlocks items */
  uint8_t *d_entriesVisibleType;       /* GetEntriesVisibleType(): one byte per hash entry */
  b200_vec2f *d_minmax;                /* renderingRangeImage, w*h, 1/8-res corner used */
  b200_vec4f *d_raycastResult;         /* raycastResult, w*h */
  b200_vec4f *d_forwardProjection;     /* forwardProjection, w*h (may be NULL) */
  int32_t *d_fwdProjMissingPoints;     /* fwdProjMissingPoints, w*h (may be NULL) */
  b200_vec4u *d_raycastImage;          /* raycastImage, w*h */
  int32_t img_w, img_h;
  int32_t noVisibleBlocks;             /* host-visible, in/out */
  int32_t noFwdProjMissingPoints;      /* host-visible, out */
} b200_render_state;

/* ---- per-frame inputs (ITMView + ITMTrackingState::pose_d + calib) ----------------------- */

typedef struct {
  const float *d_depth;          /* view->depth, metres, w*h */
  const b200_vec4u *d_rgb;       /* view->rgb, RGBA8 */
  int32_t depth_w, depth_h, rgb_w, rgb_h;
  float M_d[16];                 /* trackingState->pose_d->GetM() */
  float invM_d[16];              /* its inverse (Matrix4::inv, ORUtils/Matrix.h:162-224) */
  float M_rgb[16];               /* calib.trafo_rgb_to_depth.calib_inv * M_d */
  float proj_d[4];               /* intrinsics_d.projectionParamsSimple.all = fx,fy,cx,cy */
  float proj_rgb[4];
  int32_t depthWeighting;        /* WeightParams, Engine/ITMSceneReconstructionEngine.h:21-23 */
  int32_t requiresFullRendering; /* trackingState->requiresFullRendering (approx. integration off) */
} b200_view;

typedef struct {               /* pose + intrinsics pair used by the visualisation calls */
  float M[16];
  float invM[16];
  float proj[4];
} b200_camera;

typedef enum {                 /* IITMVisualisationEngine::RenderImageType, Vis.h:22-32 */
  B200_RENDER_SHADED_GREYSCALE = 0,
  B200_RENDER_COLOUR_FROM_VOLUME = 1,
  B200_RENDER_COLOUR_FROM_NORMAL = 2,
  B200_RENDER_COLOUR_FROM_DEPTH_WEIGHT = 3,
  B200_RENDER_DEPTH_MAP = 4
} b200_render_type;

/* ---- engine handle ---------------------------------------------------------------------- */

/* One engine per volume. Engines on one device may have any of their calls in flight at the same time, each on its own
   stream: no kernel of the library waits on a CTA that has not started, so a volume's work completes whatever other engines'
   kernels hold the GPU, and its results are byte for byte those of the same calls run alone. The order between volumes is the
   caller's, set with b200_engine_wait_engine. (An engine alone on its device runs a faster form of the allocation's list pass
   that needs its whole grid resident; creating a second engine on the device waits once for the device, b200_engine_create,
   after which every engine there runs the form that does not. Create engines from the thread that enqueues their work.)
   DynSLAM's frame (static map + K car volumes, one GPU), with no host wait:
     1. b200_process_silhouettes_async on the static engine's stream (cuts the car frames out of the input);
     2. every car engine: b200_engine_wait_engine(car, static), then b200_process_frame_async of its volume;
     3. b200_process_frame_async of the static map;
     4. b200_engine_wait_engine(static, car) for every car, then b200_composite_instances on the static engine.
   Stand-alone calls (b200_decay with forceAllVoxels for Reap, b200_mesh_scene, b200_checkpoint_save) on one engine may run
   while the other engines' frames are in flight; they wait for their own engine's stream only. The volume group (b200_group_*,
   below) enqueues this sequence as one call and keeps the car volumes in a pool of slots restarted on the device. */
typedef struct b200_engine b200_engine;

typedef struct {
  int32_t device;              /* CUDA ordinal */
  int32_t numBlocks;           /* capacity the scratch is sized for */
  int32_t numBuckets;
  int32_t excessSize;
  int32_t img_w, img_h;
  int64_t decayRingItems;      /* capacity (visible-list items) of the decay snapshot ring; 0 = default 24*numBlocks.
                                  The reference keeps one copy of the visible list per frame in an unbounded std::queue
                                  (Reco_CUDA.cu:302-317); here the queue holds at most 4095 frames and decayRingItems list
                                  items. Beyond either bound the OLDEST snapshots are dropped (a Decay() that would have
                                  swept a dropped snapshot sweeps nothing; b200_frame_stats.droppedSnapshots counts them) —
                                  size it as min_decay_age x (visible blocks per frame) with headroom. Never an error. */
  void *stream;                /* optional caller cudaStream_t; NULL = engine-owned stream */
} b200_engine_config;

/* On failure nothing is left allocated, *out is NULL and b200_last_error(NULL) gives the reason (thread-local). */
b200_status b200_engine_create(const b200_engine_config *cfg, b200_engine **out);
void b200_engine_destroy(b200_engine *e);
const char *b200_last_error(const b200_engine *e);
void *b200_engine_stream(b200_engine *e);
int32_t b200_frame_index(const b200_engine *e);      /* frameIdx, Reco_CUDA.h:37-45 */

/* ---- ITMSceneReconstructionEngine ------------------------------------------------------- */

/* ResetScene — Reco_CUDA.cu:145-172 */
b200_status b200_reset_scene(b200_engine *e, b200_scene *scene);
/* Restart a volume on the device (no reference twin: what a new InfiniTamDriver for a new track would be). Afterwards e, scene
   and rs behave byte for byte like a newly created engine on a newly allocated scene that b200_reset_scene reset, with a newly
   allocated (zeroed) render state: frame index 0; decay queue and ring empty; decayed total and dropped-snapshot count 0;
   allocation request keys (tagged with frame indices) cleared; hash table, voxel blocks, free lists and counters reset as
   ResetScene resets them, swap states zeroed; every buffer of rs zeroed (entriesVisibleType, the visible list, the images,
   the forward-projection buffers when present) and noVisibleBlocks 0. Unlike b200_reset_scene, which keeps the frame index as
   the reference's ResetScene does, the frame index restarts.
   Stream-ordered on e's stream: no host wait, no allocation, only memsets and one reset kernel, so it may be enqueued while
   other engines' frames are in flight and inside a stream capture. The host fields of scene and rs are set to the reset
   values; b200_sync() refreshes them as usual. B200_ERR_INVALID, with nothing enqueued: a scene that does not fit the engine,
   rs or one of its buffers missing, a host-frame slot (b200_host_frame_submit*) or a preview slot (b200_render_view_submit)
   not yet waited for. */
b200_status b200_volume_restart_async(b200_engine *e, b200_scene *scene, b200_render_state *rs);
/* AllocateSceneFromDepth — Reco_CUDA.cu:175-358 */
b200_status b200_allocate_from_depth(b200_engine *e, b200_scene *scene, b200_render_state *rs,
                                     const b200_view *view, int onlyUpdateVisibleList);
/* IntegrateIntoScene — Reco_CUDA.cu:361-427 */
b200_status b200_integrate(b200_engine *e, b200_scene *scene, b200_render_state *rs,
                           const b200_view *view);
/* Decay — Reco_CUDA.cu:509-560 */
b200_status b200_decay(b200_engine *e, b200_scene *scene, b200_render_state *rs, int maxWeight,
                       int minAge, int forceAllVoxels);
/* GetDecayedBlockCount — Reco_CUDA.cu:563-566 */
size_t b200_decayed_block_count(const b200_engine *e);

/* ---- ITMVisualisationEngine ---------------------------------------------------------------- */

/* FindVisibleBlocks — Vis_CUDA.cu:151-180.
   Constraint on free-view use of this call (and of b200_expected_depths after it) beside the fused path: the list's length
   goes through the engine's one device-side visible count, which is the LIVE render state's list length for the next fused
   frame, and the call marks the host counters as current although it refreshes none of the scene's. So (1) with frames of
   b200_process_frame_async / b200_host_frame_submit* outstanding, call b200_sync() first: without it the next frame re-marks
   the wrong number of blocks and allocates from stale free-list counters (seen on an H100: hash table, voxels and lists all
   differ from a run without the render); (2) after these calls do not call b200_sync() again before the next frame: it would
   hand the free view's count to the live render state. b200_render_view_async has neither constraint. */
b200_status b200_find_visible_blocks(b200_engine *e, const b200_scene *scene,
                                     b200_render_state *rs, const b200_camera *cam);
/* CreateExpectedDepths — Vis_CUDA.cu:194-240 */
b200_status b200_expected_depths(b200_engine *e, const b200_scene *scene, b200_render_state *rs,
                                 const b200_camera *cam);
/* FindSurface / GenericRaycast — Vis_CUDA.cu:242-265, :484-489 */
b200_status b200_find_surface(b200_engine *e, const b200_scene *scene, b200_render_state *rs,
                              const b200_camera *cam);
/* RenderImage — Vis_CUDA.cu:267-343 */
b200_status b200_render_image(b200_engine *e, const b200_scene *scene, b200_render_state *rs,
                              const b200_camera *cam, b200_vec4u *d_outChar, float *d_outFloat,
                              int out_w, int out_h, b200_render_type type);
/* CreateICPMaps — Vis_CUDA.cu:372-390. d_points/d_normals = pointCloud->locations/colours */
b200_status b200_icp_maps(b200_engine *e, const b200_scene *scene, b200_render_state *rs,
                          const b200_view *view, b200_vec4f *d_points, b200_vec4f *d_normals);
/* ForwardRender — Vis_CUDA.cu:393-453 */
b200_status b200_forward_render(b200_engine *e, const b200_scene *scene, b200_render_state *rs,
                                const b200_view *view);
/* CreatePointCloud — Vis_CUDA.cu:346-369. *noTotalPoints = pointCloud->noTotalPoints */
b200_status b200_point_cloud(b200_engine *e, const b200_scene *scene, b200_render_state *rs,
                             const b200_view *view, const float *calib_rgb_to_depth,
                             int skipPoints, b200_vec4f *d_locations, b200_vec4f *d_colours,
                             uint32_t *noTotalPoints);

/* ---- ITMSwappingEngine ------------------------------------------------------------------- */

typedef struct {               /* the device half of ITMGlobalCache, Objects/ITMGlobalCache.h */
  b200_voxel *d_syncedVoxelBlocks;  /* SDF_TRANSFER_BLOCK_NUM blocks */
  uint8_t *d_hasSyncedData;         /* bool per transfer slot */
  int32_t *d_neededEntryIDs;        /* SDF_TRANSFER_BLOCK_NUM ints */
} b200_transfer_buffers;

/* IntegrateGlobalIntoLocal, device half — Swap_CUDA.cu:44-124.
   step 1: list entries to swap in; returns the count (<= SDF_TRANSFER_BLOCK_NUM) */
b200_status b200_swap_list_in(b200_engine *e, b200_scene *scene, b200_transfer_buffers *tb,
                              int *noNeeded);
/* step 2: merge the blocks the host has copied into tb into the local VBA */
b200_status b200_swap_integrate_in(b200_engine *e, b200_scene *scene, b200_transfer_buffers *tb,
                                   int noNeeded);
/* SaveToGlobalMemory, device half — Swap_CUDA.cu:126-216 */
b200_status b200_swap_out(b200_engine *e, b200_scene *scene, b200_render_state *rs,
                          b200_transfer_buffers *tb, int *noNeeded);

/* ---- fused fast path (no reference twin: removes the per-call blocking copies, SURVEY 3A) */

typedef struct {
  int32_t doDecay, decayMaxWeight, decayMinAge;
  int32_t doRaycast;           /* CreateExpectedDepths + CreateICPMaps */
  /* Optional per-frame renders for compositing (the multi-volume configuration): shaded from the ray points of THIS frame's
     raycast (same pose), i.e. RenderImage's shading pass without a second raycast, before Decay touches the volume.
     NULL = not rendered. d_colourRender: RENDER_COLOUR_FROM_VOLUME (w*h RGBA8); d_depthRender: RENDER_DEPTH_MAP (w*h f32). */
  b200_vec4u *d_colourRender;
  float *d_depthRender;
} b200_frame_opts;

/* Enqueue allocate -> integrate -> expected depths -> ICP maps -> decay for one frame on the
   engine stream without any host synchronisation. Counters live on the device; the host
   fields of scene / rs are refreshed by b200_sync(). */
b200_status b200_process_frame_async(b200_engine *e, b200_scene *scene, b200_render_state *rs,
                                     const b200_view *view, b200_vec4f *d_points,
                                     b200_vec4f *d_normals, const b200_frame_opts *opts);
b200_status b200_sync(b200_engine *e, b200_scene *scene, b200_render_state *rs);

/* Same, from host buffers: depth (float metres) and rgb are copied H2D from pinned staging
   inside the call and the grey raycast image is copied back to h_outImage (may be NULL). */
b200_status b200_process_frame_host(b200_engine *e, b200_scene *scene, b200_render_state *rs,
                                    b200_view *view, const float *h_depth,
                                    const b200_vec4u *h_rgb, float *d_depth_stage,
                                    b200_vec4u *d_rgb_stage, b200_vec4f *d_points,
                                    b200_vec4f *d_normals, const b200_frame_opts *opts,
                                    b200_vec4u *h_outImage);

/* Pipelined variant for streams of host frames: two staging slots and a copy stream inside the engine, so that the
   H2D copy of frame f+1 and the D2H copy of frame f's image overlap the kernels of the neighbouring frames.
   b200_host_frame_submit(slot) enqueues {H2D depth+RGB from (pinned) host memory, the fused frame, D2H of the grey raycast
   image into h_outImage} without blocking; b200_host_frame_wait(slot) blocks until that slot's image has landed.
   A slot may be resubmitted only after it has been waited for. Host counters are refreshed by b200_sync(). */
b200_status b200_host_frame_submit(b200_engine *e, b200_scene *scene, b200_render_state *rs, b200_view *view,
                                   const float *h_depth, const b200_vec4u *h_rgb, b200_vec4f *d_points, b200_vec4f *d_normals,
                                   const b200_frame_opts *opts, b200_vec4u *h_outImage, int slot);
b200_status b200_host_frame_wait(b200_engine *e, int slot);

/* ---- free-view preview (no reference twin: ITMMainEngine::GetImage's FREECAMERA branch, ITMMainEngine.cpp:231-278, which
   DynSLAM runs twice per volume and preview, once for the RGBA image and once for the depth) -----------------------------
   b200_render_view_async is FindVisibleBlocks + CreateExpectedDepths + RenderImage(type) + RenderImage(RENDER_DEPTH_MAP) from
   one pose as one enqueue: five launches on e's stream, the kernels of the stand-alone calls (table sweep that lists, image
   reset, one pass over the list that projects and rasterises, the raycast, one shading pass with two outputs), no host
   synchronisation, one raycast.

   rs is a free-view render state: never the live one of a volume that is being fused (rejected when the engine can tell).
   The outputs have rs's size, img_w x img_h. d_outChar (RGBA8) receives `type`, which is any render type but
   B200_RENDER_DEPTH_MAP; d_outDepth (f32) receives the depth map; either may be NULL, not both. RENDER_COLOUR_FROM_NORMAL
   leaves the alpha of found pixels as it is in d_outChar, as RenderImage does.

   Valid once the work has run (stream order on e's stream, or after b200_render_view_sync): rs->d_visibleBlockPositions,
   rs->d_minmax (the whole image), rs->d_raycastResult, d_outChar and d_outDepth, byte for byte what b200_find_visible_blocks,
   b200_expected_depths, b200_render_image(type) and b200_render_image(B200_RENDER_DEPTH_MAP) leave for the same scene, render
   state and camera; the MAX_RENDERING_BLOCKS rule is decided on the device. rs->noVisibleBlocks is a host field: only
   b200_render_view_sync refreshes it.

   It reads the scene and writes rs's buffers, the outputs and scratch of its own: none of the volume's counters, nothing a
   fused frame or a checkpoint reads. It may be enqueued with asynchronous frames outstanding, before or after them, any number
   of times; the frames' results do not change. (It counts as launched work for b200_checkpoint_save's kept classification: a
   save after it classifies afresh.)

   B200_ERR_INVALID, before anything is allocated or enqueued: a scene that does not fit the engine, rs, one of the three
   buffers named above or cam missing, a non-positive size, both outputs NULL, B200_RENDER_DEPTH_MAP or an unknown value as
   type, the live render state of the last fused frame as rs. */
b200_status b200_render_view_async(b200_engine *e, const b200_scene *scene, b200_render_state *rs, const b200_camera *cam,
                                   b200_render_type type, b200_vec4u *d_outChar, float *d_outDepth);
/* The host waits for e's stream and sets rs->noVisibleBlocks to the count of the latest b200_render_view_async, whose render
   state rs must be (B200_ERR_INVALID otherwise). Touches no other host field: the volume's counters stay as b200_sync() or
   the asynchronous frames left them. */
b200_status b200_render_view_sync(b200_engine *e, b200_render_state *rs);

/* The same render with the images landing in host memory (pinned, or pageable at the price cudaMemcpyAsync charges for it):
   the render goes to staging inside the engine, then a device-to-host copy on a copy stream of the preview's own, so that
   preview k's download runs under preview k+1's, or the next fused frame's, kernels. Only enqueues. slot in {0, 1}; a slot may
   be resubmitted only after b200_render_view_wait(slot) (B200_ERR_INVALID otherwise, nothing enqueued), and these slots are
   not b200_host_frame_submit's: neither blocks the other. h_outChar / h_outDepth: as d_outChar / d_outDepth above, valid when
   b200_render_view_wait(slot) returns; the alpha RENDER_COLOUR_FROM_NORMAL leaves on found pixels is 0 here. rs's buffers are
   valid in stream order as above. A larger image than the slots have held needs both slots waited for first. */
b200_status b200_render_view_submit(b200_engine *e, const b200_scene *scene, b200_render_state *rs, const b200_camera *cam,
                                    b200_render_type type, b200_vec4u *h_outChar, float *h_outDepth, int slot);
b200_status b200_render_view_wait(b200_engine *e, int slot);   /* the host waits for slot's images; OK when nothing is in flight */

/* e's stream waits, on the device, for everything enqueued so far on producer's stream (an event record and a
   cudaStreamWaitEvent; the host does not wait). This is what lets one engine composite layers other engines rendered
   (b200_composite_instances, b200_composite_depth) with no host synchronisation between the renders and the composite.
   Engines on the same device or on peers. It is the only ordering between engines: calls of engines on one device that do
   not wait for each other run concurrently (see the engine handle above for the frame sequence of one GPU). */
b200_status b200_engine_wait_engine(b200_engine *e, b200_engine *producer);

/* ---- view builder (SURVEY 8(f) rank 1): the step immediately before fusion ------------------------
   Replaces ITMViewBuilder_CUDA (Engine/DeviceSpecific/CUDA/ITMViewBuilder_CUDA.cu). All images are
   device pointers, row-major, w*h elements. Border semantics are the CUDA reference's (the filter leaves
   the two outermost rows/columns of its TARGET untouched, :196-209). */

typedef struct {
  int32_t trafoType;           /* ITMDisparityCalib::TrafoType (Objects/ITMDisparityCalib.h:24-29): 0 TRAFO_KINECT, 1 TRAFO_AFFINE */
  float params[2];             /* disparityCalib.params */
  float fx_depth;              /* intrinsics_d.projectionParamsSimple.fx (TRAFO_KINECT only) */
  float intrinsics_d[4];       /* intrinsics_d.projectionParamsSimple.all, for ComputeNormalAndWeights */
  int32_t useBilateralFilter;  /* ITMLibSettings::useBilateralFilter (default true, Utils/ITMLibSettings.cpp:63) */
  int32_t modelSensorNoise;    /* ITMLibSettings::modelSensorNoise (TRACKER_WICP only, :74-75) */
} b200_view_calib;

/* ITMViewBuilder::ConvertDisparityToDepth (ITMViewBuilder_CUDA.cu:120-135, DA/ITMViewBuilder.h:7-20) */
b200_status b200_convert_disparity_to_depth(b200_engine *e, float *d_out, const int16_t *d_in, int w, int h,
                                            float p0, float p1, float fx_depth);
/* ITMViewBuilder::ConvertDepthAffineToFloat (ITMViewBuilder_CUDA.cu:137-148, DA/ITMViewBuilder.h:22-28) */
b200_status b200_convert_depth_affine_to_float(b200_engine *e, float *d_out, const int16_t *d_in, int w, int h,
                                               float p0, float p1);
/* ITMViewBuilder::DepthFiltering — ONE pass (ITMViewBuilder_CUDA.cu:150-161, :196-209, DA/ITMViewBuilder.h:31-56);
   d_out's 2-pixel border is left untouched */
b200_status b200_depth_filtering(b200_engine *e, float *d_out, const float *d_in, int w, int h);
/* ITMViewBuilder::ComputeNormalAndWeights (ITMViewBuilder_CUDA.cu:163-178, :211-227, DA/ITMViewBuilder.h:59-114) */
b200_status b200_compute_normal_and_weights(b200_engine *e, b200_vec4f *d_normal, float *d_sigmaZ, const float *d_depth,
                                            int w, int h, const float intrinsic[4]);
/* ITMViewBuilder::UpdateView(view, rgb, rawDepth, useBilateralFilter, modelSensorNoise) without its two H2D
   copies (ITMViewBuilder_CUDA.cu:33-84): conversion + five filter passes + copy back in one kernel.
   d_depthNormal / d_depthUncertainty are used only with modelSensorNoise. The _async form only enqueues
   on the engine stream (the fused frame that follows is ordered behind it). */
b200_status b200_update_view(b200_engine *e, const int16_t *d_rawDepth, int w, int h, const b200_view_calib *calib,
                             float *d_depth, b200_vec4f *d_depthNormal, float *d_depthUncertainty);
b200_status b200_update_view_async(b200_engine *e, const int16_t *d_rawDepth, int w, int h, const b200_view_calib *calib,
                                   float *d_depth, b200_vec4f *d_depthNormal, float *d_depthUncertainty);
/* b200_host_frame_submit for a RAW sensor frame: h_rawDepth (int16, e.g. millimetres) and h_rgb are copied H2D,
   UpdateView runs on the device into the slot's float depth image, then the fused frame. Halves the depth upload. */
b200_status b200_host_frame_submit_raw(b200_engine *e, b200_scene *scene, b200_render_state *rs, b200_view *view,
                                       const int16_t *h_rawDepth, const b200_vec4u *h_rgb, const b200_view_calib *calib,
                                       b200_vec4f *d_points, b200_vec4f *d_normals, const b200_frame_opts *opts,
                                       b200_vec4u *h_outImage, int slot);

/* ---- DynSLAM's stored stereo input (DS/Input.cpp:41-97 -> DS/InfiniTamDriver.cpp:81-100) -------------------------------
   The two host loops every DynSLAM frame passes through before InfiniTamDriver::UpdateView, on the device and bit-exact:
   the int16 millimetre depth image from the stored DispNet disparity (DepthProvider::DepthFromDisparityMap<float> with
   scale 1, DS/DepthProvider.h:94-137, around PrecomputedDepthProvider::DepthFromDisparity, DS/PrecomputedDepthProvider.cpp:
   77-80) or from the stored ELAS depth (the max-depth clamp of PrecomputedDepthProvider::ReadPrecomputed, :52-74), and the
   RGBA8 colour image from OpenCV's BGR8 frame (CvToItm(const cv::Mat3b &, ...), DS/InfiniTamDriver.cpp:81-100). */

enum { B200_DEPTH_IN_DISPARITY_F32 = 0, B200_DEPTH_IN_DEPTH_MM_S16 = 1 };

typedef struct {
  int32_t kind;                /* B200_DEPTH_IN_*: 0 float32 disparity in px (DispNet PFM), 1 int16 depth in mm (ELAS XML) */
  float baseline_m;            /* dynslam::StereoCalibration::baseline_meters (DS/DepthProvider.h:22-28; kind 0 only) */
  float focal_length_px;       /* dynslam::StereoCalibration::focal_length_px (kind 0 only) */
  float min_depth_m;           /* DepthProvider::min_depth_m_ (kind 0 only: the clamp of kind 1 has no lower bound) */
  float max_depth_m;           /* DepthProvider::max_depth_m_; (int32)(max_depth_m * 1000) must be below 32767 */
} b200_depth_input;

/* d_out_mm (w*h int16) from d_in (w*h float disparities or int16 millimetres, per kind). A depth of (int32)(1000 * focal *
   baseline / disp) outside [(int32)(min_depth_m * 1000), (int32)(max_depth_m * 1000)] becomes 0, as does every |disp| < 1
   (the reference's unqualified abs() is int abs(int)); kind 1 sets values above (int16)round(max_depth_m * 1000) to 0.
   d_out_mm may equal d_in for kind 1. Synchronous. */
b200_status b200_depth_mm_from_input(b200_engine *e, int16_t *d_out_mm, const void *d_in, int w, int h, const b200_depth_input *in);
/* CvToItm(const cv::Mat3b &, ITMUChar4Image *): d_bgr (w*h*3 bytes) into d_out (w*h RGBA8, a = 255). Synchronous. */
b200_status b200_bgr_to_rgba(b200_engine *e, b200_vec4u *d_out, const uint8_t *d_bgr, int w, int h);
/* b200_host_frame_submit_raw from the stored stereo input: h_depthIn (view->depth_w x depth_h, float disparity or int16 mm
   per in->kind) and h_bgr (view->rgb_w x rgb_h BGR8) are copied H2D; on the copy stream one kernel turns them into the int16
   mm depth and the RGBA8 colour image; then UpdateView and the fused frame run as in b200_host_frame_submit_raw. If
   d_depthMmOut is not NULL it receives the frame's int16 mm depth (the input depth of b200_evaluate_depth); it is complete
   when b200_host_frame_wait(slot) returns. Same slot rules as b200_host_frame_submit; modelSensorNoise is rejected. */
b200_status b200_host_frame_submit_stereo(b200_engine *e, b200_scene *scene, b200_render_state *rs, b200_view *view,
                                          const uint8_t *h_bgr, const void *h_depthIn, const b200_depth_input *in,
                                          const b200_view_calib *calib, b200_vec4f *d_points, b200_vec4f *d_normals,
                                          const b200_frame_opts *opts, b200_vec4u *h_outImage, int16_t *d_depthMmOut, int slot);

/* ---- instance frame splitting (SURVEY 8(f) rank 2) ---------------------------------------------------
   Replaces the download / CPU masking / upload round trip of InstanceReconstructor::ProcessFrame
   (DS/InstRecLib/InstanceReconstructor.cpp:180-197) around ProcessSilhouette_CPU / RemoveSilhouette_CPU
   (:59-170). The frame (view->rgb, view->depth) and the instance frames stay on the device. */

typedef struct {
  int32_t x0, y0, x1, y1;      /* instreclib::utils::BoundingBox::r, inclusive (Utils/BoundingBox.h:35-37) */
  const uint8_t *d_data;       /* Mask::mask_data_ (cv::Mat1b, box-sized, row-major; 1 = inside) on the DEVICE */
} b200_mask;

typedef struct {
  int32_t action;              /* what InstanceReconstructor::ProcessSilhouette (:226-285) decides for the track:
                                  0 = keep in the main map (static / static class),
                                  1 = RemoveSilhouette_CPU(delete_mask) only (uncertain or unreconstructable),
                                  2 = ProcessSilhouette_CPU(copy_mask -> instance frame) then RemoveSilhouette_CPU(delete_mask) */
  b200_mask copy_mask, delete_mask;
  b200_vec4u *d_dest_rgb;      /* instance_view->rgb, full frame size (action 2) */
  float *d_dest_depth;         /* instance_view->depth */
} b200_silhouette_op;

/* Applies ops[0..n) in order to the frame, exactly like the reference's loop over the active tracks
   (InstanceReconstructor::UpdateTracks, :210-224): a later op sees the pixels an earlier one blanked. */
b200_status b200_process_silhouettes(b200_engine *e, b200_vec4u *d_rgb, float *d_depth, int w, int h,
                                     const b200_silhouette_op *ops, int n);
b200_status b200_process_silhouettes_async(b200_engine *e, b200_vec4u *d_rgb, float *d_depth, int w, int h,
                                           const b200_silhouette_op *ops, int n);

/* ---- compositing of per-volume renders (SURVEY 8(f) rank 3, the consumer of the multi-GPU gather) ------ */

typedef struct {
  const b200_vec4u *d_color;   /* the instance's render (GetImage) */
  const float *d_depth;        /* its depth render (GetFloatImage kDepth); 0 = nothing */
  int32_t tint[4];             /* kMatplotlib2Palette[track id % size] (InstanceReconstructor.cpp:43-55) */
} b200_instance_layer;

/* CompositeDepth (InstanceReconstructor.cpp:850-869) */
b200_status b200_composite_depth(b200_engine *e, float *d_target, const float *d_source, int n);
/* CompositeColor (InstanceReconstructor.cpp:873-905) */
b200_status b200_composite_color(b200_engine *e, b200_vec4u *d_target_color, float *d_target_depth,
                                 const b200_vec4u *d_instance_color, const float *d_instance_depth, int n,
                                 const int32_t tint[4], float tint_strength);
/* CompositeInstances (InstanceReconstructor.cpp:932-987) without the renders: dims the background by
   dim_factor (< 0: no dimming) and composites layers[0..n_layers) in order, all in one pass over the image. */
b200_status b200_composite_instances(b200_engine *e, b200_vec4u *d_out_color, float *d_out_depth, int n,
                                     const b200_instance_layer *layers, int n_layers, float dim_factor,
                                     float tint_strength);

/* ---- volume group: the static map and a pool of car-volume slots on one GPU (InstanceReconstructor's one ITMScene per car
   track, DS/InstRecLib/InstanceReconstructor.cpp:363-389) --------------------------------------------------------------------
   b200_group_create makes max_cars slots up front, each with an engine, a scene, a render state, an instance frame (RGBA8 and
   f32 depth), a colour and a depth render for the composite and the ICP point and normal maps. So the device waits of
   b200_engine_create happen there only, and slot engines are destroyed only by b200_group_destroy: a track that starts takes a
   slot and restarts it on the device (b200_group_track_start), a track that ends leaves its slot for the next one.
   Memory per slot (arithmetic from the buffer sizes, not a measurement), at the defaults and a 1242 x 375 image: voxel blocks
   29.3 MB, hash table 31.5 MB, excess and allocation lists 2.1 MB, visibility bytes 1.6 MB, the render state's images 13.0 MB,
   instance frame and renders 7.5 MB, ICP maps 14.9 MB, engine scratch about 19 MB: about 119 MB.

   Every per-engine call works on a slot's engine, scene and render state (b200_group_slot) unchanged: b200_decay with
   forceAllVoxels for Reap, b200_mesh_scene, b200_checkpoint_save / _load, b200_render_view_async. They are ordered after the
   slot's own work only, as between any engines. */
typedef struct b200_group b200_group;

typedef struct {
  b200_engine *static_engine;          /* the caller's static map: engine, scene and live render state, kept by pointer for the */
  b200_scene *static_scene;            /* group's life; its host counters are written by b200_group_sync */
  b200_render_state *static_rs;
  b200_vec4f *static_points, *static_normals;   /* the static map's ICP maps (w*h each) */
  int32_t max_cars;                    /* slots */
  /* the car volumes; a field <= 0 takes the default in brackets (bench.py configs[2]: InstanceReconstructor.cpp:365-389's
     5 x 5 x 10 m at 0.035 m, with the full-size table) */
  int32_t numBlocks;                   /* [7142] */
  int32_t numBuckets, excessSize;      /* [0x100000, 0x80000] */
  float voxelSize, mu;                 /* [0.035, 1.0]; viewFrustum and stopIntegratingAtMaxW are the static scene's */
  int32_t maxW;                        /* [50] */
  int32_t img_w, img_h;                /* [the static render state's]; must equal it */
  int64_t decayRingItems;              /* as b200_engine_config's [24 x numBlocks] */
  int32_t shared_stream;               /* 1: every slot on the static engine's stream; 0: a stream per slot */
  float dim_factor, tint_strength;     /* the composite's, as b200_composite_instances takes them */
} b200_group_config;

typedef struct {                       /* a slot's device images, owned by the group (img_w x img_h each) */
  b200_vec4u *d_instance_rgb; float *d_instance_depth;   /* the instance frame the silhouettes cut out */
  b200_vec4u *d_colour_render; float *d_depth_render;    /* RENDER_COLOUR_FROM_VOLUME and RENDER_DEPTH_MAP of its latest frame */
  b200_vec4f *d_points, *d_normals;                      /* its ICP maps */
} b200_group_images;

typedef struct {                       /* one car of a frame */
  int32_t slot;
  int32_t action;                      /* b200_silhouette_op.action, with its masks (device data, the caller's) */
  b200_mask copy_mask, delete_mask;
  b200_camera cam;                     /* the car's pose (M and its inverse) and the depth intrinsics of its instance frame */
  int32_t fuse;                        /* nonzero: fuse the instance frame into the slot's volume and composite its layer */
  int32_t tint[4];                     /* the layer's tint (kMatplotlib2Palette[track id % 10] in DynSLAM) */
} b200_group_car;

/* On failure nothing is left allocated, *out is NULL and b200_group_last_error(NULL) gives the reason (thread-local). Waits for
   the device. */
b200_status b200_group_create(const b200_group_config *cfg, b200_group **out);
void b200_group_destroy(b200_group *g);
const char *b200_group_last_error(const b200_group *g);
/* slot i's engine, scene and render state (pointers into the group; any output may be NULL) */
b200_status b200_group_slot(b200_group *g, int slot, b200_engine **engine, b200_scene **scene, b200_render_state **rs);
b200_status b200_group_slot_images(b200_group *g, int slot, b200_group_images *out);
/* A new track in slot: b200_volume_restart_async of the slot's volume on its stream, after everything the group has enqueued
   so far (the slot's stream waits for the static engine's). No host wait, no allocation. */
b200_status b200_group_track_start(b200_group *g, int slot);
/* One frame of every volume as one enqueue, DynSLAM's sequence of the engine handle's comment above:
     1. one silhouette launch on the static engine's stream, cars[0..n) in order (action 2 extracts into the slot's instance
        frame; a fused car with action 0 or 1 gets an empty instance frame, white with depth 0, as ProcessSilhouette leaves it);
     2. for every fused car: its stream waits for the static engine's, then b200_process_frame_async of its volume (pose and
        intrinsics from cam, decay as below) with the slot's colour and depth renders;
     3. b200_process_frame_async of the static map with static_view (normally d_depth and d_rgb after step 1), its depth render
        into d_out_depth;
     4. the static engine's stream waits for every slot that has work it has not waited for;
     5. the static map's shaded raycast image and depth under the fused cars' layers, in cars order, dimmed and tinted as
        b200_composite_instances does, into d_out_color / d_out_depth.
   d_rgb / d_depth: the frame (img_w x img_h), updated in place by the silhouettes. decay: NULL, or {maxWeight, minAge} for
   every volume. No host wait, no allocation, no copy from host memory. B200_ERR_INVALID, before anything is enqueued: a null
   pointer, n < 0 or n > max_cars, a static view of another size, a slot out of range, a slot twice in one frame, a slot that
   was never started, an unknown action or a mask it needs missing. Host counters are refreshed by b200_group_sync. */
b200_status b200_group_frame_async(b200_group *g, b200_vec4u *d_rgb, float *d_depth, const b200_view *static_view,
                                   const b200_group_car *cars, int n, const int32_t *decay, b200_vec4u *d_out_color,
                                   float *d_out_depth);
/* b200_sync of the static map and of every slot */
b200_status b200_group_sync(b200_group *g);

/* ---- evaluation consumer of the float raycast (SURVEY 8(f) rank 3): Evaluation::EvaluateDepth ----------------------------
   DS/Evaluation/Evaluation.cpp:241-304 with ProjectLidar (:214-238) and EvaluationCallback::ProcessLidarPoint /
   ComputeAccuracy (DS/Evaluation/EvaluationCallback.cpp:15-103): every LIDAR return of a frame is projected into the left
   and right colour cameras (double precision), the rendered depth (the float raycast / composite preview, metres) and the
   input depth (int16 millimetres) under it become disparities, and each callback — one per delta_max, plus the KITTI-style
   one — counts the point as missing, erroneous or correct for the fused and for the input depth. One launch for all points
   and all callbacks; only the counters come back. */

typedef struct b200_eval_params {
  double velo_to_cam[16];      /* Evaluation::velo_to_left_gray_cam_ (Eigen::Matrix4d, column-major) */
  double proj_left[12];        /* proj_left_color_  (Eigen::Matrix<double, 3, 4>, column-major) */
  double proj_right[12];       /* proj_right_color_ */
  float baseline_m, left_focal_length_px, min_depth_m, max_depth_m;
  int32_t frame_width, frame_height;
} b200_eval_params;

typedef struct b200_eval_callback {   /* EvaluationCallback's constructor arguments (EvaluationCallback.h:14-24) */
  float delta_max;
  int32_t compare_on_intersection, kitti_style;
} b200_eval_callback;

typedef struct b200_eval_stats { int64_t missing, error, correct, missing_separate; } b200_eval_stats;   /* Evaluation.h:27-33 */
typedef struct b200_eval_result { int64_t measurement_count; b200_eval_stats rendered, input; } b200_eval_result;
typedef struct b200_eval_summary { int64_t valid_lidar_points, epi_errors, negative_disparities, skipped_lidar_points; } b200_eval_summary;

/* SegmentedCallback::GetPointAssociation's verdict for the pixel a point falls on (SegmentedCallback.h), one byte per pixel */
enum { B200_EVAL_STATIC = 0, B200_EVAL_DYNAMIC = 1, B200_EVAL_NEITHER = 2 };
#define B200_EVAL_MAX_CALLBACKS 16

/* d_lidar: n points of four floats (x, y, z, reflectance — the KITTI velodyne .bin record); d_rendered_depth, d_input_depth_mm:
   frame_width x frame_height; d_association: one byte per pixel or NULL (every point static: Evaluation::EvaluateFrame);
   callbacks / out_static / out_dynamic: host arrays of n_callbacks (out_dynamic may be NULL: dynamic points are skipped).
   Synchronous, like the reference. A negative ground-truth disparity returns B200_ERR_NEGATIVE_DISPARITY (the reference
   throws at the first one; the counts are then unspecified). */
b200_status b200_evaluate_depth(b200_engine *e, const b200_eval_params *params, const float *d_lidar, int n,
                                const float *d_rendered_depth, const int16_t *d_input_depth_mm, const uint8_t *d_association,
                                const b200_eval_callback *callbacks, int n_callbacks, b200_eval_result *out_static,
                                b200_eval_result *out_dynamic, b200_eval_summary *summary);

/* ---- meshing (SURVEY 8(f) rank 4): ITMMeshingEngine<TVoxel, ITMVoxelBlockHash>::MeshScene --------------------------------
   Engine/DeviceSpecific/CUDA/ITMMeshingEngine_CUDA.cu:37-81 with DeviceAgnostic/ITMMeshingEngine.h. d_triangles is
   mesh->triangles->GetData(MEMORYDEVICE_CUDA) (ITMMesh::Triangle, Objects/ITMMesh.h:20-23: six Vector3f), noMaxTriangles
   mesh->noMaxTriangles; *noTotalTriangles receives mesh->noTotalTriangles. Triangles come out in the order of the reference's
   serial CPU engine (ascending hash entry, then z, y, x, then the case table), not in the CUDA engine's atomicAdd order. */

typedef struct { float p0[3], p1[3], p2[3], c0[3], c1[3], c2[3]; } b200_triangle;

b200_status b200_mesh_scene(b200_engine *e, const b200_scene *scene, b200_triangle *d_triangles, uint32_t noMaxTriangles,
                            uint32_t *noTotalTriangles);

/* ---- checkpoints: one volume's state saved to a host buffer and loaded back (no reference twin) ------------------------
   A checkpoint holds everything that decides the future of one volume and nothing that can be derived: after a load, fusion
   continues bit for bit as if the process had never stopped. It holds no device pointers or ordinals, so it can be loaded on
   another GPU or in another process; the same state always gives the same bytes (save -> load -> save is identical).

   Layout (little-endian). A 512-byte b200_checkpoint_header, then the sections below in this order, each 16-byte aligned, the
   voxel payload 4096-byte aligned; the header's section table gives every offset and length, padding bytes are zero:
     HASH_INDEX      uint32 x noEntries       ascending indices of the hash entries that differ from the reset entry
                                              {pos 0, pad 0, offset 0, ptr -2, allocatedTime 0} (stale pos/offset of freed heads count)
     HASH_ENTRIES    20 B x noEntries         those entries (b200_hash_entry)
     ALLOCATION_LIST int32 x numBlocks        localVBA's free list, in full
     EXCESS_LIST     int32 x excessSize       the excess list, in full
     SWAP_STATES     uint8 x (numBuckets + excessSize), only with B200_CK_HAS_SWAP_STATES
     VIS_INDEX       uint32 x noVisBytes      ascending indices of the nonzero entriesVisibleType bytes
     VIS_VALUE       uint8 x noVisBytes       their values
     VISIBLE_LIST    12 B x min(noVisibleBlocks, numBlocks)
     MINMAX          8 B x img_w*img_h        renderingRangeImage
     RAYCAST_RESULT  16 B x img_w*img_h
     RAYCAST_IMAGE   4 B x img_w*img_h
     FWD_PROJECTION  16 B x img_w*img_h, FWD_MISSING int32 x img_w*img_h: only with B200_CK_HAS_FORWARD
     QUEUE_COUNTS    int32 x noSnapshots      the decay queue, oldest first: items per snapshot, -1 = overwritten in the ring
                                              before the save (b200_engine_config.decayRingItems; its Decay sweeps nothing)
     QUEUE_ITEMS     12 B x noQueueItems      the snapshots' block positions, oldest first
     BLOCK_IDS       uint32 x noBlocks        ascending ids of the voxel blocks that differ from a reset block {sdf 32767, 0...},
                                              allocated or not (decay can free a block whose voxels still hold sdf and colour)
     BLOCK_DATA      4096 B x noBlocks        those blocks
   Not saved: the engine's cache of the visible list's VBA pointers (the next integration looks the blocks up itself). */

#define B200_CHECKPOINT_MAGIC "B200CKPT"
#define B200_CHECKPOINT_VERSION 1
#define B200_CHECKPOINT_HEADER_BYTES 512
enum {
  B200_CK_HASH_INDEX, B200_CK_HASH_ENTRIES, B200_CK_ALLOCATION_LIST, B200_CK_EXCESS_LIST, B200_CK_SWAP_STATES, B200_CK_VIS_INDEX,
  B200_CK_VIS_VALUE, B200_CK_VISIBLE_LIST, B200_CK_MINMAX, B200_CK_RAYCAST_RESULT, B200_CK_RAYCAST_IMAGE, B200_CK_FWD_PROJECTION,
  B200_CK_FWD_MISSING, B200_CK_QUEUE_COUNTS, B200_CK_QUEUE_ITEMS, B200_CK_BLOCK_IDS, B200_CK_BLOCK_DATA, B200_CK_SECTIONS
};
#define B200_CK_HAS_SWAP_STATES 1u
#define B200_CK_HAS_FORWARD 2u

typedef struct {
  char magic[8];                       /* B200_CHECKPOINT_MAGIC, no terminator */
  uint32_t version, flags;             /* B200_CHECKPOINT_VERSION; B200_CK_HAS_* */
  int32_t numBlocks, numBuckets, excessSize, img_w, img_h;   /* geometry: must equal the loading scene's and render state's */
  float voxelSize, mu;                 /* must equal the loading scene's, bit for bit */
  int32_t maxW; float viewFrustum_min, viewFrustum_max; int32_t stopIntegratingAtMaxW, useSwapping;   /* for information only */
  int32_t lastFreeBlockId, lastFreeExcessListId, noVisibleBlocks, noFwdProjMissingPoints;
  int32_t frameIdx, noSnapshots;
  int64_t totalDecayed, droppedSnapshots;
  int64_t noEntries, noVisBytes, noBlocks, noQueueItems;
  uint64_t totalBytes;
  uint64_t section[B200_CK_SECTIONS][2];   /* offset, length in bytes */
  uint8_t reserved[96];
} b200_checkpoint_header;

/* Save. First brings the engine to the b200_sync() state (outstanding frames finished, the expected-depth image complete).
   h_out == NULL: only *size is set. Every such size query classifies the state afresh, and the save with h_out that
   immediately follows it reuses that classification instead of sweeping the voxel block array again (any engine call that
   launches work in between discards it; a save with h_out != NULL and no size query before it classifies on its own). After
   a change the caller makes to the buffers itself, which the engine cannot see, a size query therefore brings the saved
   state up to date. h_out may be pageable or pinned; capacity below *size is B200_ERR_INVALID and nothing is written.
   Synchronous. */
b200_status b200_checkpoint_save(b200_engine *e, b200_scene *scene, b200_render_state *rs, void *h_out, size_t capacity,
                                 size_t *size);
/* Load into a scene and render state of the same geometry, voxelSize and mu, with the same optional buffers (swap states,
   forward projection). Writes every saved buffer (the rest of the voxel blocks, hash entries and visibility bytes get their
   reset values), the host counters of scene and rs, and the engine's frame index, decay counters and queue. A queue longer
   than this engine's ring or 4095-frame queue holds drops its oldest snapshots, as a running engine does. Every rejection
   (B200_ERR_INVALID: bad magic or version, a truncated buffer or section table, a geometry, voxelSize, mu or optional-buffer
   mismatch, an index or count out of range or out of order, a host-frame slot not yet waited for) is made before anything
   is written. A checkpoint is trusted data beyond that: the values inside its sections (hash entries, free-list entries,
   voxels, images) are loaded as they are, without range checks or a checksum. Clears the engine's allocation request keys,
   which are tagged with frame indices, so a checkpoint of an earlier frame loads into an engine that has run past it.
   Synchronous. */
b200_status b200_checkpoint_load(b200_engine *e, b200_scene *scene, b200_render_state *rs, const void *h_in, size_t size);

/* ---- the exchange step of the multi-volume configuration (SURVEY 8e) -----------------------------------------------
   One volume per GPU, one process per GPU: the static map on rank 0, one ITMScene per car on the other ranks
   (DS/InstRecLib/InstanceReconstructor.cpp:363-389). Fusion, allocation and decay need no communication; per frame every
   rank hands the colour (RGBA8) and depth (f32) renders of its volume to rank 0, which z-composites them over its own render
   (CompositeInstances, InstanceReconstructor.cpp:932-987). NCCL send/recv over NVLink on the communicator's own stream,
   double-buffered, so the next frame's kernels never wait for this frame's rendez-vous. libnccl.so.2 is loaded at run time. */

#define B200_COMM_ID_BYTES 128
typedef struct b200_comm b200_comm;

/* rank 0 makes the rendez-vous id (ncclGetUniqueId); the host distributes it to the other ranks over any channel */
b200_status b200_comm_unique_id(char id[B200_COMM_ID_BYTES]);
b200_status b200_comm_create(int device, int nranks, int rank, const char id[B200_COMM_ID_BYTES], int img_w, int img_h,
                             b200_comm **out);
void b200_comm_destroy(b200_comm *c);
const char *b200_comm_last_error(const b200_comm *c);   /* c == NULL: why the last create / unique_id failed on this thread */
/* Per frame, every rank: d_color / d_depth (w*h each) are this volume's renders, produced by work already enqueued on e's
   stream. Ranks > 0 send them to rank 0. Rank 0 receives the other ranks' layers, copies its own render to d_out_color /
   d_out_depth and composites the layers over it in rank order (tints: 4 ints per layer, rank r at tints[4*(r-1)];
   dim_factor < 0: no dimming). Only enqueues. slot in {0, 1} double-buffers the hand-over. */
b200_status b200_gather_composite_submit(b200_comm *c, b200_engine *e, const b200_vec4u *d_color, const float *d_depth,
                                         b200_vec4u *d_out_color, float *d_out_depth, const int32_t *tints, float dim_factor,
                                         float tint_strength, int slot);
/* e's stream waits on the device until slot's exchange has drained (call before overwriting the buffers handed over with it) */
b200_status b200_gather_composite_release(b200_comm *c, b200_engine *e, int slot);
/* the host waits until slot's exchange (on rank 0: and the composite) has finished */
b200_status b200_gather_composite_wait(b200_comm *c, int slot);

#ifdef __cplusplus
}
#endif
#endif /* B200FUSION_H */
