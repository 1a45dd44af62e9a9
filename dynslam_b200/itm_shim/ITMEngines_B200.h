// ITMEngines_B200.h — C++ host side of the drop-in: ITMLib engine subclasses that forward to the
// C-ABI of libb200fusion (include/b200fusion.h). Header-only; compiled against the UNMODIFIED
// reference headers (-I <DynSLAM>/src/InfiniTAM/InfiniTAM), nothing from the reference is copied.
//
//   ITMSceneReconstructionEngine_B200<TVoxel, ITMVoxelBlockHash>  : ITMSceneReconstructionEngine  (Engine/ITMSceneReconstructionEngine.h:33-78)
//   ITMVisualisationEngine_B200<TVoxel, ITMVoxelBlockHash>        : ITMVisualisationEngine        (Engine/ITMVisualisationEngine.h:112-127)
//   ITMSwappingEngine_B200<TVoxel, ITMVoxelBlockHash>             : ITMSwappingEngine             (Engine/ITMSwappingEngine.h:22-31)
//
// All ITMLib objects (ITMScene, ITMRenderState_VH, ITMView, ITMTrackingState) are allocated
// exactly as today with MEMORYDEVICE_CUDA; the shim only unpacks their raw device pointers.
// Error convention: capacity errors re-throw std::runtime_error with the reference's messages
// (Reco_CUDA.cu:348-357) so InstanceReconstructor.cpp:662-671 keeps working; CUDA errors print and
// exit(-1) like ORcudaSafeCall (ORUtils/CUDADefines.cpp:9-47).
// One b200_engine handle is shared by the three engines of a volume (B200EngineHandle).
#pragma once

#include <cstdio>
#include <cstdlib>
#include <map>
#include <memory>
#include <stdexcept>

#include "ITMLib/Utils/ITMLibSettings.h"

#include "ITMLib/Engine/ITMMeshingEngine.h"
#include "ITMLib/Engine/ITMSceneReconstructionEngine.h"
#include "ITMLib/Engine/ITMSwappingEngine.h"
#include "ITMLib/Engine/ITMVisualisationEngine.h"
#include "ITMLib/Objects/ITMRenderState_VH.h"

#include "b200fusion.h"

namespace ITMLib {
namespace Engine {

static_assert(sizeof(ITMHashEntry) == sizeof(b200_hash_entry), "ITMHashEntry layout");
static_assert(sizeof(Vector3i) == sizeof(b200_vec3i) && sizeof(Vector4f) == sizeof(b200_vec4f), "vector layouts");

/// Owns the opaque engine (scratch, decay ring, stream) of ONE volume.
class B200EngineHandle {
 public:
  b200_engine *e = nullptr;
  /// decayRingItems: capacity of the engine's decay-snapshot ring in visible-list items (0 = 24 x sdfLocalBlockNum); size it as
  /// min_decay_age x visible blocks per frame with headroom. When it (or the 4095-frame queue) is full, the oldest snapshots
  /// are dropped instead of growing without bound like the reference's std::queue (Reco_CUDA.cu:302-317).
  B200EngineHandle(int device, long sdfLocalBlockNum, Vector2i imgSize, long long decayRingItems = 0) {
    b200_engine_config cfg{};
    cfg.decayRingItems = decayRingItems;
    cfg.device = device;
    cfg.numBlocks = (int)sdfLocalBlockNum;
    cfg.numBuckets = (int)SDF_BUCKET_NUM;
    cfg.excessSize = (int)SDF_EXCESS_LIST_SIZE;
    cfg.img_w = imgSize.x; cfg.img_h = imgSize.y;
    const b200_status st = b200_engine_create(&cfg, &e);
    if (st != B200_OK) { fprintf(stderr, "b200fusion: engine create failed (%d): %s\n", (int)st, b200_last_error(nullptr)); exit(-1); }
  }
  ~B200EngineHandle() { b200_engine_destroy(e); }
  void check(b200_status st) const {
    switch (st) {
    case B200_OK: return;
    case B200_ERR_VBA_FULL:
      throw std::runtime_error("Invalid free voxel block ID. InfiniTAM has run out of space in the Voxel Block Array.");
    case B200_ERR_EXCESS_FULL:
      throw std::runtime_error("Invalid free excess list slot ID. InfiniTAM has run out of slots in the hash table excess list. "
                               "Consider increasing the size of the excess list or the number of buckets.");
    default:
      fprintf(stderr, "b200fusion error %d: %s\n", (int)st, b200_last_error(e));
      exit(-1);
    }
  }
};

/// The engine handle of the volume configured by `settings` (one ITMLibSettings object per ITMMainEngine / InfiniTamDriver,
/// i.e. per volume, in DynSLAM: DS/InfiniTamDriver.h, DS/InstRecLib/InstanceReconstructor.cpp:363-389). ITMMainEngine's
/// constructor calls it first, with the image size (integration/itmlib_b200.patch); ITMDenseMapper's constructor, which only
/// receives the settings, then picks the same handle up. Entries die with their last engine (weak references).
inline std::shared_ptr<B200EngineHandle> B200HandleFor(const ITMLibSettings *settings, Vector2i imgSize = Vector2i(0, 0)) {
  static std::map<const ITMLibSettings *, std::weak_ptr<B200EngineHandle>> registry;
  std::shared_ptr<B200EngineHandle> h = registry[settings].lock();
  if (!h) {
    if (imgSize.x <= 0 || imgSize.y <= 0) throw std::runtime_error("B200HandleFor: no engine yet for these settings and no image size given");
    int device = 0;
    cudaGetDevice(&device);
    h = std::make_shared<B200EngineHandle>(device, settings->sdfLocalBlockNum, imgSize);
    registry[settings] = h;
  }
  return h;
}

namespace b200_detail {

template <class TVoxel>
inline b200_scene PackScene(ITMScene<TVoxel, ITMVoxelBlockHash> *scene) {
  static_assert(sizeof(TVoxel) == sizeof(b200_voxel), "libb200fusion is built for ITMVoxel_s_rgb (Utils/ITMLibDefines.h:233)");
  b200_scene s{};
  s.d_voxels = (b200_voxel *)scene->localVBA.GetVoxelBlocks();
  s.d_allocationList = scene->localVBA.GetAllocationList();
  s.d_hash = (b200_hash_entry *)scene->index.GetEntries();
  s.d_excessList = scene->index.GetExcessAllocationList();
  s.d_swapStates = scene->useSwapping ? (uint8_t *)scene->globalCache->GetSwapStates(true) : nullptr;
  s.numBlocks = scene->index.getNumAllocatedVoxelBlocks();
  s.numBuckets = (int)SDF_BUCKET_NUM;
  s.excessSize = (int)SDF_EXCESS_LIST_SIZE;
  s.lastFreeBlockId = scene->localVBA.lastFreeBlockId;
  s.lastFreeExcessListId = scene->index.GetLastFreeExcessListId();
  const ITMSceneParams *p = scene->sceneParams;
  s.voxelSize = p->voxelSize; s.mu = p->mu; s.maxW = p->maxW;
  s.viewFrustum_min = p->viewFrustum_min; s.viewFrustum_max = p->viewFrustum_max;
  s.stopIntegratingAtMaxW = p->stopIntegratingAtMaxW ? 1 : 0;
  s.useSwapping = scene->useSwapping ? 1 : 0;
  return s;
}

template <class TVoxel>
inline void UnpackScene(const b200_scene &s, ITMScene<TVoxel, ITMVoxelBlockHash> *scene) {
  scene->localVBA.lastFreeBlockId = s.lastFreeBlockId;
  scene->index.SetLastFreeExcessListId(s.lastFreeExcessListId);
}

inline b200_render_state PackRenderState(ITMRenderState *renderState) {
  ITMRenderState_VH *vh = (ITMRenderState_VH *)renderState;
  b200_render_state r{};
  r.d_visibleBlockPositions = (b200_vec3i *)vh->GetVisibleBlockPositions();
  r.d_entriesVisibleType = vh->GetEntriesVisibleType();
  r.d_minmax = (b200_vec2f *)vh->renderingRangeImage->GetData(MEMORYDEVICE_CUDA);
  r.d_raycastResult = (b200_vec4f *)vh->raycastResult->GetData(MEMORYDEVICE_CUDA);
  r.d_forwardProjection = (b200_vec4f *)vh->forwardProjection->GetData(MEMORYDEVICE_CUDA);
  r.d_fwdProjMissingPoints = vh->fwdProjMissingPoints->GetData(MEMORYDEVICE_CUDA);
  r.d_raycastImage = (b200_vec4u *)vh->raycastImage->GetData(MEMORYDEVICE_CUDA);
  r.img_w = vh->renderingRangeImage->noDims.x; r.img_h = vh->renderingRangeImage->noDims.y;
  r.noVisibleBlocks = vh->noVisibleBlocks;
  r.noFwdProjMissingPoints = vh->noFwdProjMissingPoints;
  return r;
}

inline void UnpackRenderState(const b200_render_state &r, ITMRenderState *renderState) {
  ITMRenderState_VH *vh = (ITMRenderState_VH *)renderState;
  vh->noVisibleBlocks = r.noVisibleBlocks;
  vh->noFwdProjMissingPoints = r.noFwdProjMissingPoints;
}

inline void CopyM(const Matrix4f &M, float *out) { for (int i = 0; i < 16; ++i) out[i] = M.m[i]; }
inline void CopyV(const Vector4f &v, float *out) { out[0] = v.x; out[1] = v.y; out[2] = v.z; out[3] = v.w; }

inline b200_view PackView(const ITMView *view, const ITMTrackingState *trackingState, bool depthWeighting) {
  b200_view v{};
  v.d_depth = view->depth->GetData(MEMORYDEVICE_CUDA);
  v.d_rgb = (const b200_vec4u *)view->rgb->GetData(MEMORYDEVICE_CUDA);
  v.depth_w = view->depth->noDims.x; v.depth_h = view->depth->noDims.y;
  v.rgb_w = view->rgb->noDims.x; v.rgb_h = view->rgb->noDims.y;
  Matrix4f M_d = trackingState->pose_d->GetM(), invM_d;
  M_d.inv(invM_d);                                                        // Reco_CUDA.cu:190
  Matrix4f M_rgb = view->calib->trafo_rgb_to_depth.calib_inv * M_d;        // Reco_CUDA.cu:381
  CopyM(M_d, v.M_d); CopyM(invM_d, v.invM_d); CopyM(M_rgb, v.M_rgb);
  CopyV(view->calib->intrinsics_d.projectionParamsSimple.all, v.proj_d);
  CopyV(view->calib->intrinsics_rgb.projectionParamsSimple.all, v.proj_rgb);
  v.depthWeighting = depthWeighting ? 1 : 0;
  v.requiresFullRendering = trackingState->requiresFullRendering ? 1 : 0;
  return v;
}

inline b200_camera PackCamera(const ITMPose *pose, const ITMIntrinsics *intrinsics) {
  b200_camera c{};
  CopyM(pose->GetM(), c.M); CopyM(pose->GetInvM(), c.invM);
  CopyV(intrinsics->projectionParamsSimple.all, c.proj);
  return c;
}

}  // namespace b200_detail

// --------------------------------------------------------------------------------------------------
template <class TVoxel, class TIndex> class ITMSceneReconstructionEngine_B200;

template <class TVoxel>
class ITMSceneReconstructionEngine_B200<TVoxel, ITMVoxelBlockHash> : public ITMSceneReconstructionEngine<TVoxel, ITMVoxelBlockHash> {
  std::shared_ptr<B200EngineHandle> h;

 public:
  explicit ITMSceneReconstructionEngine_B200(std::shared_ptr<B200EngineHandle> handle) : h(handle) {}

  void ResetScene(ITMScene<TVoxel, ITMVoxelBlockHash> *scene) override {
    b200_scene s = b200_detail::PackScene(scene);
    h->check(b200_reset_scene(h->e, &s));
    b200_detail::UnpackScene(s, scene);
  }

  /// What a new InfiniTamDriver for a new track would be, without building one: the engine, scene and render state behave like a
  /// newly created engine on a newly allocated, reset scene with a new render state (frame index 0, empty decay queue).
  /// Stream-ordered on the engine's stream; the host waits for nothing and nothing is allocated (b200_volume_restart_async).
  void RestartScene(ITMScene<TVoxel, ITMVoxelBlockHash> *scene, ITMRenderState *renderState) {
    b200_scene s = b200_detail::PackScene(scene);
    b200_render_state r = b200_detail::PackRenderState(renderState);
    h->check(b200_volume_restart_async(h->e, &s, &r));
    b200_detail::UnpackScene(s, scene);
    b200_detail::UnpackRenderState(r, renderState);
  }

  void AllocateSceneFromDepth(ITMScene<TVoxel, ITMVoxelBlockHash> *scene, const ITMView *view, const ITMTrackingState *trackingState,
                              const ITMRenderState *renderState, bool onlyUpdateVisibleList = false) override {
    b200_scene s = b200_detail::PackScene(scene);
    b200_render_state r = b200_detail::PackRenderState((ITMRenderState *)renderState);
    b200_view v = b200_detail::PackView(view, trackingState, this->GetFusionWeightParams().depthWeighting);
    b200_status st = b200_allocate_from_depth(h->e, &s, &r, &v, onlyUpdateVisibleList ? 1 : 0);
    b200_detail::UnpackScene(s, scene);                       // the reference updates the host fields before it throws
    b200_detail::UnpackRenderState(r, (ITMRenderState *)renderState);
    h->check(st);
  }

  void IntegrateIntoScene(ITMScene<TVoxel, ITMVoxelBlockHash> *scene, const ITMView *view, const ITMTrackingState *trackingState,
                          const ITMRenderState *renderState) override {
    b200_scene s = b200_detail::PackScene(scene);
    b200_render_state r = b200_detail::PackRenderState((ITMRenderState *)renderState);
    b200_view v = b200_detail::PackView(view, trackingState, this->GetFusionWeightParams().depthWeighting);
    h->check(b200_integrate(h->e, &s, &r, &v));
  }

  void Decay(ITMScene<TVoxel, ITMVoxelBlockHash> *scene, const ITMRenderState *renderState, int maxWeight, int minAge,
             bool forceAllVoxels) override {
    b200_scene s = b200_detail::PackScene(scene);
    b200_render_state r = b200_detail::PackRenderState((ITMRenderState *)renderState);
    h->check(b200_decay(h->e, &s, &r, maxWeight, minAge, forceAllVoxels ? 1 : 0));
    b200_detail::UnpackScene(s, scene);
  }

  size_t GetDecayedBlockCount() override { return b200_decayed_block_count(h->e); }

  /// Writes the volume's checkpoint (include/b200fusion.h: scene, render state, frame index, decay queue) to `path`, the
  /// buffer verbatim. Returns false if the file cannot be written.
  bool SaveScene(ITMScene<TVoxel, ITMVoxelBlockHash> *scene, ITMRenderState *renderState, const char *path) {
    b200_scene s = b200_detail::PackScene(scene);
    b200_render_state r = b200_detail::PackRenderState(renderState);
    size_t size = 0;
    h->check(b200_checkpoint_save(h->e, &s, &r, nullptr, 0, &size));
    std::unique_ptr<char[]> buf(new char[size]);
    h->check(b200_checkpoint_save(h->e, &s, &r, buf.get(), size, &size));
    FILE *f = fopen(path, "wb");
    if (!f) return false;
    const bool ok = fwrite(buf.get(), 1, size, f) == size;
    return (fclose(f) == 0) && ok;
  }

  /// Replaces the volume's state with the checkpoint in `path` (same scene geometry, voxelSize and mu); fusion then continues
  /// bit for bit as in the process that saved it. Returns false, with the volume untouched, if the file cannot be read or is
  /// not a checkpoint that fits this scene (the reason is printed and stays in b200_last_error); CUDA errors exit as elsewhere.
  bool LoadScene(ITMScene<TVoxel, ITMVoxelBlockHash> *scene, ITMRenderState *renderState, const char *path) {
    FILE *f = fopen(path, "rb");
    if (!f) return false;
    fseek(f, 0, SEEK_END);
    const long size = ftell(f);
    fseek(f, 0, SEEK_SET);
    std::unique_ptr<char[]> buf(new char[size > 0 ? size : 1]);
    const bool ok = size > 0 && fread(buf.get(), 1, (size_t)size, f) == (size_t)size;
    fclose(f);
    if (!ok) return false;
    b200_scene s = b200_detail::PackScene(scene);
    b200_render_state r = b200_detail::PackRenderState(renderState);
    const b200_status st = b200_checkpoint_load(h->e, &s, &r, buf.get(), (size_t)size);
    if (st == B200_ERR_INVALID) { fprintf(stderr, "b200fusion: %s: %s\n", path, b200_last_error(h->e)); return false; }
    h->check(st);
    b200_detail::UnpackScene(s, scene);
    b200_detail::UnpackRenderState(r, renderState);
    return true;
  }
};

// --------------------------------------------------------------------------------------------------
template <class TVoxel, class TIndex> class ITMVisualisationEngine_B200;

template <class TVoxel>
class ITMVisualisationEngine_B200<TVoxel, ITMVoxelBlockHash> : public ITMVisualisationEngine<TVoxel, ITMVoxelBlockHash> {
  std::shared_ptr<B200EngineHandle> h;
  typedef ITMScene<TVoxel, ITMVoxelBlockHash> Scene;
  Scene *mutableScene() const { return const_cast<Scene *>(this->scene); }

 public:
  ITMVisualisationEngine_B200(const Scene *scene, const ITMLibSettings *settings, std::shared_ptr<B200EngineHandle> handle)
      : ITMVisualisationEngine<TVoxel, ITMVoxelBlockHash>(scene, settings), h(handle) {}

  ITMRenderState_VH *CreateRenderState(const Vector2i &imgSize) const override {
    return new ITMRenderState_VH(ITMVoxelBlockHash::noTotalEntries, imgSize, this->scene->sceneParams->viewFrustum_min,
                                 this->scene->sceneParams->viewFrustum_max, this->settings->sdfLocalBlockNum, MEMORYDEVICE_CUDA);
  }

  void FindVisibleBlocks(const ITMPose *pose, const ITMIntrinsics *intrinsics, ITMRenderState *renderState) const override {
    b200_scene s = b200_detail::PackScene(mutableScene());
    b200_render_state r = b200_detail::PackRenderState(renderState);
    b200_camera c = b200_detail::PackCamera(pose, intrinsics);
    h->check(b200_find_visible_blocks(h->e, &s, &r, &c));
    b200_detail::UnpackRenderState(r, renderState);
  }

  void CreateExpectedDepths(const ITMPose *pose, const ITMIntrinsics *intrinsics, ITMRenderState *renderState) const override {
    b200_scene s = b200_detail::PackScene(mutableScene());
    b200_render_state r = b200_detail::PackRenderState(renderState);
    b200_camera c = b200_detail::PackCamera(pose, intrinsics);
    h->check(b200_expected_depths(h->e, &s, &r, &c));
  }

  void RenderImage(const ITMPose *pose, const ITMIntrinsics *intrinsics, const ITMRenderState *renderState, ITMUChar4Image *outputCharImage,
                   ITMFloatImage *outputFloatImage, IITMVisualisationEngine::RenderImageType type) const override {
    b200_scene s = b200_detail::PackScene(mutableScene());
    b200_render_state r = b200_detail::PackRenderState((ITMRenderState *)renderState);
    b200_camera c = b200_detail::PackCamera(pose, intrinsics);
    h->check(b200_render_image(h->e, &s, &r, &c, (b200_vec4u *)outputCharImage->GetData(MEMORYDEVICE_CUDA),
                               outputFloatImage->GetData(MEMORYDEVICE_CUDA), outputCharImage->noDims.x, outputCharImage->noDims.y,
                               (b200_render_type)type));
  }

  // Not an ITMLib virtual: FindVisibleBlocks + CreateExpectedDepths + RenderImage(type) + RenderImage(RENDER_DEPTH_MAP) from one
  // pose as one enqueue and one raycast (b200_render_view_async), then the wait that refreshes renderState->noVisibleBlocks.
  // renderState is a free-view render state sized like the output images; either image may be NULL.
  void RenderFreeView(const ITMPose *pose, const ITMIntrinsics *intrinsics, ITMRenderState *renderState, ITMUChar4Image *outputCharImage,
                      ITMFloatImage *outputFloatImage, IITMVisualisationEngine::RenderImageType type) const {
    b200_scene s = b200_detail::PackScene(mutableScene());
    b200_render_state r = b200_detail::PackRenderState(renderState);
    b200_camera c = b200_detail::PackCamera(pose, intrinsics);
    h->check(b200_render_view_async(h->e, &s, &r, &c, (b200_render_type)type,
                                    outputCharImage ? (b200_vec4u *)outputCharImage->GetData(MEMORYDEVICE_CUDA) : NULL,
                                    outputFloatImage ? outputFloatImage->GetData(MEMORYDEVICE_CUDA) : NULL));
    h->check(b200_render_view_sync(h->e, &r));
    b200_detail::UnpackRenderState(r, renderState);
  }

  void FindSurface(const ITMPose *pose, const ITMIntrinsics *intrinsics, const ITMRenderState *renderState) const override {
    b200_scene s = b200_detail::PackScene(mutableScene());
    b200_render_state r = b200_detail::PackRenderState((ITMRenderState *)renderState);
    b200_camera c = b200_detail::PackCamera(pose, intrinsics);
    h->check(b200_find_surface(h->e, &s, &r, &c));
  }

  void CreatePointCloud(const ITMView *view, ITMTrackingState *trackingState, ITMRenderState *renderState, bool skipPoints) const override {
    b200_scene s = b200_detail::PackScene(mutableScene());
    b200_render_state r = b200_detail::PackRenderState(renderState);
    b200_view v = b200_detail::PackView(view, trackingState, false);
    float calib[16];
    b200_detail::CopyM(view->calib->trafo_rgb_to_depth.calib, calib);
    uint32_t n = 0;
    h->check(b200_point_cloud(h->e, &s, &r, &v, calib, skipPoints ? 1 : 0,
                              (b200_vec4f *)trackingState->pointCloud->locations->GetData(MEMORYDEVICE_CUDA),
                              (b200_vec4f *)trackingState->pointCloud->colours->GetData(MEMORYDEVICE_CUDA), &n));
    trackingState->pointCloud->noTotalPoints = n;
    trackingState->pose_pointCloud->SetFrom(trackingState->pose_d);       // Vis_CUDA.cu:353
  }

  void CreateICPMaps(const ITMView *view, ITMTrackingState *trackingState, ITMRenderState *renderState) const override {
    b200_scene s = b200_detail::PackScene(mutableScene());
    b200_render_state r = b200_detail::PackRenderState(renderState);
    b200_view v = b200_detail::PackView(view, trackingState, false);
    h->check(b200_icp_maps(h->e, &s, &r, &v, (b200_vec4f *)trackingState->pointCloud->locations->GetData(MEMORYDEVICE_CUDA),
                           (b200_vec4f *)trackingState->pointCloud->colours->GetData(MEMORYDEVICE_CUDA)));
    trackingState->pose_pointCloud->SetFrom(trackingState->pose_d);       // Vis_CUDA.cu:378
  }

  void ForwardRender(const ITMView *view, ITMTrackingState *trackingState, ITMRenderState *renderState) const override {
    b200_scene s = b200_detail::PackScene(mutableScene());
    b200_render_state r = b200_detail::PackRenderState(renderState);
    b200_view v = b200_detail::PackView(view, trackingState, false);
    h->check(b200_forward_render(h->e, &s, &r, &v));
    b200_detail::UnpackRenderState(r, renderState);
  }
};

// --------------------------------------------------------------------------------------------------
template <class TVoxel, class TIndex> class ITMSwappingEngine_B200;

template <class TVoxel>
class ITMSwappingEngine_B200<TVoxel, ITMVoxelBlockHash> : public ITMSwappingEngine<TVoxel, ITMVoxelBlockHash> {
  std::shared_ptr<B200EngineHandle> h;

  static b200_transfer_buffers Buffers(ITMGlobalCache<TVoxel> *gc) {
    b200_transfer_buffers t{};
    t.d_syncedVoxelBlocks = (b200_voxel *)gc->GetSyncedVoxelBlocks(true);
    t.d_hasSyncedData = (uint8_t *)gc->GetHasSyncedData(true);
    t.d_neededEntryIDs = gc->GetNeededEntryIDs(true);
    return t;
  }

 public:
  explicit ITMSwappingEngine_B200(std::shared_ptr<B200EngineHandle> handle) : h(handle) {}

  // Swap_CUDA.cu:44-124: the host half (gathering stored blocks, PCIe copies) stays in C++
  void IntegrateGlobalIntoLocal(ITMScene<TVoxel, ITMVoxelBlockHash> *scene, ITMRenderState *renderState) override {
    ITMGlobalCache<TVoxel> *gc = scene->globalCache;
    b200_scene s = b200_detail::PackScene(scene);
    b200_transfer_buffers t = Buffers(gc);
    int n = 0;
    h->check(b200_swap_list_in(h->e, &s, &t, &n));
    if (n <= 0) return;
    int *ids = gc->GetNeededEntryIDs(false);
    TVoxel *blocks = gc->GetSyncedVoxelBlocks(false);
    bool *has = gc->GetHasSyncedData(false);
    ORcudaSafeCall(cudaMemcpy(ids, gc->GetNeededEntryIDs(true), sizeof(int) * n, cudaMemcpyDeviceToHost));
    memset(blocks, 0, (size_t)n * SDF_BLOCK_SIZE3 * sizeof(TVoxel));
    memset(has, 0, n * sizeof(bool));
    for (int i = 0; i < n; i++) if (gc->HasStoredData(ids[i])) {
      has[i] = true;
      memcpy(blocks + (size_t)i * SDF_BLOCK_SIZE3, gc->GetStoredVoxelBlock(ids[i]), SDF_BLOCK_SIZE3 * sizeof(TVoxel));
    }
    ORcudaSafeCall(cudaMemcpy(gc->GetHasSyncedData(true), has, sizeof(bool) * n, cudaMemcpyHostToDevice));
    ORcudaSafeCall(cudaMemcpy(gc->GetSyncedVoxelBlocks(true), blocks, sizeof(TVoxel) * SDF_BLOCK_SIZE3 * n, cudaMemcpyHostToDevice));
    h->check(b200_swap_integrate_in(h->e, &s, &t, n));
  }

  // Swap_CUDA.cu:126-216
  void SaveToGlobalMemory(ITMScene<TVoxel, ITMVoxelBlockHash> *scene, ITMRenderState *renderState) override {
    ITMGlobalCache<TVoxel> *gc = scene->globalCache;
    b200_scene s = b200_detail::PackScene(scene);
    b200_render_state r = b200_detail::PackRenderState(renderState);
    b200_transfer_buffers t = Buffers(gc);
    int n = 0;
    h->check(b200_swap_out(h->e, &s, &r, &t, &n));
    b200_detail::UnpackScene(s, scene);
    if (n <= 0) return;
    int *ids = gc->GetNeededEntryIDs(false);
    TVoxel *blocks = gc->GetSyncedVoxelBlocks(false);
    bool *has = gc->GetHasSyncedData(false);
    ORcudaSafeCall(cudaMemcpy(ids, gc->GetNeededEntryIDs(true), sizeof(int) * n, cudaMemcpyDeviceToHost));
    ORcudaSafeCall(cudaMemcpy(has, gc->GetHasSyncedData(true), sizeof(bool) * n, cudaMemcpyDeviceToHost));
    ORcudaSafeCall(cudaMemcpy(blocks, gc->GetSyncedVoxelBlocks(true), sizeof(TVoxel) * SDF_BLOCK_SIZE3 * n, cudaMemcpyDeviceToHost));
    for (int i = 0; i < n; i++) if (has[i]) gc->SetStoredData(ids[i], blocks + (size_t)i * SDF_BLOCK_SIZE3);
  }
};

// ---- ITMMeshingEngine (Engine/ITMMeshingEngine.h:18-27) ---------------------------------------------------------------
template <class TVoxel, class TIndex> class ITMMeshingEngine_B200;

template <class TVoxel>
class ITMMeshingEngine_B200<TVoxel, ITMVoxelBlockHash> : public ITMMeshingEngine<TVoxel, ITMVoxelBlockHash> {
  std::shared_ptr<B200EngineHandle> h;

 public:
  explicit ITMMeshingEngine_B200(std::shared_ptr<B200EngineHandle> handle) : h(handle) {}

  // ITMMeshingEngine_CUDA.cu:37-81; the triangles arrive in the CPU engine's (deterministic) order
  void MeshScene(ITMMesh *mesh, const ITMScene<TVoxel, ITMVoxelBlockHash> *scene) override {
    static_assert(sizeof(ITMMesh::Triangle) == sizeof(b200_triangle), "ITMMesh::Triangle layout");
    b200_scene s = b200_detail::PackScene(const_cast<ITMScene<TVoxel, ITMVoxelBlockHash> *>(scene));
    uint32_t n = 0;
    h->check(b200_mesh_scene(h->e, &s, (b200_triangle *)mesh->triangles->GetData(MEMORYDEVICE_CUDA), mesh->noMaxTriangles, &n));
    mesh->noTotalTriangles = n;
    printf("Meshing done: %d/%d triangles in mesh.\n", mesh->noTotalTriangles, mesh->noMaxTriangles);
  }
};

}  // namespace Engine
}  // namespace ITMLib
