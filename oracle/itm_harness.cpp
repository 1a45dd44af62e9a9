// itm_harness.cpp — TEST / BASELINE INFRASTRUCTURE. Headless driver of the REAL ITMLib objects
// (ITMScene, ITMRenderState_VH, ITMView, ITMTrackingState) through the abstract engine interfaces,
// with either back-end behind them:
//   impl 0: the UNMODIFIED reference CUDA engines (ITMSceneReconstructionEngine_CUDA /
//           ITMVisualisationEngine_CUDA), compiled for sm_90a from the reference's source tree — the "reference CUDA build" that north_star's >=10x is measured against;
//   impl 1: the B200 shim classes (dynslam_b200/itm_shim/ITMEngines_B200.h) over libb200fusion.
// The call sequence per frame is the reference's own: ITMDenseMapper::ProcessFrame
// (Engine/ITMDenseMapper.cpp:53-69), ITMTrackingController::Prepare (Engine/ITMTrackingController.cpp:23-51)
// and ITMDenseMapper::Decay (:78-86), i.e. what InfiniTamDriver::Integrate / PrepareNextStep / Decay
// run (DS/InfiniTamDriver.h:137-158, :201-206). View building is outside the path (SURVEY 2.1 #11):
// the float depth and RGBA frames are copied straight into the ITMView images.
// Built by oracle/build_ref.sh into oracle/_ref/libitmharness.so (git-ignored, ships via gpurun).
#include <cstdio>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <unistd.h>
#include <fcntl.h>

#include "ITMLib/Engine/DeviceSpecific/CUDA/ITMSceneReconstructionEngine_CUDA.h"
#include "ITMLib/Engine/DeviceSpecific/CUDA/ITMVisualisationEngine_CUDA.h"
#include "ITMLib/Objects/ITMRGBDCalib.h"
#include "ITMLib/Objects/ITMTrackingState.h"
#include "ITMLib/Objects/ITMView.h"
#include "ITMLib/Utils/ITMLibSettings.h"

#include "ITMLib/Engine/DeviceSpecific/CUDA/ITMViewBuilder_CUDA.h"

#include "ITMEngines_B200.h"
#include "ITMViewBuilder_B200.h"

#include <chrono>

using namespace ITMLib::Engine;
using namespace ITMLib::Objects;

struct Harness {
  int impl;
  ITMLibSettings *settings;
  ITMScene<ITMVoxel, ITMVoxelIndex> *scene;
  ITMSceneReconstructionEngine<ITMVoxel, ITMVoxelIndex> *reco;
  IITMVisualisationEngine *vis;
  ITMRenderState *renderState;
  ITMRGBDCalib calib;
  ITMView *view;
  ITMTrackingState *trackingState;
  Vector2i imgSize;
  std::shared_ptr<B200EngineHandle> handle;
  int savedStdout;
  char err[256];
};

extern "C" {

// stdout of the reference is chatty (two printf lines per frame, Reco_CUDA.cu:338-346, :546-559);
// it is part of the reference's cost but must not pollute a caller that prints JSON on stdout.
void harness_mute_stdout(Harness *H, int mute) {
  fflush(stdout);
  if (mute && H->savedStdout < 0) {
    H->savedStdout = dup(1);
    int nul = open("/dev/null", O_WRONLY);
    dup2(nul, 1);
    close(nul);
  } else if (!mute && H->savedStdout >= 0) {
    dup2(H->savedStdout, 1);
    close(H->savedStdout);
    H->savedStdout = -1;
  }
}

Harness *harness_create(int impl, int w, int h, float fx, float fy, float cx, float cy, float voxelSize, float mu, int maxW,
                        long numBlocks) {
  Harness *H = new Harness();
  H->impl = impl; H->savedStdout = -1; H->err[0] = 0;
  H->imgSize = Vector2i(w, h);
  H->settings = new ITMLibSettings();
  H->settings->sceneParams.voxelSize = voxelSize;
  H->settings->sceneParams.mu = mu;
  H->settings->sceneParams.maxW = maxW;
  H->settings->sdfLocalBlockNum = numBlocks;
  H->calib.intrinsics_d.SetFrom(fx, fy, cx, cy, (float)w, (float)h);
  H->calib.intrinsics_rgb.SetFrom(fx, fy, cx, cy, (float)w, (float)h);
  H->scene = new ITMScene<ITMVoxel, ITMVoxelIndex>(&H->settings->sceneParams, false, MEMORYDEVICE_CUDA, numBlocks);
  if (impl == 0) {
    H->reco = new ITMSceneReconstructionEngine_CUDA<ITMVoxel, ITMVoxelIndex>(numBlocks);
    H->vis = new ITMVisualisationEngine_CUDA<ITMVoxel, ITMVoxelIndex>(H->scene, H->settings);
  } else {
    H->handle = std::make_shared<B200EngineHandle>(0, numBlocks, H->imgSize);
    H->reco = new ITMSceneReconstructionEngine_B200<ITMVoxel, ITMVoxelIndex>(H->handle);
    H->vis = new ITMVisualisationEngine_B200<ITMVoxel, ITMVoxelIndex>(H->scene, H->settings, H->handle);
  }
  H->renderState = H->vis->CreateRenderState(H->imgSize);
  H->view = new ITMView(&H->calib, H->imgSize, H->imgSize, true);
  H->trackingState = new ITMTrackingState(H->imgSize, MEMORYDEVICE_CUDA);
  H->reco->ResetScene(H->scene);
  return H;
}

void harness_destroy(Harness *H) {
  harness_mute_stdout(H, 0);
  delete H->trackingState; delete H->view; delete H->renderState; delete H->vis; delete H->reco; delete H->scene; delete H->settings;
  delete H;
}

const char *harness_error(Harness *H) { return H->err; }

// One frame: H2D of the frame into the ITMView, then the reference's call sequence.
// Returns 0, or 2 when the engine threw std::runtime_error (VBA / excess exhaustion).
int harness_process_frame(Harness *H, const float *depth, const unsigned char *rgba, const float *M_d, int decayMaxWeight,
                          int decayMinAge, int doDecay, int doRaycast) {
  const size_t n = (size_t)H->imgSize.x * H->imgSize.y;
  ORcudaSafeCall(cudaMemcpy(H->view->depth->GetData(MEMORYDEVICE_CUDA), depth, n * sizeof(float), cudaMemcpyHostToDevice));
  ORcudaSafeCall(cudaMemcpy(H->view->rgb->GetData(MEMORYDEVICE_CUDA), rgba, n * 4, cudaMemcpyHostToDevice));
  Matrix4f M; for (int i = 0; i < 16; ++i) M.m[i] = M_d[i];
  H->trackingState->pose_d->SetM(M);
  H->trackingState->requiresFullRendering = true;            // useApproximateRaycast == false (ITMLibSettings.cpp:58)
  try {
    H->reco->AllocateSceneFromDepth(H->scene, H->view, H->trackingState, H->renderState);
    H->reco->IntegrateIntoScene(H->scene, H->view, H->trackingState, H->renderState);
    if (doRaycast) {
      H->vis->CreateExpectedDepths(H->trackingState->pose_d, &(H->view->calib->intrinsics_d), H->renderState);
      H->vis->CreateICPMaps(H->view, H->trackingState, H->renderState);
      H->trackingState->pose_pointCloud->SetFrom(H->trackingState->pose_d);
    }
    if (doDecay) H->reco->Decay(H->scene, H->renderState, decayMaxWeight, decayMinAge, false);
  } catch (std::runtime_error &e) {
    snprintf(H->err, sizeof(H->err), "%s", e.what());
    return 2;
  }
  return 0;
}

void harness_sync(Harness *H) { ORcudaSafeCall(cudaDeviceSynchronize()); }
// The same frame with a device synchronise + wall clock after every call: where the synchronous ITMLib loop spends its time
// (bench.py `itmlib_harness.stages_us`). stage_us[6] += {H2D of the frame, AllocateSceneFromDepth, IntegrateIntoScene,
// CreateExpectedDepths, CreateICPMaps, Decay} in microseconds.
int harness_process_frame_timed(Harness *H, const float *depth, const unsigned char *rgba, const float *M_d, int decayMaxWeight,
                                int decayMinAge, int doDecay, double *stage_us) {
  const size_t n = (size_t)H->imgSize.x * H->imgSize.y;
  auto now = [] { return std::chrono::steady_clock::now(); };
  auto us = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) {
    return std::chrono::duration<double, std::micro>(b - a).count();
  };
  ORcudaSafeCall(cudaDeviceSynchronize());
  auto t0 = now();
  ORcudaSafeCall(cudaMemcpy(H->view->depth->GetData(MEMORYDEVICE_CUDA), depth, n * sizeof(float), cudaMemcpyHostToDevice));
  ORcudaSafeCall(cudaMemcpy(H->view->rgb->GetData(MEMORYDEVICE_CUDA), rgba, n * 4, cudaMemcpyHostToDevice));
  Matrix4f M; for (int i = 0; i < 16; ++i) M.m[i] = M_d[i];
  H->trackingState->pose_d->SetM(M);
  H->trackingState->requiresFullRendering = true;
  ORcudaSafeCall(cudaDeviceSynchronize());
  auto t1 = now(); stage_us[0] += us(t0, t1);
  try {
    H->reco->AllocateSceneFromDepth(H->scene, H->view, H->trackingState, H->renderState);
    ORcudaSafeCall(cudaDeviceSynchronize());
    auto t2 = now(); stage_us[1] += us(t1, t2);
    H->reco->IntegrateIntoScene(H->scene, H->view, H->trackingState, H->renderState);
    ORcudaSafeCall(cudaDeviceSynchronize());
    auto t3 = now(); stage_us[2] += us(t2, t3);
    H->vis->CreateExpectedDepths(H->trackingState->pose_d, &(H->view->calib->intrinsics_d), H->renderState);
    ORcudaSafeCall(cudaDeviceSynchronize());
    auto t4 = now(); stage_us[3] += us(t3, t4);
    H->vis->CreateICPMaps(H->view, H->trackingState, H->renderState);
    H->trackingState->pose_pointCloud->SetFrom(H->trackingState->pose_d);
    ORcudaSafeCall(cudaDeviceSynchronize());
    auto t5 = now(); stage_us[4] += us(t4, t5);
    if (doDecay) H->reco->Decay(H->scene, H->renderState, decayMaxWeight, decayMinAge, false);
    ORcudaSafeCall(cudaDeviceSynchronize());
    stage_us[5] += us(t5, now());
  } catch (std::runtime_error &e) {
    snprintf(H->err, sizeof(H->err), "%s", e.what());
    return 2;
  }
  return 0;
}

// page-lock a caller buffer (frames held in numpy arrays) so that the per-frame cudaMemcpy is a DMA from pinned memory
int harness_pin(void *p, size_t bytes) { return (int)cudaHostRegister(p, bytes, cudaHostRegisterDefault); }
int harness_unpin(void *p) { return (int)cudaHostUnregister(p); }


void harness_counters(Harness *H, int *lastFreeBlockId, int *lastFreeExcess, int *noVisible, long *decayed) {
  *lastFreeBlockId = H->scene->localVBA.lastFreeBlockId;
  *lastFreeExcess = H->scene->index.GetLastFreeExcessListId();
  *noVisible = ((ITMRenderState_VH *)H->renderState)->noVisibleBlocks;
  *decayed = (long)H->reco->GetDecayedBlockCount();
}

int harness_table_entries(void) { return ITMVoxelBlockHash::noTotalEntries; }

// device -> host copies for order-free comparisons
void harness_download(Harness *H, void *hashOut, void *voxelsOut, void *rayOut, void *imgOut) {
  ORcudaSafeCall(cudaDeviceSynchronize());
  if (hashOut) ORcudaSafeCall(cudaMemcpy(hashOut, H->scene->index.GetEntries(), sizeof(ITMHashEntry) * (size_t)ITMVoxelBlockHash::noTotalEntries, cudaMemcpyDeviceToHost));
  if (voxelsOut) ORcudaSafeCall(cudaMemcpy(voxelsOut, H->scene->localVBA.GetVoxelBlocks(), sizeof(ITMVoxel) * (size_t)H->scene->localVBA.allocatedSize, cudaMemcpyDeviceToHost));
  const size_t n = (size_t)H->imgSize.x * H->imgSize.y;
  if (rayOut) ORcudaSafeCall(cudaMemcpy(rayOut, H->renderState->raycastResult->GetData(MEMORYDEVICE_CUDA), n * sizeof(Vector4f), cudaMemcpyDeviceToHost));
  if (imgOut) ORcudaSafeCall(cudaMemcpy(imgOut, H->renderState->raycastImage->GetData(MEMORYDEVICE_CUDA), n * 4, cudaMemcpyDeviceToHost));
}

void harness_download_lists(Harness *H, int *allocationList, int *excessList, unsigned char *visType) {
  ORcudaSafeCall(cudaDeviceSynchronize());
  if (allocationList) ORcudaSafeCall(cudaMemcpy(allocationList, H->scene->localVBA.GetAllocationList(), sizeof(int) * (size_t)H->settings->sdfLocalBlockNum, cudaMemcpyDeviceToHost));
  if (excessList) ORcudaSafeCall(cudaMemcpy(excessList, H->scene->index.GetExcessAllocationList(), sizeof(int) * (size_t)SDF_EXCESS_LIST_SIZE, cudaMemcpyDeviceToHost));
  if (visType) ORcudaSafeCall(cudaMemcpy(visType, ((ITMRenderState_VH *)H->renderState)->GetEntriesVisibleType(), (size_t)ITMVoxelBlockHash::noTotalEntries, cudaMemcpyDeviceToHost));
}

// ---- the reference's own Decay on a state the caller supplies (impl 0 only) ----
// The reference's allocation is nondeterministic, so a test cannot let it build its own map and compare: it hands the
// reference exactly the state the oracle decays. The decay queue (frameVisibleBlocks) and the frame index are private
// members of ITMSceneReconstructionEngine_CUDA. They are reached with pointers-to-member formed in explicit template
// instantiations, where C++ does not check access ([temp.explicit]/12 of C++14): the reference's headers are included
// unmodified.
}  // extern "C"
typedef ITMSceneReconstructionEngine_CUDA<ITMVoxel, ITMVoxelBlockHash> RefReco;
template <class Tag, typename Tag::type Member> struct ExposeMember { friend typename Tag::type member(Tag) { return Member; } };
struct DecayQueueOf { typedef std::queue<VisibleBlockInfo> RefReco::*type; friend type member(DecayQueueOf); };
struct FrameIdxOf { typedef size_t RefReco::*type; friend type member(FrameIdxOf); };
template struct ExposeMember<DecayQueueOf, &RefReco::frameVisibleBlocks>;
template struct ExposeMember<FrameIdxOf, &RefReco::frameIdx>;
extern "C" {

static RefReco *ref_reco(Harness *H) {
  if (H->impl != 0) { snprintf(H->err, sizeof(H->err), "the decay entry points drive the reference engine (impl 0) only"); return nullptr; }
  return static_cast<RefReco *>(H->reco);
}

// ResetScene (empties the decay queue and the decayed-block count, keeps frameIdx; Reco_CUDA.cu:145-172), then the caller's
// hash table, voxel block array, allocation list, excess list and visibility bytes, and the two free-list cursors. Decay
// copies localVBA.lastFreeBlockId to the device itself (:516-519).
int harness_upload_state(Harness *H, const void *hash, const void *voxels, const int *allocationList, const int *excessList,
                         const unsigned char *visType, int lastFreeBlockId, int lastFreeExcessListId) {
  RefReco *reco = ref_reco(H);
  if (!reco) return 1;
  reco->ResetScene(H->scene);
  ORcudaSafeCall(cudaMemcpy(H->scene->index.GetEntries(), hash, sizeof(ITMHashEntry) * (size_t)ITMVoxelBlockHash::noTotalEntries, cudaMemcpyHostToDevice));
  ORcudaSafeCall(cudaMemcpy(H->scene->localVBA.GetVoxelBlocks(), voxels, sizeof(ITMVoxel) * (size_t)H->scene->localVBA.allocatedSize, cudaMemcpyHostToDevice));
  ORcudaSafeCall(cudaMemcpy(H->scene->localVBA.GetAllocationList(), allocationList, sizeof(int) * (size_t)H->settings->sdfLocalBlockNum, cudaMemcpyHostToDevice));
  ORcudaSafeCall(cudaMemcpy(H->scene->index.GetExcessAllocationList(), excessList, sizeof(int) * (size_t)SDF_EXCESS_LIST_SIZE, cudaMemcpyHostToDevice));
  ORcudaSafeCall(cudaMemcpy(((ITMRenderState_VH *)H->renderState)->GetEntriesVisibleType(), visType, (size_t)ITMVoxelBlockHash::noTotalEntries, cudaMemcpyHostToDevice));
  H->scene->localVBA.lastFreeBlockId = lastFreeBlockId;
  H->scene->index.SetLastFreeExcessListId(lastFreeExcessListId);
  return 0;
}

// frameVisibleBlocks.push({count, frameIdx, device copy of the positions}), as AllocateSceneFromDepth does (:302-316),
// including its null block for an empty list
int harness_push_snapshot(Harness *H, const int *positions, long n) {
  RefReco *reco = ref_reco(H);
  if (!reco) return 1;
  ORUtils::MemoryBlock<Vector3i> *copy = nullptr;
  if (n > 0) {
    copy = new ORUtils::MemoryBlock<Vector3i>((size_t)n, MEMORYDEVICE_CUDA);
    ORcudaSafeCall(cudaMemcpy(copy->GetData(MEMORYDEVICE_CUDA), positions, sizeof(Vector3i) * (size_t)n, cudaMemcpyHostToDevice));
  }
  const size_t f = reco->*member(FrameIdxOf());
  (reco->*member(DecayQueueOf())).push(VisibleBlockInfo{(size_t)n, f, copy});
  return 0;
}

int harness_set_frame_index(Harness *H, long f) {
  RefReco *reco = ref_reco(H);
  if (!reco) return 1;
  reco->*member(FrameIdxOf()) = (size_t)f;
  return 0;
}

long harness_queue_size(Harness *H) {
  RefReco *reco = ref_reco(H);
  return reco ? (long)(reco->*member(DecayQueueOf())).size() : -1;
}

// the reference's own ITMSceneReconstructionEngine_CUDA::Decay (host method and kernels, :509-560); *decayed receives
// GetDecayedBlockCount() (blocks freed since the upload's ResetScene)
int harness_decay(Harness *H, int maxWeight, int minAge, int forceAll, long *decayed) {
  RefReco *reco = ref_reco(H);
  if (!reco) return 1;
  reco->Decay(H->scene, H->renderState, maxWeight, minAge, forceAll != 0);
  ORcudaSafeCall(cudaDeviceSynchronize());
  *decayed = (long)reco->GetDecayedBlockCount();
  return 0;
}

// ---- view builder (SURVEY 8(f) rank 1): ITMViewBuilder_CUDA (impl 0) vs ITMViewBuilder_B200 (impl 1) ----
struct VBHarness {
  int impl;
  ITMRGBDCalib calib;
  ITMViewBuilder *vb;
  ITMView *view;
  ITMUChar4Image *rgb;
  ITMShortImage *raw;
  ITMFloatImage *scratch;      // device-only timing of the reference: stands in for its floatImage
  std::shared_ptr<B200EngineHandle> handle;
  Vector2i imgSize;
};

VBHarness *vbh_create(int impl, int w, int h, float fx, float fy, float cx, float cy) {
  VBHarness *V = new VBHarness();
  V->impl = impl; V->imgSize = Vector2i(w, h); V->view = NULL;
  V->calib.intrinsics_d.SetFrom(fx, fy, cx, cy, (float)w, (float)h);
  V->calib.intrinsics_rgb.SetFrom(fx, fy, cx, cy, (float)w, (float)h);     // disparityCalib default: affine mm -> m
  if (impl == 0) V->vb = new ITMViewBuilder_CUDA(&V->calib);
  else { V->handle = std::make_shared<B200EngineHandle>(0, 2048, V->imgSize); V->vb = new ITMViewBuilder_B200(&V->calib, V->handle); }
  V->rgb = new ITMUChar4Image(V->imgSize, true, false);
  V->raw = new ITMShortImage(V->imgSize, true, false);
  V->scratch = new ITMFloatImage(V->imgSize, true, true);
  return V;
}

void vbh_destroy(VBHarness *V) { delete V->view; delete V->vb; delete V->rgb; delete V->raw; delete V->scratch; delete V; }

// ITMMainEngine::ProcessFrame's call (Engine/ITMMainEngine.cpp:152): host images in, view on the device
void vbh_update_view(VBHarness *V, const short *raw, const unsigned char *rgba, int useBilateralFilter, int modelSensorNoise) {
  const size_t n = (size_t)V->imgSize.x * V->imgSize.y;
  memcpy(V->raw->GetData(MEMORYDEVICE_CPU), raw, n * sizeof(short));
  memcpy(V->rgb->GetData(MEMORYDEVICE_CPU), rgba, n * 4);
  V->vb->UpdateView(&V->view, V->rgb, V->raw, useBilateralFilter != 0, modelSensorNoise != 0);
  ORcudaSafeCall(cudaDeviceSynchronize());
}

// wall-clock milliseconds per UpdateView (host images already in ITMLib's host buffers), device synchronised
double vbh_time_update_view(VBHarness *V, int useBilateralFilter, int iters) {
  ORcudaSafeCall(cudaDeviceSynchronize());
  auto t0 = std::chrono::steady_clock::now();
  for (int i = 0; i < iters; ++i) V->vb->UpdateView(&V->view, V->rgb, V->raw, useBilateralFilter != 0, false);
  ORcudaSafeCall(cudaDeviceSynchronize());
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count() / iters;
}

// device part only: for the reference its own public stages in UpdateView's order on the device-resident short image
// (ITMViewBuilder_CUDA.cu:56-79); for the B200 builder the fused kernel. Milliseconds per call.
double vbh_time_device_only(VBHarness *V, int iters) {
  if (!V->view) return -1.0;
  ITMShortImage dshort(V->imgSize, true, true);
  dshort.SetFrom(V->raw, ORUtils::MemoryBlock<short>::CPU_TO_CUDA);
  ORcudaSafeCall(cudaDeviceSynchronize());
  auto t0 = std::chrono::steady_clock::now();
  for (int i = 0; i < iters; ++i) {
    if (V->impl == 0) {
      V->vb->ConvertDepthAffineToFloat(V->view->depth, &dshort, V->calib.disparityCalib.params);
      V->vb->DepthFiltering(V->scratch, V->view->depth);
      V->vb->DepthFiltering(V->view->depth, V->scratch);
      V->vb->DepthFiltering(V->scratch, V->view->depth);
      V->vb->DepthFiltering(V->view->depth, V->scratch);
      V->vb->DepthFiltering(V->scratch, V->view->depth);
      V->view->depth->SetFrom(V->scratch, ORUtils::MemoryBlock<float>::CUDA_TO_CUDA);
    } else {
      b200_view_calib c{};
      c.trafoType = 1; c.params[0] = V->calib.disparityCalib.params.x; c.params[1] = V->calib.disparityCalib.params.y;
      c.useBilateralFilter = 1;
      V->handle->check(b200_update_view_async(V->handle->e, dshort.GetData(MEMORYDEVICE_CUDA), V->imgSize.x, V->imgSize.y, &c,
                                              V->view->depth->GetData(MEMORYDEVICE_CUDA), nullptr, nullptr));
    }
  }
  ORcudaSafeCall(cudaDeviceSynchronize());
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count() / iters;
}

void vbh_download(VBHarness *V, float *depthOut) {
  ORcudaSafeCall(cudaDeviceSynchronize());
  ORcudaSafeCall(cudaMemcpy(depthOut, V->view->depth->GetData(MEMORYDEVICE_CUDA), (size_t)V->imgSize.x * V->imgSize.y * sizeof(float), cudaMemcpyDeviceToHost));
}

}  // extern "C"
