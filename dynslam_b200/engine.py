"""Host-side mirror of the reference's engine interfaces for the hot path, over the C-ABI.

Class and method names follow ITMLib (src/InfiniTAM/InfiniTAM/ITMLib/):
  ITMScene / ITMRenderState_VH / ITMView              Objects/ITMScene.h, ITMRenderState_VH.h, ITMView.h
  ITMSceneReconstructionEngine                         Engine/ITMSceneReconstructionEngine.h:33-78
  ITMVisualisationEngine                               Engine/ITMVisualisationEngine.h:19-127
  ITMSwappingEngine (+ ITMGlobalCache host store)      Engine/ITMSwappingEngine.h:22-31
Error behaviour mirrors the reference: capacity exhaustion raises RuntimeError (the reference
throws std::runtime_error, Reco_CUDA.cu:348-357, caught by InstanceReconstructor.cpp:662-671);
CUDA failures raise CudaError (the reference prints and exits, OR/CUDADefines.cpp:9-47).

torch is used for device memory only. There is no CPU path: constructing an engine without the
CUDA library or without a GPU raises.
"""
import ctypes as C

import numpy as np
import torch

from . import abi


class CudaError(RuntimeError):
    pass


def _ptr(t):
    return t.data_ptr() if t is not None else None


class SceneParams:
    """ITMSceneParams (Objects/ITMSceneParams.h:14-71); defaults of ITMLibSettings.cpp:23."""

    def __init__(self, voxelSize=0.05, mu=0.75, maxW=50, viewFrustum_min=0.1, viewFrustum_max=300.0,
                 stopIntegratingAtMaxW=False):
        self.voxelSize, self.mu, self.maxW = voxelSize, mu, maxW
        self.viewFrustum_min, self.viewFrustum_max = viewFrustum_min, viewFrustum_max
        self.stopIntegratingAtMaxW = stopIntegratingAtMaxW


class Scene:
    """ITMScene<ITMVoxel_s_rgb, ITMVoxelBlockHash>: hash table + excess list + VBA + free list."""

    def __init__(self, params, numBlocks=0x60000, numBuckets=0x100000, excessSize=0x80000, device="cuda:0",
                 useSwapping=False):
        self.params = params
        self.device = torch.device(device)
        self.numBlocks, self.numBuckets, self.excessSize = numBlocks, numBuckets, excessSize
        self.noTotalEntries = numBuckets + excessSize
        dev = self.device
        self.voxels = torch.empty(numBlocks * abi.SDF_BLOCK_SIZE3 * 8, dtype=torch.uint8, device=dev)
        self.allocationList = torch.empty(numBlocks, dtype=torch.int32, device=dev)
        self.hash = torch.empty(self.noTotalEntries * 20, dtype=torch.uint8, device=dev)
        self.excessList = torch.empty(excessSize, dtype=torch.int32, device=dev)
        self.swapStates = torch.zeros(self.noTotalEntries, dtype=torch.uint8, device=dev) if useSwapping else None
        s = abi.Scene()
        s.d_voxels, s.d_allocationList = _ptr(self.voxels), _ptr(self.allocationList)
        s.d_hash, s.d_excessList, s.d_swapStates = _ptr(self.hash), _ptr(self.excessList), _ptr(self.swapStates)
        s.numBlocks, s.numBuckets, s.excessSize = numBlocks, numBuckets, excessSize
        s.lastFreeBlockId, s.lastFreeExcessListId = numBlocks - 1, excessSize - 1
        s.voxelSize, s.mu, s.maxW = params.voxelSize, params.mu, params.maxW
        s.viewFrustum_min, s.viewFrustum_max = params.viewFrustum_min, params.viewFrustum_max
        s.stopIntegratingAtMaxW, s.useSwapping = int(params.stopIntegratingAtMaxW), int(useSwapping)
        self.c = s

    @property
    def lastFreeBlockId(self):
        return self.c.lastFreeBlockId

    @property
    def lastFreeExcessListId(self):
        return self.c.lastFreeExcessListId

    def to_host(self):
        """numpy copies of every persistent buffer (for parity checks)."""
        return dict(hash=self.hash.cpu().numpy().view(abi.HASH_ENTRY_DTYPE).copy(),
                    voxels=self.voxels.cpu().numpy().view(abi.VOXEL_DTYPE).copy(),
                    allocationList=self.allocationList.cpu().numpy().copy(),
                    excessList=self.excessList.cpu().numpy().copy(),
                    lastFreeBlockId=self.c.lastFreeBlockId, lastFreeExcessListId=self.c.lastFreeExcessListId)


class RenderStateVH:
    """ITMRenderState_VH (+ base): visible list, visibility bytes, min/max image, raycast images."""

    def __init__(self, scene, imgSize, forward=False):
        w, h = imgSize
        dev = scene.device
        self.w, self.h = w, h
        self.visibleBlockPositions = torch.zeros(scene.numBlocks * 3, dtype=torch.int32, device=dev)
        self.entriesVisibleType = torch.zeros(scene.noTotalEntries, dtype=torch.uint8, device=dev)
        self.renderingRangeImage = torch.zeros(h * w * 2, dtype=torch.float32, device=dev)
        self.raycastResult = torch.zeros(h * w * 4, dtype=torch.float32, device=dev)
        self.raycastImage = torch.zeros(h * w * 4, dtype=torch.uint8, device=dev)
        self.forwardProjection = torch.zeros(h * w * 4, dtype=torch.float32, device=dev) if forward else None
        self.fwdProjMissingPoints = torch.zeros(h * w, dtype=torch.int32, device=dev) if forward else None
        r = abi.RenderState()
        r.d_visibleBlockPositions, r.d_entriesVisibleType = _ptr(self.visibleBlockPositions), _ptr(self.entriesVisibleType)
        r.d_minmax, r.d_raycastResult, r.d_raycastImage = _ptr(self.renderingRangeImage), _ptr(self.raycastResult), _ptr(self.raycastImage)
        r.d_forwardProjection, r.d_fwdProjMissingPoints = _ptr(self.forwardProjection), _ptr(self.fwdProjMissingPoints)
        r.img_w, r.img_h, r.noVisibleBlocks = w, h, 0
        self.c = r

    @property
    def noVisibleBlocks(self):
        return self.c.noVisibleBlocks

    def to_host(self):
        n = max(self.c.noVisibleBlocks, 0)
        return dict(visType=self.entriesVisibleType.cpu().numpy().copy(),
                    visiblePos=self.visibleBlockPositions.cpu().numpy().reshape(-1, 3)[:n].copy(),
                    noVisibleBlocks=self.c.noVisibleBlocks)


class View:
    """ITMView + pose_d + calibration: device depth (float metres) / rgb (RGBA8) and matrices."""

    def __init__(self, depth, rgb, M_d, proj_d, M_rgb=None, proj_rgb=None, depthWeighting=False,
                 requiresFullRendering=True):
        self.depth, self.rgb = depth, rgb
        v = abi.View()
        v.d_depth, v.d_rgb = _ptr(depth), _ptr(rgb)
        v.depth_h, v.depth_w = depth.shape[:2]
        v.rgb_h, v.rgb_w = rgb.shape[:2]
        v.proj_d = abi.f4(*[float(x) for x in proj_d])
        v.proj_rgb = abi.f4(*[float(x) for x in (proj_rgb if proj_rgb is not None else proj_d)])
        v.depthWeighting, v.requiresFullRendering = int(depthWeighting), int(requiresFullRendering)
        self.c = v
        self.set_pose(M_d, M_rgb)

    def set_pose(self, M_d, M_rgb=None):
        lib = abi.host_library()
        self.c.M_d = abi.mat_to_c(M_d)
        inv = abi.f16()
        if not lib.b200h_mat4_inv(self.c.M_d, inv):
            raise ValueError("singular pose")
        self.c.invM_d = inv
        self.c.M_rgb = abi.mat_to_c(M_rgb if M_rgb is not None else M_d)


def make_camera(M, proj):
    lib = abi.host_library()
    c = abi.Camera()
    c.M = abi.mat_to_c(M)
    inv = abi.f16()
    if not lib.b200h_mat4_inv(c.M, inv):
        raise ValueError("singular pose")
    c.invM = inv
    c.proj = abi.f4(*[float(x) for x in proj])
    return c


class Engine:
    """Opaque per-volume engine handle (owns scratch, decay ring, stream)."""

    def __init__(self, scene, imgSize, decayRingItems=0, stream=None):
        if not torch.cuda.is_available():
            raise RuntimeError("dynslam_b200 needs a CUDA device; there is no CPU fallback")
        self.lib = abi.load_library()
        cfg = abi.EngineConfig()
        cfg.device = scene.device.index or 0
        cfg.numBlocks, cfg.numBuckets, cfg.excessSize = scene.numBlocks, scene.numBuckets, scene.excessSize
        cfg.img_w, cfg.img_h = imgSize
        cfg.decayRingItems = decayRingItems
        cfg.stream = stream
        h = C.c_void_p()
        rc = self.lib.b200_engine_create(C.byref(cfg), C.byref(h))
        self.h = h if rc == abi.OK else None
        if rc:      # a failed create leaves nothing allocated; the reason is in b200_last_error(NULL)
            msg = self.lib.b200_last_error(None).decode()
            raise (CudaError if rc == abi.ERR_CUDA else ValueError)(msg)
        self.scene = scene
        self._ext = torch.cuda.ExternalStream(self.lib.b200_engine_stream(self.h), device=scene.device)

    def after_torch(self):
        """Order the engine's stream behind the work already enqueued on torch's current stream (tensor fills, uploads,
        torch kernels that produced depth / rgb): the engine runs on its own non-blocking stream and would otherwise race
        with them. One event record + one stream wait, no host synchronisation; a no-op when both are the same stream."""
        cur = torch.cuda.current_stream(self.scene.device)
        if cur.cuda_stream != self._ext.cuda_stream:
            self._ext.wait_stream(cur)

    def close(self):
        if getattr(self, "h", None):
            self.lib.b200_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def check(self, rc):
        if rc == abi.OK:
            return
        msg = self.lib.b200_last_error(self.h).decode()
        if rc in (abi.ERR_VBA_FULL, abi.ERR_EXCESS_FULL, abi.ERR_DECAY_RING_FULL):
            raise RuntimeError(msg)
        if rc == abi.ERR_CUDA:
            raise CudaError(msg)
        raise ValueError(msg)

    @property
    def frameIdx(self):
        return self.lib.b200_frame_index(self.h)

    @property
    def stream(self):
        return self.lib.b200_engine_stream(self.h)

    def stats(self):
        st = abi.FrameStats()
        self.check(self.lib.b200_get_stats(self.h, C.byref(st)))
        return st

    def set_timing(self, on):
        self.lib.b200_set_timing(self.h, int(on))

    def set_max_rendering_blocks(self, n):
        """test hook (include/b200fusion_diag.h): lower MAX_RENDERING_BLOCKS to reach the cap rule with small scenes"""
        self.lib.b200_diag_set_max_rendering_blocks(self.h, int(n))

    def set_grid_scale(self, k):
        """test hook (include/b200fusion_diag.h): launch the kernels whose CTAs wait on one another on k times their grid,
        more CTAs than the GPU holds at once; k <= 1 restores the default"""
        self.lib.b200_diag_set_grid_scale(self.h, int(k))

    def last_integrate(self):
        """test hook (include/b200fusion_diag.h): (kernel, grid) of the last integrate launch; kernel 1 TMA, 2 V3, 3 V4 with
        two voxels per lane, 4 V4 with four, + 8 in tolerance mode"""
        k, g = C.c_int(), C.c_int()
        self.lib.b200_diag_last_integrate(self.h, C.byref(k), C.byref(g))
        return k.value, g.value

    def push_decay_snapshot(self, positions):
        """test hook (include/b200fusion_diag.h): append a snapshot of block positions (int32 (n, 3) tensor on the engine's
        device) to the decay queue, as an allocation does, without advancing the frame index"""
        positions = positions.to(device=self.scene.device, dtype=torch.int32).contiguous()
        self.after_torch()
        self.check(self.lib.b200_diag_push_decay_snapshot(self.h, _ptr(positions) if positions.numel() else None,
                                                          positions.shape[0]))

    def save_checkpoint(self, scene, renderState):
        """b200_checkpoint_save: the volume's state (scene, render state, frame index, decay queue) as a uint8 array, laid out as
        include/b200fusion.h documents; load_checkpoint resumes fusion from it bit for bit. Finishes outstanding frames first."""
        n = C.c_size_t()
        self.after_torch()
        self.check(self.lib.b200_checkpoint_save(self.h, C.byref(scene.c), C.byref(renderState.c), None, 0, C.byref(n)))
        buf = np.empty(n.value, dtype=np.uint8)
        self.check(self.lib.b200_checkpoint_save(self.h, C.byref(scene.c), C.byref(renderState.c), buf.ctypes.data, buf.size,
                                                 C.byref(n)))
        return buf

    def load_checkpoint(self, scene, renderState, buf):
        """b200_checkpoint_load: replaces the state of scene and renderState (same geometry, voxelSize, mu and optional buffers)
        and this engine's frame index and decay queue with a checkpoint's. Raises ValueError, with nothing written, on a buffer
        that does not fit."""
        b = np.ascontiguousarray(np.frombuffer(memoryview(buf).cast("B"), dtype=np.uint8))
        self.after_torch()
        self.check(self.lib.b200_checkpoint_load(self.h, C.byref(scene.c), C.byref(renderState.c), b.ctypes.data, b.size))

    def restart_volume(self, scene, renderState):
        """b200_volume_restart_async: on this engine's stream, with no host wait and no allocation, the engine, scene and render
        state become what a newly created engine on a newly allocated, reset scene with a new render state is (frame index 0)."""
        self.after_torch()
        self.check(self.lib.b200_volume_restart_async(self.h, C.byref(scene.c), C.byref(renderState.c)))

    def set_frame_index(self, f):
        """test hook (include/b200fusion_diag.h): the frame index Decay measures block ages against"""
        self.lib.b200_diag_set_frame_index(self.h, int(f))

    # ---- fused fast path --------------------------------------------------------------------
    def process_frame_async(self, renderState, view, points=None, normals=None, decay=None, raycast=True, colour_out=None,
                            depth_out=None):
        """colour_out / depth_out: optional renders (RENDER_COLOUR_FROM_VOLUME / RENDER_DEPTH_MAP) shaded from this frame's ray
        points, for compositing (multi-volume configuration)."""
        o = abi.FrameOpts()
        o.doRaycast = int(raycast)
        o.d_colourRender, o.d_depthRender = _ptr(colour_out), _ptr(depth_out)
        if decay is not None:
            o.doDecay, o.decayMaxWeight, o.decayMinAge = 1, decay[0], decay[1]
        self.after_torch()
        self.check(self.lib.b200_process_frame_async(self.h, C.byref(self.scene.c), C.byref(renderState.c), C.byref(view.c),
                                                      _ptr(points), _ptr(normals), C.byref(o)))

    def sync(self, renderState):
        self.check(self.lib.b200_sync(self.h, C.byref(self.scene.c), C.byref(renderState.c)))

    def process_frame_host(self, renderState, view, h_depth, h_rgb, d_depth_stage, d_rgb_stage, points=None, normals=None,
                           decay=None, raycast=True, h_out=None):
        o = abi.FrameOpts()
        o.doRaycast = int(raycast)
        if decay is not None:
            o.doDecay, o.decayMaxWeight, o.decayMinAge = 1, decay[0], decay[1]
        self.check(self.lib.b200_process_frame_host(self.h, C.byref(self.scene.c), C.byref(renderState.c), C.byref(view.c),
                                                     _ptr(h_depth), _ptr(h_rgb), _ptr(d_depth_stage), _ptr(d_rgb_stage),
                                                     _ptr(points), _ptr(normals), C.byref(o), _ptr(h_out)))


    def host_frame_submit(self, renderState, view, h_depth, h_rgb, points=None, normals=None, decay=None, raycast=True, h_out=None,
                          slot=0, colour_out=None, depth_out=None):
        """Pipelined host frames: H2D, fused frame and D2H of the grey image are enqueued without blocking."""
        o = abi.FrameOpts()
        o.doRaycast = int(raycast)
        o.d_colourRender, o.d_depthRender = _ptr(colour_out), _ptr(depth_out)
        if decay is not None:
            o.doDecay, o.decayMaxWeight, o.decayMinAge = 1, decay[0], decay[1]
        self.check(self.lib.b200_host_frame_submit(self.h, C.byref(self.scene.c), C.byref(renderState.c), C.byref(view.c),
                                                    _ptr(h_depth), _ptr(h_rgb), _ptr(points), _ptr(normals), C.byref(o), _ptr(h_out), slot))

    def host_frame_submit_raw(self, renderState, view, h_raw, h_rgb, calib, points=None, normals=None, decay=None, raycast=True,
                              h_out=None, slot=0):
        """As host_frame_submit, from a RAW int16 depth frame: UpdateView (conversion + bilateral filter) runs on the device."""
        o = abi.FrameOpts()
        o.doRaycast = int(raycast)
        if decay is not None:
            o.doDecay, o.decayMaxWeight, o.decayMinAge = 1, decay[0], decay[1]
        self.check(self.lib.b200_host_frame_submit_raw(self.h, C.byref(self.scene.c), C.byref(renderState.c), C.byref(view.c),
                                                        _ptr(h_raw), _ptr(h_rgb), C.byref(calib), _ptr(points), _ptr(normals),
                                                        C.byref(o), _ptr(h_out), slot))

    def host_frame_submit_stereo(self, renderState, view, h_bgr, h_depth_in, depth_input, calib, points=None, normals=None, decay=None,
                                 raycast=True, h_out=None, depth_mm_out=None, slot=0):
        """As host_frame_submit_raw, from DynSLAM's stored stereo input: h_bgr (h, w, 3 uint8, OpenCV's BGR) and h_depth_in (a float32
        disparity map or int16 millimetres, per depth_input.kind; see make_depth_input). The int16 mm depth and the RGBA colour are
        made on the device; depth_mm_out (an int16 CUDA tensor, optional) receives the frame's int16 mm depth once
        host_frame_wait(slot) returns."""
        o = abi.FrameOpts()
        o.doRaycast = int(raycast)
        if decay is not None:
            o.doDecay, o.decayMaxWeight, o.decayMinAge = 1, decay[0], decay[1]
        self.check(self.lib.b200_host_frame_submit_stereo(self.h, C.byref(self.scene.c), C.byref(renderState.c), C.byref(view.c),
                                                           _ptr(h_bgr), _ptr(h_depth_in), C.byref(depth_input), C.byref(calib),
                                                           _ptr(points), _ptr(normals), C.byref(o), _ptr(h_out), _ptr(depth_mm_out), slot))

    def trace(self):
        """Launch trace collected since set_timing(3): list of (kernel, start_us, end_us)."""
        buf = C.create_string_buffer(1 << 20)
        n = self.lib.b200_get_trace(self.h, buf, len(buf))
        out = []
        for ln in buf.raw[:n].decode().splitlines():
            name, a, b = ln.split()
            out.append((name, float(a), float(b)))
        return out

    def host_frame_wait(self, slot):
        self.check(self.lib.b200_host_frame_wait(self.h, slot))

    def wait_engine(self, other):
        """b200_engine_wait_engine: this engine's stream waits, on the device, for what is enqueued on other's stream so far
        (compositing layers another engine rendered without a host synchronisation in between)."""
        self.check(self.lib.b200_engine_wait_engine(self.h, other.h))


def make_view_calib(trafoType=1, params=(1.0 / 1000.0, 0.0), fx_depth=0.0, intrinsics_d=(0.0, 0.0, 0.0, 0.0), useBilateralFilter=True,
                    modelSensorNoise=False):
    """b200_view_calib. Defaults: ITMDisparityCalib() = affine mm -> m (Objects/ITMDisparityCalib.h:40-45),
    useBilateralFilter true, modelSensorNoise false (Utils/ITMLibSettings.cpp:63, :74)."""
    c = abi.ViewCalib()
    c.trafoType = int(trafoType)
    c.params = (C.c_float * 2)(float(params[0]), float(params[1]))
    c.fx_depth = float(fx_depth)
    c.intrinsics_d = (C.c_float * 4)(*[float(x) for x in intrinsics_d])
    c.useBilateralFilter, c.modelSensorNoise = int(useBilateralFilter), int(modelSensorNoise)
    return c


def make_depth_input(kind=abi.DEPTH_IN_DISPARITY_F32, baseline_m=0.0, focal_length_px=0.0, min_depth_m=0.5, max_depth_m=20.0):
    """b200_depth_input. kind 0: a DispNet float disparity map with the rig's StereoCalibration (DS/DepthProvider.h:22-28);
    kind 1: an ELAS int16 millimetre depth map. min/max: DepthProvider's depth bounds (the KITTI configurations' 0.5 m and 20 m, DS/Input.h:71-72)."""
    d = abi.DepthInput()
    d.kind, d.baseline_m, d.focal_length_px = int(kind), float(baseline_m), float(focal_length_px)
    d.min_depth_m, d.max_depth_m = float(min_depth_m), float(max_depth_m)
    return d


class StereoInput:
    """DynSLAM's per-frame input conversions on the device (images are torch CUDA tensors), named after the reference's functions."""

    def __init__(self, engine, depth_input):
        self.e, self.depth_input = engine, depth_input

    def DepthFromDisparityMap(self, out_depth, disparity):
        """DepthProvider::DepthFromDisparityMap<float> with scale 1 (kind 0), or ReadPrecomputed's max-depth clamp of a stored int16
        depth map (kind 1; out_depth may be the input): int16 millimetres into out_depth."""
        ViewBuilder._inputs_ready()
        h, w = disparity.shape
        self.e.check(self.e.lib.b200_depth_mm_from_input(self.e.h, _ptr(out_depth), _ptr(disparity), w, h, C.byref(self.depth_input)))

    def CvToItm(self, out_rgba, bgr):
        """CvToItm(const cv::Mat3b &, ITMUChar4Image *): (h, w, 3) BGR8 into (h, w, 4) RGBA8 with alpha 255."""
        ViewBuilder._inputs_ready()
        h, w = bgr.shape[:2]
        self.e.check(self.e.lib.b200_bgr_to_rgba(self.e.h, _ptr(out_rgba), _ptr(bgr), w, h))


class ViewBuilder:
    """ITMViewBuilder (B200 back-end, Engine/ITMViewBuilder.h:19-58). Images are torch CUDA tensors."""

    def __init__(self, engine, calib):
        self.e, self.calib = engine, calib

    @staticmethod
    def _inputs_ready():
        # the images are torch tensors produced on torch's stream; the engine works on its own stream
        torch.cuda.current_stream().synchronize()

    def ConvertDisparityToDepth(self, depth_out, disp_in, fx_depth, params):
        self._inputs_ready()
        h, w = disp_in.shape
        self.e.check(self.e.lib.b200_convert_disparity_to_depth(self.e.h, _ptr(depth_out), _ptr(disp_in), w, h, params[0], params[1], fx_depth))

    def ConvertDepthAffineToFloat(self, depth_out, depth_in, params):
        self._inputs_ready()
        h, w = depth_in.shape
        self.e.check(self.e.lib.b200_convert_depth_affine_to_float(self.e.h, _ptr(depth_out), _ptr(depth_in), w, h, params[0], params[1]))

    def DepthFiltering(self, image_out, image_in):
        self._inputs_ready()
        h, w = image_in.shape
        self.e.check(self.e.lib.b200_depth_filtering(self.e.h, _ptr(image_out), _ptr(image_in), w, h))

    def ComputeNormalAndWeights(self, normal_out, sigmaZ_out, depth_in, intrinsic):
        self._inputs_ready()
        h, w = depth_in.shape
        self.e.check(self.e.lib.b200_compute_normal_and_weights(self.e.h, _ptr(normal_out), _ptr(sigmaZ_out), _ptr(depth_in), w, h,
                                                                (C.c_float * 4)(*[float(x) for x in intrinsic])))

    def UpdateView(self, depth_out, rawDepth, depthNormal=None, depthUncertainty=None, sync=True):
        """UpdateView(view, rgb, rawDepth, useBilateralFilter, modelSensorNoise) on device-resident images."""
        self._inputs_ready()
        h, w = rawDepth.shape
        f = self.e.lib.b200_update_view if sync else self.e.lib.b200_update_view_async
        self.e.check(f(self.e.h, _ptr(rawDepth), w, h, C.byref(self.calib), _ptr(depth_out), _ptr(depthNormal), _ptr(depthUncertainty)))


# kMatplotlib2Palette (DS/InstRecLib/InstanceReconstructor.cpp:43-55)
MATPLOTLIB2_PALETTE = [(0x1f, 0x77, 0xb4, 255), (0xff, 0x7f, 0x0e, 255), (0x2c, 0xa0, 0x2c, 255), (0xd6, 0x27, 0x28, 255),
                       (0x94, 0x67, 0xbd, 255), (0x8c, 0x56, 0x4b, 255), (0xe3, 0x77, 0xc2, 255), (0x71, 0x71, 0x71, 255),
                       (0xbc, 0xbd, 0x22, 255), (0x17, 0xbe, 0xcf, 255)]

KEEP, REMOVE, EXTRACT = 0, 1, 2   # b200_silhouette_op.action


def make_mask(bbox, data):
    """b200_mask from an inclusive (x0, y0, x1, y1) box and a box-sized uint8 CUDA tensor (1 = inside)."""
    x0, y0, x1, y1 = [int(v) for v in bbox]
    assert data.dtype == torch.uint8 and tuple(data.shape) == (y1 - y0 + 1, x1 - x0 + 1) and data.is_contiguous()
    m = abi.Mask()
    m.x0, m.y0, m.x1, m.y1, m.d_data = x0, y0, x1, y1, data.data_ptr()
    m._keep = data
    return m


class InstanceFrames:
    """The image work of InstanceReconstructor (DS/InstRecLib/InstanceReconstructor.cpp) that touches full frames:
    cutting detections out of the main frame into per-instance frames, and compositing the per-volume renders."""

    def __init__(self, engine):
        self.e = engine

    def ProcessSilhouettes(self, rgb, depth, ops, sync=True, wait_inputs=True):
        """ops: list of (action, copy_mask, delete_mask, dest_rgb, dest_depth) in the order of the active tracks.
        wait_inputs=False: the caller already orders the tensors on the engine's stream."""
        if wait_inputs:
            torch.cuda.current_stream().synchronize()
        h, w = depth.shape
        arr, n = ops if isinstance(ops, tuple) else self.prepare_ops(ops)
        f = self.e.lib.b200_process_silhouettes if sync else self.e.lib.b200_process_silhouettes_async
        self.e.check(f(self.e.h, _ptr(rgb), _ptr(depth), w, h, arr, n))

    @staticmethod
    def prepare_ops(ops):
        """the b200_silhouette_op array of a list of ops — build it once for a frame that is processed more than once (or ahead of
        time: a Python host spends longer marshalling the array than the GPU spends on the launch)"""
        arr = (abi.SilhouetteOp * max(len(ops), 1))()
        for k, (action, cm, dm, drgb, ddepth) in enumerate(ops):
            arr[k].action = int(action)
            if cm is not None:
                arr[k].copy_mask = cm
            if dm is not None:
                arr[k].delete_mask = dm
            arr[k].d_dest_rgb, arr[k].d_dest_depth = _ptr(drgb), _ptr(ddepth)
        return arr, len(ops)

    def CompositeDepth(self, target, source):
        torch.cuda.current_stream().synchronize()
        self.e.check(self.e.lib.b200_composite_depth(self.e.h, _ptr(target), _ptr(source), target.numel()))

    def CompositeColor(self, target_color, target_depth, instance_color, instance_depth, tint, tint_strength):
        torch.cuda.current_stream().synchronize()
        self.e.check(self.e.lib.b200_composite_color(self.e.h, _ptr(target_color), _ptr(target_depth), _ptr(instance_color),
                                                      _ptr(instance_depth), target_depth.numel(),
                                                      (C.c_int32 * 4)(*[int(t) for t in tint]), float(tint_strength)))

    def CompositeInstances(self, out_color, out_depth, layers, dim_factor=0.10, tint_strength=1.0, wait_inputs=True):
        """layers: list of (color, depth, tint) in the order of the active tracks; dim_factor < 0 skips the dimming."""
        if wait_inputs:
            torch.cuda.current_stream().synchronize()
        arr = (abi.InstanceLayer * max(len(layers), 1))()
        for k, (col, dep, tint) in enumerate(layers):
            arr[k].d_color, arr[k].d_depth = _ptr(col), _ptr(dep)
            arr[k].tint = (C.c_int32 * 4)(*[int(t) for t in tint])
        self.e.check(self.e.lib.b200_composite_instances(self.e.h, _ptr(out_color), _ptr(out_depth), out_depth.numel(), arr, len(layers),
                                                          float(dim_factor), float(tint_strength)))


class SceneReconstructionEngine:
    """ITMSceneReconstructionEngine<ITMVoxel, ITMVoxelBlockHash> (B200 back-end)."""

    def __init__(self, engine):
        self.e = engine
        self.fusionWeightParams = dict(depthWeighting=False)

    def SetFusionWeightParams(self, depthWeighting):
        self.fusionWeightParams["depthWeighting"] = bool(depthWeighting)

    def ResetScene(self, scene):
        self.e.after_torch()
        self.e.check(self.e.lib.b200_reset_scene(self.e.h, C.byref(scene.c)))

    def AllocateSceneFromDepth(self, scene, view, renderState, onlyUpdateVisibleList=False):
        self.e.after_torch()
        self.e.check(self.e.lib.b200_allocate_from_depth(self.e.h, C.byref(scene.c), C.byref(renderState.c), C.byref(view.c),
                                                          int(onlyUpdateVisibleList)))

    def IntegrateIntoScene(self, scene, view, renderState):
        view.c.depthWeighting = int(self.fusionWeightParams["depthWeighting"])
        self.e.after_torch()
        self.e.check(self.e.lib.b200_integrate(self.e.h, C.byref(scene.c), C.byref(renderState.c), C.byref(view.c)))

    def Decay(self, scene, renderState, maxWeight, minAge, forceAllVoxels=False):
        self.e.after_torch()
        self.e.check(self.e.lib.b200_decay(self.e.h, C.byref(scene.c), C.byref(renderState.c), maxWeight, minAge,
                                           int(forceAllVoxels)))

    def GetDecayedBlockCount(self):
        return self.e.lib.b200_decayed_block_count(self.e.h)


class VisualisationEngine:
    """ITMVisualisationEngine<ITMVoxel, ITMVoxelBlockHash> (B200 back-end)."""

    def __init__(self, engine, scene):
        self.e, self.scene = engine, scene

    def CreateRenderState(self, imgSize, forward=False):
        return RenderStateVH(self.scene, imgSize, forward=forward)

    def FindVisibleBlocks(self, camera, renderState):
        self.e.after_torch()
        self.e.check(self.e.lib.b200_find_visible_blocks(self.e.h, C.byref(self.scene.c), C.byref(renderState.c), C.byref(camera)))

    def CreateExpectedDepths(self, camera, renderState):
        self.e.after_torch()
        self.e.check(self.e.lib.b200_expected_depths(self.e.h, C.byref(self.scene.c), C.byref(renderState.c), C.byref(camera)))

    def FindSurface(self, camera, renderState):
        self.e.after_torch()
        self.e.check(self.e.lib.b200_find_surface(self.e.h, C.byref(self.scene.c), C.byref(renderState.c), C.byref(camera)))

    def RenderImage(self, camera, renderState, outputCharImage, outputFloatImage, type=abi.RENDER_SHADED_GREYSCALE):
        self.e.after_torch()
        self.e.check(self.e.lib.b200_render_image(self.e.h, C.byref(self.scene.c), C.byref(renderState.c), C.byref(camera),
                                                   _ptr(outputCharImage), _ptr(outputFloatImage), renderState.w, renderState.h, type))

    def RenderFreeView(self, camera, renderState, outputCharImage, outputFloatImage, type=abi.RENDER_SHADED_GREYSCALE, sync=True):
        """b200_render_view_async: FindVisibleBlocks + CreateExpectedDepths + RenderImage(type) + RenderImage(RENDER_DEPTH_MAP) from
        one pose as one enqueue and one raycast, into a free-view render state. Either image may be None. sync=False only
        enqueues (renderState.noVisibleBlocks is then refreshed by RenderFreeViewSync)."""
        self.e.after_torch()
        self.e.check(self.e.lib.b200_render_view_async(self.e.h, C.byref(self.scene.c), C.byref(renderState.c), C.byref(camera), type,
                                                        _ptr(outputCharImage), _ptr(outputFloatImage)))
        if sync:
            self.RenderFreeViewSync(renderState)

    def RenderFreeViewSync(self, renderState):
        self.e.check(self.e.lib.b200_render_view_sync(self.e.h, C.byref(renderState.c)))

    def RenderFreeViewSubmit(self, camera, renderState, h_outChar, h_outFloat, type=abi.RENDER_SHADED_GREYSCALE, slot=0):
        """b200_render_view_submit: the same render, the images landing in the host tensors h_outChar / h_outFloat (pinned or
        pageable; either may be None) once RenderFreeViewWait(slot) returns."""
        self.e.after_torch()
        self.e.check(self.e.lib.b200_render_view_submit(self.e.h, C.byref(self.scene.c), C.byref(renderState.c), C.byref(camera), type,
                                                         _ptr(h_outChar), _ptr(h_outFloat), slot))

    def RenderFreeViewWait(self, slot):
        self.e.check(self.e.lib.b200_render_view_wait(self.e.h, slot))

    def CreateICPMaps(self, view, renderState, points, normals):
        self.e.after_torch()
        self.e.check(self.e.lib.b200_icp_maps(self.e.h, C.byref(self.scene.c), C.byref(renderState.c), C.byref(view.c),
                                               _ptr(points), _ptr(normals)))

    def ForwardRender(self, view, renderState):
        self.e.after_torch()
        self.e.check(self.e.lib.b200_forward_render(self.e.h, C.byref(self.scene.c), C.byref(renderState.c), C.byref(view.c)))
        return renderState.c.noFwdProjMissingPoints

    def CreatePointCloud(self, view, renderState, locations, colours, skipPoints=False, calib_rgb_to_depth=None):
        calib = abi.mat_to_c(calib_rgb_to_depth if calib_rgb_to_depth is not None else np.eye(4, dtype=np.float32))
        n = C.c_uint32()
        self.e.after_torch()
        self.e.check(self.e.lib.b200_point_cloud(self.e.h, C.byref(self.scene.c), C.byref(renderState.c), C.byref(view.c), calib,
                                                  int(skipPoints), _ptr(locations), _ptr(colours), C.byref(n)))
        return n.value


class Mesh:
    """ITMMesh (Objects/ITMMesh.h:15-42): noMaxTriangles = sdfLocalBlockNum * 512 / 16 triangles of six Vector3f on the device."""

    def __init__(self, scene, noMaxTriangles=None):
        self.noMaxTriangles = int(noMaxTriangles if noMaxTriangles is not None else scene.numBlocks * abi.SDF_BLOCK_SIZE3 // 16)
        self.triangles = torch.zeros(self.noMaxTriangles * 18, dtype=torch.float32, device=scene.device)
        self.noTotalTriangles = 0

    def to_host(self):
        n = min(self.noTotalTriangles, self.noMaxTriangles - 1)
        return self.triangles.cpu().numpy().view(abi.TRIANGLE_DTYPE)[:n].copy()

    def WriteOBJ(self, fileName):
        """ITMMesh::WriteOBJ (Objects/ITMMesh.h:46-122): `v x y z r g b` per vertex, then `f 3i+3 3i+2 3i+1`, printf's %f."""
        if self.noTotalTriangles > self.noMaxTriangles:
            raise RuntimeError(f"Unable to save mesh to file [{fileName}]. Too many triangles: {self.noTotalTriangles} while the maximum is {self.noMaxTriangles}.")
        t = self.triangles.cpu().numpy().view(abi.TRIANGLE_DTYPE)[:self.noTotalTriangles]
        with open(fileName, "w") as f:
            for tr in t:
                for p, c in ((tr["p0"], tr["c0"]), (tr["p1"], tr["c1"]), (tr["p2"], tr["c2"])):
                    f.write("v %f %f %f %f %f %f\n" % (p[0], p[1], p[2], c[0], c[1], c[2]))
            for i in range(len(t)):
                f.write("f %d %d %d\n" % (i * 3 + 2 + 1, i * 3 + 1 + 1, i * 3 + 0 + 1))


class MeshingEngine:
    """ITMMeshingEngine<ITMVoxel, ITMVoxelBlockHash> (B200 back-end)."""

    def __init__(self, engine):
        self.e = engine

    def MeshScene(self, mesh, scene):
        n = C.c_uint32()
        self.e.after_torch()
        self.e.check(self.e.lib.b200_mesh_scene(self.e.h, C.byref(scene.c), _ptr(mesh.triangles), mesh.noMaxTriangles, C.byref(n)))
        mesh.noTotalTriangles = n.value
        return n.value


class Evaluation:
    """dynslam::eval::Evaluation's depth evaluation (DS/Evaluation/Evaluation.h:52-190, Evaluation.cpp:150-304) on the B200
    back-end: the rendered depth stays on the device, one launch evaluates every LIDAR return against every callback."""

    def __init__(self, engine, velo_to_left_gray_cam, proj_left_color, proj_right_color, baseline_m, frame_width, frame_height,
                 min_depth_m, max_depth_m):
        self.e = engine
        p = abi.EvalParams()
        p.velo_to_cam[:] = list(np.asarray(velo_to_left_gray_cam, dtype=np.float64).reshape(4, 4).T.reshape(-1))   # column-major, like Eigen
        p.proj_left[:] = list(np.asarray(proj_left_color, dtype=np.float64).reshape(3, 4).T.reshape(-1))
        p.proj_right[:] = list(np.asarray(proj_right_color, dtype=np.float64).reshape(3, 4).T.reshape(-1))
        p.baseline_m = float(baseline_m)
        p.left_focal_length_px = float(np.float32(np.asarray(proj_left_color, dtype=np.float64).reshape(3, 4)[0, 0]))   # Evaluation.h:174
        p.min_depth_m, p.max_depth_m = float(min_depth_m), float(max_depth_m)
        p.frame_width, p.frame_height = int(frame_width), int(frame_height)
        self.params = p

    @staticmethod
    def default_callbacks(compare_on_intersection=True):
        """the callback list of Evaluation::EvaluateFrame (Evaluation.cpp:176-195): delta_max 0.5, 1..12, then the KITTI-style 3 px / 5 %"""
        return [(0.5, compare_on_intersection, False)] + [(float(d), compare_on_intersection, False) for d in range(1, 13)] + \
               [(3.0, compare_on_intersection, True)]

    def EvaluateDepth(self, lidar_points, rendered_depth, input_depth_mm, callbacks=None, association=None, with_dynamic=False):
        """lidar_points: cuda float32 [n, 4] (KITTI .bin records); rendered_depth: cuda float32 [h, w] metres; input_depth_mm: cuda
        int16 [h, w]; association: cuda uint8 [h, w] or None. Returns (static results, dynamic results or None, summary)."""
        cbs = callbacks if callbacks is not None else self.default_callbacks()
        n = len(cbs)
        arr = (abi.EvalCallback * n)(*[abi.EvalCallback(float(d), int(bool(c)), int(bool(k))) for d, c, k in cbs])
        out_s = (abi.EvalResult * n)()
        out_d = (abi.EvalResult * n)() if with_dynamic else None
        summ = abi.EvalSummary()
        self.e.after_torch()
        rc = self.e.lib.b200_evaluate_depth(self.e.h, C.byref(self.params), _ptr(lidar_points), int(lidar_points.shape[0]), _ptr(rendered_depth),
                                            _ptr(input_depth_mm), _ptr(association) if association is not None else None, arr, n, out_s,
                                            out_d, C.byref(summ))
        if rc == abi.ERR_NEGATIVE_DISPARITY:
            raise RuntimeError(self.e.lib.b200_last_error(self.e.h).decode())      # the reference throws std::runtime_error
        self.e.check(rc)
        summary = dict(valid_lidar_points=summ.valid_lidar_points, epi_errors=summ.epi_errors, skipped_lidar_points=summ.skipped_lidar_points)
        return [r.as_dict() for r in out_s], ([r.as_dict() for r in out_d] if with_dynamic else None), summary


class GlobalCache:
    """Host half of ITMGlobalCache (Objects/ITMGlobalCache.h:17-129): stored blocks per entry."""

    def __init__(self, scene):
        dev = scene.device
        self.stored = {}
        n = abi.TRANSFER_BLOCK_NUM
        self.syncedVoxelBlocks = torch.zeros(n * abi.SDF_BLOCK_SIZE3 * 8, dtype=torch.uint8, device=dev)
        self.hasSyncedData = torch.zeros(n, dtype=torch.uint8, device=dev)
        self.neededEntryIDs = torch.zeros(n, dtype=torch.int32, device=dev)
        t = abi.TransferBuffers()
        t.d_syncedVoxelBlocks, t.d_hasSyncedData, t.d_neededEntryIDs = _ptr(self.syncedVoxelBlocks), _ptr(self.hasSyncedData), _ptr(self.neededEntryIDs)
        self.c = t


class SwappingEngine:
    """ITMSwappingEngine<ITMVoxel, ITMVoxelBlockHash>: host orchestration of Swap_CUDA.cu:44-216."""

    def __init__(self, engine):
        self.e = engine

    def IntegrateGlobalIntoLocal(self, scene, cache):
        n = C.c_int()
        self.e.check(self.e.lib.b200_swap_list_in(self.e.h, C.byref(scene.c), C.byref(cache.c), C.byref(n)))
        n = n.value
        if n > 0:
            ids = cache.neededEntryIDs[:n].cpu().numpy()
            blocks = np.zeros((n, abi.SDF_BLOCK_SIZE3 * 8), dtype=np.uint8)
            for i, entry in enumerate(ids):
                if int(entry) in cache.stored:
                    blocks[i] = cache.stored[int(entry)]
            cache.syncedVoxelBlocks[:n * abi.SDF_BLOCK_SIZE3 * 8].copy_(torch.from_numpy(blocks.reshape(-1)))
            self.e.check(self.e.lib.b200_swap_integrate_in(self.e.h, C.byref(scene.c), C.byref(cache.c), n))
        return n

    def SaveToGlobalMemory(self, scene, renderState, cache):
        n = C.c_int()
        self.e.check(self.e.lib.b200_swap_out(self.e.h, C.byref(scene.c), C.byref(renderState.c), C.byref(cache.c), C.byref(n)))
        n = n.value
        if n > 0:
            ids = cache.neededEntryIDs[:n].cpu().numpy()
            has = cache.hasSyncedData[:n].cpu().numpy()
            blocks = cache.syncedVoxelBlocks[:n * abi.SDF_BLOCK_SIZE3 * 8].cpu().numpy().reshape(n, -1)
            for i, entry in enumerate(ids):
                if has[i]:
                    cache.stored[int(entry)] = blocks[i].copy()
        return n


class _DeviceBuffer:
    """a device allocation the library owns, seen by torch without a copy (__cuda_array_interface__)"""

    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 3, "strides": None}


def _device_view(ptr, n, dtype, device):
    typestr = {torch.uint8: "|u1", torch.int32: "<i4", torch.float32: "<f4"}[dtype]
    return torch.as_tensor(_DeviceBuffer(ptr, n, typestr), device=device)


class _SlotScene:
    """a group slot's scene: the group's b200_scene and views of its buffers"""

    def __init__(self, cptr, device):
        self.c = cptr.contents
        self.device = device
        self.numBlocks, self.numBuckets, self.excessSize = self.c.numBlocks, self.c.numBuckets, self.c.excessSize
        self.noTotalEntries = self.numBuckets + self.excessSize
        self.params = SceneParams(voxelSize=self.c.voxelSize, mu=self.c.mu, maxW=self.c.maxW)

    @property
    def lastFreeBlockId(self):
        return self.c.lastFreeBlockId

    @property
    def lastFreeExcessListId(self):
        return self.c.lastFreeExcessListId


class _SlotRenderState:
    """a group slot's render state: the group's b200_render_state and views of its buffers"""

    def __init__(self, cptr, scene, device):
        r = cptr.contents
        self.c, self.w, self.h = r, r.img_w, r.img_h
        px = r.img_w * r.img_h
        self.visibleBlockPositions = _device_view(r.d_visibleBlockPositions, scene.numBlocks * 3, torch.int32, device)
        self.entriesVisibleType = _device_view(r.d_entriesVisibleType, scene.noTotalEntries, torch.uint8, device)
        self.renderingRangeImage = _device_view(r.d_minmax, px * 2, torch.float32, device)
        self.raycastResult = _device_view(r.d_raycastResult, px * 4, torch.float32, device)
        self.raycastImage = _device_view(r.d_raycastImage, px * 4, torch.uint8, device)

    @property
    def noVisibleBlocks(self):
        return self.c.noVisibleBlocks


class _SlotEngine(Engine):
    """a group slot's engine: every Engine method works on it; the group owns and destroys it"""

    def __init__(self, lib, handle, scene):
        self.lib, self.h, self.scene = lib, C.c_void_p(handle), scene
        self._ext = torch.cuda.ExternalStream(self.lib.b200_engine_stream(self.h), device=scene.device)

    def close(self):
        self.h = None


class VolumeSlot:
    """one slot of a VolumeGroup: its engine, scene, render state and images (torch views of the group's buffers)"""

    def __init__(self, group, i):
        lib, dev = group.lib, group.device
        eng, sc, rs = C.c_void_p(), C.POINTER(abi.Scene)(), C.POINTER(abi.RenderState)()
        group.check(lib.b200_group_slot(group.h, i, C.byref(eng), C.byref(sc), C.byref(rs)))
        im = abi.GroupImages()
        group.check(lib.b200_group_slot_images(group.h, i, C.byref(im)))
        self.scene = _SlotScene(sc, dev)
        self.engine = _SlotEngine(lib, eng.value, self.scene)
        self.rs = _SlotRenderState(rs, self.scene, dev)
        px = self.rs.w * self.rs.h
        self.instance_rgb = _device_view(im.d_instance_rgb, px * 4, torch.uint8, dev)
        self.instance_depth = _device_view(im.d_instance_depth, px, torch.float32, dev)
        self.colour_render = _device_view(im.d_colour_render, px * 4, torch.uint8, dev)
        self.depth_render = _device_view(im.d_depth_render, px, torch.float32, dev)
        self.points = _device_view(im.d_points, px * 4, torch.float32, dev)
        self.normals = _device_view(im.d_normals, px * 4, torch.float32, dev)


class GroupCar:
    """one car of a VolumeGroup frame (b200_group_car): its slot, silhouette action and masks (make_mask), pose, depth
    intrinsics, whether it is fused, and its layer's tint. prepare() builds the C array once for reuse."""

    def __init__(self, slot, action, copy_mask, delete_mask, M, proj, fuse=True, tint=(0, 0, 0, 255)):
        self.slot, self.action, self.copy_mask, self.delete_mask = slot, action, copy_mask, delete_mask
        self.M, self.proj, self.fuse, self.tint = M, proj, fuse, tint


class VolumeGroup:
    """b200_group_*: the static map (an Engine, its Scene and live RenderStateVH) and max_cars car-volume slots created up front
    (include/b200fusion.h, "volume group"). frame() enqueues DynSLAM's whole multi-volume frame as one call; track_start(i)
    restarts slot i for a new track on the device. slots[i] gives each slot's Engine, scene, render state and images, on which
    every per-engine call works."""

    def __init__(self, static_engine, static_rs, static_points, static_normals, max_cars, shared_stream=False, numBlocks=0,
                 numBuckets=0, excessSize=0, voxelSize=0.0, mu=0.0, maxW=0, decayRingItems=0, dim_factor=0.10, tint_strength=1.0):
        self.lib = static_engine.lib
        self.static, self.static_rs = static_engine, static_rs
        self.device = static_engine.scene.device
        self._keep = (static_points, static_normals)
        cfg = abi.GroupConfig()
        cfg.static_engine = static_engine.h.value
        cfg.static_scene = C.addressof(static_engine.scene.c)
        cfg.static_rs = C.addressof(static_rs.c)
        cfg.static_points, cfg.static_normals = _ptr(static_points), _ptr(static_normals)
        cfg.max_cars = max_cars
        cfg.numBlocks, cfg.numBuckets, cfg.excessSize = numBlocks, numBuckets, excessSize
        cfg.voxelSize, cfg.mu, cfg.maxW = voxelSize, mu, maxW
        cfg.decayRingItems, cfg.shared_stream = decayRingItems, int(shared_stream)
        cfg.dim_factor, cfg.tint_strength = dim_factor, tint_strength
        static_engine.after_torch()
        h = C.c_void_p()
        rc = self.lib.b200_group_create(C.byref(cfg), C.byref(h))
        self.h = h if rc == abi.OK else None
        if rc:
            msg = self.lib.b200_group_last_error(None).decode()
            raise (CudaError if rc == abi.ERR_CUDA else ValueError)(msg)
        self.max_cars = max_cars
        self.slots = [VolumeSlot(self, i) for i in range(max_cars)]

    def check(self, rc):
        if rc == abi.OK:
            return
        msg = self.lib.b200_group_last_error(self.h).decode()
        if rc in (abi.ERR_VBA_FULL, abi.ERR_EXCESS_FULL):
            raise RuntimeError(msg)
        raise (CudaError if rc == abi.ERR_CUDA else ValueError)(msg)

    def close(self):
        if getattr(self, "h", None):
            self.lib.b200_group_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def track_start(self, slot):
        """b200_group_track_start: slot's volume restarted for a new track, after everything the group enqueued so far"""
        self.static.after_torch()
        self.check(self.lib.b200_group_track_start(self.h, int(slot)))

    @staticmethod
    def prepare(cars):
        """the b200_group_car array of a list of GroupCar (build it once for a frame enqueued more than once)"""
        arr = (abi.GroupCar * max(len(cars), 1))()
        for k, c in enumerate(cars):
            a = arr[k]
            a.slot, a.action, a.fuse = int(c.slot), int(c.action), int(bool(c.fuse))
            if c.copy_mask is not None:
                a.copy_mask = c.copy_mask
            if c.delete_mask is not None:
                a.delete_mask = c.delete_mask
            a.cam = make_camera(c.M, c.proj)
            a.tint = (C.c_int32 * 4)(*[int(t) for t in c.tint])
        return arr, len(cars)

    def frame(self, rgb, depth, static_view, cars, out_color, out_depth, decay=None, wait_inputs=True):
        """b200_group_frame_async. cars: a list of GroupCar or prepare()'s result. rgb / depth: the frame, updated in place by the
        silhouettes; static_view normally views them. wait_inputs=False: the caller already orders the tensors on the static
        engine's stream."""
        arr, n = cars if isinstance(cars, tuple) else self.prepare(cars)
        dec = (C.c_int32 * 2)(int(decay[0]), int(decay[1])) if decay is not None else None
        if wait_inputs:
            self.static.after_torch()
        self.check(self.lib.b200_group_frame_async(self.h, _ptr(rgb), _ptr(depth), C.byref(static_view.c), arr, n, dec, _ptr(out_color),
                                                   _ptr(out_depth)))

    def sync(self):
        """b200_group_sync: host counters of the static map and of every slot"""
        self.check(self.lib.b200_group_sync(self.h))
