"""ctypes mirror of include/b200fusion.h and loader for the in-tree CUDA library.

The structures are byte-for-byte the C-ABI PODs (which are themselves byte-for-byte the
reference's ITMHashEntry / ITMVoxel_s_rgb / Vector* types, Utils/ITMLibDefines.h:69-84,
:138-169). There is NO fallback: if dynslam_b200/csrc/libb200fusion.so is missing or fails to
load, importing the engine raises.
"""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "csrc", "libb200fusion.so")
HOST_LIB_PATH = os.path.join(HERE, "csrc", "libb200host.so")   # host-side helpers of this mirror (csrc/hostmath.c), not the C-ABI

SDF_BLOCK_SIZE = 8
SDF_BLOCK_SIZE3 = 512
MAX_RENDERING_BLOCKS = 65536 * 4
TRANSFER_BLOCK_NUM = 0x1000

OK, ERR_CUDA, ERR_VBA_FULL, ERR_EXCESS_FULL, ERR_INVALID, ERR_DECAY_RING_FULL, ERR_UNSUPPORTED, ERR_NEGATIVE_DISPARITY = range(8)

RENDER_SHADED_GREYSCALE, RENDER_COLOUR_FROM_VOLUME, RENDER_COLOUR_FROM_NORMAL, \
    RENDER_COLOUR_FROM_DEPTH_WEIGHT, RENDER_DEPTH_MAP = range(5)

# numpy dtypes of the PODs (itemsize asserts below pin the layout)
TRIANGLE_DTYPE = np.dtype([("p0", np.float32, 3), ("p1", np.float32, 3), ("p2", np.float32, 3),
                           ("c0", np.float32, 3), ("c1", np.float32, 3), ("c2", np.float32, 3)])   # ITMMesh::Triangle, 72 bytes
HASH_ENTRY_DTYPE = np.dtype([("pos", np.int16, 3), ("_pad", np.int16), ("offset", np.int32),
                             ("ptr", np.int32), ("allocatedTime", np.int32)])
VOXEL_DTYPE = np.dtype([("sdf", np.int16), ("w_depth", np.uint8), ("clr", np.uint8, 3),
                        ("w_color", np.uint8), ("_pad", np.uint8)])
assert HASH_ENTRY_DTYPE.itemsize == 20 and VOXEL_DTYPE.itemsize == 8

# b200_checkpoint_header and its section order (include/b200fusion.h)
CHECKPOINT_MAGIC, CHECKPOINT_VERSION, CHECKPOINT_HEADER_BYTES = b"B200CKPT", 1, 512
CHECKPOINT_SECTIONS = ["HASH_INDEX", "HASH_ENTRIES", "ALLOCATION_LIST", "EXCESS_LIST", "SWAP_STATES", "VIS_INDEX", "VIS_VALUE",
                       "VISIBLE_LIST", "MINMAX", "RAYCAST_RESULT", "RAYCAST_IMAGE", "FWD_PROJECTION", "FWD_MISSING", "QUEUE_COUNTS",
                       "QUEUE_ITEMS", "BLOCK_IDS", "BLOCK_DATA"]
CK_HAS_SWAP_STATES, CK_HAS_FORWARD = 1, 2
CHECKPOINT_HEADER_DTYPE = np.dtype([
    ("magic", "S8"), ("version", "<u4"), ("flags", "<u4"),
    ("numBlocks", "<i4"), ("numBuckets", "<i4"), ("excessSize", "<i4"), ("img_w", "<i4"), ("img_h", "<i4"),
    ("voxelSize", "<f4"), ("mu", "<f4"), ("maxW", "<i4"), ("viewFrustum_min", "<f4"), ("viewFrustum_max", "<f4"),
    ("stopIntegratingAtMaxW", "<i4"), ("useSwapping", "<i4"),
    ("lastFreeBlockId", "<i4"), ("lastFreeExcessListId", "<i4"), ("noVisibleBlocks", "<i4"), ("noFwdProjMissingPoints", "<i4"),
    ("frameIdx", "<i4"), ("noSnapshots", "<i4"), ("totalDecayed", "<i8"), ("droppedSnapshots", "<i8"),
    ("noEntries", "<i8"), ("noVisBytes", "<i8"), ("noBlocks", "<i8"), ("noQueueItems", "<i8"), ("totalBytes", "<u8"),
    ("section", "<u8", (len(CHECKPOINT_SECTIONS), 2)), ("reserved", "u1", 96)])
assert CHECKPOINT_HEADER_DTYPE.itemsize == CHECKPOINT_HEADER_BYTES

f16 = C.c_float * 16
f4 = C.c_float * 4


class EvalParams(C.Structure):          # b200_eval_params
    _fields_ = [("velo_to_cam", C.c_double * 16), ("proj_left", C.c_double * 12), ("proj_right", C.c_double * 12),
                ("baseline_m", C.c_float), ("left_focal_length_px", C.c_float), ("min_depth_m", C.c_float), ("max_depth_m", C.c_float),
                ("frame_width", C.c_int32), ("frame_height", C.c_int32)]


class EvalCallback(C.Structure):        # b200_eval_callback
    _fields_ = [("delta_max", C.c_float), ("compare_on_intersection", C.c_int32), ("kitti_style", C.c_int32)]


class EvalStats(C.Structure):
    _fields_ = [("missing", C.c_int64), ("error", C.c_int64), ("correct", C.c_int64), ("missing_separate", C.c_int64)]


class EvalResult(C.Structure):
    _fields_ = [("measurement_count", C.c_int64), ("rendered", EvalStats), ("input", EvalStats)]

    def as_dict(self):
        f = lambda s: dict(missing=s.missing, error=s.error, correct=s.correct, missing_separate=s.missing_separate)
        return dict(measurement_count=self.measurement_count, rendered=f(self.rendered), input=f(self.input))


class EvalSummary(C.Structure):
    _fields_ = [("valid_lidar_points", C.c_int64), ("epi_errors", C.c_int64), ("negative_disparities", C.c_int64),
                ("skipped_lidar_points", C.c_int64)]


EVAL_STATIC, EVAL_DYNAMIC, EVAL_NEITHER = 0, 1, 2
EVAL_MAX_CALLBACKS = 16


class Scene(C.Structure):
    _fields_ = [("d_voxels", C.c_void_p), ("d_allocationList", C.c_void_p), ("d_hash", C.c_void_p),
                ("d_excessList", C.c_void_p), ("d_swapStates", C.c_void_p),
                ("numBlocks", C.c_int32), ("numBuckets", C.c_int32), ("excessSize", C.c_int32),
                ("lastFreeBlockId", C.c_int32), ("lastFreeExcessListId", C.c_int32),
                ("voxelSize", C.c_float), ("mu", C.c_float), ("maxW", C.c_int32),
                ("viewFrustum_min", C.c_float), ("viewFrustum_max", C.c_float),
                ("stopIntegratingAtMaxW", C.c_int32), ("useSwapping", C.c_int32)]


class RenderState(C.Structure):
    _fields_ = [("d_visibleBlockPositions", C.c_void_p), ("d_entriesVisibleType", C.c_void_p),
                ("d_minmax", C.c_void_p), ("d_raycastResult", C.c_void_p),
                ("d_forwardProjection", C.c_void_p), ("d_fwdProjMissingPoints", C.c_void_p),
                ("d_raycastImage", C.c_void_p), ("img_w", C.c_int32), ("img_h", C.c_int32),
                ("noVisibleBlocks", C.c_int32), ("noFwdProjMissingPoints", C.c_int32)]


class View(C.Structure):
    _fields_ = [("d_depth", C.c_void_p), ("d_rgb", C.c_void_p),
                ("depth_w", C.c_int32), ("depth_h", C.c_int32), ("rgb_w", C.c_int32), ("rgb_h", C.c_int32),
                ("M_d", f16), ("invM_d", f16), ("M_rgb", f16), ("proj_d", f4), ("proj_rgb", f4),
                ("depthWeighting", C.c_int32), ("requiresFullRendering", C.c_int32)]


class Camera(C.Structure):
    _fields_ = [("M", f16), ("invM", f16), ("proj", f4)]


class EngineConfig(C.Structure):
    _fields_ = [("device", C.c_int32), ("numBlocks", C.c_int32), ("numBuckets", C.c_int32),
                ("excessSize", C.c_int32), ("img_w", C.c_int32), ("img_h", C.c_int32),
                ("decayRingItems", C.c_int64), ("stream", C.c_void_p)]


class TransferBuffers(C.Structure):
    _fields_ = [("d_syncedVoxelBlocks", C.c_void_p), ("d_hasSyncedData", C.c_void_p),
                ("d_neededEntryIDs", C.c_void_p)]


class FrameOpts(C.Structure):
    _fields_ = [("doDecay", C.c_int32), ("decayMaxWeight", C.c_int32), ("decayMinAge", C.c_int32),
                ("doRaycast", C.c_int32), ("d_colourRender", C.c_void_p), ("d_depthRender", C.c_void_p)]


class ViewCalib(C.Structure):
    """b200_view_calib: ITMDisparityCalib + depth intrinsics + the two ITMLibSettings switches UpdateView reads."""
    _fields_ = [("trafoType", C.c_int32), ("params", C.c_float * 2), ("fx_depth", C.c_float),
                ("intrinsics_d", C.c_float * 4), ("useBilateralFilter", C.c_int32), ("modelSensorNoise", C.c_int32)]


class DepthInput(C.Structure):
    """b200_depth_input: which stored depth a stereo-input frame carries, the stereo rig and DepthProvider's depth bounds."""
    _fields_ = [("kind", C.c_int32), ("baseline_m", C.c_float), ("focal_length_px", C.c_float), ("min_depth_m", C.c_float),
                ("max_depth_m", C.c_float)]


DEPTH_IN_DISPARITY_F32, DEPTH_IN_DEPTH_MM_S16 = 0, 1


class Mask(C.Structure):
    """b200_mask: inclusive bounding box + box-sized u8 mask (1 = inside)."""
    _fields_ = [("x0", C.c_int32), ("y0", C.c_int32), ("x1", C.c_int32), ("y1", C.c_int32), ("d_data", C.c_void_p)]


class SilhouetteOp(C.Structure):
    _fields_ = [("action", C.c_int32), ("copy_mask", Mask), ("delete_mask", Mask), ("d_dest_rgb", C.c_void_p),
                ("d_dest_depth", C.c_void_p)]


class InstanceLayer(C.Structure):
    _fields_ = [("d_color", C.c_void_p), ("d_depth", C.c_void_p), ("tint", C.c_int32 * 4)]


class GroupConfig(C.Structure):         # b200_group_config
    _fields_ = [("static_engine", C.c_void_p), ("static_scene", C.c_void_p), ("static_rs", C.c_void_p),
                ("static_points", C.c_void_p), ("static_normals", C.c_void_p), ("max_cars", C.c_int32),
                ("numBlocks", C.c_int32), ("numBuckets", C.c_int32), ("excessSize", C.c_int32), ("voxelSize", C.c_float),
                ("mu", C.c_float), ("maxW", C.c_int32), ("img_w", C.c_int32), ("img_h", C.c_int32), ("decayRingItems", C.c_int64),
                ("shared_stream", C.c_int32), ("dim_factor", C.c_float), ("tint_strength", C.c_float)]


class GroupImages(C.Structure):         # b200_group_images
    _fields_ = [("d_instance_rgb", C.c_void_p), ("d_instance_depth", C.c_void_p), ("d_colour_render", C.c_void_p),
                ("d_depth_render", C.c_void_p), ("d_points", C.c_void_p), ("d_normals", C.c_void_p)]


class GroupCar(C.Structure):            # b200_group_car
    _fields_ = [("slot", C.c_int32), ("action", C.c_int32), ("copy_mask", Mask), ("delete_mask", Mask), ("cam", Camera),
                ("fuse", C.c_int32), ("tint", C.c_int32 * 4)]


class FrameStats(C.Structure):
    _fields_ = [("ms_allocate", C.c_float), ("ms_integrate", C.c_float), ("ms_expected", C.c_float),
                ("ms_raycast", C.c_float), ("ms_decay", C.c_float), ("ms_total", C.c_float),
                ("launches", C.c_int64), ("noVisibleBlocks", C.c_int32), ("noIntegratedBlocks", C.c_int32),
                ("ring_ms_integrate", C.c_float), ("ring_count", C.c_int32), ("totalIntegratedBlocks", C.c_int64),
                ("droppedSnapshots", C.c_int64), ("decayReplays", C.c_int64)]


# every symbol include/b200fusion.h declares; tests assert the .so exports all of them
EXPORTS = [
    "b200_engine_create", "b200_engine_destroy", "b200_last_error", "b200_engine_stream",
    "b200_frame_index", "b200_reset_scene",
    "b200_allocate_from_depth", "b200_integrate", "b200_decay", "b200_decayed_block_count",
    "b200_find_visible_blocks", "b200_expected_depths", "b200_find_surface", "b200_render_image",
    "b200_icp_maps", "b200_forward_render", "b200_point_cloud", "b200_swap_list_in",
    "b200_swap_integrate_in", "b200_swap_out", "b200_process_frame_async", "b200_sync",
    "b200_process_frame_host", "b200_host_frame_submit", "b200_host_frame_wait",
    "b200_convert_disparity_to_depth", "b200_convert_depth_affine_to_float", "b200_depth_filtering",
    "b200_compute_normal_and_weights", "b200_update_view", "b200_update_view_async", "b200_host_frame_submit_raw",
    "b200_depth_mm_from_input", "b200_bgr_to_rgba", "b200_host_frame_submit_stereo",
    "b200_process_silhouettes", "b200_process_silhouettes_async", "b200_composite_depth", "b200_composite_color",
    "b200_composite_instances", "b200_evaluate_depth",
    "b200_mesh_scene", "b200_checkpoint_save", "b200_checkpoint_load", "b200_comm_unique_id", "b200_comm_create", "b200_comm_destroy", "b200_comm_last_error", "b200_gather_composite_submit",
    "b200_gather_composite_release", "b200_gather_composite_wait",
    "b200_render_view_async", "b200_render_view_sync", "b200_render_view_submit", "b200_render_view_wait", "b200_engine_wait_engine",
    "b200_volume_restart_async", "b200_group_create", "b200_group_destroy", "b200_group_last_error", "b200_group_slot",
    "b200_group_slot_images", "b200_group_track_start", "b200_group_frame_async", "b200_group_sync",
]
# measurement / test hooks (include/b200fusion_diag.h): exported by the same library, not part of the drop-in boundary
DIAG_EXPORTS = ["b200_set_timing", "b200_get_trace", "b200_get_stats", "b200_selftest_divide", "b200_diag_set_max_rendering_blocks", "b200_diag_set_grid_scale",
                "b200_diag_read_debug", "b200_diag_read_spans", "b200_diag_last_integrate", "b200_diag_push_decay_snapshot", "b200_diag_set_frame_index"]

_lib = None


def load_library():
    """Load libb200fusion.so (CDLL only: no CUDA call happens until an engine is created)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'`. "
            "dynslam_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    P = C.POINTER
    vp = C.c_void_p
    lib.b200_engine_create.argtypes = [P(EngineConfig), P(vp)]
    lib.b200_engine_destroy.argtypes = [vp]
    lib.b200_engine_destroy.restype = None
    lib.b200_last_error.argtypes = [vp]
    lib.b200_last_error.restype = C.c_char_p
    lib.b200_engine_stream.argtypes = [vp]
    lib.b200_engine_stream.restype = vp
    lib.b200_frame_index.argtypes = [vp]
    lib.b200_reset_scene.argtypes = [vp, P(Scene)]
    lib.b200_allocate_from_depth.argtypes = [vp, P(Scene), P(RenderState), P(View), C.c_int]
    lib.b200_integrate.argtypes = [vp, P(Scene), P(RenderState), P(View)]
    lib.b200_decay.argtypes = [vp, P(Scene), P(RenderState), C.c_int, C.c_int, C.c_int]
    lib.b200_decayed_block_count.argtypes = [vp]
    lib.b200_decayed_block_count.restype = C.c_size_t
    lib.b200_find_visible_blocks.argtypes = [vp, P(Scene), P(RenderState), P(Camera)]
    lib.b200_expected_depths.argtypes = [vp, P(Scene), P(RenderState), P(Camera)]
    lib.b200_find_surface.argtypes = [vp, P(Scene), P(RenderState), P(Camera)]
    lib.b200_render_image.argtypes = [vp, P(Scene), P(RenderState), P(Camera), vp, vp, C.c_int, C.c_int, C.c_int]
    lib.b200_icp_maps.argtypes = [vp, P(Scene), P(RenderState), P(View), vp, vp]
    lib.b200_forward_render.argtypes = [vp, P(Scene), P(RenderState), P(View)]
    lib.b200_point_cloud.argtypes = [vp, P(Scene), P(RenderState), P(View), P(C.c_float), C.c_int, vp, vp,
                                     P(C.c_uint32)]
    lib.b200_swap_list_in.argtypes = [vp, P(Scene), P(TransferBuffers), P(C.c_int)]
    lib.b200_swap_integrate_in.argtypes = [vp, P(Scene), P(TransferBuffers), C.c_int]
    lib.b200_swap_out.argtypes = [vp, P(Scene), P(RenderState), P(TransferBuffers), P(C.c_int)]
    lib.b200_process_frame_async.argtypes = [vp, P(Scene), P(RenderState), P(View), vp, vp, P(FrameOpts)]
    lib.b200_sync.argtypes = [vp, P(Scene), P(RenderState)]
    lib.b200_process_frame_host.argtypes = [vp, P(Scene), P(RenderState), P(View), vp, vp, vp, vp, vp, vp,
                                            P(FrameOpts), vp]
    lib.b200_host_frame_submit.argtypes = [vp, P(Scene), P(RenderState), P(View), vp, vp, vp, vp, P(FrameOpts), vp, C.c_int]
    lib.b200_host_frame_wait.argtypes = [vp, C.c_int]
    lib.b200_convert_disparity_to_depth.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float]
    lib.b200_convert_depth_affine_to_float.argtypes = [vp, vp, vp, C.c_int, C.c_int, C.c_float, C.c_float]
    lib.b200_depth_filtering.argtypes = [vp, vp, vp, C.c_int, C.c_int]
    lib.b200_compute_normal_and_weights.argtypes = [vp, vp, vp, vp, C.c_int, C.c_int, P(C.c_float)]
    lib.b200_update_view.argtypes = [vp, vp, C.c_int, C.c_int, P(ViewCalib), vp, vp, vp]
    lib.b200_update_view_async.argtypes = [vp, vp, C.c_int, C.c_int, P(ViewCalib), vp, vp, vp]
    lib.b200_host_frame_submit_raw.argtypes = [vp, P(Scene), P(RenderState), P(View), vp, vp, P(ViewCalib), vp, vp, P(FrameOpts),
                                               vp, C.c_int]
    lib.b200_depth_mm_from_input.argtypes = [vp, vp, vp, C.c_int, C.c_int, P(DepthInput)]
    lib.b200_bgr_to_rgba.argtypes = [vp, vp, vp, C.c_int, C.c_int]
    lib.b200_host_frame_submit_stereo.argtypes = [vp, P(Scene), P(RenderState), P(View), vp, vp, P(DepthInput), P(ViewCalib), vp, vp,
                                                  P(FrameOpts), vp, vp, C.c_int]
    lib.b200_process_silhouettes.argtypes = [vp, vp, vp, C.c_int, C.c_int, P(SilhouetteOp), C.c_int]
    lib.b200_process_silhouettes_async.argtypes = [vp, vp, vp, C.c_int, C.c_int, P(SilhouetteOp), C.c_int]
    lib.b200_composite_depth.argtypes = [vp, vp, vp, C.c_int]
    lib.b200_composite_color.argtypes = [vp, vp, vp, vp, vp, C.c_int, P(C.c_int32), C.c_float]
    lib.b200_composite_instances.argtypes = [vp, vp, vp, C.c_int, P(InstanceLayer), C.c_int, C.c_float, C.c_float]
    lib.b200_mesh_scene.argtypes = [vp, P(Scene), vp, C.c_uint32, P(C.c_uint32)]
    lib.b200_checkpoint_save.argtypes = [vp, P(Scene), P(RenderState), vp, C.c_size_t, P(C.c_size_t)]
    lib.b200_checkpoint_load.argtypes = [vp, P(Scene), P(RenderState), vp, C.c_size_t]
    lib.b200_evaluate_depth.argtypes = [vp, P(EvalParams), vp, C.c_int, vp, vp, vp, P(EvalCallback), C.c_int, P(EvalResult), P(EvalResult), P(EvalSummary)]
    lib.b200_comm_unique_id.argtypes = [C.c_char_p]
    lib.b200_comm_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_char_p, C.c_int, C.c_int, P(vp)]
    lib.b200_comm_destroy.argtypes = [vp]
    lib.b200_comm_destroy.restype = None
    lib.b200_comm_last_error.argtypes = [vp]
    lib.b200_comm_last_error.restype = C.c_char_p
    lib.b200_gather_composite_submit.argtypes = [vp, vp, vp, vp, vp, vp, P(C.c_int32), C.c_float, C.c_float, C.c_int]
    lib.b200_gather_composite_release.argtypes = [vp, vp, C.c_int]
    lib.b200_gather_composite_wait.argtypes = [vp, C.c_int]
    lib.b200_render_view_async.argtypes = [vp, P(Scene), P(RenderState), P(Camera), C.c_int, vp, vp]
    lib.b200_render_view_sync.argtypes = [vp, P(RenderState)]
    lib.b200_render_view_submit.argtypes = [vp, P(Scene), P(RenderState), P(Camera), C.c_int, vp, vp, C.c_int]
    lib.b200_render_view_wait.argtypes = [vp, C.c_int]
    lib.b200_engine_wait_engine.argtypes = [vp, vp]
    lib.b200_volume_restart_async.argtypes = [vp, P(Scene), P(RenderState)]
    lib.b200_group_create.argtypes = [P(GroupConfig), P(vp)]
    lib.b200_group_destroy.argtypes = [vp]
    lib.b200_group_destroy.restype = None
    lib.b200_group_last_error.argtypes = [vp]
    lib.b200_group_last_error.restype = C.c_char_p
    lib.b200_group_slot.argtypes = [vp, C.c_int, P(vp), P(P(Scene)), P(P(RenderState))]
    lib.b200_group_slot_images.argtypes = [vp, C.c_int, P(GroupImages)]
    lib.b200_group_track_start.argtypes = [vp, C.c_int]
    lib.b200_group_frame_async.argtypes = [vp, vp, vp, P(View), P(GroupCar), C.c_int, P(C.c_int32), vp, vp]
    lib.b200_group_sync.argtypes = [vp]
    lib.b200_set_timing.argtypes = [vp, C.c_int]
    lib.b200_set_timing.restype = None
    lib.b200_get_stats.argtypes = [vp, P(FrameStats)]
    lib.b200_get_trace.argtypes = [vp, C.c_char_p, C.c_int]
    lib.b200_selftest_divide.argtypes = [vp, C.c_uint64, C.c_uint64, C.c_float, P(C.c_uint64)]
    lib.b200_diag_set_max_rendering_blocks.argtypes = [vp, C.c_int]
    lib.b200_diag_set_max_rendering_blocks.restype = None
    lib.b200_diag_set_grid_scale.argtypes = [vp, C.c_int]
    lib.b200_diag_set_grid_scale.restype = None
    lib.b200_diag_read_debug.argtypes = [vp, P(C.c_uint64), C.c_int]
    lib.b200_diag_read_spans.argtypes = [vp, P(C.c_uint64), C.c_int]
    lib.b200_diag_read_spans.restype = C.c_int
    lib.b200_diag_last_integrate.argtypes = [vp, P(C.c_int), P(C.c_int)]
    lib.b200_diag_last_integrate.restype = None
    lib.b200_diag_push_decay_snapshot.argtypes = [vp, vp, C.c_int]
    lib.b200_diag_set_frame_index.argtypes = [vp, C.c_int32]
    lib.b200_diag_set_frame_index.restype = None
    _lib = lib
    return lib


_host = None


def host_library():
    """libb200host.so: Matrix4f::inv / operator* in the reference's operation order for hosts without ORUtils."""
    global _host
    if _host is None:
        if not os.path.exists(HOST_LIB_PATH):
            raise RuntimeError(f"{HOST_LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'`")
        h = C.CDLL(HOST_LIB_PATH)
        P = C.POINTER
        h.b200h_mat4_inv.argtypes = [P(C.c_float), P(C.c_float)]
        h.b200h_mat4_mul.argtypes = [P(C.c_float), P(C.c_float), P(C.c_float)]
        h.b200h_mat4_mul.restype = None
        vp = C.c_void_p
        h.b200h_free.argtypes = [vp]; h.b200h_free.restype = None
        h.b200h_read_pfm.argtypes = [C.c_char_p, P(C.c_int), P(C.c_int), P(C.c_int), P(P(C.c_float))]
        h.b200h_read_depth_xml.argtypes = [C.c_char_p, P(C.c_int), P(C.c_int), P(P(C.c_int16))]
        h.b200h_clamp_max_depth_s16.argtypes = [vp, C.c_size_t, C.c_float]; h.b200h_clamp_max_depth_s16.restype = None
        h.b200h_clamp_max_depth_f32.argtypes = [vp, C.c_size_t, C.c_float]; h.b200h_clamp_max_depth_f32.restype = None
        h.b200h_read_mask_txt.argtypes = [C.c_char_p, C.c_int, C.c_int, vp]
        h.b200h_write_obj.argtypes = [C.c_char_p, vp, C.c_uint32, C.c_uint32]
        _host = h
    return _host


def mat_to_c(m):
    """4x4 row-major numpy matrix -> ITM column-major float[16] (m[col*4+row], OR/Matrix.h:23-33)."""
    a = np.asarray(m, dtype=np.float32)
    assert a.shape == (4, 4)
    return f16(*a.T.reshape(-1).tolist())


def c_to_mat(c):
    return np.array(list(c), dtype=np.float32).reshape(4, 4).T.copy()
