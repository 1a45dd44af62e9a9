"""Test infrastructure: ctypes bindings of the CPU oracle (oracle/liboracle.so) and of the
reference-function driver (oracle/_ref/libitmref.so), plus numpy-backed host copies of the scene /
render-state buffers laid out exactly like the device ones (same C structs, host pointers)."""
import ctypes as C
import os
import subprocess

import numpy as np

from dynslam_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_SO = os.path.join(ROOT, "oracle", "liboracle.so")
REF_SO = os.path.join(ROOT, "oracle", "_ref", "libitmref.so")

_oracle = None
_ref = None


def build_oracle():
    subprocess.run(["make", "-C", os.path.join(ROOT, "oracle"), "liboracle.so"], check=True,
                   stdout=subprocess.DEVNULL)


def oracle():
    global _oracle
    if _oracle is not None:
        return _oracle
    srcs = [os.path.join(ROOT, "oracle", f) for f in ("tsdf_oracle.c", "view_oracle.c", "frames_oracle.c", "mesh_oracle.c", "eval_oracle.c")]
    if not os.path.exists(ORACLE_SO) or os.path.getmtime(ORACLE_SO) < max(os.path.getmtime(s) for s in srcs):
        build_oracle()
    L = C.CDLL(ORACLE_SO)
    P, vp = C.POINTER, C.c_void_p
    L.oracle_engine_create.argtypes = [C.c_int, C.c_int, C.c_int]
    L.oracle_engine_create.restype = vp
    L.oracle_engine_destroy.argtypes = [vp]
    L.oracle_engine_destroy.restype = None
    L.oracle_frame_index.argtypes = [vp]
    L.oracle_decayed_block_count.argtypes = [vp]
    L.oracle_decayed_block_count.restype = C.c_long
    L.oracle_queue_size.argtypes = [vp]
    L.oracle_integrated_blocks.argtypes = [vp]
    L.oracle_mesh_scene.argtypes = [P(abi.Scene), vp, C.c_uint32]
    L.oracle_mesh_scene.restype = C.c_uint32
    L.oracle_evaluate_depth.argtypes = [P(abi.EvalParams), vp, C.c_int, vp, vp, vp, P(abi.EvalCallback), C.c_int, P(abi.EvalResult), P(abi.EvalResult),
                                        P(abi.EvalSummary)]
    L.oracle_mat4_inv.argtypes = [P(C.c_float), P(C.c_float)]
    L.oracle_mat4_mul.argtypes = [P(C.c_float), P(C.c_float), P(C.c_float)]
    L.oracle_mat4_mul.restype = None
    L.oracle_reset_scene.argtypes = [vp, P(abi.Scene)]
    L.oracle_reset_scene.restype = None
    L.oracle_allocate_from_depth.argtypes = [vp, P(abi.Scene), P(abi.RenderState), P(abi.View), C.c_int, C.c_int]
    L.oracle_integrate.argtypes = [vp, P(abi.Scene), P(abi.RenderState), P(abi.View), C.c_int]
    L.oracle_integrate.restype = None
    L.oracle_decay.argtypes = [vp, P(abi.Scene), P(abi.RenderState), C.c_int, C.c_int, C.c_int]
    L.oracle_push_snapshot.argtypes = [vp, vp, C.c_int]
    L.oracle_push_snapshot.restype = None
    L.oracle_peek_snapshot.argtypes = [vp, vp, C.c_int]
    L.oracle_set_frame_index.argtypes = [vp, C.c_int]
    L.oracle_set_frame_index.restype = None
    L.oracle_decay_branches.argtypes = [P(C.c_long)]
    L.oracle_decay_branches.restype = None
    L.oracle_find_visible_blocks.argtypes = [P(abi.Scene), P(abi.RenderState), P(abi.Camera)]
    L.oracle_find_visible_blocks.restype = None
    L.oracle_expected_depths.argtypes = [P(abi.Scene), P(abi.RenderState), P(abi.Camera)]
    L.oracle_expected_depths.restype = None
    L.oracle_raycast.argtypes = [P(abi.Scene), P(abi.RenderState), P(C.c_float), P(C.c_float), C.c_int]
    L.oracle_raycast.restype = None
    L.oracle_render_image.argtypes = [P(abi.Scene), P(abi.RenderState), P(abi.Camera), vp, vp, C.c_int, C.c_int]
    L.oracle_render_image.restype = None
    L.oracle_icp_maps.argtypes = [P(abi.Scene), P(abi.RenderState), P(abi.View), vp, vp, C.c_int]
    L.oracle_icp_maps.restype = None
    L.oracle_forward_render.argtypes = [P(abi.Scene), P(abi.RenderState), P(abi.View)]
    L.oracle_forward_render.restype = None
    L.oracle_point_cloud.argtypes = [P(abi.Scene), P(abi.RenderState), P(abi.View), P(C.c_float), C.c_int, vp, vp]
    L.oracle_point_cloud.restype = C.c_uint
    L.oracle_swap_list_in.argtypes = [P(abi.Scene), vp]
    L.oracle_swap_integrate_in.argtypes = [P(abi.Scene), vp, vp, C.c_int]
    L.oracle_swap_integrate_in.restype = None
    L.oracle_swap_out.argtypes = [P(abi.Scene), P(abi.RenderState), vp, vp, vp]
    L.oracle_convert_disparity_to_depth.argtypes = [vp, vp, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float]
    L.oracle_convert_disparity_to_depth.restype = None
    L.oracle_convert_depth_affine_to_float.argtypes = [vp, vp, C.c_int, C.c_int, C.c_float, C.c_float]
    L.oracle_convert_depth_affine_to_float.restype = None
    L.oracle_depth_filtering.argtypes = [vp, vp, C.c_int, C.c_int]
    L.oracle_depth_filtering.restype = None
    L.oracle_compute_normal_and_weights.argtypes = [vp, vp, vp, C.c_int, C.c_int, P(C.c_float)]
    L.oracle_compute_normal_and_weights.restype = None
    L.oracle_update_view.argtypes = [vp, C.c_int, C.c_int, P(abi.ViewCalib), vp, vp, vp, vp]
    L.oracle_update_view.restype = None
    L.oracle_process_silhouettes.argtypes = [vp, vp, C.c_int, C.c_int, P(abi.SilhouetteOp), C.c_int]
    L.oracle_process_silhouettes.restype = None
    L.oracle_composite_depth.argtypes = [vp, vp, C.c_int]
    L.oracle_composite_depth.restype = None
    L.oracle_composite_color.argtypes = [vp, vp, vp, vp, C.c_int, P(C.c_int32), C.c_float]
    L.oracle_composite_color.restype = None
    L.oracle_composite_instances.argtypes = [vp, vp, C.c_int, P(abi.InstanceLayer), C.c_int, C.c_float, C.c_float]
    L.oracle_composite_instances.restype = None
    L.oracle_set_max_rendering_blocks.argtypes = [C.c_int]
    L.oracle_set_max_rendering_blocks.restype = None
    L.oracle_num_threads.restype = C.c_int
    L.oracle_set_threads.argtypes = [C.c_int]
    L.oracle_set_threads.restype = None
    _oracle = L
    return L


def ref_available():
    return os.path.exists(REF_SO)


def ref():
    global _ref
    if _ref is not None:
        return _ref
    L = C.CDLL(REF_SO)
    P, vp = C.POINTER, C.c_void_p
    L.ref_table_sizes.argtypes = [P(C.c_int), P(C.c_int)]
    L.ref_mesh_scene.argtypes = [vp, vp, C.c_long, C.c_float, vp, C.c_uint]
    L.ref_mesh_scene.restype = C.c_uint
    L.ref_mat4_inv.argtypes = [P(C.c_float), P(C.c_float)]
    L.ref_mat4_mul.argtypes = [P(C.c_float), P(C.c_float), P(C.c_float)]
    L.ref_mat4_mul.restype = None
    L.ref_find_block.argtypes = [vp, C.c_int, C.c_int, C.c_int]
    L.ref_mark_image.argtypes = [vp, vp, vp, P(abi.Scene), P(abi.View)]
    L.ref_mark_image.restype = None
    L.ref_block_visible.argtypes = [vp, P(C.c_float), P(C.c_float), C.c_float, C.c_int, C.c_int]
    L.ref_integrate_block.argtypes = [vp, vp, P(abi.Scene), P(abi.View)]
    L.ref_integrate_block.restype = None
    L.ref_project_single_block.argtypes = [vp, P(C.c_float), P(C.c_float), C.c_int, C.c_int, C.c_float,
                                           P(C.c_int), P(C.c_int), P(C.c_float)]
    L.ref_raycast.argtypes = [P(abi.Scene), P(abi.RenderState), P(C.c_float), P(C.c_float)]
    L.ref_raycast.restype = None
    L.ref_shade.argtypes = [P(abi.Scene), P(abi.RenderState), P(abi.Camera), vp, vp, C.c_int]
    L.ref_shade.restype = None
    L.ref_icp.argtypes = [P(abi.Scene), P(abi.RenderState), P(C.c_float), vp, vp]
    L.ref_icp.restype = None
    L.ref_combine_block.argtypes = [vp, vp, C.c_int]
    L.ref_combine_block.restype = None
    L.ref_forward_project_pixel.argtypes = [P(C.c_float), P(C.c_float), P(C.c_float), C.c_int, C.c_int]
    L.ref_view_convert_disparity.argtypes = [vp, vp, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float]
    L.ref_view_convert_disparity.restype = None
    L.ref_view_convert_affine.argtypes = [vp, vp, C.c_int, C.c_int, C.c_float, C.c_float]
    L.ref_view_convert_affine.restype = None
    L.ref_view_filter_pass.argtypes = [vp, vp, C.c_int, C.c_int]
    L.ref_view_filter_pass.restype = None
    L.ref_view_normal_weight.argtypes = [vp, vp, vp, C.c_int, C.c_int, P(C.c_float)]
    L.ref_view_normal_weight.restype = None
    _ref = L
    return L


def fptr(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def vptr(a):
    return C.c_void_p(a.ctypes.data)


class SceneParams:
    def __init__(self, voxelSize=0.05, mu=0.75, maxW=50, vf_min=0.1, vf_max=300.0, stopIntegratingAtMaxW=0):
        self.voxelSize, self.mu, self.maxW = voxelSize, mu, maxW
        self.vf_min, self.vf_max, self.stopIntegratingAtMaxW = vf_min, vf_max, stopIntegratingAtMaxW


class HostVolume:
    """numpy-backed ITMScene + ITMRenderState_VH on the host, for the oracle / reference driver."""

    def __init__(self, numBlocks, numBuckets, excessSize, w, h, params=None, swapping=False):
        p = params or SceneParams()
        self.params = p
        self.numBlocks, self.numBuckets, self.excessSize, self.w, self.h = numBlocks, numBuckets, excessSize, w, h
        n = numBuckets + excessSize
        self.voxels = np.zeros(numBlocks * 512, dtype=abi.VOXEL_DTYPE)
        self.allocationList = np.zeros(numBlocks, dtype=np.int32)
        self.hash = np.zeros(n, dtype=abi.HASH_ENTRY_DTYPE)
        self.excessList = np.zeros(excessSize, dtype=np.int32)
        self.swapStates = np.zeros(n, dtype=np.uint8) if swapping else None
        self.visiblePos = np.zeros((numBlocks, 3), dtype=np.int32)
        self.visType = np.zeros(n, dtype=np.uint8)
        self.minmax = np.zeros((h, w, 2), dtype=np.float32)
        self.raycastResult = np.zeros((h, w, 4), dtype=np.float32)
        self.forwardProjection = np.zeros((h, w, 4), dtype=np.float32)
        self.fwdMissing = np.zeros(h * w, dtype=np.int32)
        self.raycastImage = np.zeros((h, w, 4), dtype=np.uint8)
        self.points = np.zeros((h, w, 4), dtype=np.float32)
        self.normals = np.zeros((h, w, 4), dtype=np.float32)
        s = abi.Scene()
        s.d_voxels, s.d_allocationList = self.voxels.ctypes.data, self.allocationList.ctypes.data
        s.d_hash, s.d_excessList = self.hash.ctypes.data, self.excessList.ctypes.data
        s.d_swapStates = self.swapStates.ctypes.data if swapping else None
        s.numBlocks, s.numBuckets, s.excessSize = numBlocks, numBuckets, excessSize
        s.voxelSize, s.mu, s.maxW = p.voxelSize, p.mu, p.maxW
        s.viewFrustum_min, s.viewFrustum_max = p.vf_min, p.vf_max
        s.stopIntegratingAtMaxW, s.useSwapping = p.stopIntegratingAtMaxW, int(swapping)
        self.scene = s
        r = abi.RenderState()
        r.d_visibleBlockPositions, r.d_entriesVisibleType = self.visiblePos.ctypes.data, self.visType.ctypes.data
        r.d_minmax, r.d_raycastResult = self.minmax.ctypes.data, self.raycastResult.ctypes.data
        r.d_forwardProjection, r.d_fwdProjMissingPoints = self.forwardProjection.ctypes.data, self.fwdMissing.ctypes.data
        r.d_raycastImage = self.raycastImage.ctypes.data
        r.img_w, r.img_h = w, h
        self.rs = r
        self.engine = oracle().oracle_engine_create(numBlocks, numBuckets, excessSize)
        oracle().oracle_reset_scene(self.engine, C.byref(s))

    def __del__(self):
        try:
            oracle().oracle_engine_destroy(self.engine)
        except Exception:
            pass

    def state(self):
        """dict of every piece of persistent state (copies), for byte-exact comparisons."""
        n = self.rs.noVisibleBlocks
        return dict(hash=self.hash.copy(), voxels=self.voxels.copy(), allocationList=self.allocationList.copy(),
                    excessList=self.excessList.copy(), visType=self.visType.copy(),
                    visiblePos=self.visiblePos[:max(n, 0)].copy(), noVisibleBlocks=n,
                    lastFreeBlockId=self.scene.lastFreeBlockId,
                    lastFreeExcessListId=self.scene.lastFreeExcessListId)


def make_view(depth, rgb, M_d, proj, M_rgb=None, depthWeighting=0, requiresFullRendering=1, inv=None, proj_rgb=None):
    """Host-pointer b200_view. Keeps references to the arrays on the returned object. M_rgb / proj_rgb default to the depth
    camera's."""
    L = oracle()
    depth = np.ascontiguousarray(depth, dtype=np.float32)
    rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
    v = abi.View()
    v.d_depth, v.d_rgb = depth.ctypes.data, rgb.ctypes.data
    v.depth_h, v.depth_w = depth.shape
    v.rgb_h, v.rgb_w = rgb.shape[:2]
    v.M_d = abi.mat_to_c(M_d)
    invc = abi.f16()
    L.oracle_mat4_inv(v.M_d, invc)
    v.invM_d = invc
    v.M_rgb = abi.mat_to_c(M_rgb if M_rgb is not None else M_d)
    v.proj_d = abi.f4(*[float(x) for x in proj])
    v.proj_rgb = abi.f4(*[float(x) for x in (proj_rgb if proj_rgb is not None else proj)])
    v.depthWeighting, v.requiresFullRendering = depthWeighting, int(requiresFullRendering)
    v._keep = (depth, rgb)
    return v


def make_camera(M, proj):
    L = oracle()
    c = abi.Camera()
    c.M = abi.mat_to_c(M)
    inv = abi.f16()
    L.oracle_mat4_inv(c.M, inv)
    c.invM = inv
    c.proj = abi.f4(*[float(x) for x in proj])
    return c
