"""Pins the oracle (oracle/tsdf_oracle.c) against the reference's own DeviceAgnostic functions
(oracle/_ref/libitmref.so, compiled from the reference's source by oracle/build_ref.sh): every stage bit-exact on a short
KITTI-shaped synthetic sequence. CPU only. The reference's outputs are stored as digests (tests/refpins.py); where
oracle/_ref is built the reference also runs live."""
import ctypes as C

import numpy as np
import pytest

from dynslam_b200 import abi, synth
from tests import hostlib as H
from tests import refpins


def _ref_or_none():
    return H.ref() if H.ref_available() else None

NB, NE = 0x100000, 0x80000  # compile-time sizes of the reference (Utils/ITMLibDefines.h:42-53)
SCALE = 0.25


def _hooks():
    L = H.oracle()
    L.oracle_mark_only.argtypes = [C.c_void_p, C.POINTER(abi.Scene), C.c_void_p, C.POINTER(abi.View)]
    L.oracle_mark_only.restype = None
    L.oracle_alloc_type.argtypes = [C.c_void_p]
    L.oracle_alloc_type.restype = C.POINTER(C.c_uint8)
    L.oracle_block_coords.argtypes = [C.c_void_p]
    L.oracle_block_coords.restype = C.POINTER(C.c_int16)
    L.oracle_block_visible.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_float, C.c_int, C.c_int]
    L.oracle_project_single_block.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_int, C.c_int,
                                              C.c_float, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_float)]
    L.oracle_combine_block.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    L.oracle_combine_block.restype = None
    return L


@pytest.fixture(scope="module")
def seq():
    """Runs 6 frames through the oracle, keeping per-frame views and pre-integration voxel copies."""
    L = _hooks()
    R = _ref_or_none()
    if R:
        nb, ne = C.c_int(), C.c_int()
        assert R.ref_table_sizes(C.byref(nb), C.byref(ne)) == 20
        assert (nb.value, ne.value) == (NB, NE)
    scene = synth.StreetScene(seed=6, length_m=80.0)
    w, h = int(round(synth.KITTI_W * SCALE)), int(round(synth.KITTI_H * SCALE))
    vol = H.HostVolume(20000, NB, NE, w, h, H.SceneParams(voxelSize=0.05, mu=0.75, maxW=50))
    frames = []
    for f in range(6):
        depth, rgb, M, proj = synth.kitti_frame(scene, f * 3, scale=SCALE)
        view = H.make_view(depth, rgb, M, proj, depthWeighting=(f % 2))
        # stage pin 1: marking, on the table state before this frame's allocation
        vis_o = vol.visType.copy()
        L.oracle_mark_only(vol.engine, C.byref(vol.scene), H.vptr(vis_o), C.byref(view))
        n = NB + NE
        at_o = np.ctypeslib.as_array(L.oracle_alloc_type(vol.engine), shape=(n,)).copy()
        bc_o = np.ctypeslib.as_array(L.oracle_block_coords(vol.engine), shape=(n * 4,)).copy()
        req = np.nonzero(at_o)[0]
        ref = None
        if R:
            vis_r = vol.visType.copy()
            at_r = np.zeros(n, dtype=np.uint8)
            bc_r = np.zeros(n * 4, dtype=np.int16)
            R.ref_mark_image(H.vptr(at_r), H.vptr(vis_r), H.vptr(bc_r), C.byref(vol.scene), C.byref(view))
            assert np.array_equal(at_o, at_r)
            assert np.array_equal(vis_o, vis_r)
            assert np.array_equal(bc_o.reshape(-1, 4)[req], bc_r.reshape(-1, 4)[req])
            ref = at_r.tobytes() + vis_r.tobytes() + bc_r.reshape(-1, 4)[req].tobytes()
        refpins.check(f"oracle_vs_ref/mark/frame{f}", at_o.tobytes() + vis_o.tobytes() + bc_o.reshape(-1, 4)[req].tobytes(), ref)
        if f == 0:
            assert len(req) > 500
        rc = L.oracle_allocate_from_depth(vol.engine, C.byref(vol.scene), C.byref(vol.rs), C.byref(view), 0, 0)
        assert rc == 0
        pre = vol.voxels.copy()
        L.oracle_integrate(vol.engine, C.byref(vol.scene), C.byref(vol.rs), C.byref(view), 0)
        frames.append((view, pre, vol.voxels.copy(), vol.visiblePos[:vol.rs.noVisibleBlocks].copy()))
    return vol, frames


def test_mat4_inv_and_mul():
    L, R = H.oracle(), _ref_or_none()
    rng = np.random.RandomState(0)
    ours, refs = [], []
    for i in range(50):
        M = synth.kitti_pose(i * 7).astype(np.float32)
        M[:3, 3] += rng.randn(3).astype(np.float32)
        c = abi.mat_to_c(M)
        a, b = abi.f16(), abi.f16()
        assert L.oracle_mat4_inv(c, a) == 1
        m1, m2 = abi.f16(), abi.f16()
        L.oracle_mat4_mul(c, a, m1)
        ours += [bytes(a), bytes(m1)]
        if R:
            assert R.ref_mat4_inv(c, b) == 1
            R.ref_mat4_mul(c, a, m2)
            refs += [bytes(b), bytes(m2)]
    refpins.check("oracle_vs_ref/mat4_inv_mul", b"".join(ours), b"".join(refs) if R else None)


def test_integrate_blocks_bit_exact(seq):
    vol, frames = seq
    R = _ref_or_none()
    rng = np.random.RandomState(1)
    live = np.nonzero(vol.hash["ptr"] >= 0)[0]
    ptr_of = {tuple(int(t) for t in vol.hash[i]["pos"]): int(vol.hash[i]["ptr"]) for i in live}
    checked = changed = 0
    ours, refs = [], []
    for view, pre, post, vis in frames:
        pick = rng.choice(len(vis), size=min(400, len(vis)), replace=False)
        for i in pick:
            x, y, z = (int(t) for t in vis[i])
            # the final table may have moved the block (no decay here, so ptr is stable)
            ptr = ptr_of.get((x, y, z), -1)
            if R:
                idx = R.ref_find_block(H.vptr(vol.hash), x, y, z)
                assert ptr == (int(vol.hash[idx]["ptr"]) if idx >= 0 else -1)
            if ptr < 0:
                continue
            want = post[ptr * 512:(ptr + 1) * 512]
            ours.append(want.tobytes())
            if R:
                blk = pre[ptr * 512:(ptr + 1) * 512].copy()
                pos = np.array([x, y, z], dtype=np.int16)
                R.ref_integrate_block(H.vptr(blk), H.vptr(pos), C.byref(vol.scene), C.byref(view))
                assert blk.tobytes() == want.tobytes()
                refs.append(blk.tobytes())
            checked += 1
            changed += int(want.tobytes() != pre[ptr * 512:(ptr + 1) * 512].tobytes())
    assert checked > 1000 and changed > 300
    refpins.check("oracle_vs_ref/integrate_blocks", b"".join(ours), b"".join(refs) if R else None)


def test_integrate_blocks_approximate_and_colour_camera_bit_exact():
    """the two integration branches the default views never take: approximate integration (requiresFullRendering = false: only
    voxels with w_depth == 0 are updated) and a colour camera of its own (M_rgb, proj_rgb and an RGB image size that differ from
    the depth camera's: colours are re-projected). Frame 0 fills the volume with the default view, frames 1-3 use the branches."""
    L, R = H.oracle(), _ref_or_none()
    scene = synth.StreetScene(seed=6, length_m=80.0)
    w, h = int(round(synth.KITTI_W * SCALE)), int(round(synth.KITTI_H * SCALE))
    vol = H.HostVolume(20000, NB, NE, w, h, H.SceneParams(voxelSize=0.05, mu=0.75, maxW=50))
    offset = np.array([[0.9998, -0.0050, 0.0200, -0.54], [0.0054, 0.9999, -0.0100, 0.05], [-0.0199, 0.0101, 0.9998, 0.02],
                       [0, 0, 0, 1]], dtype=np.float64)
    proj_rgb = np.array([707.0912 * 0.3, 707.0912 * 0.3, 601.8873 * 0.3 + 4.0, 183.1104 * 0.3 - 2.5], dtype=np.float32)
    rng = np.random.RandomState(5)
    ours, refs = [], []
    kept = written = recoloured = 0
    for f, (approx, own_rgb) in enumerate(((False, False), (True, False), (False, True), (True, True))):
        depth, rgb, M, proj = synth.kitti_frame(scene, f * 2, scale=SCALE)
        M_rgb, pr = None, None
        if own_rgb:
            M_rgb, pr = (offset @ M.astype(np.float64)).astype(np.float32), proj_rgb
            rgb = scene.render(M_rgb, 373, 113, *[float(x) for x in pr])[1]
        view = H.make_view(depth, rgb, M, proj, M_rgb=M_rgb, proj_rgb=pr, requiresFullRendering=int(not approx))
        assert L.oracle_allocate_from_depth(vol.engine, C.byref(vol.scene), C.byref(vol.rs), C.byref(view), 0, 0) == 0
        pre = vol.voxels.copy()
        L.oracle_integrate(vol.engine, C.byref(vol.scene), C.byref(vol.rs), C.byref(view), 0)
        if f == 0:
            continue
        vis = vol.visiblePos[:vol.rs.noVisibleBlocks]
        for i in rng.choice(len(vis), size=min(300, len(vis)), replace=False):
            x, y, z = (int(t) for t in vis[i])
            idx = L.oracle_find_block(H.vptr(vol.hash), NB, x, y, z)
            if idx < 0:
                continue
            ptr = int(vol.hash[idx]["ptr"])
            a, b = pre[ptr * 512:(ptr + 1) * 512], vol.voxels[ptr * 512:(ptr + 1) * 512]
            ours.append(b.tobytes())
            if approx:
                kept += int(((a["w_depth"] != 0) & (a["w_depth"] == b["w_depth"])).sum())
                written += int(((a["w_depth"] == 0) & (b["w_depth"] != 0)).sum())
            if own_rgb:
                recoloured += int((a["clr"] != b["clr"]).any(axis=1).sum())
            if R:
                blk = a.copy()
                pos = np.array([x, y, z], dtype=np.int16)
                R.ref_integrate_block(H.vptr(blk), H.vptr(pos), C.byref(vol.scene), C.byref(view))
                assert blk.tobytes() == b.tobytes(), (f, x, y, z)
                refs.append(blk.tobytes())
    assert kept > 10000 and written > 1000 and recoloured > 10000, (kept, written, recoloured)
    refpins.check("oracle_vs_ref/integrate_blocks_approx_colour_camera", b"".join(ours), b"".join(refs) if R else None)


def test_block_visibility_and_projection(seq):
    vol, frames = seq
    L, R = _hooks(), _ref_or_none()
    used = np.nonzero(vol.hash["ptr"] >= 0)[0]
    rng = np.random.RandomState(2)
    w, h = vol.w, vol.h
    n_vis = n_proj = 0
    ours, refs = [], []

    def rec(vis, o, ul, lr, zr):
        return np.array([vis, o] + (list(ul) + list(lr) if o else []), np.int32).tobytes() + (bytes(zr) if o else b"")

    for view, _, _, _ in frames[::2]:
        for i in rng.choice(used, size=600, replace=False):
            pos = vol.hash[i]["pos"].astype(np.int16).copy()
            a = L.oracle_block_visible(H.vptr(pos), view.M_d, view.proj_d, vol.scene.voxelSize, w, h)
            n_vis += a
            ul1, lr1, zr1 = (C.c_int * 2)(), (C.c_int * 2)(), (C.c_float * 2)()
            o1 = L.oracle_project_single_block(H.vptr(pos), view.M_d, view.proj_d, w, h, vol.scene.voxelSize, ul1, lr1, zr1)
            ours.append(rec(a, o1, ul1, lr1, zr1))
            if o1:
                n_proj += 1
            if R:
                b = R.ref_block_visible(H.vptr(pos), view.M_d, view.proj_d, vol.scene.voxelSize, w, h)
                ul2, lr2, zr2 = (C.c_int * 2)(), (C.c_int * 2)(), (C.c_float * 2)()
                o2 = R.ref_project_single_block(H.vptr(pos), view.M_d, view.proj_d, w, h, vol.scene.voxelSize, ul2, lr2, zr2)
                refs.append(rec(b, o2, ul2, lr2, zr2))
                assert ours[-1] == refs[-1]
    assert n_vis > 100 and n_proj > 100
    refpins.check("oracle_vs_ref/block_visibility_projection", b"".join(ours), b"".join(refs) if R else None)


def test_raycast_shading_icp_bit_exact(seq):
    vol, frames = seq
    L, R = H.oracle(), _ref_or_none()
    view = frames[-1][0]
    cam = abi.Camera()
    cam.M, cam.invM, cam.proj = view.M_d, view.invM_d, view.proj_d
    L.oracle_expected_depths(C.byref(vol.scene), C.byref(vol.rs), C.byref(cam))
    mm = vol.minmax.copy()
    assert (mm[..., 0] < mm[..., 1]).sum() > 200  # some 1/8-res cells are covered
    # raycast
    L.oracle_raycast(C.byref(vol.scene), C.byref(vol.rs), view.invM_d, view.proj_d, 0)
    ray_o = vol.raycastResult.copy()
    ray_r = None
    if R:
        vol.raycastResult[:] = 0
        R.ref_raycast(C.byref(vol.scene), C.byref(vol.rs), view.invM_d, view.proj_d)
        ray_r = vol.raycastResult.tobytes()
        assert ray_o.tobytes() == ray_r
    refpins.check("oracle_vs_ref/raycast", ray_o.tobytes(), ray_r)
    assert (ray_o[..., 3] > 0).mean() > 0.3
    # all five render types
    for t in range(5):
        oc = np.zeros((vol.h, vol.w, 4), dtype=np.uint8)
        of = np.zeros((vol.h, vol.w), dtype=np.float32)
        L.oracle_render_image(C.byref(vol.scene), C.byref(vol.rs), C.byref(cam), H.vptr(oc), H.vptr(of), t, 0)
        # drawPixelNormal leaves alpha untouched (DA/ITMVisualisationEngine.h:283-288)
        rgb = (lambda c: c[..., :3]) if t == abi.RENDER_COLOUR_FROM_NORMAL else (lambda c: c)
        ref = None
        if R:
            rc_ = np.zeros_like(oc)
            rf = np.zeros_like(of)
            R.ref_shade(C.byref(vol.scene), C.byref(vol.rs), C.byref(cam), H.vptr(rc_), H.vptr(rf), t)
            assert rgb(oc).tobytes() == rgb(rc_).tobytes(), t
            assert of.tobytes() == rf.tobytes()
            ref = rgb(rc_).tobytes() + rf.tobytes()
        refpins.check(f"oracle_vs_ref/shade/type{t}", rgb(oc).tobytes() + of.tobytes(), ref)
        if t == abi.RENDER_DEPTH_MAP:
            assert (of > 0).mean() > 0.3
        else:
            assert oc[..., :3].any()
    # ICP maps
    L.oracle_icp_maps(C.byref(vol.scene), C.byref(vol.rs), C.byref(view), H.vptr(vol.points), H.vptr(vol.normals), 0)
    img_o, p_o, n_o = vol.raycastImage.copy(), vol.points.copy(), vol.normals.copy()
    ref = None
    if R:
        vol.raycastImage[:] = 0
        p_r, n_r = np.zeros_like(p_o), np.zeros_like(n_o)
        R.ref_icp(C.byref(vol.scene), C.byref(vol.rs), view.invM_d, H.vptr(p_r), H.vptr(n_r))
        assert img_o.tobytes() == vol.raycastImage.tobytes()
        assert p_o.tobytes() == p_r.tobytes() and n_o.tobytes() == n_r.tobytes()
        ref = vol.raycastImage.tobytes() + p_r.tobytes() + n_r.tobytes()
    refpins.check("oracle_vs_ref/icp_maps", img_o.tobytes() + p_o.tobytes() + n_o.tobytes(), ref)
    assert (p_o[..., 3] > 0).mean() > 0.2


def test_combine_voxels(seq):
    vol, frames = seq
    L, R = _hooks(), _ref_or_none()
    used = np.nonzero(vol.hash["ptr"] >= 0)[0][:64]
    ours, refs = [], []
    for k, i in enumerate(used[:-1]):
        a = vol.voxels[int(vol.hash[i]["ptr"]) * 512:][:512].copy()
        b = vol.voxels[int(vol.hash[used[k + 1]]["ptr"]) * 512:][:512].copy()
        d1, d2 = b.copy(), b.copy()
        L.oracle_combine_block(H.vptr(a), H.vptr(d1), 50)
        ours.append(d1.tobytes())
        if R:
            R.ref_combine_block(H.vptr(a), H.vptr(d2), 50)
            assert d1.tobytes() == d2.tobytes()
            refs.append(d2.tobytes())
    refpins.check("oracle_vs_ref/combine_voxels", b"".join(ours), b"".join(refs) if R else None)


# ---- view builder (oracle/view_oracle.c vs DeviceAgnostic/ITMViewBuilder.h) ---------------------------
def _vb_inputs():
    from tests import viewlib
    raw, _ = viewlib.raw_kitti_frame(scale=0.25)
    return [raw, viewlib.raw_noise_frame()]


def test_view_convert_bit_exact():
    L, R = H.oracle(), _ref_or_none()
    for k, raw in enumerate(_vb_inputs()):
        h, w = raw.shape
        a, b = np.zeros((h, w), np.float32), np.zeros((h, w), np.float32)
        L.oracle_convert_depth_affine_to_float(H.vptr(a), H.vptr(raw), w, h, 1.0 / 1000.0, 0.0)
        if R:
            R.ref_view_convert_affine(H.vptr(b), H.vptr(raw), w, h, 1.0 / 1000.0, 0.0)
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
        refpins.check(f"oracle_vs_ref/view_convert_affine/input{k}", a.tobytes(), b.tobytes() if R else None)
        assert (a == -1.0).any() and (a > 0).any()
        # Kinect disparity trafo (Objects/ITMDisparityCalib.h:25-26) with the calib-file style parameters
        disp = (raw // 4).astype(np.int16)
        disp[0, :5] = 1135                                   # disparity_tmp == 0 -> depth 0 -> -1
        L.oracle_convert_disparity_to_depth(H.vptr(a), H.vptr(disp), w, h, 1135.09, 0.0819141, 573.71)
        if R:
            R.ref_view_convert_disparity(H.vptr(b), H.vptr(disp), w, h, 1135.09, 0.0819141, 573.71)
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
        refpins.check(f"oracle_vs_ref/view_convert_disparity/input{k}", a.tobytes(), b.tobytes() if R else None)


def test_view_filter_and_update_view_bit_exact():
    L, R = H.oracle(), _ref_or_none()
    for k, raw in enumerate(_vb_inputs()):
        h, w = raw.shape
        d0 = np.zeros((h, w), np.float32)
        L.oracle_convert_depth_affine_to_float(H.vptr(d0), H.vptr(raw), w, h, 1.0 / 1000.0, 0.0)   # pinned in the test above
        # one pass: the target's 2-pixel border must stay what it was
        a, b = np.full((h, w), 7.0, np.float32), np.full((h, w), 7.0, np.float32)
        L.oracle_depth_filtering(H.vptr(a), H.vptr(d0), w, h)
        if R:
            R.ref_view_filter_pass(H.vptr(b), H.vptr(d0), w, h)
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
        refpins.check(f"oracle_vs_ref/view_filter_pass/input{k}", a.tobytes(), b.tobytes() if R else None)
        assert (a[:2] == 7.0).all() and (a[:, -2:] == 7.0).all()
        calib = abi.ViewCalib()
        calib.trafoType, calib.useBilateralFilter, calib.modelSensorNoise = 1, 1, 1
        calib.params = (C.c_float * 2)(1.0 / 1000.0, 0.0)
        calib.intrinsics_d = (C.c_float * 4)(707.0912, 707.0912, w / 2.0, h / 2.0)
        depth_o, float_o = np.zeros((h, w), np.float32), np.zeros((h, w), np.float32)
        nrm_o, sig_o = np.zeros((h, w, 4), np.float32), np.zeros((h, w), np.float32)
        L.oracle_update_view(H.vptr(raw), w, h, C.byref(calib), H.vptr(depth_o), H.vptr(float_o), H.vptr(nrm_o), H.vptr(sig_o))
        assert (depth_o[:2] == 0).all() and (depth_o[-2:] == 0).all() and (depth_o[:, :2] == 0).all()   # floatImage's border
        ref = None
        if R:
            # UpdateView: the reference's own sequence (ITMViewBuilder_CUDA.cu:64-79) composed from its functions
            depth_r, float_r = d0.copy(), np.zeros((h, w), np.float32)
            for _ in range(2):
                R.ref_view_filter_pass(H.vptr(float_r), H.vptr(depth_r), w, h)
                R.ref_view_filter_pass(H.vptr(depth_r), H.vptr(float_r), w, h)
            R.ref_view_filter_pass(H.vptr(float_r), H.vptr(depth_r), w, h)
            assert np.array_equal(depth_o.view(np.uint32), float_r.view(np.uint32))
            nrm_r, sig_r = np.zeros((h, w, 4), np.float32), np.zeros((h, w), np.float32)
            R.ref_view_normal_weight(H.vptr(float_r), H.vptr(nrm_r), H.vptr(sig_r), w, h, calib.intrinsics_d)
            assert np.array_equal(nrm_o.view(np.uint32), nrm_r.view(np.uint32))
            assert np.array_equal(sig_o.view(np.uint32), sig_r.view(np.uint32))
            ref = float_r.tobytes() + nrm_r.tobytes() + sig_r.tobytes()
        refpins.check(f"oracle_vs_ref/update_view/input{k}", depth_o.tobytes() + nrm_o.tobytes() + sig_o.tobytes(), ref)
        assert (nrm_o[..., 3] == 1.0).sum() > 0.3 * w * h


def test_mesh_oracle_equals_reference_cpu_engine():
    """Meshing (SURVEY 8(f) rank 4): oracle/mesh_oracle.c against the reference's OWN serial engine,
    ITMMeshingEngine_CPU<ITMVoxel, ITMVoxelBlockHash>::MeshScene (Engine/DeviceSpecific/CPU/ITMMeshingEngine_CPU.cpp:19-80, live
    code, compiled from its source into oracle/_ref/libitmref.so), on a map fused by the oracle: same triangle count, every
    vertex and colour bit for bit, same order."""
    from dynslam_b200 import abi, synth
    from tests import parity as P
    L, R = H.oracle(), _ref_or_none()
    cfg = P.Cfg(scale=0.25, frames=4, numBlocks=16384, numBuckets=0x100000, excessSize=0x80000)    # the reference's compile-time table size
    w, h = int(round(synth.KITTI_W * cfg.scale)), int(round(synth.KITTI_H * cfg.scale))
    vol = H.HostVolume(cfg.numBlocks, cfg.numBuckets, cfg.excessSize, w, h)
    for depth, rgb, M, proj in P.frames_of(cfg):
        hv = H.make_view(depth, rgb, M, proj)
        assert L.oracle_allocate_from_depth(vol.engine, C.byref(vol.scene), C.byref(vol.rs), C.byref(hv), 0, 0) == 0
        L.oracle_integrate(vol.engine, C.byref(vol.scene), C.byref(vol.rs), C.byref(hv), 0)
    nmax = cfg.numBlocks * 512 // 16
    a = np.zeros(nmax, dtype=abi.TRIANGLE_DTYPE)
    b = np.zeros(nmax, dtype=abi.TRIANGLE_DTYPE)
    na = L.oracle_mesh_scene(C.byref(vol.scene), H.vptr(a), nmax)
    assert na > 20000
    ref = None
    if R:
        nb = R.ref_mesh_scene(H.vptr(vol.hash), H.vptr(vol.voxels), cfg.numBlocks, C.c_float(cfg.voxelSize), H.vptr(b), nmax)
        assert na == nb
        assert a[:na].tobytes() == b[:na].tobytes()
        ref = np.int64(nb).tobytes() + b[:nb].tobytes()
    refpins.check("oracle_vs_ref/mesh_scene", np.int64(na).tobytes() + a[:na].tobytes(), ref)
    # colours are really interpolated from the volume, vertices lie inside the fused region
    assert a["c0"][:na].max() > 0.2 and np.isfinite(a["p0"][:na]).all()
