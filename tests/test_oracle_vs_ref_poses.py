"""Pins the oracle (oracle/tsdf_oracle.c) against the reference's own DeviceAgnostic functions on the general-pose trajectories
of tests/poselib.py: reversing, turning in place, pitched and rolled, upside down, 1 m above the ground and kilometres from
the origin, with fx != fy and principal points off the image centre. Block coordinates of every sign, rays marching in every
direction. Same pattern as tests/test_oracle_vs_ref.py: marking, integrated blocks, block visibility and projection, raycast,
the five shade types and the ICP maps, bit for bit, at the reference's compile-time table sizes. The reference's outputs are
stored as digests (tests/refpins.py, keys oracle_vs_ref/poses/<trajectory>/...); where oracle/_ref is built it also runs live.

The fused surface is also checked against the analytic scene it was rendered from, in float64 (test_surface_distance)."""
import ctypes as C

import numpy as np
import pytest

from dynslam_b200 import abi
from tests import hostlib as H
from tests import poselib as PL
from tests import refpins
from tests.test_oracle_vs_ref import NB, NE, _hooks, _ref_or_none

_runs = {}


def _fuse(name):
    """every frame of the trajectory through the oracle, marking pinned on the way; per frame the view and the voxels before and
    after integration"""
    if name in _runs:
        return _runs[name]
    L, R, t = _hooks(), _ref_or_none(), PL.get(name)
    if R:
        nb, ne = C.c_int(), C.c_int()
        assert R.ref_table_sizes(C.byref(nb), C.byref(ne)) == 20 and (nb.value, ne.value) == (NB, NE)
    vol = H.HostVolume(20000, NB, NE, t.w, t.h, H.SceneParams(voxelSize=PL.VOXEL, mu=t.mu, maxW=50))
    frames, marks, refs = [], [], []
    n = NB + NE
    for f, (depth, rgb, M, proj) in enumerate(t.frames()):
        view = H.make_view(depth, rgb, M, proj, depthWeighting=(f % 2))
        vis_o = vol.visType.copy()
        L.oracle_mark_only(vol.engine, C.byref(vol.scene), H.vptr(vis_o), C.byref(view))
        at_o = np.ctypeslib.as_array(L.oracle_alloc_type(vol.engine), shape=(n,)).copy()
        bc_o = np.ctypeslib.as_array(L.oracle_block_coords(vol.engine), shape=(n * 4,)).copy()
        req = np.nonzero(at_o)[0]
        marks.append(at_o.tobytes() + vis_o.tobytes() + bc_o.reshape(-1, 4)[req].tobytes())
        if R:
            vis_r, at_r, bc_r = vol.visType.copy(), np.zeros(n, dtype=np.uint8), np.zeros(n * 4, dtype=np.int16)
            R.ref_mark_image(H.vptr(at_r), H.vptr(vis_r), H.vptr(bc_r), C.byref(vol.scene), C.byref(view))
            refs.append(at_r.tobytes() + vis_r.tobytes() + bc_r.reshape(-1, 4)[req].tobytes())
            assert marks[-1] == refs[-1], (name, f)
        assert L.oracle_allocate_from_depth(vol.engine, C.byref(vol.scene), C.byref(vol.rs), C.byref(view), 0, 0) == 0
        pre = vol.voxels.copy()
        L.oracle_integrate(vol.engine, C.byref(vol.scene), C.byref(vol.rs), C.byref(view), 0)
        frames.append((view, pre, vol.voxels.copy(), vol.visiblePos[:vol.rs.noVisibleBlocks].copy()))
    _runs[name] = (t, vol, frames, b"".join(marks), b"".join(refs) if R else None)
    return _runs[name]


@pytest.mark.parametrize("name", PL.NAMES)
def test_marking(name):
    t, vol, frames, ours, ref = _fuse(name)
    refpins.check(f"oracle_vs_ref/poses/{name}/mark", ours, ref)
    live = vol.hash[vol.hash["ptr"] >= 0]["pos"]
    assert len(live) > 80
    if name in ("reverse", "far"):
        assert (live[:, 0] < 0).all() and (live[:, 2] < 0).all()          # every block at negative x and z
    if name == "far":
        assert np.abs(live).min(axis=0).min() > 1000                       # block coordinates in the thousands
    if name == "turn_in_place":
        assert ((live < 0).any(axis=0) & (live > 0).any(axis=0)).all()     # both signs on every axis


@pytest.mark.parametrize("name", PL.NAMES)
def test_integrate_blocks(name):
    t, vol, frames, _, _ = _fuse(name)
    L, R = H.oracle(), _ref_or_none()
    rng = np.random.RandomState(1)
    ours, refs = [], []
    changed = 0
    for view, pre, post, vis in frames:
        for i in rng.choice(len(vis), size=min(200, len(vis)), replace=False):
            x, y, z = (int(v) for v in vis[i])
            idx = L.oracle_find_block(H.vptr(vol.hash), NB, x, y, z)      # no decay here: a block's ptr never changes
            if idx < 0:
                continue
            ptr = int(vol.hash[idx]["ptr"])
            want = post[ptr * 512:(ptr + 1) * 512]
            ours.append(want.tobytes())
            changed += int(want.tobytes() != pre[ptr * 512:(ptr + 1) * 512].tobytes())
            if R:
                blk = pre[ptr * 512:(ptr + 1) * 512].copy()
                R.ref_integrate_block(H.vptr(blk), H.vptr(np.array([x, y, z], dtype=np.int16)), C.byref(vol.scene), C.byref(view))
                assert blk.tobytes() == want.tobytes(), (name, x, y, z)
                refs.append(blk.tobytes())
    assert changed > 100, changed
    refpins.check(f"oracle_vs_ref/poses/{name}/integrate_blocks", b"".join(ours), b"".join(refs) if R else None)


def _views(t, frames):
    """(invM, M, proj) of every frame and of the last camera turned 90 and 180 degrees"""
    out = [(v.M_d, v.proj_d) for v, _, _, _ in frames]
    for deg in (90.0, 180.0):
        c = H.make_camera(t.turned(deg), t.proj)
        out.append((c.M, c.proj))
    return out


@pytest.mark.parametrize("name", PL.NAMES)
def test_block_visibility_and_projection(name):
    t, vol, frames, _, _ = _fuse(name)
    L, R = _hooks(), _ref_or_none()
    used = np.nonzero(vol.hash["ptr"] >= 0)[0]
    rng = np.random.RandomState(2)
    n_vis = n_proj = 0
    ours, refs = [], []

    def rec(vis, o, ul, lr, zr):
        return np.array([vis, o] + (list(ul) + list(lr) if o else []), np.int32).tobytes() + (bytes(zr) if o else b"")

    for M, proj in _views(t, frames):
        for i in rng.choice(used, size=min(300, len(used)), replace=False):
            pos = vol.hash[i]["pos"].astype(np.int16).copy()
            a = L.oracle_block_visible(H.vptr(pos), M, proj, vol.scene.voxelSize, t.w, t.h)
            ul1, lr1, zr1 = (C.c_int * 2)(), (C.c_int * 2)(), (C.c_float * 2)()
            o1 = L.oracle_project_single_block(H.vptr(pos), M, proj, t.w, t.h, vol.scene.voxelSize, ul1, lr1, zr1)
            ours.append(rec(a, o1, ul1, lr1, zr1))
            n_vis, n_proj = n_vis + a, n_proj + bool(o1)
            if R:
                b = R.ref_block_visible(H.vptr(pos), M, proj, vol.scene.voxelSize, t.w, t.h)
                ul2, lr2, zr2 = (C.c_int * 2)(), (C.c_int * 2)(), (C.c_float * 2)()
                o2 = R.ref_project_single_block(H.vptr(pos), M, proj, t.w, t.h, vol.scene.voxelSize, ul2, lr2, zr2)
                refs.append(rec(b, o2, ul2, lr2, zr2))
                assert ours[-1] == refs[-1], (name, tuple(pos))
    assert n_vis > 100 and n_proj > 100, (n_vis, n_proj)
    refpins.check(f"oracle_vs_ref/poses/{name}/block_visibility_projection", b"".join(ours), b"".join(refs) if R else None)


@pytest.mark.parametrize("name", PL.NAMES)
def test_raycast_shading_icp(name):
    """at the last frame's pose (the allocation's list) and from the last camera turned 35 degrees (FindVisibleBlocks' list):
    expected depths, raycast, all five render types, and the ICP maps at the last frame's pose"""
    t, vol, frames, _, _ = _fuse(name)
    L, R = H.oracle(), _ref_or_none()
    view = frames[-1][0]
    last = abi.Camera()
    last.M, last.invM, last.proj = view.M_d, view.invM_d, view.proj_d
    ours, refs = [], []
    for k, cam in enumerate((last, H.make_camera(t.turned(35.0), t.proj))):
        if k:
            L.oracle_find_visible_blocks(C.byref(vol.scene), C.byref(vol.rs), C.byref(cam))
        L.oracle_expected_depths(C.byref(vol.scene), C.byref(vol.rs), C.byref(cam))
        assert (vol.minmax[..., 0] < vol.minmax[..., 1]).sum() > 10
        L.oracle_raycast(C.byref(vol.scene), C.byref(vol.rs), cam.invM, cam.proj, 0)
        ours.append(vol.raycastResult.tobytes())
        assert (vol.raycastResult[..., 3] > 0).mean() > 0.2, (name, k)
        if R:
            vol.raycastResult[:] = 0
            R.ref_raycast(C.byref(vol.scene), C.byref(vol.rs), cam.invM, cam.proj)
            refs.append(vol.raycastResult.tobytes())
            assert ours[-1] == refs[-1], (name, k)
        for ty in range(5):
            oc, of = np.zeros((t.h, t.w, 4), dtype=np.uint8), np.zeros((t.h, t.w), dtype=np.float32)
            L.oracle_render_image(C.byref(vol.scene), C.byref(vol.rs), C.byref(cam), H.vptr(oc), H.vptr(of), ty, 0)
            rgb = (lambda c: c[..., :3]) if ty == abi.RENDER_COLOUR_FROM_NORMAL else (lambda c: c)   # normals leave alpha alone
            ours.append(rgb(oc).tobytes() + of.tobytes())
            if R:
                rc_, rf = np.zeros_like(oc), np.zeros_like(of)
                R.ref_shade(C.byref(vol.scene), C.byref(vol.rs), C.byref(cam), H.vptr(rc_), H.vptr(rf), ty)
                refs.append(rgb(rc_).tobytes() + rf.tobytes())
                assert ours[-1] == refs[-1], (name, k, ty)
    refpins.check(f"oracle_vs_ref/poses/{name}/raycast_shade", b"".join(ours), b"".join(refs) if R else None)
    # ICP maps at the last frame's pose
    L.oracle_find_visible_blocks(C.byref(vol.scene), C.byref(vol.rs), C.byref(last))
    L.oracle_expected_depths(C.byref(vol.scene), C.byref(vol.rs), C.byref(last))
    L.oracle_icp_maps(C.byref(vol.scene), C.byref(vol.rs), C.byref(view), H.vptr(vol.points), H.vptr(vol.normals), 0)
    mine = vol.raycastImage.tobytes() + vol.points.tobytes() + vol.normals.tobytes()
    ref = None
    if R:
        img = vol.raycastImage.copy()
        vol.raycastImage[:] = 0
        p_r, n_r = np.zeros_like(vol.points), np.zeros_like(vol.normals)
        R.ref_icp(C.byref(vol.scene), C.byref(vol.rs), view.invM_d, H.vptr(p_r), H.vptr(n_r))
        assert img.tobytes() == vol.raycastImage.tobytes()
        ref = vol.raycastImage.tobytes() + p_r.tobytes() + n_r.tobytes()
    refpins.check(f"oracle_vs_ref/poses/{name}/icp_maps", mine, ref)
    assert (vol.points[..., 3] > 0).mean() > 0.1


# Distances (voxels) of the found raycast points at the last frame's pose to the analytic scene, float64, as measured when
# these bounds were set: median / p99 / found fraction of the pixels, on the oracle's map (FindVisibleBlocks' list) and, in
# brackets, on the tolerance-mode kernel's chained frames (the allocation's list, tests/test_gpu_poses.py, H100). The bounds
# leave a margin of 1.3-2x. The maximum is not bounded: silhouette edges interpolate across depth discontinuities and give
# several voxels. ground_close fuses with mu = 1 m (20 voxels): where its band passes under a box's edge the views disagree
# and about 3 % of the points lie up to half a metre under the ground, so its p99 is the band's, not the surface's.
#   reverse        0.052 / 0.32 / 57 %  (0.052 / 0.31 / 56 %)      turn_in_place  0.005 / 1.36 / 78 %  (0.005 / 1.94 / 76 %)
#   pitch_roll     0.059 / 1.15 / 74 %  (0.062 / 1.61 / 70 %)      ground_close   0.005 / 7.77 / 99 %  (0.005 / 7.77 / 99 %)
#   far            0.149 / 1.15 / 80 %  (0.117 / 0.90 / 81 %)
SURFACE_BOUNDS = {"reverse": (0.15, 0.6, 0.45), "turn_in_place": (0.15, 3.0, 0.65), "pitch_roll": (0.15, 2.5, 0.6),
                  "ground_close": (0.15, 10.0, 0.9), "far": (0.3, 2.0, 0.7)}


def check_surface(name, rays, bounds=None):
    """the found points of a raycast of a map fused from trajectory `name` lie on the analytic scene"""
    med, p99, found = PL.distance_stats(rays, PL.VOXEL, PL.get(name).offset)
    bmed, bp99, bfound = bounds or SURFACE_BOUNDS[name]
    print(f"{name}: distance to the scene median {med:.3f} voxel, p99 {p99:.2f} voxels, {found:.0%} of the pixels found")
    assert med <= bmed and p99 <= bp99 and found >= bfound, (name, med, p99, found)


@pytest.mark.parametrize("name", PL.NAMES)
def test_surface_distance(name):
    """float64 distance of the oracle's surface to the scene it was fused from: an error the oracle and the CUDA path shared
    (both are pinned to each other and to the reference only in float32) would show here"""
    t, vol, frames, _, _ = _fuse(name)
    L = H.oracle()
    view = frames[-1][0]
    cam = abi.Camera()
    cam.M, cam.invM, cam.proj = view.M_d, view.invM_d, view.proj_d
    L.oracle_find_visible_blocks(C.byref(vol.scene), C.byref(vol.rs), C.byref(cam))
    L.oracle_expected_depths(C.byref(vol.scene), C.byref(vol.rs), C.byref(cam))
    L.oracle_raycast(C.byref(vol.scene), C.byref(vol.rs), cam.invM, cam.proj, 0)
    check_surface(name, vol.raycastResult)
