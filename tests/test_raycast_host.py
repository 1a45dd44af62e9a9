"""CPU test of the raycast kernel's per-ray code: dynslam_b200/csrc/raycast_ray.cuh (`__host__ __device__`: one-entry block
cache incl. remembered misses, single-face trilinear path, bucket prefetch, castRay) compiled for the host by tests/hostcheck
and run over whole images of an oracle-built map; every ray must equal the CPU oracle's castRay (which is pinned to the
reference's DA/ITMVisualisationEngine.h:93-179), bit for bit."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from dynslam_b200 import abi, synth
from tests import hostlib as H
from tests import poselib as PL

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostcheck")


@pytest.fixture(scope="module")
def lib():
    subprocess.run(["make", "-C", HERE, "all"], check=True, stdout=subprocess.DEVNULL)
    L = C.CDLL(os.path.join(HERE, "libhostcheck.so"))
    vp = C.c_void_p
    L.hostcheck_raycast.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_float), C.c_float, C.c_float, vp, vp, C.c_int]
    L.hostcheck_raycast.restype = None
    return L


@pytest.mark.parametrize("voxel,mu,nbuckets,frames", [(0.05, 0.75, 0x4000, 4), (0.05, 0.75, 0x400, 3), (0.1, 0.4, 0x2000, 3)])
def test_cast_ray_equals_oracle(lib, voxel, mu, nbuckets, frames):
    """Second case: 1024 buckets, so most lookups walk excess chains; third: a thin band, rays leave it again."""
    L = H.oracle()
    scale = 0.25
    w, h = int(round(synth.KITTI_W * scale)), int(round(synth.KITTI_H * scale))
    vol = H.HostVolume(16384, nbuckets, 0x4000, w, h, H.SceneParams(voxel, mu, 50, 0.1, 300.0, 0))
    street = synth.StreetScene(seed=6, length_m=60.0)
    for f in range(frames):
        depth, rgb, M, proj = synth.kitti_frame(street, 2 * f, scale=scale)
        hv = H.make_view(depth, rgb, M, proj)
        assert L.oracle_allocate_from_depth(vol.engine, C.byref(vol.scene), C.byref(vol.rs), C.byref(hv), 0, 0) == 0
        L.oracle_integrate(vol.engine, C.byref(vol.scene), C.byref(vol.rs), C.byref(hv), 0)
    # render from the last pose and from a pose the map was not built from
    Mfree = synth.kitti_pose(2 * frames + 1).copy()
    Mfree[0, 3] += 0.3
    for Mv in (M, Mfree):
        hv = H.make_view(depth, rgb, Mv, proj)
        cam = H.make_camera(Mv, proj)
        L.oracle_find_visible_blocks(C.byref(vol.scene), C.byref(vol.rs), C.byref(cam))
        L.oracle_expected_depths(C.byref(vol.scene), C.byref(vol.rs), C.byref(cam))
        L.oracle_icp_maps(C.byref(vol.scene), C.byref(vol.rs), C.byref(hv), H.vptr(vol.points), H.vptr(vol.normals), 0)
        for variant in (0, 1):      # 0: cast_ray (one-entry cache), 1: cast_ray_nbr (neighbourhood cache, k_raycast's default)
            out = np.zeros((h, w, 4), np.float32)
            lib.hostcheck_raycast(H.vptr(vol.voxels), H.vptr(vol.hash), nbuckets, w, h, hv.invM_d, hv.proj_d, voxel, mu, H.vptr(vol.minmax), H.vptr(out), variant)
            hit = int((out[..., 3] > 0).sum())
            assert hit > w * h // 4
            assert out.tobytes() == vol.raycastResult.tobytes(), variant


@pytest.mark.parametrize("name", PL.NAMES)
def test_cast_ray_general_poses_equals_oracle(lib, name):
    """the general-pose trajectories of tests/poselib.py: negative and far-from-zero block coordinates, rays marching in every
    direction through the block-neighbourhood cache (per-axis carries and re-keying at block boundaries both ways), fx != fy,
    off-centre and off-image principal points. Rendered from the last pose and from the last camera turned 35 and 90 degrees."""
    L, t = H.oracle(), PL.get(name)
    nb = 0x2000
    vol = H.HostVolume(16384, nb, 0x4000, t.w, t.h, H.SceneParams(PL.VOXEL, t.mu, 50, 0.1, 300.0, 0))
    for depth, rgb, M, proj in t.frames():
        hv = H.make_view(depth, rgb, M, proj)
        assert L.oracle_allocate_from_depth(vol.engine, C.byref(vol.scene), C.byref(vol.rs), C.byref(hv), 0, 0) == 0
        L.oracle_integrate(vol.engine, C.byref(vol.scene), C.byref(vol.rs), C.byref(hv), 0)
    hits = []
    for Mv in (M, t.turned(35.0), t.turned(90.0)):
        hv = H.make_view(depth, rgb, Mv, t.proj)
        cam = H.make_camera(Mv, t.proj)
        L.oracle_find_visible_blocks(C.byref(vol.scene), C.byref(vol.rs), C.byref(cam))
        L.oracle_expected_depths(C.byref(vol.scene), C.byref(vol.rs), C.byref(cam))
        L.oracle_icp_maps(C.byref(vol.scene), C.byref(vol.rs), C.byref(hv), H.vptr(vol.points), H.vptr(vol.normals), 0)
        for variant in (0, 1):
            out = np.zeros((t.h, t.w, 4), np.float32)
            lib.hostcheck_raycast(H.vptr(vol.voxels), H.vptr(vol.hash), nb, t.w, t.h, hv.invM_d, hv.proj_d, PL.VOXEL, t.mu,
                                  H.vptr(vol.minmax), H.vptr(out), variant)
            assert out.tobytes() == vol.raycastResult.tobytes(), (name, variant)
        hits.append(int((vol.raycastResult[..., 3] > 0).sum()))
    assert hits[0] > t.w * t.h // 3, hits
