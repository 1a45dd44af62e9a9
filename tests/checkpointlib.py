"""Checkpoint test infrastructure: bindings of the checkpoint oracle (oracle/libcheckpointoracle.so, built by build()) and
helpers that run the CPU oracle over a street sequence and compare whole volumes."""
import ctypes as C
import os

import numpy as np

from dynslam_b200 import abi, synth
from tests import hostlib as H

CK_SO = os.path.join(H.ROOT, "oracle", "libcheckpointoracle.so")
_ck = None


def ck_oracle():
    global _ck
    if _ck is None:
        L = C.CDLL(CK_SO)
        P, vp = C.POINTER, C.c_void_p
        L.oracle_checkpoint_save.argtypes = [vp, P(abi.Scene), P(abi.RenderState), vp, C.c_size_t, P(C.c_size_t)]
        L.oracle_checkpoint_load.argtypes = [vp, P(abi.Scene), P(abi.RenderState), vp, C.c_size_t, P(C.c_int)]
        _ck = L
    return _ck


def oracle_save(vol):
    L, n = ck_oracle(), C.c_size_t()
    assert L.oracle_checkpoint_save(vol.engine, C.byref(vol.scene), C.byref(vol.rs), None, 0, C.byref(n)) == 0
    buf = np.zeros(n.value, np.uint8)
    assert L.oracle_checkpoint_save(vol.engine, C.byref(vol.scene), C.byref(vol.rs), H.vptr(buf), buf.size, C.byref(n)) == 0
    return buf


def oracle_load(vol, buf):
    """(status, which check refused it: 0 = none)"""
    b = np.ascontiguousarray(buf, np.uint8)
    why = C.c_int()
    rc = ck_oracle().oracle_checkpoint_load(vol.engine, C.byref(vol.scene), C.byref(vol.rs), H.vptr(b), b.size, C.byref(why))
    return rc, why.value


def host_volume(cfg, w, h, fill=None):
    """a HostVolume of cfg's geometry; fill: byte every buffer is set to after the oracle's ResetScene (a caller's garbage)"""
    vol = H.HostVolume(cfg.numBlocks, cfg.numBuckets, cfg.excessSize, w, h,
                       H.SceneParams(cfg.voxelSize, cfg.mu, cfg.maxW, cfg.vf_min, cfg.vf_max, int(cfg.stopMaxW)))
    if fill is not None:
        for a in volume_arrays(vol).values():
            a.view(np.uint8)[...] = fill
    return vol


def volume_arrays(vol):
    return dict(hash=vol.hash, voxels=vol.voxels, allocationList=vol.allocationList, excessList=vol.excessList, visType=vol.visType,
                visiblePos=vol.visiblePos, minmax=vol.minmax, raycastResult=vol.raycastResult, raycastImage=vol.raycastImage,
                forwardProjection=vol.forwardProjection, fwdMissing=vol.fwdMissing)


def oracle_frame(vol, depth, rgb, M, proj, decay):
    """one fused frame on the oracle: allocate, integrate, expected depths, ICP maps, Decay(decay)"""
    L = H.oracle()
    hv = H.make_view(depth, rgb, M, proj)
    assert L.oracle_allocate_from_depth(vol.engine, C.byref(vol.scene), C.byref(vol.rs), C.byref(hv), 0, 0) == 0
    L.oracle_integrate(vol.engine, C.byref(vol.scene), C.byref(vol.rs), C.byref(hv), 0)
    L.oracle_expected_depths(C.byref(vol.scene), C.byref(vol.rs), C.byref(H.make_camera(M, proj)))
    L.oracle_icp_maps(C.byref(vol.scene), C.byref(vol.rs), C.byref(hv), H.vptr(vol.points), H.vptr(vol.normals), 0)
    if decay is not None:
        L.oracle_decay(vol.engine, C.byref(vol.scene), C.byref(vol.rs), decay[0], decay[1], 0)


def street_frames(n, scale=0.2, seed=6, step=2):
    scene = synth.StreetScene(seed=seed, length_m=max(60.0, n * step * 0.8 + 40.0))
    return [synth.kitti_frame(scene, f * step, scale=scale, zmax=20.0) for f in range(n)]


def volume_state(vol):
    """every piece of a host volume's state: arrays (the visible list up to its count), counters, frame index, decayed count"""
    L = H.oracle()
    d = {k: a.copy() for k, a in volume_arrays(vol).items()}
    d["visiblePos"] = vol.visiblePos[:max(vol.rs.noVisibleBlocks, 0)].copy()
    d.update(lastFreeBlockId=vol.scene.lastFreeBlockId, lastFreeExcessListId=vol.scene.lastFreeExcessListId,
             noVisibleBlocks=vol.rs.noVisibleBlocks, noFwd=vol.rs.noFwdProjMissingPoints, frameIdx=L.oracle_frame_index(vol.engine),
             decayed=L.oracle_decayed_block_count(vol.engine), queue=L.oracle_queue_size(vol.engine))
    return d


def assert_same(a, b, what=""):
    assert a.keys() == b.keys()
    for k in a:
        if isinstance(a[k], np.ndarray):
            assert a[k].tobytes() == b[k].tobytes(), f"{what}{k} differs"
        else:
            assert a[k] == b[k], f"{what}{k}: {a[k]} != {b[k]}"
