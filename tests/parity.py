"""GPU-vs-oracle parity harness (test infrastructure; also used by __graft_entry__.smoke()).

Runs the same seeded frame sequence through the CUDA engine (via the C-ABI) and through the CPU
oracle and compares EVERY piece of state after every stage, bit for bit:
hash table, visibility bytes, visible list, counters, free lists, the whole voxel block array,
min/max image, ray points, ICP maps and the grey raycast image."""
import ctypes as C
import json
import os

import numpy as np
import torch

from dynslam_b200 import abi, engine as E, synth
from tests import hostlib as H


class Cfg:
    def __init__(self, **kw):
        self.scale = 0.25
        self.numBlocks, self.numBuckets, self.excessSize = 16384, 0x4000, 0x2000
        self.voxelSize, self.mu, self.maxW = 0.05, 0.75, 50
        self.vf_min, self.vf_max = 0.1, 300.0
        self.frames, self.frame_step = 6, 2
        self.decay = None            # (maxWeight, minAge)
        self.depthWeighting = False
        self.stopMaxW = False
        self.zmax = 20.0
        self.maxRenderingBlocks = 0   # > 0: lower MAX_RENDERING_BLOCKS on the engine (diag hook) to reach the cap rule
        self.decayRingItems = 0
        self.scene_seed = 6
        self.raycast = True
        self.workload = "kitti"
        self.requiresFullRendering = True   # False: approximate integration (only voxels with w_depth == 0 are updated)
        # separate colour camera: rgb_offset = 4x4 rigid depth-camera -> colour-camera transform (M_rgb = rgb_offset @ M_d),
        # proj_rgb = its intrinsics, rgb_size = (w, h) of its image; None = the depth camera's
        self.rgb_offset = None
        self.proj_rgb = None
        self.rgb_size = None
        self.size = None              # (w, h) of the depth image; None: the workload's (KITTI scaled by `scale`, or the plane's)
        self.source = None            # callable returning the (depth, rgb, M, proj) frames; None: the workload's sequence
        self.__dict__.update(kw)

    def colour_camera(self, M, proj, w, h):
        """(M_rgb, proj_rgb, (w, h)) of the frame whose depth camera is (M, proj, w, h)"""
        M_rgb = M if self.rgb_offset is None else (np.asarray(self.rgb_offset, np.float64) @ np.asarray(M, np.float64)).astype(np.float32)
        proj_rgb = proj if self.proj_rgb is None else np.asarray(self.proj_rgb, np.float32)
        return M_rgb, proj_rgb, (self.rgb_size or (w, h))


def _cmp(name, a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    if a.shape != b.shape or a.tobytes() != b.tobytes():
        av, bv = a.reshape(-1).view(np.uint8), b.reshape(-1).view(np.uint8)
        n = min(av.size, bv.size)
        bad = np.nonzero(av[:n] != bv[:n])[0]
        raise AssertionError(f"{name}: {bad.size} differing bytes of {n} (shapes {a.shape} vs {b.shape}); first at byte "
                             f"{bad[0] if bad.size else -1}")


class Pair:
    """One volume on the GPU and its oracle twin."""

    def __init__(self, cfg, device="cuda:0"):
        self.cfg = cfg
        if cfg.size is not None:
            self.w, self.h = cfg.size
        elif cfg.workload == "plane":
            self.w, self.h = 640, 480
        else:
            self.w, self.h = int(round(synth.KITTI_W * cfg.scale)), int(round(synth.KITTI_H * cfg.scale))
        p = E.SceneParams(cfg.voxelSize, cfg.mu, cfg.maxW, cfg.vf_min, cfg.vf_max, cfg.stopMaxW)
        self.scene = E.Scene(p, cfg.numBlocks, cfg.numBuckets, cfg.excessSize, device=device)
        self.eng = E.Engine(self.scene, (self.w, self.h), decayRingItems=cfg.decayRingItems)
        if cfg.maxRenderingBlocks > 0:
            self.eng.set_max_rendering_blocks(cfg.maxRenderingBlocks)
        self.reco = E.SceneReconstructionEngine(self.eng)
        self.reco.SetFusionWeightParams(cfg.depthWeighting)
        self.vis = E.VisualisationEngine(self.eng, self.scene)
        self.rs = self.vis.CreateRenderState((self.w, self.h))
        self.reco.ResetScene(self.scene)
        dev = self.scene.device
        self.points = torch.zeros(self.h * self.w * 4, dtype=torch.float32, device=dev)
        self.normals = torch.zeros(self.h * self.w * 4, dtype=torch.float32, device=dev)
        self.host = H.HostVolume(cfg.numBlocks, cfg.numBuckets, cfg.excessSize, self.w, self.h,
                                 H.SceneParams(cfg.voxelSize, cfg.mu, cfg.maxW, cfg.vf_min, cfg.vf_max, int(cfg.stopMaxW)))
        self.L = H.oracle()

    def views(self, depth, rgb, M, proj):
        cfg, dev = self.cfg, self.scene.device
        M_rgb, proj_rgb, _ = cfg.colour_camera(M, proj, self.w, self.h)
        d = torch.from_numpy(np.ascontiguousarray(depth)).to(dev)
        c = torch.from_numpy(np.ascontiguousarray(rgb)).to(dev)
        gv = E.View(d, c, M, proj, M_rgb=M_rgb, proj_rgb=proj_rgb, depthWeighting=cfg.depthWeighting,
                    requiresFullRendering=cfg.requiresFullRendering)
        hv = H.make_view(depth, rgb, M, proj, M_rgb=M_rgb, proj_rgb=proj_rgb, depthWeighting=int(cfg.depthWeighting),
                         requiresFullRendering=int(cfg.requiresFullRendering))
        assert bytes(gv.c.invM_d) == bytes(hv.invM_d), "b200_mat4_inv differs from the oracle's"
        return gv, hv

    def compare_scene(self, tag, voxels=True):
        g, r = self.scene.to_host(), self.rs.to_host()
        o = self.host.state()
        assert g["lastFreeBlockId"] == o["lastFreeBlockId"], (tag, g["lastFreeBlockId"], o["lastFreeBlockId"])
        assert g["lastFreeExcessListId"] == o["lastFreeExcessListId"], tag
        assert r["noVisibleBlocks"] == o["noVisibleBlocks"], (tag, r["noVisibleBlocks"], o["noVisibleBlocks"])
        for f in ("pos", "offset", "ptr", "allocatedTime"):
            _cmp(f"{tag}: hash.{f}", g["hash"][f], o["hash"][f])
        _cmp(f"{tag}: entriesVisibleType", r["visType"], o["visType"])
        _cmp(f"{tag}: visible list", r["visiblePos"], o["visiblePos"])
        _cmp(f"{tag}: allocationList", g["allocationList"], o["allocationList"])
        _cmp(f"{tag}: excessList", g["excessList"], o["excessList"])
        if voxels:
            _cmp(f"{tag}: voxels", g["voxels"], o["voxels"])

    def step(self, depth, rgb, M, proj, frame_no, on_allocated=None):
        """one frame through both sides, compared after every stage; on_allocated(pair, hv) runs between allocation and
        integration"""
        cfg, L, hv_ = self.cfg, self.L, None
        gv, hv = self.views(depth, rgb, M, proj)
        tag = f"frame {frame_no}"
        self.reco.AllocateSceneFromDepth(self.scene, gv, self.rs)
        rc = L.oracle_allocate_from_depth(self.host.engine, C.byref(self.host.scene), C.byref(self.host.rs), C.byref(hv), 0, 0)
        assert rc == 0
        self.compare_scene(tag + " allocate", voxels=False)
        if on_allocated is not None:
            on_allocated(self, hv)
        self.reco.IntegrateIntoScene(self.scene, gv, self.rs)
        L.oracle_integrate(self.host.engine, C.byref(self.host.scene), C.byref(self.host.rs), C.byref(hv), 0)
        self.compare_scene(tag + " integrate")
        if cfg.raycast:
            cam = E.make_camera(M, proj)
            self.vis.CreateExpectedDepths(cam, self.rs)
            L.oracle_expected_depths(C.byref(self.host.scene), C.byref(self.host.rs), C.byref(H.make_camera(M, proj)))
            _cmp(tag + ": minmax", self.rs.renderingRangeImage.cpu().numpy(), self.host.minmax.reshape(-1))
            self.vis.CreateICPMaps(gv, self.rs, self.points, self.normals)
            L.oracle_icp_maps(C.byref(self.host.scene), C.byref(self.host.rs), C.byref(hv), H.vptr(self.host.points),
                              H.vptr(self.host.normals), 0)
            _cmp(tag + ": raycastResult", self.rs.raycastResult.cpu().numpy(), self.host.raycastResult.reshape(-1))
            _cmp(tag + ": raycastImage", self.rs.raycastImage.cpu().numpy(), self.host.raycastImage.reshape(-1))
            _cmp(tag + ": points", self.points.cpu().numpy(), self.host.points.reshape(-1))
            _cmp(tag + ": normals", self.normals.cpu().numpy(), self.host.normals.reshape(-1))
        if cfg.decay is not None:
            self.reco.Decay(self.scene, self.rs, cfg.decay[0], cfg.decay[1], False)
            L.oracle_decay(self.host.engine, C.byref(self.host.scene), C.byref(self.host.rs), cfg.decay[0], cfg.decay[1], 0)
            self.compare_scene(tag + " decay")
            assert self.reco.GetDecayedBlockCount() == L.oracle_decayed_block_count(self.host.engine)
        return gv, hv


def check_tolerance_mode(ppl=None, cfg=None, min_changed=100000):
    """B200_INTEGRATE_IMPL=fast (and B200_V4_PPL=ppl when given) against the oracle under the tolerance bar of
    tests/test_gpu_parity.py::test_integrate_tolerance_mode: allocation bit-exact, weights exact, TSDF codes within 1 LSB and
    rarely off, colour-gate flips rarer still. Every frame starts from the oracle's voxels. cfg: the sequence (default: 5 street
    frames); min_changed: the voxel updates it must make at least."""
    os.environ["B200_INTEGRATE_IMPL"] = "fast"
    if ppl is not None:
        os.environ["B200_V4_PPL"] = str(ppl)
    try:
        cfg = cfg or Cfg(frames=5, raycast=False)
        pair = Pair(cfg)
    finally:
        os.environ.pop("B200_INTEGRATE_IMPL", None)
        os.environ.pop("B200_V4_PPL", None)
    L = pair.L
    changed = flips = gate = 0
    for i, (depth, rgb, M, proj) in enumerate(frames_of(cfg)):
        gv, hv = pair.views(depth, rgb, M, proj)
        pair.reco.AllocateSceneFromDepth(pair.scene, gv, pair.rs)
        assert L.oracle_allocate_from_depth(pair.host.engine, C.byref(pair.host.scene), C.byref(pair.host.rs), C.byref(hv), 0, 0) == 0
        pair.compare_scene(f"frame {i} allocate", voxels=False)          # hash, lists, visibility, counters: bit-exact
        before = pair.host.voxels.copy()
        pair.reco.IntegrateIntoScene(pair.scene, gv, pair.rs)
        L.oracle_integrate(pair.host.engine, C.byref(pair.host.scene), C.byref(pair.host.rs), C.byref(hv), 0)
        g, o = pair.scene.to_host()["voxels"], pair.host.voxels
        assert np.array_equal(g["w_depth"], o["w_depth"])                # which voxels were updated, and their weights
        ds = g["sdf"].astype(np.int32) - o["sdf"].astype(np.int32)
        assert np.abs(ds).max() <= 1
        upd = (o["sdf"] != before["sdf"]) | (o["w_depth"] != before["w_depth"])
        changed += int(upd.sum()); flips += int((ds != 0).sum())
        colour_diff = (g["clr"] != o["clr"]).any(axis=1) | (g["w_color"] != o["w_color"])
        gate += int(colour_diff.sum())
        assert np.abs(g["sdf"].astype(np.float32) / 32767.0 - o["sdf"].astype(np.float32) / 32767.0).max() <= 3.06e-5
        pair.scene.voxels.copy_(torch.from_numpy(pair.host.voxels.view(np.uint8).reshape(-1)).to(pair.scene.device))
    assert changed > min_changed, changed
    assert flips < 0.02 * changed, (flips, changed)                      # a TSDF code on the other side of a rounding boundary
    assert gate < 0.002 * changed, (gate, changed)                       # colour gate |eta/mu| <= 0.25 decided differently on a tie
    kernel = pair.eng.last_integrate()[0]
    assert kernel >= 8 and (ppl is None or kernel == 8 + 2 + ppl), kernel   # V4 in tolerance mode, in the form asked for
    print(f"tolerance mode: {changed} voxel updates, {flips} TSDF codes off by one LSB, {gate} colour-gate flips")
    return pair


def frames_of(cfg):
    if cfg.source is not None:
        yield from cfg.source()
        return
    if cfg.workload == "plane":
        depth, rgb, M, proj = synth.plane_frame(seed=1)
        for f in range(cfg.frames):
            yield depth, rgb, M, proj
        return
    scene = synth.StreetScene(seed=cfg.scene_seed, length_m=max(60.0, cfg.frames * cfg.frame_step * 0.8 + 40.0))
    for f in range(cfg.frames):
        depth, rgb, M, proj = synth.kitti_frame(scene, f * cfg.frame_step, scale=cfg.scale, zmax=cfg.zmax)
        if cfg.rgb_offset is not None or cfg.proj_rgb is not None or cfg.rgb_size is not None:
            # the colour image as the colour camera sees the street: its own pose, intrinsics and size
            M_rgb, pr, (rw, rh) = cfg.colour_camera(M, proj, depth.shape[1], depth.shape[0])
            rgb = scene.render(M_rgb, rw, rh, float(pr[0]), float(pr[1]), float(pr[2]), float(pr[3]), zmax=cfg.zmax)[1]
        yield depth, rgb, M, proj


def run_sequence(cfg, device="cuda:0"):
    pair = Pair(cfg, device)
    last = None
    for i, (depth, rgb, M, proj) in enumerate(frames_of(cfg)):
        last = pair.step(depth, rgb, M, proj, i)
    return pair, last


def run_smoke():
    cfg = Cfg(scale=0.2, frames=3, frame_step=3, decay=(1, 1), numBlocks=8192, numBuckets=0x2000, excessSize=0x1000)
    pair, _ = run_sequence(cfg)
    assert pair.rs.noVisibleBlocks > 100
    return pair


# ---- golden fixtures (tests/golden/) -----------------------------------------------------------
import hashlib


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()[:32]


GOLDEN_CFG = dict(scale=0.25, frames=6, frame_step=2, numBlocks=16384, numBuckets=0x1000, excessSize=0x2000, decay=(3, 2))


def state_digests(hash_, visType, visiblePos, voxels, allocationList, minmax, rays, image, points, normals, counters):
    d = {f"hash.{f}": _sha(hash_[f]) for f in ("pos", "offset", "ptr", "allocatedTime")}
    d.update(visType=_sha(visType), visiblePos=_sha(visiblePos), voxels=_sha(voxels), allocationList=_sha(allocationList),
             minmax=_sha(minmax), raycastResult=_sha(rays), raycastImage=_sha(image), points=_sha(points), normals=_sha(normals),
             counters=[int(c) for c in counters])
    return d


def oracle_sequence_digests(cfg, ref_check=False):
    """Per-frame digests of the oracle's state on the golden sequence. With ref_check=True every frame's marking,
    integration of all visible blocks, raycast and ICP output is also recomputed with the reference's own functions
    (oracle/_ref/libitmref.so) and must be identical — that is what certifies the fixture."""
    L = H.oracle()
    w, h = int(round(synth.KITTI_W * cfg.scale)), int(round(synth.KITTI_H * cfg.scale))
    vol = H.HostVolume(cfg.numBlocks, cfg.numBuckets, cfg.excessSize, w, h,
                       H.SceneParams(cfg.voxelSize, cfg.mu, cfg.maxW, cfg.vf_min, cfg.vf_max, int(cfg.stopMaxW)))
    out = []
    for i, (depth, rgb, M, proj) in enumerate(frames_of(cfg)):
        hv = H.make_view(depth, rgb, M, proj, depthWeighting=int(cfg.depthWeighting))
        cam = H.make_camera(M, proj)
        assert L.oracle_allocate_from_depth(vol.engine, C.byref(vol.scene), C.byref(vol.rs), C.byref(hv), 0, 0) == 0
        pre = vol.voxels.copy() if ref_check else None
        L.oracle_integrate(vol.engine, C.byref(vol.scene), C.byref(vol.rs), C.byref(hv), 0)
        if ref_check:
            R = H.ref()
            for p in vol.visiblePos[:vol.rs.noVisibleBlocks]:
                idx = L.oracle_find_block(H.vptr(vol.hash), cfg.numBuckets, int(p[0]), int(p[1]), int(p[2]))
                if idx < 0:
                    continue
                ptr = int(vol.hash[idx]["ptr"])
                blk = pre[ptr * 512:(ptr + 1) * 512].copy()
                pos = np.array(p, dtype=np.int16)
                R.ref_integrate_block(H.vptr(blk), H.vptr(pos), C.byref(vol.scene), C.byref(hv))
                assert blk.tobytes() == vol.voxels[ptr * 512:(ptr + 1) * 512].tobytes()
        L.oracle_expected_depths(C.byref(vol.scene), C.byref(vol.rs), C.byref(cam))
        L.oracle_icp_maps(C.byref(vol.scene), C.byref(vol.rs), C.byref(hv), H.vptr(vol.points), H.vptr(vol.normals), 0)
        if ref_check and cfg.numBuckets == 0x100000:
            pass
        d = state_digests(vol.hash, vol.visType, vol.visiblePos[:vol.rs.noVisibleBlocks], vol.voxels, vol.allocationList,
                          vol.minmax, vol.raycastResult, vol.raycastImage, vol.points, vol.normals,
                          (vol.scene.lastFreeBlockId, vol.scene.lastFreeExcessListId, vol.rs.noVisibleBlocks))
        if cfg.decay is not None:
            L.oracle_decay(vol.engine, C.byref(vol.scene), C.byref(vol.rs), cfg.decay[0], cfg.decay[1], 0)
            d["after_decay"] = {"hash.ptr": _sha(vol.hash["ptr"]), "hash.offset": _sha(vol.hash["offset"]), "voxels": _sha(vol.voxels),
                                "allocationList": _sha(vol.allocationList), "visType": _sha(vol.visType),
                                "lastFreeBlockId": int(vol.scene.lastFreeBlockId),
                                "decayed": int(L.oracle_decayed_block_count(vol.engine))}
        out.append(d)
    return out


def gpu_sequence_digests(cfg, device="cuda:0"):
    pair = Pair(cfg, device)
    out = []
    for i, (depth, rgb, M, proj) in enumerate(frames_of(cfg)):
        gv = E.View(torch.from_numpy(depth).to(pair.scene.device), torch.from_numpy(rgb).to(pair.scene.device), M, proj,
                    depthWeighting=cfg.depthWeighting)
        pair.reco.AllocateSceneFromDepth(pair.scene, gv, pair.rs)
        pair.reco.IntegrateIntoScene(pair.scene, gv, pair.rs)
        pair.vis.CreateExpectedDepths(E.make_camera(M, proj), pair.rs)
        pair.vis.CreateICPMaps(gv, pair.rs, pair.points, pair.normals)
        g, r = pair.scene.to_host(), pair.rs.to_host()
        d = state_digests(g["hash"], r["visType"], r["visiblePos"], g["voxels"], g["allocationList"],
                          pair.rs.renderingRangeImage.cpu().numpy(), pair.rs.raycastResult.cpu().numpy(),
                          pair.rs.raycastImage.cpu().numpy(), pair.points.cpu().numpy(), pair.normals.cpu().numpy(),
                          (g["lastFreeBlockId"], g["lastFreeExcessListId"], r["noVisibleBlocks"]))
        if cfg.decay is not None:
            pair.reco.Decay(pair.scene, pair.rs, cfg.decay[0], cfg.decay[1], False)
            g, r = pair.scene.to_host(), pair.rs.to_host()
            d["after_decay"] = {"hash.ptr": _sha(g["hash"]["ptr"]), "hash.offset": _sha(g["hash"]["offset"]), "voxels": _sha(g["voxels"]),
                                "allocationList": _sha(g["allocationList"]), "visType": _sha(r["visType"]),
                                "lastFreeBlockId": int(g["lastFreeBlockId"]), "decayed": int(pair.reco.GetDecayedBlockCount())}
        out.append(d)
    return out
