"""GPU: several volumes on one device. The kernels whose CTAs wait on one another hand out their tiles by ticket (draw_tile,
csrc/common.cuh), so their results must not depend on which CTAs are resident: engines fusing concurrently on their own
streams compute what they compute one after another on one stream, and grids launched larger than the GPU holds
(b200_diag_set_grid_scale) compute what the default grids do."""
import ctypes as C

import numpy as np
import pytest
import torch

from dynslam_b200 import abi, engine as E, synth, volumes as V
from tests import hostlib as H
from tests import parity as P

pytestmark = pytest.mark.gpu

W, H_ = 414, 125                      # a third of KITTI's frame: the test's frames render quickly on the host
SMALL = dict(static_blocks=0x8000, car_blocks=7142, num_buckets=0x20000, excess=0x8000)
DECAY = (1, 5)                        # partial decay live after five frames


@pytest.fixture(scope="module")
def street():
    """40 frames of the street with three followed cars (car streams: one per volume in the concurrent run)"""
    return V.street_frames(0, 40, 3, w=W, h=H_)


def _free_camera(fr):
    M = np.array(fr.M, dtype=np.float32, copy=True)
    M[0, 3] += 0.6                    # a camera beside the ego camera, as a free-view preview would place it
    return E.make_camera(M, fr.proj)


def _run(frames, shared_stream, between=True):
    vol = V.StreetVolumes(3, W, H_, shared_stream, decay=DECAY, **SMALL)
    dev_frames = vol.upload(frames)
    views = []
    for i in range(1 + vol.ncars):
        vis = E.VisualisationEngine(vol.engines[i], vol.scenes[i])
        rs = vis.CreateRenderState((W, H_))
        views.append((vis, rs, torch.zeros((H_, W, 4), dtype=torch.uint8, device=vol.dev), torch.zeros((H_, W), dtype=torch.float32, device=vol.dev)))
    frame = [None]

    def renders(v):
        # a free view of the static map and of every car, interleaved with the frames (b200_render_view_async)
        for i, (vis, rs, col, dep) in enumerate(views):
            with torch.cuda.stream(v.streams[i]):
                vis.RenderFreeView(_free_camera(frame[0]), rs, col, dep, sync=False)

    for fr in dev_frames:
        frame[0] = fr
        vol.step(fr, renders if between else None)
    vol.synchronize()
    out = [vol.state(i) for i in range(1 + vol.ncars)]
    for i, (vis, rs, col, dep) in enumerate(views):
        out[i]["free colour"] = col.cpu().numpy().tobytes()
        out[i]["free depth"] = dep.cpu().numpy().tobytes()
    out.append({"composite colour": vol.out_color.cpu().numpy().tobytes(), "composite depth": vol.out_depth.cpu().numpy().tobytes()})
    decayed = [e.lib.b200_decayed_block_count(e.h) for e in vol.engines]
    vol.close()
    return out, decayed


@pytest.mark.parametrize("graph", [0, 1])
def test_concurrent_volumes_match_one_stream(street, graph, monkeypatch):
    """static map + 3 car volumes, one stream each, fork / join through b200_engine_wait_engine and no host synchronisation
    until the end, against the same volumes run one after another on one shared stream"""
    monkeypatch.setenv("B200_GRAPH", str(graph))       # read when an engine is created
    shared, dec_s = _run(street, True)
    conc, dec_c = _run(street, False)
    assert dec_s == dec_c and dec_s[0] > 0              # the partial decay was live
    for i, (a, b) in enumerate(zip(shared, conc)):
        for k in a:
            assert np.array_equal(np.frombuffer(bytes(a[k]), np.uint8), np.frombuffer(bytes(b[k]), np.uint8)), (i, k)


# ---- oversubscribed grids ----------------------------------------------------------------------------------------------

def _everything(scale, cap=150):
    """every kernel that hands out tiles by ticket, on one small volume with excess-list requests (1024 buckets) and
    MAX_RENDERING_BLOCKS lowered to `cap`: allocation and the fused path, FindVisibleBlocks, ForwardRender, CreatePointCloud,
    checkpoint save, meshing, the swap-out list and full Decay (Reap). Returns the named outputs as bytes and the counts.

    With scale k > 1 every one of them (k_serve_list, k_freeview_list, k_fwd_gather_missing, k_point_cloud, k_ck_classify,
    k_mesh_list, k_mesh_blocks, k_swap_list, k_decay_rank) is launched on k x SMs x its CTAs per SM, whatever its tile count:
    at k = 8 that is at least 16 CTAs of 256 threads (or 16 of 512) per SM, where an SM holds at most 2048 threads, 8 (or 4) of
    them. Most CTAs of every launch start only after others have retired. An engine with a scaled grid runs k_serve_list in its
    ticketed form even when it is alone on the device."""
    cfg = P.Cfg(frames=5, numBuckets=0x400, excessSize=0x4000, numBlocks=16384)
    w, h = int(round(synth.KITTI_W * cfg.scale)), int(round(synth.KITTI_H * cfg.scale))
    scene = E.Scene(E.SceneParams(cfg.voxelSize, cfg.mu, cfg.maxW), cfg.numBlocks, cfg.numBuckets, cfg.excessSize)
    eng = E.Engine(scene, (w, h))
    eng.set_grid_scale(scale)
    eng.set_max_rendering_blocks(cap)
    reco, vis = E.SceneReconstructionEngine(eng), E.VisualisationEngine(eng, scene)
    rs = vis.CreateRenderState((w, h), forward=True)
    reco.ResetScene(scene)
    dev = scene.device
    points = torch.zeros(h * w * 4, dtype=torch.float32, device=dev)
    normals = torch.zeros(h * w * 4, dtype=torch.float32, device=dev)
    out = {}
    excess_free = [scene.lastFreeExcessListId]
    frames = list(P.frames_of(cfg))
    for i, (depth, rgb, M, proj) in enumerate(frames):
        gv = E.View(torch.from_numpy(depth).to(dev), torch.from_numpy(rgb).to(dev), M, proj)
        eng.process_frame_async(rs, gv, points, normals, decay=(1, 2))
        eng.sync(rs)
        excess_free.append(scene.lastFreeExcessListId)
        st = scene.to_host()
        out[f"frame {i} hash"] = st["hash"].tobytes()
        out[f"frame {i} voxels"] = st["voxels"].tobytes()
        out[f"frame {i} visible"] = rs.to_host()["visiblePos"].tobytes()
        out[f"frame {i} minmax"] = rs.renderingRangeImage.cpu().numpy().tobytes()
        out[f"frame {i} rays"] = rs.raycastResult.cpu().numpy().tobytes()
        out[f"frame {i} points"] = points.cpu().numpy().tobytes()
    out["checkpoint"] = eng.save_checkpoint(scene, rs).tobytes()
    free = vis.CreateRenderState((w, h))
    vis.FindVisibleBlocks(E.make_camera(frames[-1][2], frames[-1][3]), free)
    out["find visible"] = free.visibleBlockPositions.cpu().numpy()[:free.noVisibleBlocks * 3].tobytes()
    M2 = synth.kitti_pose(len(frames) * cfg.frame_step + 1)
    g2 = E.View(gv.depth, gv.rgb, M2, frames[-1][3])
    n_fwd = vis.ForwardRender(g2, rs)
    out["forward"] = rs.forwardProjection.cpu().numpy().tobytes()
    out["forward missing"] = rs.fwdProjMissingPoints.cpu().numpy()[:n_fwd].tobytes()
    loc = torch.zeros(h * w * 4, dtype=torch.float32, device=dev)
    col = torch.zeros(h * w * 4, dtype=torch.float32, device=dev)
    n_pc = vis.CreatePointCloud(gv, rs, loc, col)
    out["point cloud"] = loc.cpu().numpy()[:n_pc * 4].tobytes() + col.cpu().numpy()[:n_pc * 4].tobytes()
    mesh = E.Mesh(scene)
    n_tri = E.MeshingEngine(eng).MeshScene(mesh, scene)
    out["mesh"] = mesh.to_host()[:n_tri].tobytes()
    # swap-out list: every allocated entry in active memory, half of them invisible
    st = scene.to_host()
    used = np.nonzero(st["hash"]["ptr"] >= 0)[0]
    states = np.zeros(cfg.numBuckets + cfg.excessSize, dtype=np.uint8)
    states[used] = 2
    vt = rs.entriesVisibleType.cpu().numpy().copy()
    vt[used[::2]] = 0
    rs.entriesVisibleType.copy_(torch.from_numpy(vt).to(dev))
    d_states = torch.from_numpy(states).to(dev)
    scene.swapStates = d_states
    scene.c.d_swapStates = d_states.data_ptr()
    cache = E.GlobalCache(scene)
    n_out = E.SwappingEngine(eng).SaveToGlobalMemory(scene, rs, cache)
    out["swap out ids"] = cache.neededEntryIDs.cpu().numpy()[:n_out].tobytes()
    out["swap out blocks"] = cache.syncedVoxelBlocks.cpu().numpy()[:n_out * 4096].tobytes()
    reco.Decay(scene, rs, 1, 0, forceAllVoxels=True)        # Reap
    st = scene.to_host()
    for k in ("hash", "voxels", "allocationList", "excessList"):
        out[f"reap {k}"] = st[k].tobytes()
    out["counts"] = repr((n_fwd, n_pc, n_tri, n_out, reco.GetDecayedBlockCount(), scene.lastFreeBlockId)).encode()
    eng.close()
    # excess-list requests were served in frames after the first, where the list pass defers the excess part of the table
    excess_frames = sum(1 for a, b in zip(excess_free[1:], excess_free[2:]) if b < a)
    return out, (n_fwd, n_pc, n_tri, n_out, excess_frames)


def test_oversubscribed_grids_match_default():
    ref, counts = _everything(1)
    got, _ = _everything(8)
    assert all(c > 0 for c in counts), counts
    for k in ref:
        assert ref[k] == got[k], k
    # the lowered MAX_RENDERING_BLOCKS bit: without it the expected-depth images differ
    uncapped, _ = _everything(1, cap=0)
    assert any(ref[f"frame {i} minmax"] != uncapped[f"frame {i} minmax"] for i in range(5))


def test_oversubscribed_grids_against_oracle():
    """the allocation pair with excess-list requests, the fused path's raycast and partial decay, and meshing on 8x grids,
    stage by stage against the CPU oracle"""
    cfg = P.Cfg(frames=4, numBuckets=0x400, excessSize=0x4000, numBlocks=16384, decay=(1, 2), maxRenderingBlocks=150)
    H.oracle().oracle_set_max_rendering_blocks(150)
    try:
        pair = P.Pair(cfg)
        pair.eng.set_grid_scale(8)
        for i, (depth, rgb, M, proj) in enumerate(P.frames_of(cfg)):
            pair.step(depth, rgb, M, proj, i)
    finally:
        H.oracle().oracle_set_max_rendering_blocks(0)
    mesh = E.Mesh(pair.scene)
    n = E.MeshingEngine(pair.eng).MeshScene(mesh, pair.scene)
    tri = np.zeros(mesh.noMaxTriangles, dtype=abi.TRIANGLE_DTYPE)
    no = pair.L.oracle_mesh_scene(C.byref(pair.host.scene), H.vptr(tri), mesh.noMaxTriangles)
    assert n == no > 1000 and mesh.to_host()[:n].tobytes() == tri[:n].tobytes()


# ---- stand-alone calls beside frames -----------------------------------------------------------------------------------

def _reap_and_mesh(frames, beside):
    """the cars fuse 30 frames, then car 0 runs Reap (full Decay) and meshes; beside=True: while the static map's next
    frames are in flight on its own stream, beside=False: alone"""
    vol = V.StreetVolumes(3, W, H_, False, decay=DECAY, **SMALL)
    dev_frames = vol.upload(frames)
    for fr in dev_frames[:30]:
        vol.step(fr)
    vol.synchronize()
    car, sc, rs = vol.engines[1], vol.scenes[1], vol.rs[1]
    if beside:
        with torch.cuda.stream(vol.streams[0]):
            for fr in dev_frames[30:]:
                vol.engines[0].process_frame_async(vol.rs[0], E.View(fr.depth, fr.rgb, fr.M, fr.proj), vol.points[0], vol.normals[0],
                                                   decay=DECAY)
    with torch.cuda.stream(vol.streams[1]):
        E.SceneReconstructionEngine(car).Decay(sc, rs, 1, 0, forceAllVoxels=True)
        mesh = E.Mesh(sc)
        n = E.MeshingEngine(car).MeshScene(mesh, sc)
    vol.synchronize()
    st = sc.to_host()
    out = {k: st[k].tobytes() for k in ("hash", "voxels", "allocationList", "excessList")}
    out["mesh"] = mesh.to_host()[:n].tobytes()
    out["lastFree"] = repr((sc.lastFreeBlockId, sc.lastFreeExcessListId, car.lib.b200_decayed_block_count(car.h))).encode()
    vol.close()
    return out, n


def test_reap_and_mesh_beside_frames(street):
    alone, n = _reap_and_mesh(street, False)
    beside, _ = _reap_and_mesh(street, True)
    assert n > 0
    for k in alone:
        assert alone[k] == beside[k], k
