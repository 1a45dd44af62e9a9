"""GPU: the free-view preview (csrc/preview.cu) — b200_render_view_async / _sync / _submit / _wait and
b200_engine_wait_engine — against the three-call sequence it fuses (b200_find_visible_blocks, b200_expected_depths,
b200_render_image twice) and against the CPU oracle, byte for byte: list, count, min/max image, ray points, RGBA and depth."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from dynslam_b200 import abi, engine as E, synth
from tests import evallib as V
from tests import hostlib as H
from tests import parity as P

pytestmark = pytest.mark.gpu
RGBA_TYPES = (abi.RENDER_SHADED_GREYSCALE, abi.RENDER_COLOUR_FROM_VOLUME, abi.RENDER_COLOUR_FROM_NORMAL,
              abi.RENDER_COLOUR_FROM_DEPTH_WEIGHT)
FILL = 7   # what the RGBA outputs hold before a render: RENDER_COLOUR_FROM_NORMAL keeps it as the alpha of found pixels


def _turn_back(M):
    """the same camera centre, looking the other way (half a turn about the camera's y axis)"""
    R = np.diag([-1.0, 1.0, -1.0, 1.0]).astype(np.float32)
    return (R @ M).astype(np.float32)


def _poses():
    off = synth.kitti_pose(9).copy()
    off[0, 3] += 0.4
    off[1, 3] -= 0.2
    back = _turn_back(synth.kitti_pose(22))       # past the end of the trajectory, looking back along it
    nothing = synth.kitti_pose(3).copy()
    nothing[0, 3] += 1000.0                       # the whole street a kilometre to the right of the frustum
    return [("offset", off), ("back", back), ("nothing", nothing)]


@pytest.fixture(scope="module")
def street():
    cfg = P.Cfg(frames=5)
    pair, _ = P.run_sequence(cfg)
    return pair


def _proj(pair):
    return synth.kitti_intrinsics() * np.float32(pair.cfg.scale)


class Render:
    """device outputs + free-view render state of one render"""

    def __init__(self, pair, fill=FILL):
        dev = pair.scene.device
        self.rs = pair.vis.CreateRenderState((pair.w, pair.h))
        self.col = torch.full((pair.h * pair.w * 4,), fill, dtype=torch.uint8, device=dev)
        self.dep = torch.full((pair.h * pair.w,), -1.0, dtype=torch.float32, device=dev)

    def state(self):
        n = self.rs.noVisibleBlocks
        return dict(n=n, list=self.rs.visibleBlockPositions.cpu().numpy().reshape(-1, 3)[:n].copy(),
                    minmax=self.rs.renderingRangeImage.cpu().numpy(), rays=self.rs.raycastResult.cpu().numpy(),
                    col=self.col.cpu().numpy(), dep=self.dep.cpu().numpy())


def _three_calls(pair, cam, t, fill=FILL):
    r = Render(pair, fill)
    pair.vis.FindVisibleBlocks(cam, r.rs)
    pair.vis.CreateExpectedDepths(cam, r.rs)
    pair.vis.RenderImage(cam, r.rs, r.col, r.dep, t)
    pair.vis.RenderImage(cam, r.rs, r.col, r.dep, abi.RENDER_DEPTH_MAP)
    return r


def _same(tag, a, b):
    assert a["n"] == b["n"], (tag, a["n"], b["n"])
    for k in ("list", "minmax", "rays", "col", "dep"):
        P._cmp(f"{tag}: {k}", a[k], b[k])


def _oracle_state(pair, M, proj, t, fill=FILL):
    L, ocam = pair.L, H.make_camera(M, proj)
    pos = np.zeros((pair.cfg.numBlocks, 3), dtype=np.int32)
    hrs = abi.RenderState()
    C.memmove(C.byref(hrs), C.byref(pair.host.rs), C.sizeof(hrs))
    hrs.d_visibleBlockPositions = pos.ctypes.data
    L.oracle_find_visible_blocks(C.byref(pair.host.scene), C.byref(hrs), C.byref(ocam))
    L.oracle_expected_depths(C.byref(pair.host.scene), C.byref(hrs), C.byref(ocam))
    hc = np.full((pair.h, pair.w, 4), fill, dtype=np.uint8)
    hf = np.zeros((pair.h, pair.w), dtype=np.float32)
    L.oracle_render_image(C.byref(pair.host.scene), C.byref(hrs), C.byref(ocam), H.vptr(hc), H.vptr(hf), t, 0)
    L.oracle_render_image(C.byref(pair.host.scene), C.byref(hrs), C.byref(ocam), H.vptr(hc), H.vptr(hf), abi.RENDER_DEPTH_MAP, 0)
    n = hrs.noVisibleBlocks
    return dict(n=n, list=pos[:n].copy(), minmax=pair.host.minmax.reshape(-1).copy(), rays=pair.host.raycastResult.reshape(-1).copy(),
                col=hc.reshape(-1), dep=hf.reshape(-1))


def test_equals_three_call_sequence_and_oracle(street):
    pair, proj = street, _proj(street)
    for name, M in _poses():
        cam = E.make_camera(M, proj)
        for t in RGBA_TYPES:
            new = Render(pair)
            pair.vis.RenderFreeView(cam, new.rs, new.col, new.dep, t)
            got = new.state()
            _same(f"{name} type {t} vs three calls", got, _three_calls(pair, cam, t).state())
            _same(f"{name} type {t} vs oracle", got, _oracle_state(pair, M, proj, t))
            if name == "nothing":
                assert got["n"] == 0 and not got["dep"].any()
            else:
                assert got["n"] > 200 and (name == "back" or (got["dep"] > 0).any()), (name, got["n"])


def test_single_output_and_empty_volume():
    cfg = P.Cfg(frames=0)
    pair = P.Pair(cfg)
    cam = E.make_camera(synth.kitti_pose(2), _proj(pair))
    new = Render(pair)
    pair.vis.RenderFreeView(cam, new.rs, new.col, new.dep, abi.RENDER_COLOUR_FROM_VOLUME)
    _same("empty volume", new.state(), _three_calls(pair, cam, abi.RENDER_COLOUR_FROM_VOLUME).state())
    assert new.rs.noVisibleBlocks == 0
    # one output at a time: the other image is left alone
    a, b = Render(pair), Render(pair)
    pair.vis.RenderFreeView(cam, a.rs, a.col, None, abi.RENDER_COLOUR_FROM_VOLUME)
    pair.vis.RenderFreeView(cam, b.rs, None, b.dep, abi.RENDER_COLOUR_FROM_VOLUME)
    P._cmp("colour only", a.col.cpu().numpy(), new.col.cpu().numpy())
    P._cmp("depth only", b.dep.cpu().numpy(), new.dep.cpu().numpy())
    assert (a.dep.cpu().numpy() == -1.0).all() and (b.col.cpu().numpy() == FILL).all()


def test_rendering_block_cap_decided_on_the_device():
    """More rendering tiles than MAX_RENDERING_BLOCKS (lowered to 300 by the test hook): blocks are dropped in list order."""
    H.oracle().oracle_set_max_rendering_blocks(300)
    try:
        pair, _ = P.run_sequence(P.Cfg(frames=4, maxRenderingBlocks=300))
        proj = _proj(pair)
        name, M = _poses()[0]
        cam = E.make_camera(M, proj)
        t = abi.RENDER_COLOUR_FROM_VOLUME
        new = Render(pair)
        pair.vis.RenderFreeView(cam, new.rs, new.col, new.dep, t)
        capped = new.state()
        _same("capped vs three calls", capped, _three_calls(pair, cam, t).state())
        _same("capped vs oracle", capped, _oracle_state(pair, M, proj, t))
        pair.eng.set_max_rendering_blocks(0)      # back to MAX_RENDERING_BLOCKS: the cap really bit
        free = Render(pair)
        pair.vis.RenderFreeView(cam, free.rs, free.col, free.dep, t)
        live = lambda mm: int((mm.reshape(-1, 2)[:, 0] < 999999.0).sum())
        assert live(free.state()["minmax"]) > live(capped["minmax"]) > 0
    finally:
        H.oracle().oracle_set_max_rendering_blocks(0)


def _fused_run(cfg, mode, graph):
    """mode 'plain': async frames only; 'interleaved': a free-view render enqueued after every frame, no synchronisation until the
    end; 'twin': a b200_sync and the three-call sequence after every frame."""
    if graph:
        os.environ["B200_GRAPH"] = "1"
    try:
        pair = P.Pair(cfg)
    finally:
        os.environ.pop("B200_GRAPH", None)
    proj, renders = _proj(pair), []
    fv = pair.vis.CreateRenderState((pair.w, pair.h))
    for i, (depth, rgb, M, pr) in enumerate(P.frames_of(cfg)):
        gv, _ = pair.views(depth, rgb, M, pr)
        pair.eng.process_frame_async(pair.rs, gv, pair.points, pair.normals, decay=cfg.decay)
        Mv = M.copy()
        Mv[0, 3] += 0.3
        cam = E.make_camera(Mv, proj)
        t = RGBA_TYPES[i % len(RGBA_TYPES)]
        if mode == "interleaved":
            r = Render(pair)
            r.rs = fv                              # one free-view render state, reused by every preview
            pair.vis.RenderFreeView(cam, fv, r.col, r.dep, t, sync=False)
            renders.append(r)
        elif mode == "twin":
            pair.eng.sync(pair.rs)
            renders.append(_three_calls(pair, cam, t))
    if mode != "twin":                             # (the twin is synchronised already; its device-side visible count is the free view's now)
        pair.eng.sync(pair.rs)
    return pair, renders


@pytest.mark.parametrize("graph", [0, 1])
def test_interleaved_with_async_frames(graph):
    cfg = P.Cfg(frames=6, decay=(1, 2))
    oracle, _ = P.run_sequence(cfg)                # call by call, every stage compared with the oracle
    plain, _ = _fused_run(cfg, "plain", graph)
    twin, want = _fused_run(cfg, "twin", 0)
    inter, got = _fused_run(cfg, "interleaved", graph)
    for tag, other in (("plain", plain), ("stepwise", oracle), ("twin", twin)):
        a, b = inter.scene.to_host(), other.scene.to_host()
        for k in ("hash", "voxels", "allocationList", "excessList"):
            P._cmp(f"interleaved vs {tag}: {k}", a[k], b[k])
        assert (a["lastFreeBlockId"], a["lastFreeExcessListId"]) == (b["lastFreeBlockId"], b["lastFreeExcessListId"])
        ra, rb = inter.rs.to_host(), other.rs.to_host()
        assert ra["noVisibleBlocks"] == rb["noVisibleBlocks"]
        P._cmp(f"interleaved vs {tag}: visType", ra["visType"], rb["visType"])
        P._cmp(f"interleaved vs {tag}: visible list", ra["visiblePos"], rb["visiblePos"])
        for k in ("renderingRangeImage", "raycastResult", "raycastImage"):
            P._cmp(f"interleaved vs {tag}: {k}", getattr(inter.rs, k).cpu().numpy(), getattr(other.rs, k).cpu().numpy())
        P._cmp(f"interleaved vs {tag}: points", inter.points.cpu().numpy(), other.points.cpu().numpy())
        assert inter.reco.GetDecayedBlockCount() == other.reco.GetDecayedBlockCount() > 0
    assert len(got) == len(want) == cfg.frames
    for i, (g, w) in enumerate(zip(got, want)):
        P._cmp(f"render {i}: colour", g.col.cpu().numpy(), w.col.cpu().numpy())
        P._cmp(f"render {i}: depth", g.dep.cpu().numpy(), w.dep.cpu().numpy())
    # the last preview's render state
    inter.vis.RenderFreeViewSync(got[-1].rs)
    _same("last render state", got[-1].state(), want[-1].state())


def test_checkpoint_between_size_query_and_save():
    cfg = P.Cfg(frames=4, decay=(1, 2))
    pair, _ = _fused_run(cfg, "plain", 0)
    alone = pair.eng.save_checkpoint(pair.scene, pair.rs)
    n = C.c_size_t()
    lib = pair.eng.lib
    pair.eng.check(lib.b200_checkpoint_save(pair.eng.h, C.byref(pair.scene.c), C.byref(pair.rs.c), None, 0, C.byref(n)))
    r = Render(pair)
    pair.vis.RenderFreeView(E.make_camera(_poses()[0][1], _proj(pair)), r.rs, r.col, r.dep, abi.RENDER_COLOUR_FROM_VOLUME, sync=False)
    buf = np.zeros(n.value, dtype=np.uint8)
    pair.eng.check(lib.b200_checkpoint_save(pair.eng.h, C.byref(pair.scene.c), C.byref(pair.rs.c), buf.ctypes.data, buf.size, C.byref(n)))
    assert n.value == alone.size
    P._cmp("checkpoint after a preview", buf, alone)
    pair.vis.RenderFreeViewSync(r.rs)
    assert r.rs.noVisibleBlocks > 200


def test_host_hand_over(street):
    pair, proj = street, _proj(street)
    px = pair.h * pair.w
    jobs = []
    for k, (name, M) in enumerate(_poses()[:2] * 2):
        t = RGBA_TYPES[k]
        cam = E.make_camera(M, proj)
        want = Render(pair, fill=0)                # the staging a preview is rendered into starts from alpha 0
        pair.vis.RenderFreeView(cam, want.rs, want.col, want.dep, t)
        jobs.append((cam, t, want))
    fv = [pair.vis.CreateRenderState((pair.w, pair.h)) for _ in range(2)]
    for pinned in (True, False):
        outs = []
        for k, (cam, t, want) in enumerate(jobs):
            hc, hd = torch.zeros(px * 4, dtype=torch.uint8), torch.zeros(px, dtype=torch.float32)
            if pinned:
                hc, hd = hc.pin_memory(), hd.pin_memory()
            slot = k & 1
            if k >= 2:
                pair.vis.RenderFreeViewWait(slot)   # the slot's previous preview has landed: its images are checked below
            pair.vis.RenderFreeViewSubmit(cam, fv[slot], hc, hd, t, slot)
            outs.append((hc, hd))
        with pytest.raises(ValueError, match="resubmitted"):
            pair.vis.RenderFreeViewSubmit(jobs[0][0], fv[0], outs[0][0], outs[0][1], jobs[0][1], 0)
        pair.vis.RenderFreeViewWait(0)
        pair.vis.RenderFreeViewWait(1)
        pair.vis.RenderFreeViewWait(1)              # nothing in flight: returns at once
        for k, ((hc, hd), (cam, t, want)) in enumerate(zip(outs, jobs)):
            P._cmp(f"pinned={pinned} preview {k}: colour", hc.numpy(), want.col.cpu().numpy())
            P._cmp(f"pinned={pinned} preview {k}: depth", hd.numpy(), want.dep.cpu().numpy())


def _instance_volume(seed):
    """an instance-shaped volume (InstanceReconstructor's per-car scene: voxel 0.035 m, mu 1.0, 7142 blocks) on an engine of its own"""
    cfg = P.Cfg(frames=3, voxelSize=0.035, mu=1.0, numBlocks=7142, numBuckets=0x2000, excessSize=0x1000, scene_seed=seed, zmax=8.0)
    pair, _ = P.run_sequence(cfg)
    return pair


def test_multi_volume_composite_without_host_synchronisation(street):
    static, proj = street, _proj(street)
    cars = [_instance_volume(11), _instance_volume(12)]
    M = synth.kitti_pose(3).copy()
    M[0, 3] += 0.2
    cam = E.make_camera(M, proj)
    t = abi.RENDER_COLOUR_FROM_VOLUME
    tints = E.MATPLOTLIB2_PALETTE[:2]
    n = static.h * static.w
    # all-synchronous chain, composited by the oracle
    layers_sync = [_three_calls(v, cam, t) for v in [static] + cars]
    host = [(r.col.cpu().numpy().copy(), r.dep.cpu().numpy().copy()) for r in layers_sync]
    assert all((d > 0).any() for _, d in host)
    want_c, want_d = host[0][0].copy(), host[0][1].copy()
    arr = (abi.InstanceLayer * 2)()
    for k in range(2):
        arr[k].d_color, arr[k].d_depth = host[1 + k][0].ctypes.data, host[1 + k][1].ctypes.data
        arr[k].tint = (C.c_int32 * 4)(*tints[k])
    H.oracle().oracle_composite_instances(H.vptr(want_c), H.vptr(want_d), n, arr, 2, 0.10, 1.0)
    # previews on three engines, ordered on the device, composited by the static engine
    new = [Render(v) for v in [static] + cars]
    for v, r in zip([static] + cars, new):
        v.vis.RenderFreeView(cam, r.rs, r.col, r.dep, t, sync=False)
    for v in cars:
        static.eng.wait_engine(v.eng)
    fr = E.InstanceFrames(static.eng)
    fr.CompositeInstances(new[0].col, new[0].dep, [(new[1 + k].col, new[1 + k].dep, tints[k]) for k in range(2)], wait_inputs=False)
    P._cmp("composite colour", new[0].col.cpu().numpy(), want_c)
    P._cmp("composite depth", new[0].dep.cpu().numpy(), want_d)
    # the evaluation's depth preview (CompositeInstanceDepthMaps): static depth, then every car's, into b200_evaluate_depth
    a, b = Render(static), [Render(v) for v in cars]
    static.vis.RenderFreeView(cam, a.rs, None, a.dep, t, sync=False)
    for v, r in zip(cars, b):
        v.vis.RenderFreeView(cam, r.rs, None, r.dep, t, sync=False)
        static.eng.wait_engine(v.eng)
    lib = static.eng.lib
    for r in b:
        static.eng.check(lib.b200_composite_depth(static.eng.h, a.dep.data_ptr(), r.dep.data_ptr(), n))
    sync_d = host[0][1].copy()
    for k in range(2):
        H.oracle().oracle_composite_depth(H.vptr(sync_d), H.vptr(host[1 + k][1]), n)
    P._cmp("composited depth preview", a.dep.cpu().numpy(), sync_d)
    rig = V.rig(static.w, static.h, fx=float(proj[0]))
    ev = E.Evaluation(static.eng, rig[0], rig[1], rig[2], rig[3], static.w, static.h, 0.5, 30.0)
    pts = torch.from_numpy(V.lidar_cloud(20000, 5, rig, static.w, static.h)).cuda()
    inp = torch.from_numpy(V.depth_images(static.w, static.h, 9)[1]).cuda()
    got = ev.EvaluateDepth(pts, a.dep, inp)
    want = ev.EvaluateDepth(pts, torch.from_numpy(sync_d).cuda(), inp)
    assert got == want and got[0][0]["measurement_count"] > 100


def test_rejections(street):
    pair, proj = street, _proj(street)
    cam = E.make_camera(_poses()[0][1], proj)
    r = Render(pair)
    before = pair.eng.stats().launches
    with pytest.raises(ValueError, match="both outputs"):
        pair.vis.RenderFreeView(cam, r.rs, None, None)
    with pytest.raises(ValueError, match="not an RGBA render type"):
        pair.vis.RenderFreeView(cam, r.rs, r.col, r.dep, abi.RENDER_DEPTH_MAP)
    with pytest.raises(ValueError, match="not an RGBA render type"):
        pair.vis.RenderFreeView(cam, r.rs, r.col, r.dep, 9)
    r.rs.c.img_w = 0
    with pytest.raises(ValueError, match="size"):
        pair.vis.RenderFreeView(cam, r.rs, r.col, r.dep)
    r.rs.c.img_w = pair.w
    for slot in (-1, 2):
        with pytest.raises(ValueError, match="slot"):
            pair.vis.RenderFreeViewSubmit(cam, r.rs, torch.zeros(pair.h * pair.w * 4, dtype=torch.uint8), None, slot=slot)
        with pytest.raises(ValueError, match="slot"):
            pair.vis.RenderFreeViewWait(slot)
    with pytest.raises(ValueError, match="latest free-view render"):
        pair.vis.RenderFreeViewSync(Render(pair).rs)
    with pytest.raises(ValueError, match="live render state"):   # the list the last allocation built
        pair.vis.RenderFreeView(cam, pair.rs, r.col, r.dep)
    assert pair.eng.stats().launches == before     # nothing was enqueued
    assert (r.col.cpu().numpy() == FILL).all()
