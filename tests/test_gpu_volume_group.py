"""GPU: the volume group (csrc/group.cu) and the volume restart (b200_volume_restart_async). The group's frame is the sequence of
per-engine calls StreetVolumes makes, enqueued as one call: its bytes must be that sequence's. A restarted volume must be a
brand-new one. The frame and a track start must enqueue no host wait and no allocation (a thread-local stream capture rejects
both), slots must take the per-engine calls while the other volumes fuse, and every rejection must leave every volume alone."""
import numpy as np
import pytest
import torch

from dynslam_b200 import engine as E, volumes as V

pytestmark = pytest.mark.gpu

W, H_ = 414, 125                      # a third of KITTI's frame, as in test_gpu_shared_device.py
SMALL = dict(static_blocks=0x8000, car_blocks=7142, num_buckets=0x20000, excess=0x8000)
DECAY = (1, 5)                        # partial decay live after five frames
N = 24


@pytest.fixture(scope="module")
def streets():
    return {k: V.street_frames(0, N, k, w=W, h=H_) for k in (0, 1, 3)}


def _plan(f, k, has_mask):
    """frames where a car keeps its pixels in the static map (action 0), is only removed from it (action 1), or is not fused"""
    if k == 0 and f % 6 == 2:
        return (E.KEEP, True)
    if k == 1 and f % 5 == 3 and has_mask:
        return (E.REMOVE, True)
    if k == 2 and f % 7 == 4:
        return (E.EXTRACT if has_mask else E.KEEP, False)
    return (E.EXTRACT if has_mask else E.KEEP, True)


def _frame_plan(fr, ncars, f):
    return [_plan(f, k, fr.masks[k] is not None) for k in range(ncars)]


def _reference_step(sv, fr, plan):
    """StreetVolumes.step with a plan per car: the per-engine calls of the multi-volume frame, made one by one"""
    static, s0 = sv.engines[0], sv.streams[0]
    with torch.cuda.stream(s0):
        sv.frame_depth.copy_(fr.depth)
        sv.frame_rgb.copy_(fr.rgb)
        for k in range(sv.ncars):
            sv.inst_depth[k].zero_()
            sv.inst_rgb[k].fill_(255)
        ops = [(a, fr.masks[k], fr.masks[k], sv.inst_rgb[k], sv.inst_depth[k]) for k, (a, _) in enumerate(plan) if a != E.KEEP]
        if ops:
            sv.frames_api.ProcessSilhouettes(sv.frame_rgb, sv.frame_depth, ops, sync=False, wait_inputs=False)
    fused = [k for k, (_, fuse) in enumerate(plan) if fuse]
    for k in fused:
        car = sv.engines[1 + k]
        with torch.cuda.stream(sv.streams[1 + k]):
            car.wait_engine(static)
            view = E.View(sv.inst_depth[k], sv.inst_rgb[k], fr.car_poses[k], fr.proj)
            car.process_frame_async(sv.rs[1 + k], view, sv.points[1 + k], sv.normals[1 + k], decay=sv.decay,
                                    colour_out=sv.car_colour[k], depth_out=sv.car_depth[k])
    with torch.cuda.stream(s0):
        view = E.View(sv.frame_depth, sv.frame_rgb, fr.M, fr.proj)
        static.process_frame_async(sv.rs[0], view, sv.points[0], sv.normals[0], decay=sv.decay, depth_out=sv.static_depth)
        for k in fused:
            static.wait_engine(sv.engines[1 + k])
        sv.out_color.copy_(sv._raycast_image(0))
        sv.out_depth.copy_(sv.static_depth)
        layers = [(sv.car_colour[k], sv.car_depth[k], V.TINTS[k % len(V.TINTS)]) for k in fused]
        sv.frames_api.CompositeInstances(sv.out_color, sv.out_depth, layers, wait_inputs=False)


def _states(vol, n):
    out = [vol.state(i) for i in range(n)]
    out.append({"composite colour": vol.out_color.cpu().numpy().tobytes(), "composite depth": vol.out_depth.cpu().numpy().tobytes()})
    return out


def _assert_same(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert x.keys() == y.keys()
        for k in x:
            assert np.array_equal(np.frombuffer(bytes(x[k]), np.uint8), np.frombuffer(bytes(y[k]), np.uint8)), (i, k)


@pytest.mark.parametrize("ncars", [0, 1, 3])
def test_group_frame_equals_the_call_sequence(streets, ncars):
    frames = streets[ncars]
    sv = V.StreetVolumes(ncars, W, H_, True, decay=DECAY, **SMALL)
    dev = sv.upload(frames)
    plans = [_frame_plan(fr, ncars, f) for f, fr in enumerate(dev)]
    for fr, plan in zip(dev, plans):
        _reference_step(sv, fr, plan)
    sv.synchronize()
    ref = _states(sv, 1 + ncars)
    ref_decayed = sv.engines[0].lib.b200_decayed_block_count(sv.engines[0].h)
    sv.close()
    assert ref_decayed > 0                                  # the partial decay was live
    if ncars == 3:
        assert any(p[0][0] == E.KEEP for p in plans) and any(p[1][0] == E.REMOVE for p in plans) and any(not p[2][1] for p in plans)
    for shared in (True, False):
        gv = V.GroupStreetVolumes(ncars, W, H_, shared, decay=DECAY, **SMALL)
        for fr, plan in zip(dev, plans):
            gv.step(fr, plan)
        gv.synchronize()
        got = _states(gv, 1 + ncars)
        gv.close()
        _assert_same(ref, got)


def _single(frames, graph, monkeypatch, restart_at=None):
    """one volume on the street's full frames; restart_at: fuse from frame 0, Reap, restart, go on; else a brand-new engine from
    frame 10. Returns per-frame bytes from frame 10 on."""
    monkeypatch.setenv("B200_GRAPH", str(graph))
    dev = torch.device("cuda:0")
    scene = E.Scene(E.SceneParams(), 0x8000, 0x20000, 0x8000)
    eng = E.Engine(scene, (W, H_))
    reco, vis = E.SceneReconstructionEngine(eng), E.VisualisationEngine(eng, scene)
    reco.ResetScene(scene)
    rs = vis.CreateRenderState((W, H_))
    points = torch.zeros(H_ * W * 4, dtype=torch.float32, device=dev)
    normals = torch.zeros(H_ * W * 4, dtype=torch.float32, device=dev)
    first = 0 if restart_at is not None else 10
    out = []
    for f in range(first, len(frames)):
        depth, rgb, M, proj, _ = frames[f]
        if f == restart_at:
            reco.Decay(scene, rs, 1, 0, forceAllVoxels=True)      # Reap, as DynSLAM does before it drops a track
            eng.restart_volume(scene, rs)
            out.append(eng.save_checkpoint(scene, rs).tobytes())
        elif restart_at is None and f == first:
            out.append(eng.save_checkpoint(scene, rs).tobytes())
        view = E.View(torch.from_numpy(depth).to(dev), torch.from_numpy(rgb).to(dev), M, proj)
        eng.process_frame_async(rs, view, points, normals, decay=DECAY)
        if f >= 10:
            eng.sync(rs)
            out.append(eng.save_checkpoint(scene, rs).tobytes() + rs.raycastResult.cpu().numpy().tobytes() +
                       rs.raycastImage.cpu().numpy().tobytes() + points.cpu().numpy().tobytes() + normals.cpu().numpy().tobytes())
            out.append(repr((eng.frameIdx, reco.GetDecayedBlockCount(), scene.lastFreeBlockId)).encode())
    eng.close()
    return out


@pytest.mark.parametrize("graph", [0, 1])
def test_restart_equals_new_engine(streets, graph, monkeypatch):
    frames = streets[0]
    restarted = _single(frames, graph, monkeypatch, restart_at=10)
    new = _single(frames, graph, monkeypatch)
    assert len(restarted) == len(new)
    for i, (a, b) in enumerate(zip(restarted, new)):
        assert a == b, i


def test_group_slot_restart_equals_new_engine(streets):
    """slot 0 fuses frames 0..9, is reaped and restarted at frame 10: from there its bytes are those of a brand-new car engine
    (StreetVolumes) that starts at frame 10, over more than one decay cycle"""
    frames = streets[1]
    gv = V.GroupStreetVolumes(1, W, H_, False, decay=DECAY, **SMALL)
    dev = gv.upload(frames)
    for fr in dev[:10]:
        gv.step(fr)
    sl = gv.group.slots[0]
    with torch.cuda.stream(torch.cuda.ExternalStream(sl.engine.stream)):
        E.SceneReconstructionEngine(sl.engine).Decay(sl.scene, sl.rs, 1, 0, forceAllVoxels=True)
    gv.track_start(0)
    for fr in dev[10:]:
        gv.step(fr)
    gv.synchronize()
    got = gv.state(1)
    got_idx = sl.engine.frameIdx
    gv.close()
    sv = V.StreetVolumes(1, W, H_, True, decay=DECAY, **SMALL)
    for fr in sv.upload(frames[10:], first=10):
        sv.step(fr)
    sv.synchronize()
    ref = sv.state(1)
    ref_idx = sv.engines[1].frameIdx
    sv.close()
    assert got_idx == ref_idx == N - 10
    _assert_same([ref], [got])


def test_capture_of_a_frame_with_a_track_start(streets):
    """a group frame with a track start, captured on the origin stream in thread-local mode (capture rejects host waits and
    allocations), launched once, leaves the state the same calls leave uncaptured"""
    frames = streets[3]
    out = []
    for captured in (False, True):
        gv = V.GroupStreetVolumes(3, W, H_, False, decay=DECAY, **SMALL)
        dev = gv.upload(frames)
        for fr in dev[:8]:
            gv.step(fr)
        gv.synchronize()
        prepared = gv.prepare(dev[8])
        if captured:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=gv.stream, capture_error_mode="thread_local"):
                gv.track_start(1)
                gv.step(prepared)
            with torch.cuda.stream(gv.stream):
                g.replay()
            torch.cuda.synchronize()
        else:
            gv.track_start(1)
            gv.step(prepared)
        gv.synchronize()
        out.append(_states(gv, 4))
        gv.close()
    _assert_same(out[0], out[1])


def _per_engine_calls(frames, beside):
    """cars 1 and 2 fuse frames 12..19 while slot 0 (car 0, not in those frames) runs Reap, a mesh, a checkpoint save and load and
    a free view; beside=False: the same calls with nothing else in flight"""
    gv = V.GroupStreetVolumes(3, W, H_, False, decay=DECAY, **SMALL)
    dev = gv.upload(frames)
    for fr in dev[:12]:
        gv.step(fr)
    gv.synchronize()
    rest = [gv.prepare(fr, [None if k == 0 else (E.EXTRACT if fr.masks[k] is not None else E.KEEP, True) for k in range(3)])
            for fr in dev[12:20]]
    if beside:
        for p in rest:
            gv.step(p)
    sl = gv.group.slots[0]
    out = {}
    with torch.cuda.stream(torch.cuda.ExternalStream(sl.engine.stream)):
        ck0 = sl.engine.save_checkpoint(sl.scene, sl.rs)
        reco = E.SceneReconstructionEngine(sl.engine)
        reco.Decay(sl.scene, sl.rs, 1, 0, forceAllVoxels=True)
        mesh = E.Mesh(sl.scene)
        n = E.MeshingEngine(sl.engine).MeshScene(mesh, sl.scene)
        out["mesh"] = mesh.to_host()[:n].tobytes()
        out["reaped"] = sl.engine.save_checkpoint(sl.scene, sl.rs).tobytes()
        sl.engine.load_checkpoint(sl.scene, sl.rs, ck0)
        out["loaded"] = sl.engine.save_checkpoint(sl.scene, sl.rs).tobytes()
        vis = E.VisualisationEngine(sl.engine, sl.scene)
        free = vis.CreateRenderState((W, H_))
        col = torch.zeros((H_, W, 4), dtype=torch.uint8, device=gv.dev)
        dep = torch.zeros((H_, W), dtype=torch.float32, device=gv.dev)
        M = np.array(dev[11].M, dtype=np.float32, copy=True)
        M[0, 3] += 0.6
        vis.RenderFreeView(E.make_camera(M, dev[11].proj), free, col, dep)
        out["free colour"], out["free depth"] = col.cpu().numpy().tobytes(), dep.cpu().numpy().tobytes()
    if not beside:
        for p in rest:
            gv.step(p)
    gv.synchronize()
    out["ck0"] = ck0.tobytes()
    for i in (0, 2, 3):
        out.update({f"volume {i} {k}": v.tobytes() if hasattr(v, "tobytes") else v for k, v in gv.state(i).items()})
    gv.close()
    return out, n


def test_slots_take_per_engine_calls_while_others_fuse(streets):
    alone, n = _per_engine_calls(streets[3], False)
    beside, _ = _per_engine_calls(streets[3], True)
    assert n > 0 and alone["loaded"] == alone["ck0"]
    for k in alone:
        assert alone[k] == beside[k], k


def test_rejections_leave_every_volume_alone(streets):
    frames = streets[3]
    gv = V.GroupStreetVolumes(3, W, H_, False, decay=DECAY, max_cars=4, **SMALL)   # slot 3 is never started
    dev = gv.upload(frames)
    for fr in dev[:4]:
        gv.step(fr)
    gv.synchronize()
    before = [gv.state(i)["checkpoint"].tobytes() for i in range(4)]
    frame_before = (gv.frame_rgb.cpu().numpy().tobytes(), gv.frame_depth.cpu().numpy().tobytes())
    fr = dev[4]
    cars = gv.cars(fr)

    def car(slot, like=0):
        c = cars[like]
        return E.GroupCar(slot, c.action, c.copy_mask, c.delete_mask, c.M, c.proj)

    bad = {"slot out of range": cars + [car(4)], "slot twice": [cars[0], cars[1], car(0, 2)], "never started": cars + [car(3)],
           "more cars than slots": cars + [car(3), car(0)], "negative slot": [car(-1)]}
    with torch.cuda.stream(gv.stream):
        for what, cs in bad.items():
            with pytest.raises(ValueError):
                gv.group.frame(gv.frame_rgb, gv.frame_depth, gv.static_view, cs, gv.out_color, gv.out_depth, decay=DECAY)
    # the restart refuses while a preview slot is outstanding
    sl = gv.group.slots[0]
    vis = E.VisualisationEngine(sl.engine, sl.scene)
    free = vis.CreateRenderState((W, H_))
    h_col = torch.zeros((H_, W, 4), dtype=torch.uint8).pin_memory()
    vis.RenderFreeViewSubmit(E.make_camera(fr.M, fr.proj), free, h_col, None, slot=0)
    with pytest.raises(ValueError, match="outstanding"):
        sl.engine.restart_volume(sl.scene, sl.rs)
    vis.RenderFreeViewWait(0)
    gv.synchronize()
    after = [gv.state(i)["checkpoint"].tobytes() for i in range(4)]
    assert (gv.frame_rgb.cpu().numpy().tobytes(), gv.frame_depth.cpu().numpy().tobytes()) == frame_before
    for i, (a, b) in enumerate(zip(before, after)):
        assert a == b, i
    gv.close()
