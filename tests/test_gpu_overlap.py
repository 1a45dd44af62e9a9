"""The fused frame's main-stream kernels are chained by programmatic dependent launch (engine.h, launch_chained): each kernel's
CTAs may start while the previous one drains. These tests run the headline size (1242x375, 0x100000 + 0x80000 entries) past
the decay age, so that partial decay sweeps and frees blocks under the overlap, and compare every state array and counter bit
for bit with the CPU oracle — plain, captured as a CUDA graph, with the colour and depth renders of the multi-volume path, and
through the pipelined host-buffer path. The last test checks that the chain's first kernel still sees what the caller enqueued
right before the frame."""
import ctypes as C

import numpy as np
import pytest
import torch

from dynslam_b200 import engine as E, synth
from tests import hostlib as H
from tests import parity as P

pytestmark = pytest.mark.gpu

FULL = dict(scale=1.0, numBlocks=0x60000, numBuckets=0x100000, excessSize=0x80000, frame_step=1)
DECAY = (1, 6)        # maxWeight 1, minAge 6: partial decay runs from frame 7 on and frees blocks
N_FRAMES = 12


def _frames(n, seed=6):
    street = synth.StreetScene(seed=seed, length_m=n * 0.8 + 60.0)
    return [synth.kitti_frame(street, f) for f in range(n)]


def _oracle_frame(L, vol, hv, cam, decay):
    assert L.oracle_allocate_from_depth(vol.engine, C.byref(vol.scene), C.byref(vol.rs), C.byref(hv), 0, 0) == 0
    L.oracle_integrate(vol.engine, C.byref(vol.scene), C.byref(vol.rs), C.byref(hv), 1)
    L.oracle_expected_depths(C.byref(vol.scene), C.byref(vol.rs), C.byref(cam))
    L.oracle_icp_maps(C.byref(vol.scene), C.byref(vol.rs), C.byref(hv), H.vptr(vol.points), H.vptr(vol.normals), 1)
    L.oracle_decay(vol.engine, C.byref(vol.scene), C.byref(vol.rs), decay[0], decay[1], 0)


def _compare(pair, tag):
    pair.compare_scene(tag)
    P._cmp(tag + ": minmax", pair.rs.renderingRangeImage.cpu().numpy(), pair.host.minmax.reshape(-1))
    P._cmp(tag + ": raycastResult", pair.rs.raycastResult.cpu().numpy(), pair.host.raycastResult.reshape(-1))
    P._cmp(tag + ": raycastImage", pair.rs.raycastImage.cpu().numpy(), pair.host.raycastImage.reshape(-1))
    P._cmp(tag + ": points", pair.points.cpu().numpy(), pair.host.points.reshape(-1))
    P._cmp(tag + ": normals", pair.normals.cpu().numpy(), pair.host.normals.reshape(-1))
    assert pair.reco.GetDecayedBlockCount() == pair.L.oracle_decayed_block_count(pair.host.engine), tag


@pytest.mark.parametrize("how", ["plain", "graph", "renders", "host_submit"])
def test_chained_frame_matches_oracle(how, monkeypatch):
    if how == "graph":
        monkeypatch.setenv("B200_GRAPH", "1")       # read when the engine is created
    frames = _frames(N_FRAMES)
    pair = P.Pair(P.Cfg(frames=N_FRAMES, decay=DECAY, **FULL))
    dev = pair.scene.device
    W, Hh = pair.w, pair.h
    colour = torch.zeros((Hh, W, 4), dtype=torch.uint8, device=dev)
    depth_r = torch.zeros((Hh, W), dtype=torch.float32, device=dev)
    h_out = [torch.zeros(Hh * W * 4, dtype=torch.uint8).pin_memory() for _ in range(2)]
    hv_view = E.View(torch.zeros((Hh, W), dtype=torch.float32, device=dev), torch.zeros((Hh, W, 4), dtype=torch.uint8, device=dev),
                     frames[0][2], frames[0][3])
    keep = []
    for i, (depth, rgb, M, proj) in enumerate(frames):
        if how == "host_submit":
            slot = i & 1
            pair.eng.host_frame_wait(slot)
            hd, hr = torch.from_numpy(depth).pin_memory(), torch.from_numpy(rgb).pin_memory()
            keep.append((hd, hr))
            hv_view.set_pose(M)
            pair.eng.host_frame_submit(pair.rs, hv_view, hd, hr, pair.points, pair.normals, decay=DECAY, h_out=h_out[slot], slot=slot)
        else:
            gv = E.View(torch.from_numpy(depth).to(dev), torch.from_numpy(rgb).to(dev), M, proj)
            keep.append(gv)
            if how == "renders":
                pair.eng.process_frame_async(pair.rs, gv, pair.points, pair.normals, decay=DECAY, colour_out=colour, depth_out=depth_r)
            else:
                pair.eng.process_frame_async(pair.rs, gv, pair.points, pair.normals, decay=DECAY)
        _oracle_frame(pair.L, pair.host, H.make_view(depth, rgb, M, proj), H.make_camera(M, proj), DECAY)
    if how == "host_submit":
        pair.eng.host_frame_wait(0); pair.eng.host_frame_wait(1)
    pair.eng.sync(pair.rs)
    _compare(pair, f"{how}, frame {N_FRAMES}")
    assert pair.reco.GetDecayedBlockCount() > 0
    if how == "renders":
        assert int((depth_r > 0).sum()) > 0.3 * W * Hh and int(colour[..., :3].sum()) > 0
    if how == "host_submit":
        P._cmp("host image", h_out[(N_FRAMES - 1) & 1].numpy(), pair.host.raycastImage.reshape(-1).view(np.uint8))


def test_first_launch_sees_a_depth_written_just_before_the_frame():
    """A kernel on the engine's stream rewrites the depth image right before b200_process_frame_async; the frame must fuse the
    new depth (the chain's first kernel is launched without the programmatic attribute, so it waits for that kernel)."""
    frames = _frames(N_FRAMES)
    pair = P.Pair(P.Cfg(frames=N_FRAMES, decay=DECAY, **FULL))
    dev = pair.scene.device
    stream = torch.cuda.ExternalStream(pair.eng.lib.b200_engine_stream(pair.eng.h), device=dev)
    src = [torch.from_numpy(f[0]).to(dev) for f in frames]
    gv = E.View(torch.zeros_like(src[0]), torch.from_numpy(frames[0][1]).to(dev), frames[0][2], frames[0][3])
    rgbs = [torch.from_numpy(f[1]).to(dev) for f in frames]
    torch.cuda.synchronize(dev)
    for i, (depth, rgb, M, proj) in enumerate(frames):
        gv.set_pose(M)
        with torch.cuda.stream(stream):               # kernels on the engine's stream, right before the frame
            gv.rgb.copy_(rgbs[i])
            torch.mul(src[i], 1.0, out=gv.depth)
        pair.eng.lib.b200_process_frame_async(pair.eng.h, C.byref(pair.scene.c), C.byref(pair.rs.c), C.byref(gv.c),
                                              pair.points.data_ptr(), pair.normals.data_ptr(), C.byref(_opts()))
        _oracle_frame(pair.L, pair.host, H.make_view(depth, rgb, M, proj), H.make_camera(M, proj), DECAY)
    pair.eng.sync(pair.rs)
    _compare(pair, "depth written before the frame")


def _opts():
    from dynslam_b200 import abi
    o = abi.FrameOpts()
    o.doRaycast = 1
    o.doDecay, o.decayMaxWeight, o.decayMinAge = 1, DECAY[0], DECAY[1]
    return o
