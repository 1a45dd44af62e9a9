"""GPU: DynSLAM's stored stereo input on the device (dynslam_b200/csrc/input.cu) against the oracle (oracle/input_oracle.c, pinned to
the reference's DepthProvider / PrecomputedDepthProvider / CvToItm in tests/test_stereo_input_oracle.py).

  * b200_depth_mm_from_input and b200_bgr_to_rgba equal the oracle bit for bit, in both depth modes, at the KITTI size and at
    ragged sizes, through the vector path (aligned images) and the scalar one (images one element off alignment);
  * b200_host_frame_submit_stereo over a sequence with decay and both staging slots leaves the same state, bit for bit, as the
    oracle's conversion followed by b200_host_frame_submit_raw, with the frame's int16 depth handed out per frame;
  * b200_evaluate_depth fed from that depth counts as when fed from an uploaded image;
  * every rejected argument returns its status and message.
"""
import re

import numpy as np
import pytest
import torch

from dynslam_b200 import abi, synth
from dynslam_b200 import engine as E
from tests import evallib as V
from tests import parity as P
from tests import stereolib as S

pytestmark = pytest.mark.gpu


def _engine():
    return E.Engine(E.Scene(E.SceneParams(), 2048, 0x800, 0x400, "cuda:0"), (64, 48))


def _din(calib):
    _, b, f, dmin, dmax = calib
    return E.make_depth_input(abi.DEPTH_IN_DISPARITY_F32, b, f, dmin, dmax)


def _misaligned(a, dtype):
    """a CUDA copy of `a` that starts one element past a 16-byte boundary (the kernel's scalar path)"""
    flat = torch.zeros(a.size + 1, dtype=dtype, device="cuda")
    flat[1:] = torch.from_numpy(a.reshape(-1)).cuda()
    return flat[1:].view(a.shape)


@pytest.mark.parametrize("w,h", [(1242, 375), (97, 61), (7, 5)])
def test_conversion_kernels_equal_oracle(w, h):
    eng, L = _engine(), S.oracle()
    for k, calib in enumerate(S.CALIBS):
        disp = S.disparities(calib, w, h, seed=k)
        want = S.oracle_depth(L, disp, calib)
        si = E.StereoInput(eng, _din(calib))
        out = torch.full((h, w), 77, dtype=torch.int16, device="cuda")
        si.DepthFromDisparityMap(out, torch.from_numpy(disp).cuda())
        assert np.array_equal(out.cpu().numpy(), want), f"disparity {calib[0]} {w}x{h}"
        out2 = _misaligned(np.full((h, w), 77, np.int16), torch.int16)
        si.DepthFromDisparityMap(out2, _misaligned(disp, torch.float32))
        assert np.array_equal(out2.cpu().numpy(), want), f"disparity {calib[0]} {w}x{h} (unaligned)"
    for mx in S.CLAMP_MAX:
        depth = S.depth_mm(w, h, mx, seed=w)
        want = S.oracle_clamp(L, depth, mx)
        si = E.StereoInput(eng, E.make_depth_input(abi.DEPTH_IN_DEPTH_MM_S16, max_depth_m=mx))
        d = torch.from_numpy(depth).cuda()
        out = torch.full((h, w), 77, dtype=torch.int16, device="cuda")
        si.DepthFromDisparityMap(out, d)
        assert np.array_equal(out.cpu().numpy(), want), f"clamp {mx} {w}x{h}"
        si.DepthFromDisparityMap(d, d)                                   # in place, as ReadPrecomputed does
        assert np.array_equal(d.cpu().numpy(), want), f"clamp {mx} {w}x{h} in place"
        d2 = _misaligned(depth, torch.int16)
        si.DepthFromDisparityMap(d2, d2)
        assert np.array_equal(d2.cpu().numpy(), want), f"clamp {mx} {w}x{h} (unaligned)"
    bgr = S.bgr_image(w, h, seed=h)
    want = S.oracle_rgba(L, bgr)
    si = E.StereoInput(eng, E.make_depth_input())
    out = torch.zeros((h, w, 4), dtype=torch.uint8, device="cuda")
    si.CvToItm(out, torch.from_numpy(bgr).cuda())
    assert np.array_equal(out.cpu().numpy(), want)
    flat = torch.zeros(w * h * 3 + 1, dtype=torch.uint8, device="cuda")
    flat[1:] = torch.from_numpy(bgr.reshape(-1)).cuda()
    out.zero_()
    si.CvToItm(out, flat[1:].view(h, w, 3))
    assert np.array_equal(out.cpu().numpy(), want), "bgr (unaligned)"


def _stereo_frames(cfg, kind):
    for depth, rgb, M, proj in P.frames_of(cfg):
        bgr, disp = synth.stereo_frame(depth, rgb, focal_length_px=float(proj[0]))
        if kind == abi.DEPTH_IN_DEPTH_MM_S16:
            disp = np.round(depth * 1000.0).astype(np.int16)          # an ELAS map: int16 millimetres, some beyond the maximum
            disp[::17, ::13] = 25000
        yield bgr, disp, M, proj


def _run_sequence(cfg, kind, stereo):
    """Pipelined sequence, both staging slots. Returns the final state, every frame's grey image and int16 depth."""
    L = S.oracle()
    calib = E.make_view_calib()
    din = E.make_depth_input(kind, synth.KITTI_BASELINE_M, 0.0, 0.5, 20.0)
    pair = P.Pair(cfg)
    outs, depths, keep, view = [], [], [], None
    for i, (bgr, din_img, M, proj) in enumerate(_stereo_frames(cfg, kind)):
        din.focal_length_px = float(proj[0])
        h, w = bgr.shape[:2]
        if view is None:
            view = E.View(torch.zeros((h, w), dtype=torch.float32, device="cuda"), torch.zeros((h, w, 4), dtype=torch.uint8, device="cuda"),
                          M, proj)
        view.set_pose(M)
        pair.eng.host_frame_wait(i & 1)
        out = torch.zeros(pair.h * pair.w * 4, dtype=torch.uint8).pin_memory()
        outs.append(out)
        if stereo:
            hb, hd = torch.from_numpy(bgr).pin_memory(), torch.from_numpy(din_img).pin_memory()
            dmm = torch.full((h, w), -7, dtype=torch.int16, device="cuda")
            depths.append(dmm)
            keep.append((hb, hd))
            pair.eng.host_frame_submit_stereo(pair.rs, view, hb, hd, din, calib, pair.points, pair.normals, decay=cfg.decay, h_out=out,
                                              depth_mm_out=dmm, slot=i & 1)
        else:
            if kind == abi.DEPTH_IN_DISPARITY_F32:
                raw = S.oracle_depth(L, din_img, ("", din.baseline_m, din.focal_length_px, din.min_depth_m, din.max_depth_m))
            else:
                raw = S.oracle_clamp(L, din_img, din.max_depth_m)
            depths.append(raw)
            hr, hc = torch.from_numpy(raw).pin_memory(), torch.from_numpy(S.oracle_rgba(L, bgr)).pin_memory()
            keep.append((hr, hc))
            pair.eng.host_frame_submit_raw(pair.rs, view, hr, hc, calib, pair.points, pair.normals, decay=cfg.decay, h_out=out, slot=i & 1)
    pair.eng.host_frame_wait(0)
    pair.eng.host_frame_wait(1)
    pair.eng.sync(pair.rs)
    state = dict(pair.scene.to_host(), **pair.rs.to_host())
    state.update(rays=pair.rs.raycastResult.cpu().numpy(), image=pair.rs.raycastImage.cpu().numpy(), points=pair.points.cpu().numpy(),
                 normals=pair.normals.cpu().numpy(), decayed=pair.eng.lib.b200_decayed_block_count(pair.eng.h))
    depths = [d.cpu().numpy() if torch.is_tensor(d) else d for d in depths]
    return state, [o.numpy().copy() for o in outs], depths


@pytest.mark.parametrize("kind,graph,frames", [(abi.DEPTH_IN_DISPARITY_F32, False, 40), (abi.DEPTH_IN_DISPARITY_F32, True, 40),
                                               (abi.DEPTH_IN_DEPTH_MM_S16, False, 12)], ids=["disparity", "disparity-graph", "depth_mm"])
def test_stereo_frames_equal_oracle_conversion_then_raw(monkeypatch, kind, graph, frames):
    if graph:
        monkeypatch.setenv("B200_GRAPH", "1")
    else:
        monkeypatch.delenv("B200_GRAPH", raising=False)
    cfg = P.Cfg(frames=frames, frame_step=2, decay=(1, 3), numBlocks=0x10000, numBuckets=0x10000, excessSize=0x8000)
    a, img_a, dep_a = _run_sequence(cfg, kind, True)
    b, img_b, dep_b = _run_sequence(cfg, kind, False)
    for i, (x, y) in enumerate(zip(dep_a, dep_b)):
        P._cmp(f"frame {i} int16 depth", x, y)
    for i, (x, y) in enumerate(zip(img_a, img_b)):
        P._cmp(f"frame {i} grey image", x, y)
    for k in ("hash", "voxels", "allocationList", "excessList", "visType", "visiblePos", "rays", "image", "points", "normals"):
        P._cmp("stereo sequence " + k, a[k], b[k])
    for k in ("lastFreeBlockId", "lastFreeExcessListId", "noVisibleBlocks", "decayed"):
        assert a[k] == b[k], k
    assert a["noVisibleBlocks"] > 100 and a["decayed"] > 0
    assert (dep_a[-1] > 0).sum() > 0.3 * dep_a[-1].size


def test_evaluate_depth_from_the_frames_depth():
    """the int16 depth a stereo frame hands out feeds b200_evaluate_depth like an uploaded image"""
    w, h = synth.KITTI_W, synth.KITTI_H
    cfg = P.Cfg(scale=1.0, frames=1, numBlocks=0x8000, numBuckets=0x8000, excessSize=0x4000)
    pair = P.Pair(cfg)
    depth, rgb, M, proj = next(P.frames_of(cfg))
    bgr, disp = synth.stereo_frame(depth, rgb)
    din = E.make_depth_input(abi.DEPTH_IN_DISPARITY_F32, synth.KITTI_BASELINE_M, synth.KITTI_FX, 0.5, 20.0)
    view = E.View(torch.zeros((h, w), dtype=torch.float32, device="cuda"), torch.zeros((h, w, 4), dtype=torch.uint8, device="cuda"), M, proj)
    dmm = torch.zeros((h, w), dtype=torch.int16, device="cuda")
    hb, hd = torch.from_numpy(bgr).pin_memory(), torch.from_numpy(disp).pin_memory()
    pair.eng.host_frame_submit_stereo(pair.rs, view, hb, hd, din, E.make_view_calib(), pair.points, pair.normals, depth_mm_out=dmm, slot=0)
    pair.eng.host_frame_wait(0)
    want = S.oracle_depth(S.oracle(), disp, ("", din.baseline_m, din.focal_length_px, 0.5, 20.0))
    assert np.array_equal(dmm.cpu().numpy(), want)
    p, rigt = V.params(w, h)
    pts = torch.from_numpy(V.lidar_cloud(120000, 21, rigt, w, h).reshape(-1, 4)).cuda()
    rendered = torch.from_numpy(V.depth_images(w, h, 22)[0]).cuda()
    v, pl, pr, b = rigt
    ev = E.Evaluation(pair.eng, v, pl, pr, b, w, h, 0.5, 30.0)
    cbs = E.Evaluation.default_callbacks()
    got = ev.EvaluateDepth(pts, rendered, dmm, cbs)
    ref = ev.EvaluateDepth(pts, rendered, torch.from_numpy(want).cuda(), cbs)
    assert got == ref
    assert got[0][0]["measurement_count"] > 10000


def test_rejected_arguments():
    cfg = P.Cfg(frames=1)
    pair = P.Pair(cfg)
    depth, rgb, M, proj = next(P.frames_of(cfg))
    h, w = depth.shape
    bgr, disp = synth.stereo_frame(depth, rgb, focal_length_px=float(proj[0]))
    hb, hd = torch.from_numpy(bgr).pin_memory(), torch.from_numpy(disp).pin_memory()
    view = E.View(torch.zeros((h, w), dtype=torch.float32, device="cuda"), torch.zeros((h, w, 4), dtype=torch.uint8, device="cuda"), M, proj)
    calib = E.make_view_calib()
    good = E.make_depth_input(abi.DEPTH_IN_DISPARITY_F32, synth.KITTI_BASELINE_M, float(proj[0]))

    def submit(bgr_=hb, din_img=hd, din=good, calib_=calib, slot=0):
        pair.eng.host_frame_submit_stereo(pair.rs, view, bgr_, din_img, din, calib_, pair.points, pair.normals, slot=slot)

    too_deep = E.make_depth_input(abi.DEPTH_IN_DISPARITY_F32, 0.5, 700.0, 0.5, 32.768)
    with pytest.raises(ValueError, match=re.escape(S.MAX_DEPTH_ERROR)):
        submit(din=too_deep)
    too_deep.kind = abi.DEPTH_IN_DEPTH_MM_S16
    with pytest.raises(ValueError, match=re.escape(S.MAX_DEPTH_ERROR)):
        submit(din=too_deep)
    bad = E.make_depth_input(7)
    with pytest.raises(ValueError, match="unknown depth input kind 7"):
        submit(din=bad)
    with pytest.raises(ValueError, match="colour, depth input or calibration missing"):
        submit(bgr_=None)
    with pytest.raises(ValueError, match="colour, depth input or calibration missing"):
        submit(din_img=None)
    with pytest.raises(ValueError, match="modelSensorNoise is not available"):
        submit(calib_=E.make_view_calib(modelSensorNoise=True))
    submit(slot=1)
    with pytest.raises(ValueError, match="slot 1 resubmitted before b200_host_frame_wait"):
        submit(slot=1)
    with pytest.raises(ValueError, match="slot must be 0 or 1"):
        submit(slot=2)
    pair.eng.host_frame_wait(1)
    # the stand-alone conversions
    eng = pair.eng
    d_disp, out = torch.from_numpy(disp).cuda(), torch.zeros((h, w), dtype=torch.int16, device="cuda")
    with pytest.raises(ValueError, match=re.escape(S.MAX_DEPTH_ERROR)):
        E.StereoInput(eng, E.make_depth_input(abi.DEPTH_IN_DISPARITY_F32, 0.5, 700.0, 0.5, 32.768)).DepthFromDisparityMap(out, d_disp)
    with pytest.raises(ValueError, match="unknown depth input kind 7"):
        E.StereoInput(eng, bad).DepthFromDisparityMap(out, d_disp)
    with pytest.raises(ValueError, match="smaller than 5x5"):
        E.StereoInput(eng, good).DepthFromDisparityMap(out[:4, :4], d_disp[:4, :4])
    with pytest.raises(ValueError, match="null image"):
        E.StereoInput(eng, good).DepthFromDisparityMap(None, d_disp)
    with pytest.raises(ValueError, match="null image"):
        E.StereoInput(eng, good).CvToItm(None, torch.from_numpy(bgr).cuda())
    # still usable afterwards
    submit(slot=0)
    pair.eng.host_frame_wait(0)
