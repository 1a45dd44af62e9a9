"""GPU parity on the general-pose trajectories of tests/poselib.py: cameras that reverse, turn in place, pitch, roll, turn upside
down, look down at the ground from 1 m or sit kilometres from the origin, with fx != fy, off-centre and off-image principal
points and image sizes that are not multiples of the 8 x 4 warp tile (301 x 117, 97 x 61, 1242 x 375). Block coordinates of
every sign, rays marching in every direction.

Per trajectory: the stepwise path against the CPU oracle after every stage, with a partial decay (maxWeight 3, minAge 2) that
resets and deletes blocks re-observed from another side; the chained frame (decay swept in the raycast grid), its graph form
and the pipelined host frames against the stepwise run; renders of all five types and the host-bound free-view preview from
the last camera turned 90 and 180 degrees against the oracle. On `reverse` and `pitch_roll` also the old raycast, both
raycast dispatch orders with the principal point above and right of the image, the v3 / tma integrate kernels and the
tolerance-mode kernel under its one-LSB bar. The tolerance mode and the preview, which have no bit-exact twin, are checked
against the analytic scene in float64."""
import ctypes as C

import numpy as np
import pytest
import torch

from dynslam_b200 import abi, engine as E
from tests import hostlib as H
from tests import parity as P
from tests import poselib as PL
from tests.test_gpu_free_view import _oracle_state
from tests.test_gpu_variants import IMPLS, _pipelined, assert_same_state, env, make_pair, run
from tests.test_oracle_vs_ref_poses import check_surface

pytestmark = pytest.mark.gpu
DECAY = (3, 2)
AL_TILE, AL_BIG = 8192, 64          # alloc.cu: hash entries per list-kernel tile, big boxes a list-kernel CTA takes over


def _cfg(name, **kw):
    return P.Cfg(**{**PL.get(name).cfg_kw(), "decay": DECAY, **kw})


_stepwise = {}


def stepwise(name):
    """the trajectory through Pair.step (every stage compared with the oracle), and per frame the most list items with a box of
    more than 512 live cells that one CTA of the fused frame's list kernel meets"""
    if name in _stepwise:
        return _stepwise[name]
    cfg = _cfg(name)
    pair = P.Pair(cfg)
    grid = min(2 * torch.cuda.get_device_properties(0).multi_processor_count, -(-(cfg.numBuckets + cfg.excessSize) // AL_TILE))
    big = []
    for i, (depth, rgb, M, proj) in enumerate(P.frames_of(cfg)):
        def count_big(p, hv, M=M, proj=proj):
            n = p.host.rs.noVisibleBlocks
            mask = PL.big_live_boxes(p.host.visiblePos[:n], M, proj, p.w, p.h, cfg.voxelSize)
            share = PL.list_kernel_shares(n, grid)
            big.append(max(int(mask[share == k].sum()) for k in range(grid)))
        pair.step(depth, rgb, M, proj, i, on_allocated=count_big)
    _stepwise[name] = (pair, big)
    return _stepwise[name]


@pytest.mark.parametrize("name", PL.NAMES)
def test_stepwise_equals_oracle(name):
    pair, big = stepwise(name)
    assert pair.rs.noVisibleBlocks > 40
    print(f"{name}: {pair.reco.GetDecayedBlockCount()} blocks decayed; big boxes per list-kernel CTA by frame {big}")
    if name == "turn_in_place":
        assert pair.reco.GetDecayedBlockCount() > 100                 # re-observed from other sides, reset and deleted
    if name == "ground_close":
        assert max(big) > AL_BIG, big                                 # the list kernel's AL_BIG overflow runs


def _fused(cfg, **switches):
    pair, keep = make_pair(cfg, **switches), []
    for f in P.frames_of(cfg):
        gv, _ = pair.views(*f)
        keep.append(gv)
        pair.eng.process_frame_async(pair.rs, gv, pair.points, pair.normals, decay=cfg.decay)
    pair.eng.sync(pair.rs)
    return pair


@pytest.mark.parametrize("name", PL.NAMES)
def test_chained_graph_and_host_frames_equal_stepwise(name):
    ref, _ = stepwise(name)
    cfg = _cfg(name)
    for tag, pair in (("chained", _fused(cfg)), ("graph", _fused(cfg, B200_GRAPH=1))):
        assert_same_state(f"{name} {tag}", pair, ref)
        for k in ("renderingRangeImage", "raycastResult"):
            P._cmp(f"{name} {tag}: {k}", getattr(pair.rs, k).cpu().numpy(), getattr(ref.rs, k).cpu().numpy())
        P._cmp(f"{name} {tag}: points", pair.points.cpu().numpy(), ref.points.cpu().numpy())
    pair, last = _pipelined(cfg)
    assert_same_state(f"{name} host frames", pair, ref)
    P._cmp(f"{name} host frames: image", last, ref.rs.raycastImage.cpu().numpy())


@pytest.mark.parametrize("name", PL.NAMES)
def test_turned_renders_equal_oracle(name):
    """FindVisibleBlocks, CreateExpectedDepths and RenderImage of every type, and b200_render_view_submit of every RGBA type,
    from the last camera turned 90 and 180 degrees"""
    pair, _ = stepwise(name)
    t, L, dev = PL.get(name), pair.L, pair.scene.device
    for deg in (90.0, 180.0):
        M = t.turned(deg)
        cam, ocam = E.make_camera(M, t.proj), H.make_camera(M, t.proj)
        want = _oracle_state(pair, M, t.proj, abi.RENDER_SHADED_GREYSCALE)
        fv = pair.vis.CreateRenderState((pair.w, pair.h))
        pair.vis.FindVisibleBlocks(cam, fv)
        assert fv.noVisibleBlocks == want["n"], (name, deg)
        P._cmp(f"{name} {deg}: list", fv.visibleBlockPositions.cpu().numpy().reshape(-1, 3)[:want["n"]], want["list"])
        pair.vis.CreateExpectedDepths(cam, fv)
        P._cmp(f"{name} {deg}: minmax", fv.renderingRangeImage.cpu().numpy(), want["minmax"])
        hrs = abi.RenderState()
        C.memmove(C.byref(hrs), C.byref(pair.host.rs), C.sizeof(hrs))
        pos = np.zeros((pair.cfg.numBlocks, 3), dtype=np.int32)
        hrs.d_visibleBlockPositions = pos.ctypes.data
        L.oracle_find_visible_blocks(C.byref(pair.host.scene), C.byref(hrs), C.byref(ocam))
        L.oracle_expected_depths(C.byref(pair.host.scene), C.byref(hrs), C.byref(ocam))
        for ty in range(5):
            oc = torch.zeros(pair.h * pair.w * 4, dtype=torch.uint8, device=dev)
            of = torch.zeros(pair.h * pair.w, dtype=torch.float32, device=dev)
            hc, hf = np.zeros((pair.h, pair.w, 4), dtype=np.uint8), np.zeros((pair.h, pair.w), dtype=np.float32)
            pair.vis.RenderImage(cam, fv, oc, of, ty)
            L.oracle_render_image(C.byref(pair.host.scene), C.byref(hrs), C.byref(ocam), H.vptr(hc), H.vptr(hf), ty, 0)
            P._cmp(f"{name} {deg} type {ty}: rays", fv.raycastResult.cpu().numpy(), pair.host.raycastResult.reshape(-1))
            P._cmp(f"{name} {deg} type {ty}: char", oc.cpu().numpy(), hc.reshape(-1))
            P._cmp(f"{name} {deg} type {ty}: float", of.cpu().numpy(), hf.reshape(-1))
        slots = [pair.vis.CreateRenderState((pair.w, pair.h)) for _ in range(2)]
        for k, ty in enumerate((abi.RENDER_SHADED_GREYSCALE, abi.RENDER_COLOUR_FROM_VOLUME, abi.RENDER_COLOUR_FROM_NORMAL,
                                abi.RENDER_COLOUR_FROM_DEPTH_WEIGHT)):
            hc = torch.zeros(pair.h * pair.w * 4, dtype=torch.uint8).pin_memory()
            hd = torch.zeros(pair.h * pair.w, dtype=torch.float32).pin_memory()
            pair.vis.RenderFreeViewSubmit(cam, slots[k & 1], hc, hd, ty, k & 1)
            pair.vis.RenderFreeViewWait(k & 1)
            want = _oracle_state(pair, M, t.proj, ty, fill=0)      # the staging a preview is rendered into starts from alpha 0
            P._cmp(f"{name} {deg} submit type {ty}: colour", hc.numpy(), want["col"])
            P._cmp(f"{name} {deg} submit type {ty}: depth", hd.numpy(), want["dep"])


# ---- reverse and pitch_roll only: the switches ---------------------------------------------------------------------------
SWITCHED = ["reverse", "pitch_roll"]


@pytest.mark.parametrize("name", SWITCHED)
def test_old_raycast_equals_oracle(name):
    pair = run(_cfg(name), B200_RC_IMPL="old")
    assert pair.rs.noVisibleBlocks > 40


@pytest.mark.parametrize("order", [0, 1])
@pytest.mark.parametrize("name", SWITCHED)
def test_raycast_orders_off_image_principal_point(name, order):
    """the principal point above and right of the image (cy < 0, cx > w): the dispatch order by principal-point row has no row
    of the image to start from"""
    pair, _ = stepwise(name)
    t = PL.get(name)
    proj = t.proj.copy()
    proj[2], proj[3] = t.w + 13.0, -9.5
    M = t.world_pose(t.street_poses[-1])
    want = _oracle_state(pair, M, proj, abi.RENDER_SHADED_GREYSCALE, fill=0)
    assert (want["rays"].reshape(-1, 4)[:, 3] > 0).sum() > 100
    with env(B200_RC_ORDER=order):
        eng = E.Engine(pair.scene, (pair.w, pair.h))
    try:
        vis = E.VisualisationEngine(eng, pair.scene)
        rs = vis.CreateRenderState((pair.w, pair.h))
        cam = E.make_camera(M, proj)
        vis.FindVisibleBlocks(cam, rs)
        vis.CreateExpectedDepths(cam, rs)
        rs.raycastResult.fill_(float("nan"))
        oc = torch.zeros(pair.h * pair.w * 4, dtype=torch.uint8, device=pair.scene.device)
        of = torch.zeros(pair.h * pair.w, dtype=torch.float32, device=pair.scene.device)
        vis.RenderImage(cam, rs, oc, of, abi.RENDER_SHADED_GREYSCALE)
        vis.RenderImage(cam, rs, oc, of, abi.RENDER_DEPTH_MAP)
        P._cmp(f"{name} order {order}: minmax", rs.renderingRangeImage.cpu().numpy(), want["minmax"])
        P._cmp(f"{name} order {order}: rays", rs.raycastResult.cpu().numpy(), want["rays"])
        P._cmp(f"{name} order {order}: image", oc.cpu().numpy(), want["col"])
        P._cmp(f"{name} order {order}: depth", of.cpu().numpy(), want["dep"])
    finally:
        eng.close()


@pytest.mark.parametrize("impl", ["v3", "tma"])
@pytest.mark.parametrize("name", SWITCHED)
def test_integrate_kernels_equal_oracle(name, impl):
    switches, kernel = IMPLS[impl]
    pair = run(_cfg(name, raycast=False), **switches)
    assert pair.eng.last_integrate()[0] == kernel


@pytest.mark.parametrize("name", SWITCHED)
def test_tolerance_mode(name):
    P.check_tolerance_mode(cfg=_cfg(name, raycast=False, decay=None), min_changed=400000)   # measured: 3.98 M (reverse), 0.82 M (pitch_roll)


# ---- float64: the outputs without a bit-exact twin against the analytic scene --------------------------------------------
@pytest.mark.parametrize("name", PL.NAMES)
def test_tolerance_mode_and_preview_surface(name):
    """The trajectory fused by the tolerance-mode kernel alone (chained frames, no decay), then its raycast at the last frame's
    pose and the free-view preview from the same pose: the found points lie on the scene within the bounds the oracle's surface
    was measured against (tests/test_oracle_vs_ref_poses.py::SURFACE_BOUNDS)."""
    cfg = _cfg(name, decay=None)
    pair = make_pair(cfg, B200_INTEGRATE_IMPL="fast")
    keep = []
    for f in P.frames_of(cfg):
        gv = E.View(torch.from_numpy(f[0]).to(pair.scene.device), torch.from_numpy(f[1]).to(pair.scene.device), f[2], f[3])
        keep.append(gv)
        pair.eng.process_frame_async(pair.rs, gv, pair.points, pair.normals)
    pair.eng.sync(pair.rs)
    assert pair.eng.last_integrate()[0] >= 8
    check_surface(name, pair.rs.raycastResult.cpu().numpy())
    t = PL.get(name)
    r = pair.vis.CreateRenderState((pair.w, pair.h))
    dep = torch.zeros(pair.h * pair.w, dtype=torch.float32, device=pair.scene.device)
    pair.vis.RenderFreeView(E.make_camera(t.world_pose(t.street_poses[-1]), t.proj), r, None, dep, abi.RENDER_COLOUR_FROM_VOLUME)
    check_surface(name, r.raycastResult.cpu().numpy())
