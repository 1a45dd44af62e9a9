"""GPU parity tests: the CUDA path (through the C-ABI) against the CPU oracle, bit for bit, on
seeded synthetic sequences. Tolerance: none — integer/index state must be identical and, because the
library is built without FMA contraction, so must every float (north_star only asks for 1e-5)."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from dynslam_b200 import abi, engine as E, synth
from tests import hostlib as H
from tests import parity as P

pytestmark = pytest.mark.gpu


def test_kitti_sequence_all_stages():
    pair, _ = P.run_sequence(P.Cfg(frames=6))
    assert pair.rs.noVisibleBlocks > 1000
    assert pair.scene.lastFreeBlockId < pair.cfg.numBlocks - 1000


def test_hash_collisions_excess_list():
    """1024 buckets for thousands of blocks: most allocations go through the excess list."""
    cfg = P.Cfg(frames=5, numBuckets=0x400, excessSize=0x4000, numBlocks=16384)
    pair, _ = P.run_sequence(cfg)
    used_excess = cfg.excessSize - 1 - pair.scene.lastFreeExcessListId
    assert used_excess > 1000


def test_large_table_list_kernel_in_two_passes():
    """3.1 M hash entries = 384 tiles of the list kernel, more than the 2 x 132 CTAs it launches on an H100: CTAs own several tiles, so the
    kernel runs its requests pass before its list pass (alloc.cu: twoPass) — and, in the same test, the excess list is used."""
    cfg = P.Cfg(frames=4, scale=0.25, numBlocks=16384, numBuckets=0x200000, excessSize=0x100000, decay=(3, 2))
    pair, _ = P.run_sequence(cfg)
    assert pair.rs.noVisibleBlocks > 500


def test_large_table_small_buckets_two_passes_with_excess_requests():
    """the same with a bucket part of one tile and an excess part of 300: nearly every allocation is an excess request, and the
    tiles that wait for them are spread over both passes"""
    cfg = P.Cfg(frames=4, scale=0.25, numBlocks=16384, numBuckets=0x400, excessSize=0x258000)
    pair, _ = P.run_sequence(cfg)
    assert cfg.excessSize - 1 - pair.scene.lastFreeExcessListId > 500


def test_decay_partial_with_chains():
    """minAge 2 / maxWeight 3: blocks are reset and deleted every frame, chains get unlinked."""
    cfg = P.Cfg(frames=10, frame_step=3, numBuckets=0x400, excessSize=0x4000, decay=(3, 2))
    pair, _ = P.run_sequence(cfg)
    assert pair.reco.GetDecayedBlockCount() > 200


def test_decay_partial_mass_deletion():
    """maxWeight >= maxW with minAge 1: every block seen one frame ago is emptied and deleted, thousands per call — more
    candidates than k_decay_commit's ranked fast path holds (1024), so the scan-the-whole-list path runs."""
    cfg = P.Cfg(frames=5, scale=0.5, numBlocks=32768, numBuckets=0x2000, excessSize=0x4000, decay=(50, 1), raycast=False)
    pair, _ = P.run_sequence(cfg)
    assert pair.reco.GetDecayedBlockCount() > 3 * 1024


def test_decay_default_parameters():
    cfg = P.Cfg(frames=8, decay=(1, 3), raycast=False)
    pair, _ = P.run_sequence(cfg)
    assert pair.reco.GetDecayedBlockCount() > 0


def test_depth_weighting_and_stop_at_max_w():
    P.run_sequence(P.Cfg(frames=5, depthWeighting=True, stopMaxW=True, maxW=3, frame_step=1))


def test_config1_plane_8mm():
    """BASELINE config 1: 640x480 plane at 1.5 m, 8 mm voxels (mu = 4 voxels), frustum 0.2-3 m."""
    cfg = P.Cfg(workload="plane", frames=2, voxelSize=0.008, mu=0.032, maxW=100, vf_min=0.2, vf_max=3.0,
                numBlocks=32768, numBuckets=0x8000, excessSize=0x4000)
    pair, _ = P.run_sequence(cfg)
    assert pair.rs.noVisibleBlocks > 1000


def test_integrate_ldg_variant_matches():
    """`ldg` named a kernel of earlier versions: the value now selects V4, which matches the oracle"""
    os.environ["B200_INTEGRATE_IMPL"] = "ldg"
    try:
        pair, _ = P.run_sequence(P.Cfg(frames=5, raycast=False, decay=(1, 2)))
    finally:
        os.environ.pop("B200_INTEGRATE_IMPL", None)
    assert pair.rs.noVisibleBlocks > 1000
    assert pair.eng.last_integrate()[0] == 3   # V4, two voxels per lane


def test_integrate_v3_variant_matches():
    os.environ["B200_INTEGRATE_IMPL"] = "v3"
    try:
        pair, _ = P.run_sequence(P.Cfg(frames=5, raycast=False, decay=(1, 2)))
    finally:
        os.environ.pop("B200_INTEGRATE_IMPL", None)
    assert pair.rs.noVisibleBlocks > 1000


def test_integrate_tolerance_mode():
    """B200_INTEGRATE_IMPL=fast: the V4 kernel with its TSDF update in tolerance-mode arithmetic (reciprocal multiplications,
    contracted sums). north_star's bar: allocation / indices bit-exact, TSDF and weights within 1e-5 — the weight, the depth pixel
    every voxel samples and the colours are still computed exactly; the TSDF is stored as a 16-bit code, so a result on the
    other side of a rounding boundary shows as 1 LSB (3.05e-5): counted here, must be rare and never more than 1 LSB.
    Every frame starts from the oracle's voxels, so the figures are per integration step. (The four-voxel form:
    tests/test_gpu_variants.py.)"""
    P.check_tolerance_mode()


def test_integrate_tma_variant_matches():
    os.environ["B200_INTEGRATE_IMPL"] = "tma"
    try:
        pair, _ = P.run_sequence(P.Cfg(frames=5, raycast=False, decay=(1, 2)))
    finally:
        os.environ.pop("B200_INTEGRATE_IMPL", None)
    assert pair.rs.noVisibleBlocks > 1000


def test_integrate_wide_band_colour_on_rejected_voxels():
    """mu >= 4 m: computeUpdatedVoxelDepthInfo's -1 for a rejected voxel passes the |eta / mu| <= 0.25 colour gate
    (SURVEY 8a'), so voxels outside the depth image or on depth holes still get a colour update. The default
    kernel sends those voxels to its generic per-voxel path."""
    pair, _ = P.run_sequence(P.Cfg(frames=3, mu=4.0, raycast=False, numBlocks=65536, numBuckets=0x10000, excessSize=0x4000))
    assert pair.rs.noVisibleBlocks > 1000


def test_integrate_four_resident_ctas_build():
    os.environ["B200_INTEGRATE_IMPL"] = "v3"
    os.environ["B200_V3_CTAS"] = "4"
    try:
        pair = P.Pair(P.Cfg(frames=4, raycast=False, decay=(1, 2)))   # the switches are read when the engine is created
    finally:
        os.environ.pop("B200_INTEGRATE_IMPL", None)
        os.environ.pop("B200_V3_CTAS", None)
    for i, f in enumerate(P.frames_of(pair.cfg)):
        pair.step(*f, i)
    assert pair.rs.noVisibleBlocks > 1000
    assert pair.eng.last_integrate() == (2, 4 * torch.cuda.get_device_properties(0).multi_processor_count)


def test_division_sequences_equal_ieee_division():
    """The default integrate kernel divides with the hardware's own IEEE sequence (shared reciprocals, no per-division
    slow-path call); 2^28 operand pairs x 5 divisor kinds against `/`, bit for bit."""
    p = E.SceneParams(0.05, 0.75, 50, 0.1, 300.0, False)
    scene = E.Scene(p, 1024, 0x400, 0x100, device="cuda:0")
    eng = E.Engine(scene, (64, 64))
    lib = abi.load_library()
    for mu in (0.75, 1.0, 0.016, 0.032, 4.0, 0.3333):
        bad = C.c_uint64(12345)
        assert lib.b200_selftest_divide(eng.h, 1 << 28, 7 + int(mu * 1000), C.c_float(mu), C.byref(bad)) == 0
        assert bad.value == 0, (mu, bad.value)


def _oracle_camera(M, proj):
    return H.make_camera(M, proj)


def test_free_view_render_all_types():
    """FindVisibleBlocks + CreateExpectedDepths + RenderImage (5 types) from a novel pose."""
    cfg = P.Cfg(frames=5)
    pair, (gv, hv) = P.run_sequence(cfg)
    L = pair.L
    M = synth.kitti_pose(9).copy()
    M[0, 3] += 0.4
    M[1, 3] -= 0.2
    proj = synth.kitti_intrinsics() * np.float32(cfg.scale)
    cam, ocam = E.make_camera(M, proj), _oracle_camera(M, proj)
    fv = pair.vis.CreateRenderState((pair.w, pair.h))
    fv_host_pos = np.zeros((cfg.numBlocks, 3), dtype=np.int32)
    hrs = abi.RenderState()
    C.memmove(C.byref(hrs), C.byref(pair.host.rs), C.sizeof(hrs))
    hrs.d_visibleBlockPositions = fv_host_pos.ctypes.data
    pair.vis.FindVisibleBlocks(cam, fv)
    L.oracle_find_visible_blocks(C.byref(pair.host.scene), C.byref(hrs), C.byref(ocam))
    assert fv.noVisibleBlocks == hrs.noVisibleBlocks > 500
    P._cmp("freeview list", fv.to_host()["visiblePos"], fv_host_pos[:hrs.noVisibleBlocks])
    pair.vis.CreateExpectedDepths(cam, fv)
    L.oracle_expected_depths(C.byref(pair.host.scene), C.byref(hrs), C.byref(ocam))
    P._cmp("freeview minmax", fv.renderingRangeImage.cpu().numpy(), pair.host.minmax.reshape(-1))
    dev = pair.scene.device
    for t in range(5):
        oc = torch.zeros(pair.h * pair.w * 4, dtype=torch.uint8, device=dev)
        of = torch.zeros(pair.h * pair.w, dtype=torch.float32, device=dev)
        hc = np.zeros((pair.h, pair.w, 4), dtype=np.uint8)
        hf = np.zeros((pair.h, pair.w), dtype=np.float32)
        pair.vis.RenderImage(cam, fv, oc, of, t)
        L.oracle_render_image(C.byref(pair.host.scene), C.byref(hrs), C.byref(ocam), H.vptr(hc), H.vptr(hf), t, 0)
        P._cmp(f"render type {t} rays", fv.raycastResult.cpu().numpy(), pair.host.raycastResult.reshape(-1))
        P._cmp(f"render type {t} char", oc.cpu().numpy(), hc.reshape(-1))
        P._cmp(f"render type {t} float", of.cpu().numpy(), hf.reshape(-1))
        assert (hf > 0).any() if t == abi.RENDER_DEPTH_MAP else hc[..., :3].any()


def test_full_decay_reap():
    """Decay(forceAllVoxels=true): Reap() of a finished track (DS/InfiniTamDriver.h:231-235)."""
    cfg = P.Cfg(frames=4, numBuckets=0x400, excessSize=0x4000, raycast=False)
    pair, _ = P.run_sequence(cfg)
    pair.reco.Decay(pair.scene, pair.rs, 2, 0, True)
    freed = pair.L.oracle_decay(pair.host.engine, C.byref(pair.host.scene), C.byref(pair.host.rs), 2, 0, 1)
    assert freed > 100
    pair.compare_scene("full decay")
    assert pair.reco.GetDecayedBlockCount() == freed


def test_only_update_visible_list_and_empty_frame():
    cfg = P.Cfg(frames=3, raycast=False)
    pair, (gv, hv) = P.run_sequence(cfg)
    L = pair.L
    pair.reco.AllocateSceneFromDepth(pair.scene, gv, pair.rs, onlyUpdateVisibleList=True)
    L.oracle_allocate_from_depth(pair.host.engine, C.byref(pair.host.scene), C.byref(pair.host.rs), C.byref(hv), 1, 0)
    pair.compare_scene("only visible list")
    # an all-invalid frame: nothing allocated, previous blocks stay type 3 / get demoted
    depth = np.zeros((pair.h, pair.w), dtype=np.float32)
    rgb = np.zeros((pair.h, pair.w, 4), dtype=np.uint8)
    M, proj = synth.kitti_pose(40), synth.kitti_intrinsics() * np.float32(cfg.scale)
    g2, h2 = pair.views(depth, rgb, M, proj)
    pair.reco.AllocateSceneFromDepth(pair.scene, g2, pair.rs)
    L.oracle_allocate_from_depth(pair.host.engine, C.byref(pair.host.scene), C.byref(pair.host.rs), C.byref(h2), 0, 0)
    pair.compare_scene("empty frame")
    pair.reco.IntegrateIntoScene(pair.scene, g2, pair.rs)
    L.oracle_integrate(pair.host.engine, C.byref(pair.host.scene), C.byref(pair.host.rs), C.byref(h2), 0)
    pair.compare_scene("empty frame integrate")
    assert pair.eng.frameIdx == L.oracle_frame_index(pair.host.engine)


def test_vba_exhaustion_raises_like_reference():
    """Out of VBA slots: state is mutated, counters go negative, then the call raises (Reco_CUDA.cu:348-351)."""
    cfg = P.Cfg(frames=1, numBlocks=512, raycast=False)
    pair = P.Pair(cfg)
    depth, rgb, M, proj = next(iter(P.frames_of(cfg)))
    gv, hv = pair.views(depth, rgb, M, proj)
    with pytest.raises(RuntimeError):
        pair.reco.AllocateSceneFromDepth(pair.scene, gv, pair.rs)
    rc = pair.L.oracle_allocate_from_depth(pair.host.engine, C.byref(pair.host.scene), C.byref(pair.host.rs), C.byref(hv), 0, 0)
    assert rc == abi.ERR_VBA_FULL
    assert pair.scene.lastFreeBlockId == pair.host.scene.lastFreeBlockId < 0
    pair.compare_scene("exhausted", voxels=False)


def test_fused_async_path_equals_stepwise():
    """b200_process_frame_async (no host sync inside) leaves the same state as the call-by-call path."""
    cfg = P.Cfg(frames=6, decay=(1, 2))
    stepwise, _ = P.run_sequence(cfg)
    pair = P.Pair(cfg)
    for depth, rgb, M, proj in P.frames_of(cfg):
        gv, _ = pair.views(depth, rgb, M, proj)
        pair.eng.process_frame_async(pair.rs, gv, pair.points, pair.normals, decay=cfg.decay)
    pair.eng.sync(pair.rs)
    a, b = pair.scene.to_host(), stepwise.scene.to_host()
    for k in ("hash", "voxels", "allocationList"):
        P._cmp("fused " + k, a[k], b[k])
    assert a["lastFreeBlockId"] == b["lastFreeBlockId"]
    ra, rb = pair.rs.to_host(), stepwise.rs.to_host()
    P._cmp("fused visType", ra["visType"], rb["visType"])
    P._cmp("fused visible", ra["visiblePos"], rb["visiblePos"])
    P._cmp("fused image", pair.rs.raycastImage.cpu().numpy(), stepwise.rs.raycastImage.cpu().numpy())
    P._cmp("fused minmax", pair.rs.renderingRangeImage.cpu().numpy(), stepwise.rs.renderingRangeImage.cpu().numpy())
    assert pair.reco.GetDecayedBlockCount() == stepwise.reco.GetDecayedBlockCount()


def test_rendering_block_cap_rule():
    """MAX_RENDERING_BLOCKS overflow (Vis_CUDA.cu:609): blocks whose tiles would pass the cap are dropped in list order.
    The cap is lowered to 300 tiles (test hook) so that a ~1000-block frame overflows it; both the stand-alone
    CreateExpectedDepths and the fused frame (cap applied by the last CTA of the visible-list pass) must match the oracle."""
    H.oracle().oracle_set_max_rendering_blocks(300)
    try:
        cfg = P.Cfg(frames=4, maxRenderingBlocks=300)
        stepwise, _ = P.run_sequence(cfg)            # every step is compared with the oracle, min/max image included
        mm = stepwise.rs.renderingRangeImage.cpu().numpy().reshape(-1, 2)
        live = mm[:, 0] < 999999.0
        assert 0 < live.sum()
        pair = P.Pair(cfg)
        for depth, rgb, M, proj in P.frames_of(cfg):
            gv, _ = pair.views(depth, rgb, M, proj)
            pair.eng.process_frame_async(pair.rs, gv, pair.points, pair.normals)
        pair.eng.sync(pair.rs)
        P._cmp("capped fused minmax", pair.rs.renderingRangeImage.cpu().numpy(), stepwise.rs.renderingRangeImage.cpu().numpy())
        P._cmp("capped fused rays", pair.rs.raycastResult.cpu().numpy(), stepwise.rs.raycastResult.cpu().numpy())
        # and the cap really bit: without it more of the image is covered
        H.oracle().oracle_set_max_rendering_blocks(0)
        cfg.maxRenderingBlocks = 0
        free, _ = P.run_sequence(cfg)
        mm2 = free.rs.renderingRangeImage.cpu().numpy().reshape(-1, 2)
        assert (mm2[:, 0] < 999999.0).sum() > live.sum()
    finally:
        H.oracle().oracle_set_max_rendering_blocks(0)


def test_pipelined_host_frames_equal_stepwise():
    """b200_host_frame_submit/_wait (H2D, fused frame and D2H overlapped over two slots) == the call-by-call path."""
    cfg = P.Cfg(frames=7, decay=(1, 2))
    stepwise, _ = P.run_sequence(cfg)
    pair = P.Pair(cfg)
    outs = [torch.zeros(pair.h * pair.w * 4, dtype=torch.uint8).pin_memory() for _ in range(2)]
    view = None
    keep = []
    for i, (depth, rgb, M, proj) in enumerate(P.frames_of(cfg)):
        hd, hc = torch.from_numpy(depth).pin_memory(), torch.from_numpy(rgb).pin_memory()
        keep.append((hd, hc))
        if view is None:
            view = E.View(torch.zeros_like(hd, device="cuda"), torch.zeros_like(hc, device="cuda"), M, proj)
        view.set_pose(M)
        pair.eng.host_frame_wait(i & 1)
        pair.eng.host_frame_submit(pair.rs, view, hd, hc, pair.points, pair.normals, decay=cfg.decay, h_out=outs[i & 1], slot=i & 1)
    pair.eng.host_frame_wait(0)
    pair.eng.host_frame_wait(1)
    pair.eng.sync(pair.rs)
    a, b = pair.scene.to_host(), stepwise.scene.to_host()
    for k in ("hash", "voxels", "allocationList"):
        P._cmp("pipelined " + k, a[k], b[k])
    last = outs[(cfg.frames - 1) & 1].numpy()
    P._cmp("pipelined image", last, stepwise.rs.raycastImage.cpu().numpy())
    assert pair.reco.GetDecayedBlockCount() == stepwise.reco.GetDecayedBlockCount()
