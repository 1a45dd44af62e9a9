"""GPU parity tests of the branches the default path does not reach: V4's four-voxel form, the template flags
(depthWeighting, stopIntegratingAtMaxW, approximate integration), a separate colour camera, tiny and degenerate lists, lists
without the allocation's pointer list, the integrate and raycast switches, and the fused frame's graph / no-overlap / host
modes and renders. Every case is compared with the CPU oracle (or with the stepwise path, itself compared with the oracle)
bit for bit, and asserts that the branch it is about really ran.

The switches are environment variables read when an engine is created, so a test sets them, builds its engine and removes
them again (`env`)."""
import contextlib
import ctypes as C
import os

import numpy as np
import pytest
import torch

from dynslam_b200 import abi, engine as E, synth
from tests import hostlib as H
from tests import parity as P

pytestmark = pytest.mark.gpu

# b200_diag_last_integrate's kernel ids
TMA, V3, V4_PPL1, V4_PPL2, FAST = 1, 2, 3, 4, 8
IMPLS = {"v4ppl1": (dict(B200_INTEGRATE_IMPL="v4", B200_V4_PPL=1), V4_PPL1),
         "v4ppl2": (dict(B200_INTEGRATE_IMPL="v4", B200_V4_PPL=2), V4_PPL2),
         "v3": (dict(B200_INTEGRATE_IMPL="v3"), V3),
         "tma": (dict(B200_INTEGRATE_IMPL="tma"), TMA)}


@contextlib.contextmanager
def env(**kv):
    """set (value) or remove (None) environment variables for the engines created inside the block"""
    old = {k: os.environ.get(k) for k in kv}
    try:
        for k, v in kv.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = str(v)
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def make_pair(cfg, **switches):
    with env(**switches):
        return P.Pair(cfg)


def run(cfg, **switches):
    pair = make_pair(cfg, **switches)
    for i, f in enumerate(P.frames_of(cfg)):
        pair.step(*f, i)
    return pair


def sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def rigid(rx, ry, rz, t):
    """4x4 float32 rigid transform: rotations about x, y, z (radians), then translation t"""
    cx, sx, cy, sy, cz, sz = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry), np.cos(rz), np.sin(rz)
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    T = np.eye(4)
    T[:3, :3] = Rz @ Ry @ Rx
    T[:3, 3] = t
    return T.astype(np.float32)


def oracle_clone(pair):
    """a second oracle volume holding the pair's current oracle state"""
    h, c = pair.host, pair.cfg
    o = H.HostVolume(c.numBlocks, c.numBuckets, c.excessSize, pair.w, pair.h, h.params)
    for f in ("voxels", "allocationList", "hash", "excessList", "visiblePos", "visType"):
        getattr(o, f)[...] = getattr(h, f)
    o.scene.lastFreeBlockId, o.scene.lastFreeExcessListId = h.scene.lastFreeBlockId, h.scene.lastFreeExcessListId
    o.rs.noVisibleBlocks = h.rs.noVisibleBlocks
    return o


def copy_view(hv, **fields):
    v = abi.View()
    C.memmove(C.byref(v), C.byref(hv), C.sizeof(v))
    for k, x in fields.items():
        setattr(v, k, x)
    v._keep = hv._keep
    return v


def words(voxels):
    return voxels.view(np.uint64)


def assert_same_state(tag, a, b):
    """two GPU pairs hold the same volume, lists, counters and grey image"""
    ga, gb = a.scene.to_host(), b.scene.to_host()
    for k in ("hash", "voxels", "allocationList", "excessList"):
        P._cmp(f"{tag}: {k}", ga[k], gb[k])
    assert (ga["lastFreeBlockId"], ga["lastFreeExcessListId"]) == (gb["lastFreeBlockId"], gb["lastFreeExcessListId"]), tag
    ra, rb = a.rs.to_host(), b.rs.to_host()
    assert ra["noVisibleBlocks"] == rb["noVisibleBlocks"], tag
    P._cmp(f"{tag}: visType", ra["visType"], rb["visType"])
    P._cmp(f"{tag}: visible list", ra["visiblePos"], rb["visiblePos"])
    P._cmp(f"{tag}: raycastImage", a.rs.raycastImage.cpu().numpy(), b.rs.raycastImage.cpu().numpy())
    assert a.reco.GetDecayedBlockCount() == b.reco.GetDecayedBlockCount(), tag


# ---- the switches belong to the engine ---------------------------------------------------------------------------
def test_switches_are_read_per_engine():
    """an engine keeps the switches it was created with; one created after a variable is removed gets the default"""
    cfg = P.Cfg(frames=2, raycast=False)
    frames = list(P.frames_of(cfg))
    forced = make_pair(cfg, B200_V4_PPL=2)
    forced.step(*frames[0], 0)
    default = make_pair(cfg)
    default.step(*frames[0], 0)
    forced.step(*frames[1], 1)
    assert default.rs.noVisibleBlocks < 12000 and forced.rs.noVisibleBlocks < 12000
    assert default.eng.last_integrate() == (V4_PPL1, 3 * sm_count())   # by list length
    assert forced.eng.last_integrate() == (V4_PPL2, 4 * sm_count())


# ---- 1. V4's four-voxel form --------------------------------------------------------------------------------------
def test_v4_four_voxel_form_forced_kitti_with_decay():
    pair = run(P.Cfg(frames=6, decay=(3, 2)), B200_INTEGRATE_IMPL="v4", B200_V4_PPL=2)
    assert pair.eng.last_integrate()[0] == V4_PPL2
    assert pair.reco.GetDecayedBlockCount() > 0


# 4 mm voxels (configs[4]) at 0.28 of the KITTI image size (348 x 105), depth up to 8 m: the smallest scale at which the
# visible list after allocation reaches V4_PPL2_MIN_BLOCKS (12000) from the first frame (12322 and 15283 blocks)
HIRES = dict(scale=0.28, voxelSize=0.004, mu=0.016, maxW=50, zmax=8.0, frames=2, frame_step=1, raycast=False,
             numBlocks=60000, numBuckets=0x40000, excessSize=0x20000)


@pytest.mark.parametrize("ppl", [None, 1])
def test_v4_form_by_list_length_4mm(ppl):
    """unset: the list length picks the four-voxel form; B200_V4_PPL=1 forces the two-voxel form at the same size"""
    cfg = P.Cfg(**HIRES)
    pair = make_pair(cfg, B200_V4_PPL=ppl)
    for i, f in enumerate(P.frames_of(cfg)):
        pair.step(*f, i)
        assert pair.rs.noVisibleBlocks >= 12000
        assert pair.eng.last_integrate()[0] == (V4_PPL2 if ppl is None else V4_PPL1)
    print(f"4 mm list at scale {cfg.scale}: {pair.rs.noVisibleBlocks} blocks")


# ---- 2. the template flags of V4 ------------------------------------------------------------------------------------
FLAG_SETS = {"none": {}, "depthWeighting": dict(depthWeighting=True), "stopMaxW": dict(stopMaxW=True, maxW=3),
             "approx": dict(requiresFullRendering=False),
             "all": dict(depthWeighting=True, stopMaxW=True, maxW=3, requiresFullRendering=False)}


@pytest.mark.parametrize("flags", list(FLAG_SETS))
@pytest.mark.parametrize("ppl", [1, 2])
def test_v4_template_matrix(ppl, flags):
    """Every frame is compared with the oracle. On the last frame the oracle also integrates a copy of the volume with the
    flags turned off: the voxels where the two differ are the ones the flags decided, so the branch really fired."""
    cfg = P.Cfg(frames=5, frame_step=1, raycast=False, **FLAG_SETS[flags])
    pair = make_pair(cfg, B200_INTEGRATE_IMPL="v4", B200_V4_PPL=ppl)
    frames = list(P.frames_of(cfg))
    ev = {}

    def before_integrate(p, hv):
        ev["alt"], ev["hv"] = oracle_clone(p), hv

    for i, f in enumerate(frames):
        pair.step(*f, i, on_allocated=before_integrate if i == len(frames) - 1 else None)
    assert pair.eng.last_integrate()[0] == (V4_PPL1 if ppl == 1 else V4_PPL2)
    alt, hv = ev["alt"], ev["hv"]
    pre = alt.voxels.copy()
    post = pair.host.voxels
    assert (words(post) != words(pre)).sum() > 10000
    if flags == "none":
        return
    alt.scene.stopIntegratingAtMaxW = 0
    plain = copy_view(hv, depthWeighting=0, requiresFullRendering=1)
    pair.L.oracle_integrate(alt.engine, C.byref(alt.scene), C.byref(alt.rs), C.byref(plain), 0)
    decided = words(alt.voxels) != words(post)
    if flags == "depthWeighting":
        assert decided.sum() > 1000
    if flags == "stopMaxW":
        assert (decided & (pre["w_depth"] == cfg.maxW)).sum() > 1000          # voxels at maxW skipped
    if flags in ("approx", "all"):
        assert (decided & (pre["w_depth"] != 0)).sum() > 1000                  # weighted voxels left untouched
        assert ((pre["w_depth"] == 0) & (post["w_depth"] != 0)).sum() > 100   # while new ones were written


def test_tolerance_mode_four_voxel_form():
    """B200_INTEGRATE_IMPL=fast in V4's four-voxel form, under the same tolerance bar as the two-voxel form"""
    P.check_tolerance_mode(ppl=2)


# ---- 3. approximate integration in the other kernels and in the fused frame --------------------------------------------
@pytest.mark.parametrize("impl", ["v3", "tma"])
def test_approximate_integration_other_impls(impl):
    switches, kernel = IMPLS[impl]
    pair = run(P.Cfg(frames=4, frame_step=1, raycast=False, decay=(1, 2), requiresFullRendering=False), **switches)
    assert pair.eng.last_integrate()[0] == kernel


def test_fused_frame_approximate_view_equals_stepwise():
    cfg = P.Cfg(frames=5, decay=(1, 2), requiresFullRendering=False)
    stepwise = run(cfg)
    pair = P.Pair(cfg)
    keep = []
    for f in P.frames_of(cfg):
        gv, _ = pair.views(*f)
        keep.append(gv)
        assert gv.c.requiresFullRendering == 0
        pair.eng.process_frame_async(pair.rs, gv, pair.points, pair.normals, decay=cfg.decay)
    pair.eng.sync(pair.rs)
    assert_same_state("fused approximate", pair, stepwise)


# ---- 4. a colour camera of its own ---------------------------------------------------------------------------------
# a stereo-like colour camera: 0.54 m to the side, slightly rotated, other intrinsics and another image size than the
# depth camera's (311 x 94 at scale 0.25)
RGB_CAMERA = dict(rgb_offset=rigid(0.01, -0.02, 0.005, [-0.54, 0.05, 0.02]),
                  proj_rgb=[707.0912 * 0.3, 707.0912 * 0.3, 601.8873 * 0.3 + 4.0, 183.1104 * 0.3 - 2.5], rgb_size=(373, 113))


@pytest.mark.parametrize("impl", list(IMPLS))
def test_separate_colour_camera(impl):
    """every B200_INTEGRATE_IMPL integrates colour through the re-projecting branch (the V3 / V4 paths hand such views to the
    TMA kernel); voxels, colours included, equal the oracle's"""
    cfg = P.Cfg(frames=4, frame_step=1, raycast=False, **RGB_CAMERA)
    pair = run(cfg, **IMPLS[impl][0])
    assert (pair.host.voxels["w_color"] > 0).sum() > 20000


def test_point_cloud_with_colour_camera():
    cfg = P.Cfg(frames=4, **RGB_CAMERA)
    pair = P.Pair(cfg)
    for i, f in enumerate(P.frames_of(cfg)):
        gv, hv = pair.step(*f, i)
    L, dev, n_px = pair.L, pair.scene.device, pair.w * pair.h
    calib = rigid(-0.01, 0.015, 0.0, [0.3, -0.02, 0.05])
    for skip in (0, 1):
        loc = torch.zeros(n_px * 4, dtype=torch.float32, device=dev)
        col = torch.zeros(n_px * 4, dtype=torch.float32, device=dev)
        n = pair.vis.CreatePointCloud(gv, pair.rs, loc, col, skipPoints=bool(skip), calib_rgb_to_depth=calib)
        hl, hc = np.zeros((n_px, 4), dtype=np.float32), np.zeros((n_px, 4), dtype=np.float32)
        hn = L.oracle_point_cloud(C.byref(pair.host.scene), C.byref(pair.host.rs), C.byref(hv), abi.mat_to_c(calib), skip,
                                  H.vptr(hl), H.vptr(hc))
        assert n == hn > 100
        P._cmp("pc rays", pair.rs.raycastResult.cpu().numpy(), pair.host.raycastResult.reshape(-1))
        P._cmp("pc image", pair.rs.raycastImage.cpu().numpy(), pair.host.raycastImage.reshape(-1))
        P._cmp("pc locations", loc.cpu().numpy().reshape(-1, 4)[:n], hl[:n])
        P._cmp("pc colours", col.cpu().numpy().reshape(-1, 4)[:n], hc[:n])


# ---- 5. tiny and degenerate lists ------------------------------------------------------------------------------------
@pytest.mark.parametrize("impl", list(IMPLS))
def test_tiny_and_degenerate_lists(impl):
    switches, kernel = IMPLS[impl]
    cfg = P.Cfg(frames=1, raycast=False)
    pair = make_pair(cfg, **switches)
    L, host = pair.L, pair.host
    depth, rgb, M, proj = next(iter(P.frames_of(cfg)))

    def allocate(d):
        gv, hv = pair.views(d, rgb, M, proj)
        pair.reco.AllocateSceneFromDepth(pair.scene, gv, pair.rs)
        assert L.oracle_allocate_from_depth(host.engine, C.byref(host.scene), C.byref(host.rs), C.byref(hv), 0, 0) == 0
        return gv, hv

    def integrate(gv, hv, tag):
        pair.reco.IntegrateIntoScene(pair.scene, gv, pair.rs)
        L.oracle_integrate(host.engine, C.byref(host.scene), C.byref(host.rs), C.byref(hv), 0)
        pair.compare_scene(tag)

    # an empty frame through the fused path, which launches the kernel on a list of length 0 (the stepwise call returns early)
    gv, hv = pair.views(np.zeros_like(depth), rgb, M, proj)
    pair.eng.process_frame_async(pair.rs, gv, raycast=False)
    pair.eng.sync(pair.rs)
    assert L.oracle_allocate_from_depth(host.engine, C.byref(host.scene), C.byref(host.rs), C.byref(hv), 0, 0) == 0
    assert pair.rs.noVisibleBlocks == 0
    assert pair.eng.last_integrate()[0] == kernel
    grid = pair.eng.last_integrate()[1]
    pair.compare_scene("empty list")
    # a few valid pixels: short lists built by allocation
    valid = np.flatnonzero(depth.reshape(-1) > 0)
    rng = np.random.RandomState(3)
    for k in (1, 3):
        d = np.zeros_like(depth).reshape(-1)
        px = rng.choice(valid, size=k, replace=False)
        d[px] = depth.reshape(-1)[px]
        gv, hv = allocate(d.reshape(depth.shape))
        pair.compare_scene(f"{k} pixels allocate", voxels=False)
        assert 1 <= pair.rs.noVisibleBlocks <= 16 * k, pair.rs.noVisibleBlocks
        integrate(gv, hv, f"{k} pixels")
    # the whole frame, then lists cut to exact lengths around the kernel's grid size
    gv, hv = allocate(depth)
    full = pair.rs.noVisibleBlocks
    assert full > grid + 1
    for n in (1, 2, 5, grid - 1, grid, grid + 1, full):
        pair.rs.c.noVisibleBlocks = n
        host.rs.noVisibleBlocks = n
        integrate(gv, hv, f"list of {n}")
        assert pair.eng.last_integrate() == (kernel, grid)


# ---- 6. lists that allocation did not build ----------------------------------------------------------------------------
@pytest.mark.parametrize("impl", list(IMPLS))
def test_integrate_without_fresh_pointer_list(impl):
    """the kernels resolve every item through the hash table: (a) after a Decay that deleted some of the listed blocks,
    (b) after FindVisibleBlocks rebuilt the list in the same render state"""
    switches, kernel = IMPLS[impl]
    cfg = P.Cfg(frames=2, frame_step=2, raycast=False)
    pair = make_pair(cfg, **switches)
    L, host = pair.L, pair.host
    frames = list(P.frames_of(cfg))
    for i, f in enumerate(frames):
        gv, hv = pair.step(*f, i)
    # (a) minAge 1, maxWeight 1: the blocks of the previous frame's list that this frame did not raise above weight 1 go
    pair.reco.Decay(pair.scene, pair.rs, 1, 1, False)
    L.oracle_decay(host.engine, C.byref(host.scene), C.byref(host.rs), 1, 1, 0)
    pair.compare_scene("decay")
    listed = host.visiblePos[:host.rs.noVisibleBlocks]
    found = np.array([L.oracle_find_block(H.vptr(host.hash), cfg.numBuckets, int(x), int(y), int(z)) >= 0 for x, y, z in listed])
    assert (~found).sum() > 10 and found.sum() > 500, ((~found).sum(), found.sum())
    pair.reco.IntegrateIntoScene(pair.scene, gv, pair.rs)
    L.oracle_integrate(host.engine, C.byref(host.scene), C.byref(host.rs), C.byref(hv), 0)
    pair.compare_scene("integrate after decay")
    assert pair.eng.last_integrate()[0] == kernel
    # (b)
    M, proj = frames[-1][2], frames[-1][3]
    pair.vis.FindVisibleBlocks(E.make_camera(M, proj), pair.rs)
    L.oracle_find_visible_blocks(C.byref(host.scene), C.byref(host.rs), C.byref(H.make_camera(M, proj)))
    pair.compare_scene("find visible", voxels=False)
    assert pair.rs.noVisibleBlocks > 500
    pair.reco.IntegrateIntoScene(pair.scene, gv, pair.rs)
    L.oracle_integrate(host.engine, C.byref(host.scene), C.byref(host.rs), C.byref(hv), 0)
    pair.compare_scene("integrate after find visible")


# ---- 7. V4 and V3 switches -----------------------------------------------------------------------------------------
KNOBS = {"v4_tail1": (dict(B200_V4_TAIL=1), V4_PPL1, 3), "v4_tail2": (dict(B200_V4_TAIL=2), V4_PPL1, 3),
         "v4_tail6": (dict(B200_V4_TAIL=6), V4_PPL1, 3), "v4ppl2_tail1": (dict(B200_V4_PPL=2, B200_V4_TAIL=1), V4_PPL2, 4),
         "v4_no_prefetch": (dict(B200_V3_PREFETCH=0), V4_PPL1, 3),
         "v3_no_prefetch": (dict(B200_INTEGRATE_IMPL="v3", B200_V3_PREFETCH=0), V3, 3),
         "v3_two_ctas": (dict(B200_INTEGRATE_IMPL="v3", B200_V3_CTAS=2), V3, 2)}


@pytest.mark.parametrize("knob", list(KNOBS))
def test_integrate_switches(knob):
    switches, kernel, ctas = KNOBS[knob]
    pair = run(P.Cfg(frames=4, raycast=False, decay=(1, 2)), **switches)
    assert pair.eng.last_integrate() == (kernel, ctas * sm_count())


# ---- 8. raycast dispatch ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def raycast_views():
    """a fused street and, for cameras whose principal-point row is 0, the middle row, the last row, negative and beyond the
    image, the oracle's visible list, min/max image, ray points and grey render (311 x 94: no tile shape divides it)"""
    cfg = P.Cfg(frames=4)
    pair = run(cfg)
    L = pair.L
    M = synth.kitti_pose((cfg.frames - 1) * cfg.frame_step)
    M[0, 3] += 0.3
    base = synth.kitti_intrinsics() * np.float32(cfg.scale)
    views = []
    for name, cy in (("row0", 0.0), ("middle", pair.h / 2.0), ("last", pair.h - 1.0), ("negative", -9.5), ("beyond", pair.h + 13.0)):
        proj = base.copy()
        proj[3] = cy
        ocam = H.make_camera(M, proj)
        pos = np.zeros((cfg.numBlocks, 3), dtype=np.int32)
        hrs = abi.RenderState()
        C.memmove(C.byref(hrs), C.byref(pair.host.rs), C.sizeof(hrs))
        hrs.d_visibleBlockPositions = pos.ctypes.data
        L.oracle_find_visible_blocks(C.byref(pair.host.scene), C.byref(hrs), C.byref(ocam))
        L.oracle_expected_depths(C.byref(pair.host.scene), C.byref(hrs), C.byref(ocam))
        mm = pair.host.minmax.copy()
        hc, hf = np.zeros((pair.h, pair.w, 4), dtype=np.uint8), np.zeros((pair.h, pair.w), dtype=np.float32)
        L.oracle_render_image(C.byref(pair.host.scene), C.byref(hrs), C.byref(ocam), H.vptr(hc), H.vptr(hf),
                              abi.RENDER_SHADED_GREYSCALE, 0)
        rays = pair.host.raycastResult.copy()
        assert hrs.noVisibleBlocks > 100 and (rays[..., 3] > 0).sum() > 1000, name
        views.append((name, M, proj, hrs.noVisibleBlocks, mm, rays, hc))
    return pair, views


@pytest.mark.parametrize("tile", range(6))
@pytest.mark.parametrize("order", [0, 1])
@pytest.mark.parametrize("impl", [None, "old"])
def test_raycast_dispatch(raycast_views, impl, order, tile):
    """every tile shape, both dispatch orders and both ray caches; the ray image is filled with NaN first, so a pixel the
    dispatch never writes fails the comparison"""
    pair, views = raycast_views
    with env(B200_RC_IMPL=impl, B200_RC_ORDER=order, B200_RC_TILE=tile):
        eng = E.Engine(pair.scene, (pair.w, pair.h))
    try:
        vis = E.VisualisationEngine(eng, pair.scene)
        rs = vis.CreateRenderState((pair.w, pair.h))
        dev = pair.scene.device
        for name, M, proj, n_vis, mm, rays, hc in views:
            cam = E.make_camera(M, proj)
            vis.FindVisibleBlocks(cam, rs)
            assert rs.noVisibleBlocks == n_vis, name
            vis.CreateExpectedDepths(cam, rs)
            P._cmp(f"{name}: minmax", rs.renderingRangeImage.cpu().numpy(), mm.reshape(-1))
            rs.raycastResult.fill_(float("nan"))
            oc = torch.zeros(pair.h * pair.w * 4, dtype=torch.uint8, device=dev)
            of = torch.zeros(pair.h * pair.w, dtype=torch.float32, device=dev)
            vis.RenderImage(cam, rs, oc, of, abi.RENDER_SHADED_GREYSCALE)
            P._cmp(f"{name}: rays", rs.raycastResult.cpu().numpy(), rays.reshape(-1))
            P._cmp(f"{name}: image", oc.cpu().numpy(), hc.reshape(-1))
    finally:
        eng.close()


# ---- 9. fused-frame modes ------------------------------------------------------------------------------------------
def _fused_run(cfg, frames, decay_on, colour_on, sync_at, **switches):
    """fused frames with per-frame options; frame `sync_at` is a b200_sync followed by the synchronous calls of one frame"""
    pair = make_pair(cfg, **switches)
    dev = pair.scene.device
    keep, cols = [], []
    for i, f in enumerate(frames):
        gv, _ = pair.views(*f)
        col = torch.zeros(pair.h * pair.w * 4, dtype=torch.uint8, device=dev) if colour_on[i] else None
        keep.append(gv)
        cols.append(col)
        decay = cfg.decay if decay_on[i] else None
        if i == sync_at:
            pair.eng.sync(pair.rs)
            pair.reco.AllocateSceneFromDepth(pair.scene, gv, pair.rs)
            pair.reco.IntegrateIntoScene(pair.scene, gv, pair.rs)
            pair.vis.CreateExpectedDepths(E.make_camera(f[2], f[3]), pair.rs)
            pair.vis.CreateICPMaps(gv, pair.rs, pair.points, pair.normals)
            if decay:
                pair.reco.Decay(pair.scene, pair.rs, decay[0], decay[1], False)
        else:
            pair.eng.process_frame_async(pair.rs, gv, pair.points, pair.normals, decay=decay, colour_out=col)
    pair.eng.sync(pair.rs)
    return pair, cols


def _stepwise(frames, decay_on, decay):
    cfg = P.Cfg(frames=len(frames))
    pair = P.Pair(cfg)
    for i, f in enumerate(frames):
        cfg.decay = decay if decay_on[i] else None
        pair.step(*f, i)
    return pair


def test_graph_mode_changing_topology_equals_stepwise():
    """B200_GRAPH=1 over 9 frames: decay and the colour render switched on and off (a new graph topology: the executable graph
    cannot be updated and is instantiated again), a b200_sync and a synchronous frame in the middle"""
    cfg = P.Cfg(frames=9, decay=(1, 2))
    frames = list(P.frames_of(cfg))
    decay_on = [True, True, True, False, False, True, True, True, True]
    colour_on = [False, False, True, True, False, False, True, True, False]
    stepwise = _stepwise(frames, decay_on, cfg.decay)
    graph, gcols = _fused_run(cfg, frames, decay_on, colour_on, 4, B200_GRAPH=1)
    plain, pcols = _fused_run(cfg, frames, decay_on, colour_on, 4, B200_GRAPH=None)
    assert_same_state("graph", graph, stepwise)
    assert_same_state("fused", plain, stepwise)
    for i, (a, b) in enumerate(zip(gcols, pcols)):
        if a is not None:
            assert a.cpu().numpy()[0::4].any(), i
            P._cmp(f"graph colour render, frame {i}", a.cpu().numpy(), b.cpu().numpy())


def test_no_overlap_fused_frames_equal_stepwise():
    cfg = P.Cfg(frames=6, decay=(1, 2))
    frames = list(P.frames_of(cfg))
    on = [True] * len(frames)
    stepwise = _stepwise(frames, on, cfg.decay)
    pair, _ = _fused_run(cfg, frames, on, [False] * len(frames), -1, B200_NO_OVERLAP=1)
    assert_same_state("no overlap", pair, stepwise)


def _pipelined(cfg, **switches):
    pair = make_pair(cfg, **switches)
    outs = [torch.zeros(pair.h * pair.w * 4, dtype=torch.uint8).pin_memory() for _ in range(2)]
    view, keep = None, []
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
    return pair, outs[(cfg.frames - 1) & 1].numpy()


def test_pipelined_host_frames_graph_mode_equal_stepwise():
    cfg = P.Cfg(frames=7, decay=(1, 2))
    stepwise = run(cfg)
    pair, last = _pipelined(cfg, B200_GRAPH=1)
    assert_same_state("pipelined graph", pair, stepwise)
    P._cmp("pipelined graph image", last, stepwise.rs.raycastImage.cpu().numpy())


def test_process_frame_host_equals_stepwise():
    cfg = P.Cfg(frames=5, decay=(1, 2))
    stepwise = run(cfg)
    pair = P.Pair(cfg)
    dev = pair.scene.device
    d_depth = torch.zeros((pair.h, pair.w), dtype=torch.float32, device=dev)
    d_rgb = torch.zeros((pair.h, pair.w, 4), dtype=torch.uint8, device=dev)
    out = torch.zeros(pair.h * pair.w * 4, dtype=torch.uint8).pin_memory()
    torch.cuda.synchronize(dev)
    for depth, rgb, M, proj in P.frames_of(cfg):
        hd, hc = torch.from_numpy(np.ascontiguousarray(depth)), torch.from_numpy(np.ascontiguousarray(rgb))
        view = E.View(d_depth, d_rgb, M, proj)
        pair.eng.process_frame_host(pair.rs, view, hd, hc, d_depth, d_rgb, pair.points, pair.normals, decay=cfg.decay, h_out=out)
    assert_same_state("host frames", pair, stepwise)
    P._cmp("host frame image", out.numpy(), stepwise.rs.raycastImage.cpu().numpy())


# ---- 10. the fused frame's colour and depth renders ------------------------------------------------------------------
def test_fused_renders_equal_oracle_before_decay():
    """colour_out / depth_out against the oracle's RenderImage (types 1 and 4) at the frame's pose, taken after integration
    and before decay. The decay (maxWeight >= maxW, minAge 1) empties the previous frame's blocks, most of which the current
    image sees, so the oracle's colour render after it differs: the comparison sees on which side of the decay it ran."""
    cfg = P.Cfg(frames=4, decay=(50, 1))
    pair = P.Pair(cfg)
    L, host, dev = pair.L, pair.host, pair.scene.device
    keep, sensitive = [], 0
    for i, (depth, rgb, M, proj) in enumerate(P.frames_of(cfg)):
        gv, hv = pair.views(depth, rgb, M, proj)
        col = torch.zeros(pair.h * pair.w * 4, dtype=torch.uint8, device=dev)
        dep = torch.zeros(pair.h * pair.w, dtype=torch.float32, device=dev)
        keep.append((gv, col, dep))
        pair.eng.process_frame_async(pair.rs, gv, pair.points, pair.normals, decay=cfg.decay, colour_out=col, depth_out=dep)
        pair.eng.sync(pair.rs)
        assert L.oracle_allocate_from_depth(host.engine, C.byref(host.scene), C.byref(host.rs), C.byref(hv), 0, 0) == 0
        L.oracle_integrate(host.engine, C.byref(host.scene), C.byref(host.rs), C.byref(hv), 0)
        ocam = H.make_camera(M, proj)
        L.oracle_expected_depths(C.byref(host.scene), C.byref(host.rs), C.byref(ocam))

        def render(t):
            hc, hf = np.zeros((pair.h, pair.w, 4), dtype=np.uint8), np.zeros((pair.h, pair.w), dtype=np.float32)
            L.oracle_render_image(C.byref(host.scene), C.byref(host.rs), C.byref(ocam), H.vptr(hc), H.vptr(hf), t, 0)
            return hc, hf

        colour, _ = render(abi.RENDER_COLOUR_FROM_VOLUME)
        _, depth_map = render(abi.RENDER_DEPTH_MAP)
        assert colour[..., :3].any() and (depth_map > 0).any()
        P._cmp(f"frame {i}: colour_out", col.cpu().numpy(), colour.reshape(-1))
        P._cmp(f"frame {i}: depth_out", dep.cpu().numpy(), depth_map.reshape(-1))
        L.oracle_decay(host.engine, C.byref(host.scene), C.byref(host.rs), cfg.decay[0], cfg.decay[1], 0)
        pair.compare_scene(f"frame {i} decay")
        after, _ = render(abi.RENDER_COLOUR_FROM_VOLUME)
        sensitive += int(after.tobytes() != colour.tobytes())
    assert pair.reco.GetDecayedBlockCount() > 100
    assert sensitive >= 2
