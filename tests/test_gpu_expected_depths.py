"""GPU: the stand-alone CreateExpectedDepths pass (k_expected_depths, csrc/vis.cu). It draws every listed block's box and, only
when the rendering-tile total breaks MAX_RENDERING_BLOCKS, its last CTA re-applies the ordered rule (Vis_CUDA.cu:609) and
rebuilds the image. Byte for byte against the CPU oracle: a sweep of lowered caps from 1 to above the uncapped total, on a list
built by allocation (the pass reads the fresh VBA pointers) and on one built by FindVisibleBlocks (the pass looks every block up
in the hash table); and capped and uncapped calls and previews interleaved on one engine, which the list sweep's ticket and the
pass's CTA counter, both reset by the launch that used them, must survive."""
import ctypes as C

import numpy as np
import pytest
import torch

from dynslam_b200 import abi, engine as E
from tests import hostlib as H
from tests import parity as P

pytestmark = pytest.mark.gpu
SUB, FAR_AWAY, VERY_CLOSE = 8, np.float32(999999.9), np.float32(0.05)


def rendering_tiles(pos, M, proj, w, h, voxelSize):
    """CreateRenderingBlocks' tile total of the blocks at `pos`: ProjectSingleBlock (DA/ITMVisualisationEngine.h:29-71) and the
    count of :73-91, restated in float32 in the reference's operation order. It places the caps of the sweep."""
    f = np.float32
    M, proj, vs = np.asarray(M, f), np.asarray(proj, f), f(voxelSize)
    total = 0
    for bx, by, bz in pos:
        ulx, uly, lrx, lry = w // SUB, h // SUB, -1, -1
        zmin, zmax = FAR_AWAY, VERY_CLOSE
        for corner in range(8):
            c = [f(f(f(int(b) + ((corner >> k) & 1)) * f(8)) * vs) for k, b in enumerate((bx, by, bz))]
            q = [f(f(f(f(M[r, 0] * c[0]) + f(M[r, 1] * c[1])) + f(M[r, 2] * c[2])) + M[r, 3]) for r in range(3)]
            if float(q[2]) < 1e-6:
                continue
            px = f(f(f(f(proj[0] * q[0]) / q[2]) + proj[2]) / f(SUB))
            py = f(f(f(f(proj[1] * q[1]) / q[2]) + proj[3]) / f(SUB))
            ulx, lrx = min(ulx, int(np.floor(px))), max(lrx, int(np.ceil(px)))
            uly, lry = min(uly, int(np.floor(py))), max(lry, int(np.ceil(py)))
            zmin, zmax = min(zmin, q[2]), max(zmax, q[2])
        ulx, uly, lrx, lry = max(ulx, 0), max(uly, 0), min(lrx, w - 1), min(lry, h - 1)
        if ulx > lrx or uly > lry or zmax < VERY_CLOSE:
            continue
        total += int(np.ceil(f(lrx - ulx + 1) / f(16))) * int(np.ceil(f(lry - uly + 1) / f(16)))
    return total


def _set_cap(pair, cap):
    pair.eng.set_max_rendering_blocks(cap)
    H.oracle().oracle_set_max_rendering_blocks(cap)


def _oracle(pair, M, proj, find_visible=True):
    """the oracle's (count, list, image) for the pose: of the host volume's live list, or of a list FindVisibleBlocks builds"""
    L, cam = pair.L, H.make_camera(M, proj)
    hrs = abi.RenderState()
    C.memmove(C.byref(hrs), C.byref(pair.host.rs), C.sizeof(hrs))
    pos = np.zeros((pair.cfg.numBlocks, 3), dtype=np.int32)
    if find_visible:
        hrs.d_visibleBlockPositions = pos.ctypes.data
        L.oracle_find_visible_blocks(C.byref(pair.host.scene), C.byref(hrs), C.byref(cam))
    L.oracle_expected_depths(C.byref(pair.host.scene), C.byref(hrs), C.byref(cam))
    n = hrs.noVisibleBlocks
    return n, pos[:n].copy(), pair.host.minmax.reshape(-1).copy()


@pytest.fixture(scope="module")
def street():
    cfg = P.Cfg(frames=4)
    pair, _ = P.run_sequence(cfg)            # the live render state holds the last allocation's list
    *_, (_, _, M, proj) = P.frames_of(cfg)
    yield pair, M, proj
    _set_cap(pair, 0)


def _offset(M, dx):
    M = M.copy()
    M[0, 3] += dx
    return M


@pytest.mark.parametrize("listed_by", ["allocation", "find_visible"])
def test_cap_sweep(street, listed_by):
    pair, M, proj = street
    if listed_by == "allocation":
        rs, Mv = pair.rs, M
        pos = pair.host.visiblePos[:pair.host.rs.noVisibleBlocks]
    else:
        rs, Mv = pair.vis.CreateRenderState((pair.w, pair.h)), _offset(M, 0.4)
        pair.vis.FindVisibleBlocks(E.make_camera(Mv, proj), rs)
        n, pos, _ = _oracle(pair, Mv, proj)
        assert rs.noVisibleBlocks == n
        P._cmp("FindVisibleBlocks list", rs.visibleBlockPositions.cpu().numpy().reshape(-1, 3)[:n], pos)
    total = rendering_tiles(pos, Mv, proj, pair.w, pair.h, pair.cfg.voxelSize)
    assert len(pos) > 200 and total > 300, (len(pos), total)
    caps = sorted({1, 2, 3, 7, 31, 100, total // 8, total // 3, total // 2, total - 2, total - 1, total, total + 1, 2 * total})
    cam, images = E.make_camera(Mv, proj), {}
    try:
        for cap in caps + [0]:                # 0: MAX_RENDERING_BLOCKS itself
            _set_cap(pair, cap)
            pair.vis.CreateExpectedDepths(cam, rs)
            got = rs.renderingRangeImage.cpu().numpy()
            P._cmp(f"{listed_by}: cap {cap} of {total} tiles", got, _oracle(pair, Mv, proj, find_visible=listed_by == "find_visible")[2])
            images[cap] = got.tobytes()
    finally:
        _set_cap(pair, 0)
    live = lambda b: int((np.frombuffer(b, np.float32).reshape(-1, 2)[:, 0] < 999999.0).sum())
    assert images[total] == images[2 * total] == images[0]          # at and above the total nothing is dropped
    assert 0 < live(images[total // 3]) < live(images[0])           # below it the rule bites


def test_interleaved_capped_calls_and_previews(street):
    """Stand-alone calls (synchronous) and previews (enqueued, not waited for) one after the other on one engine, the cap
    changing between them; every result is compared once all have run."""
    pair, M, proj = street
    pos = pair.host.visiblePos[:pair.host.rs.noVisibleBlocks]
    total = rendering_tiles(pos, M, proj, pair.w, pair.h, pair.cfg.voxelSize)
    runs = []
    try:
        for i, cap in enumerate([total // 3, 0, 5, total // 2, 0, total + 1, 1]):
            Mv = _offset(M, 0.1 * (i % 3))
            cam = E.make_camera(Mv, proj)
            _set_cap(pair, cap)
            want = _oracle(pair, Mv, proj)
            calls = pair.vis.CreateRenderState((pair.w, pair.h))
            pair.vis.FindVisibleBlocks(cam, calls)
            pair.vis.CreateExpectedDepths(cam, calls)
            runs.append((f"call {i} (cap {cap})", calls, want, calls.renderingRangeImage.cpu().numpy()))
            view = pair.vis.CreateRenderState((pair.w, pair.h))
            dep = torch.zeros(pair.h * pair.w, dtype=torch.float32, device=pair.scene.device)
            pair.vis.RenderFreeView(cam, view, None, dep, abi.RENDER_COLOUR_FROM_VOLUME, sync=False)
            runs.append((f"preview {i} (cap {cap})", view, want, dep))   # dep: kept alive until the preview has run
        pair.vis.RenderFreeViewSync(runs[-1][1])
    finally:
        _set_cap(pair, 0)
    for tag, rs, (n, lst, mm), image in runs:
        got = rs.renderingRangeImage.cpu().numpy() if isinstance(image, torch.Tensor) else image
        P._cmp(f"{tag}: list", rs.visibleBlockPositions.cpu().numpy().reshape(-1, 3)[:n], lst)
        P._cmp(f"{tag}: minmax", got, mm)
