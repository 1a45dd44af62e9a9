"""Checkpoints on the engine (b200_checkpoint_save / b200_checkpoint_load): an engine that loads a checkpoint into buffers full of
garbage continues bit for bit like the engine that saved it, at every point of the decay queue's life, through the fused and
the ITMLib-shaped paths; its bytes equal the CPU oracle's; saves are deterministic; every rejection leaves the target alone."""
import ctypes as C

import numpy as np
import pytest
import torch

from dynslam_b200 import abi, formats
from dynslam_b200 import engine as E
from tests import checkpointlib as K
from tests import decaylib as D
from tests.parity import Cfg
from tests.test_checkpoint_oracle import rejection_cases

pytestmark = pytest.mark.gpu

NB, NBK, NEX = 16384, 0x4000, 0x2000
SCALE = 0.25


@pytest.fixture(scope="module")
def frames():
    return K.street_frames(10, scale=SCALE)


class Vol:
    """one engine with its scene and render state; fill: byte the caller's buffers hold instead of a reset volume"""

    def __init__(self, w, h, forward=False, swap=False, ring=0, fill=None, device="cuda:0", geometry=(NB, NBK, NEX),
                 params=None):
        self.scene = E.Scene(params or E.SceneParams(), *geometry, device=device, useSwapping=swap)
        self.eng = E.Engine(self.scene, (w, h), decayRingItems=ring)
        self.reco = E.SceneReconstructionEngine(self.eng)
        self.vis = E.VisualisationEngine(self.eng, self.scene)
        self.rs = self.vis.CreateRenderState((w, h), forward=forward)
        self.points = torch.zeros(h * w * 4, dtype=torch.float32, device=self.scene.device)
        self.normals = torch.zeros_like(self.points)
        if fill is None:
            self.reco.ResetScene(self.scene)
        else:
            for t in self.buffers().values():
                t.fill_(fill)
            torch.cuda.synchronize()

    def buffers(self):
        s, r = self.scene, self.rs
        d = dict(voxels=s.voxels, hash=s.hash, allocationList=s.allocationList, excessList=s.excessList,
                 visType=r.entriesVisibleType, visible=r.visibleBlockPositions, minmax=r.renderingRangeImage, rays=r.raycastResult,
                 image=r.raycastImage, points=self.points, normals=self.normals)
        if s.swapStates is not None:
            d["swap"] = s.swapStates
        if r.forwardProjection is not None:
            d.update(fwd=r.forwardProjection, fwdMissing=r.fwdProjMissingPoints)
        return d

    def view(self, depth, rgb, M, proj, full=True):
        dev = self.scene.device
        return E.View(torch.from_numpy(np.ascontiguousarray(depth)).to(dev), torch.from_numpy(np.ascontiguousarray(rgb)).to(dev), M, proj,
                      requiresFullRendering=full)

    def run(self, frames, path, decay, full=True):
        views = []      # the frames' device images stay allocated until the engine's stream has finished with them
        for depth, rgb, M, proj in frames:
            v = self.view(depth, rgb, M, proj, full)
            views.append(v)
            if path == "fused":
                self.eng.process_frame_async(self.rs, v, self.points, self.normals, decay=decay)
            else:
                self.reco.AllocateSceneFromDepth(self.scene, v, self.rs)
                self.reco.IntegrateIntoScene(self.scene, v, self.rs)
                cam = E.make_camera(M, proj)
                self.vis.CreateExpectedDepths(cam, self.rs)
                self.vis.CreateICPMaps(v, self.rs, self.points, self.normals)
                if self.rs.forwardProjection is not None:
                    self.vis.ForwardRender(v, self.rs)
                if decay is not None:
                    self.reco.Decay(self.scene, self.rs, decay[0], decay[1], False)
        self.eng.sync(self.rs)
        del views

    def state(self, outputs=True):
        """every byte of state (the visible list up to its count), the counters; outputs: also this frame's ICP maps"""
        self.eng.sync(self.rs)
        torch.cuda.synchronize()
        d = {k: t.cpu().numpy().copy() for k, t in self.buffers().items() if outputs or k not in ("points", "normals")}
        d["visible"] = d["visible"].reshape(-1, 3)[:max(self.rs.noVisibleBlocks, 0)].copy()
        st = self.eng.stats()
        d.update(lastFree=self.scene.lastFreeBlockId, lastFreeExcess=self.scene.lastFreeExcessListId, noVisible=self.rs.noVisibleBlocks,
                 noFwd=self.rs.c.noFwdProjMissingPoints, frame=self.eng.frameIdx, decayed=int(self.reco.GetDecayedBlockCount()),
                 dropped=int(st.droppedSnapshots))
        return d


def resume(frames, k, m, path="fused", decay=(3, 3), before_save=None, **kw):
    """A runs frames 0..k, saves, runs k..k+m; B (garbage buffers) loads and runs k..k+m. Returns (checkpoint, header)."""
    h, w = frames[0][0].shape
    full = kw.pop("full", True)
    a = Vol(w, h, **kw)
    a.run(frames[:k], path, decay, full)
    if before_save is not None:
        before_save(a)
    buf = a.eng.save_checkpoint(a.scene, a.rs)
    assert a.eng.save_checkpoint(a.scene, a.rs).tobytes() == buf.tobytes()           # two saves of one state
    at_save = a.state(outputs=False)
    b = Vol(w, h, fill=0xA5, **kw)
    b.eng.load_checkpoint(b.scene, b.rs, buf)
    K.assert_same(at_save, b.state(outputs=False), "right after the load: ")
    assert b.eng.save_checkpoint(b.scene, b.rs).tobytes() == buf.tobytes()           # save -> load -> save
    a.run(frames[k:k + m], path, decay, full)
    b.run(frames[k:k + m], path, decay, full)
    K.assert_same(a.state(), b.state(), f"after frame {k + m}: ")
    return buf, formats.checkpoint_header(buf)


# minAge 3: before the queue reaches it (2), at it (3), after it pops (5)
@pytest.mark.parametrize("k", [0, 2, 3, 5])
def test_resume_fused(frames, k):
    _, hdr = resume(frames, k, 4)
    assert hdr["noSnapshots"] == min(k, 3) and hdr["frameIdx"] == k
    if k == 5:
        assert hdr["totalDecayed"] > 0


@pytest.mark.parametrize("path", ["fused", "sync"])
def test_fork_reloads_an_earlier_frame(frames, path):
    """Run to k+m, load the checkpoint of frame k into the same engine (its frame index and request keys are ahead of the
    checkpoint's) and rerun k..k+m: every byte equals the first pass."""
    h, w = frames[0][0].shape
    a = Vol(w, h)
    a.run(frames[:4], path, (3, 3))
    buf = a.eng.save_checkpoint(a.scene, a.rs)
    a.run(frames[4:8], path, (3, 3))
    first = a.state()
    a.eng.load_checkpoint(a.scene, a.rs, buf)
    assert a.eng.frameIdx == 4
    a.run(frames[4:8], path, (3, 3))
    K.assert_same(first, a.state(), "rerun after reloading frame 4: ")


def test_size_query_sees_caller_writes(frames):
    """a block the caller writes directly, which the engine cannot see, is in the next save (its size query classifies again)"""
    h, w = frames[0][0].shape
    a = Vol(w, h)
    a.run(frames[:3], "fused", (3, 3))
    hdr = formats.checkpoint_header(a.eng.save_checkpoint(a.scene, a.rs))
    vox = a.scene.voxels.view(-1, 4096)
    pristine = np.nonzero((vox.cpu().numpy() == np.tile(np.array([255, 127, 0, 0, 0, 0, 0, 0], np.uint8), 512)).all(1))[0]
    vox[int(pristine[-1]), 3] = 7                       # the colour of one voxel of a free, reset block
    torch.cuda.synchronize()
    buf = a.eng.save_checkpoint(a.scene, a.rs)
    hdr2 = formats.checkpoint_header(buf)
    assert hdr2["noBlocks"] == hdr["noBlocks"] + 1
    ids = buf[hdr2["sections"]["BLOCK_IDS"][0]:][:4 * hdr2["noBlocks"]].view(np.uint32)
    assert int(pristine[-1]) in ids.tolist()


def test_resume_synchronous_calls(frames):
    resume(frames, 5, 4, path="sync")


def test_resume_graph(frames, monkeypatch):
    monkeypatch.setenv("B200_GRAPH", "1")
    resume(frames, 5, 4)


def test_resume_after_reap(frames):
    _, hdr = resume(frames, 4, 4, before_save=lambda a: a.reco.Decay(a.scene, a.rs, 3, 0, True))
    assert hdr["totalDecayed"] > 0


def test_resume_approximate_integration(frames):
    _, hdr = resume(frames, 4, 4, path="sync", full=False, forward=True)
    assert hdr["flags"] & abi.CK_HAS_FORWARD


def test_resume_swap_states(frames):
    def pattern(a):
        a.scene.swapStates.copy_(torch.arange(a.scene.swapStates.numel(), device=a.scene.device).remainder(3).to(torch.uint8))
    _, hdr = resume(frames, 4, 3, swap=True, before_save=pattern)
    assert hdr["flags"] & abi.CK_HAS_SWAP_STATES


def test_resume_overwritten_snapshot(frames):
    """ring of numBlocks items: a snapshot of numBlocks positions pushed after three frames overwrites their snapshots; they are
    saved as overwritten, and after the load their Decay sweeps nothing and counts them as dropped, as in the saving engine"""
    def big_snapshot(a):
        pos = a.rs.visibleBlockPositions.view(-1, 3)[:a.rs.noVisibleBlocks]
        a.eng.push_decay_snapshot(pos.repeat(NB // pos.shape[0] + 1, 1)[:NB])
    buf, hdr = resume(frames, 3, 5, decay=(3, 2), ring=NB, before_save=big_snapshot)
    qc = hdr["sections"]["QUEUE_COUNTS"][0]
    counts = buf[qc:qc + 4 * hdr["noSnapshots"]].view(np.int32)
    assert counts[0] == -1 and counts[-1] == NB, counts


def test_dirty_free_block():
    """Decay frees a block whose voxels have w_depth 0 but keep sdf and colour; allocation does not clear it. The checkpoint keeps
    it, and the allocation after the load that reuses it matches the saving engine's."""
    st, ops = D.crafted_case(3, 2)
    w, h = D.IMG
    a = Vol(w, h, geometry=(D.NUM_BLOCKS, D.NB, D.NE))
    s = a.scene
    for t, arr in ((s.hash, st["hash"]), (s.voxels, st["voxels"]), (s.allocationList, st["allocationList"]),
                   (s.excessList, st["excessList"]), (a.rs.entriesVisibleType, st["visType"])):
        t.copy_(torch.from_numpy(np.ascontiguousarray(arr).view(np.uint8)).view(t.dtype).reshape(t.shape).to(s.device))
    s.c.lastFreeBlockId, s.c.lastFreeExcessListId = st["lastFreeBlockId"], st["lastFreeExcessListId"]
    before = s.c.lastFreeBlockId
    for op in ops:
        if op[0] == "push":
            a.eng.push_decay_snapshot(torch.from_numpy(np.ascontiguousarray(op[1], np.int32).reshape(-1, 3)))
        elif op[0] == "frame":
            a.eng.set_frame_index(op[1])
        else:
            a.reco.Decay(s, a.rs, op[1], op[2], op[3])
    vox = s.voxels.cpu().numpy().view(abi.VOXEL_DTYPE).reshape(-1, 512)
    freed = s.allocationList.cpu().numpy()[before + 1:s.c.lastFreeBlockId + 1]
    dirty = [int(p) for p in freed if (vox[p]["w_depth"] == 0).all() and (vox[p]["sdf"] != 32767).any()]
    assert dirty, "the case frees no block with stale contents"
    buf = a.eng.save_checkpoint(s, a.rs)
    hdr = formats.checkpoint_header(buf)
    ids = buf[hdr["sections"]["BLOCK_IDS"][0]:][:4 * hdr["noBlocks"]].view(np.uint32)
    assert set(dirty) <= set(ids.tolist())
    b = Vol(w, h, fill=0xA5, geometry=(D.NUM_BLOCKS, D.NB, D.NE))
    b.eng.load_checkpoint(b.scene, b.rs, buf)
    K.assert_same(a.state(outputs=False), b.state(outputs=False))
    # the next allocation hands the freed blocks out again (from the top of the free list)
    yy, xx = np.mgrid[0:h, 0:w]
    depth = (0.6 + 0.35 * xx + 0.2 * yy).astype(np.float32)
    rgb = np.full((h, w, 4), 200, np.uint8)
    for v in (a, b):
        v.run([(depth, rgb, np.eye(4, dtype=np.float32), np.array(D.PROJ, np.float32))], "sync", None)
    sa = a.state()
    ptrs = set(np.frombuffer(sa["hash"].tobytes(), abi.HASH_ENTRY_DTYPE)["ptr"].tolist())
    assert ptrs & set(dirty), "no stale block was handed out again"
    K.assert_same(sa, b.state())


def test_engine_bytes_equal_oracle(frames):
    h, w = frames[0][0].shape
    cfg = Cfg(scale=SCALE, numBlocks=NB, numBuckets=NBK, excessSize=NEX)
    vol = K.host_volume(cfg, w, h)
    vol.rs.d_forwardProjection = None               # the engine's render state has no forward buffers here
    g = Vol(w, h)
    for f in frames[:7]:
        K.oracle_frame(vol, *f, (3, 2))
    g.run(frames[:7], "sync", (3, 2))
    assert g.eng.save_checkpoint(g.scene, g.rs).tobytes() == K.oracle_save(vol).tobytes()


def test_rejections(frames):
    h, w = frames[0][0].shape
    a = Vol(w, h, forward=True)
    a.run(frames[:5], "fused", (3, 2))
    buf = a.eng.save_checkpoint(a.scene, a.rs)
    b = Vol(w, h, forward=True)
    b.run(frames[:2], "fused", (3, 2))
    before = b.state(outputs=False)
    for name, (bad, _) in rejection_cases(buf, formats.checkpoint_header(buf)).items():
        with pytest.raises(ValueError):
            b.eng.load_checkpoint(b.scene, b.rs, bad)
        K.assert_same(before, b.state(outputs=False), f"{name}: ")
    # the target's geometry or optional buffers differ
    with pytest.raises(ValueError, match="forward"):
        c = Vol(w, h)
        c.eng.load_checkpoint(c.scene, c.rs, buf)
    # capacity below the size
    n = C.c_size_t()
    small = np.zeros(100, np.uint8)
    rc = a.eng.lib.b200_checkpoint_save(a.eng.h, C.byref(a.scene.c), C.byref(a.rs.c), small.ctypes.data, small.size, C.byref(n))
    assert rc == abi.ERR_INVALID and n.value == buf.size and not small.any()
    # a host-frame slot not yet waited for
    depth, rgb, M, proj = frames[2]
    v = b.view(depth, rgb, M, proj)
    hd, hc = torch.from_numpy(np.ascontiguousarray(depth)).pin_memory(), torch.from_numpy(np.ascontiguousarray(rgb)).pin_memory()
    b.eng.host_frame_submit(b.rs, v, hd, hc, b.points, b.normals, decay=(3, 2), slot=0)
    with pytest.raises(ValueError, match="outstanding"):
        b.eng.load_checkpoint(b.scene, b.rs, buf)
    b.eng.host_frame_wait(0)
    b.eng.load_checkpoint(b.scene, b.rs, buf)
    assert b.eng.save_checkpoint(b.scene, b.rs).tobytes() == buf.tobytes()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_other_gpu(frames):
    h, w = frames[0][0].shape
    a = Vol(w, h)
    a.run(frames[:5], "fused", (3, 3))
    buf = a.eng.save_checkpoint(a.scene, a.rs)
    b = Vol(w, h, fill=0xA5, device="cuda:1")
    b.eng.load_checkpoint(b.scene, b.rs, buf)
    a.run(frames[5:9], "fused", (3, 3))
    b.run(frames[5:9], "fused", (3, 3))
    K.assert_same(a.state(), b.state())
