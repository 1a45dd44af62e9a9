"""Voxel decay on three executors from identical inputs: the oracle, the engine (bit for bit) and the reference's own
ITMSceneReconstructionEngine_CUDA::Decay through oracle/_ref/libitmharness.so (bit for bit up to the order in which it pushes
freed blocks). The cases (tests/decaylib.py) seed a state, decay-queue snapshots and a frame index; they reach the branches
the street sequences only reach by chance: a deleted bucket head with a successor, middle and tail deletions, blocks younger
than minAge, w_depth == maxWeight and maxWeight + 1, stale zero-weight blocks, maxWeight 0 and 255, minAge 0, empty snapshots,
a queue exactly minAge deep, catch-up, ResetScene in the middle of a sequence and the allocation that follows deletions.
The reference's outcomes are also pinned in tests/golden/ref_pins.json for the CPU suite (test_oracle_vs_ref.py)."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import decaylib as D
from tests import harnesslib as HL
from tests import parity, refpins

NAMES = list(D.pinned_cases())
NO_REF = ("oracle/_ref/libitmharness.so is not built or predates the decay entry points (oracle/build_ref.sh): the reference "
          "legs do not run, the oracle stays pinned to the reference's recorded outcomes")


class GpuRun:
    """the engine on a decay case (one scene, engine and render state for the module)"""

    def __init__(self):
        from dynslam_b200 import engine as E
        p = E.SceneParams(0.05, 0.75, 50, 0.1, 300.0, False)
        self.scene = E.Scene(p, D.NUM_BLOCKS, D.NB, D.NE)
        self.eng = E.Engine(self.scene, D.IMG)
        self.reco = E.SceneReconstructionEngine(self.eng)
        self.rs = E.VisualisationEngine(self.eng, self.scene).CreateRenderState(D.IMG)

    def load(self, st):
        s, dev = self.scene, self.scene.device
        self.reco.ResetScene(s)
        for t, a in ((s.hash, st["hash"]), (s.voxels, st["voxels"]), (s.allocationList, st["allocationList"]),
                     (s.excessList, st["excessList"]), (self.rs.entriesVisibleType, st["visType"])):
            t.copy_(torch.from_numpy(np.ascontiguousarray(a).view(np.uint8)).view(t.dtype).reshape(t.shape).to(dev))
        s.c.lastFreeBlockId, s.c.lastFreeExcessListId = st["lastFreeBlockId"], st["lastFreeExcessListId"]

    def push(self, pos):
        self.eng.push_decay_snapshot(torch.from_numpy(np.ascontiguousarray(pos, np.int32).reshape(-1, 3)))

    def frame(self, f):
        self.eng.set_frame_index(f)

    def decay(self, maxWeight, minAge, forceAll):
        self.reco.Decay(self.scene, self.rs, maxWeight, minAge, forceAll)
        return int(self.reco.GetDecayedBlockCount())

    def state(self):
        g = self.scene.to_host()
        g["visType"] = self.rs.to_host()["visType"]
        return g


class RefRun:
    """the reference's CUDA engine on a decay case"""

    def __init__(self):
        self.h = HL.Harness(HL.REFERENCE_CUDA, D.IMG[0], D.IMG[1], D.PROJ, numBlocks=D.NUM_BLOCKS)
        assert self.h.noTotal == D.NB + D.NE

    def load(self, st):
        self.h.upload_state(st["hash"], st["voxels"], st["allocationList"], st["excessList"], st["visType"], st["lastFreeBlockId"],
                            st["lastFreeExcessListId"])

    def push(self, pos):
        self.h.push_snapshot(pos)

    def frame(self, f):
        self.h.set_frame_index(f)

    def decay(self, maxWeight, minAge, forceAll):
        return self.h.decay(maxWeight, minAge, forceAll)

    def state(self):
        return self.h.download_state(D.NE)


@pytest.fixture(scope="module")
def gpu():
    return GpuRun()


@pytest.fixture(scope="module")
def ref():
    if not HL.decay_available():
        pytest.skip(NO_REF)
    r = RefRun()
    yield r
    r.h.close()


def _same(tag, a, b):
    parity._cmp(tag, a, b)


def compare_exact(tag, got, want, decayed_got, decayed_want):
    """the engine against the oracle: every byte of the state"""
    assert (got["lastFreeBlockId"], got["lastFreeExcessListId"], decayed_got) == \
        (want["lastFreeBlockId"], want["lastFreeExcessListId"], decayed_want), tag
    for k in ("hash", "visType", "allocationList", "excessList", "voxels"):
        _same(f"{tag}: {k}", got[k], want[k])


def compare_reference(tag, got, want, sections, decayed_got, decayed_want):
    """the reference against the oracle: bit for bit, except that each freed section of the allocation list is compared as a
    multiset (the reference pushes with atomicAdd) and the rest of the list must be unchanged"""
    assert (got["lastFreeBlockId"], got["lastFreeExcessListId"], decayed_got) == \
        (want["lastFreeBlockId"], want["lastFreeExcessListId"], decayed_want), tag
    for k in ("hash", "visType", "excessList", "voxels"):
        _same(f"{tag}: {k}", got[k], want[k])
    _same(f"{tag}: allocationList (freed sections sorted)", D.canonical(got, sections), D.canonical(want, sections))


def check_branches(name, o):
    """the branch each case targets really ran (the oracle's counters and layouts)"""
    calls = o.calls
    br = calls[-1]["branches"]
    if name.startswith("crafted/partial"):
        c = calls[-1]
        assert c["popped"] and br["head_with_successor"] == 1 and br["excess_entry"] == 2 and br["age_skip"] == 1, br
        assert br["head_alone"] == 3, br          # w_depth == maxWeight, zero weights with stale contents, age == minAge
        # the head-with-successor chain: the successor moved into the bucket with its own visibility byte (11), its slot cleared
        pre, post = c["pre"]["hash"], c["post"]["hash"]
        moved = [b for b, ch in D.chains(pre).items() if len(ch) == 2 and post["ptr"][ch[1]] == -2 and post["ptr"][b] >= 0]
        assert len(moved) == 1
        b, nxt = moved[0], D.chains(pre)[moved[0]][1]
        assert tuple(post["pos"][b]) == tuple(pre["pos"][nxt]) and c["post"]["visType"][b] == 11 and c["post"]["visType"][nxt] == 0
        assert post["offset"][nxt] == 0
    elif name.startswith("crafted/full"):
        assert br["head_alone"] == 3 and br["head_with_successor"] == br["excess_entry"] == 0 and br["age_skip"] == 1, br
    elif name.startswith("street/partial"):
        assert calls[-1]["popped"] and len(calls[-1]["freed"]) > 0, br
        if "mw0_" not in name:
            assert br["voxel_reset"] > 0 and br["head_with_successor"] > 0, br
    elif name.startswith("street/full"):
        assert len(calls[-1]["freed"]) > 0 and br["voxel_reset"] > 0, br
        assert "age2" not in name or br["age_skip"] > 0, br


def check_queue(kind, o, blocks):
    """which of X, Y, Z each Decay reached"""
    def present(call, k):
        return D.entry_of(call["post"], blocks[k]) >= 0
    c = o.calls
    if kind == "depth":
        assert not c[0]["popped"] and len(c[0]["freed"]) == 0                 # 2 snapshots queued, minAge 2: nothing
        assert c[1]["popped"] and not present(c[1], "X") and present(c[1], "Y")   # minAge 1: the oldest (A) goes
    elif kind == "empty":
        assert c[0]["popped"] and len(c[0]["snapshot"]) == 0 and len(c[0]["freed"]) == 0 and present(c[0], "Y")
        assert c[1]["popped"] and not present(c[1], "Y")
    elif kind == "catchup":
        assert [len(x["freed"]) for x in c] == [1, 1, 1] and not any(present(c[2], k) for k in "XYZ")
    elif kind == "reset":
        assert present(c[0], "X") and not present(c[0], "Y")


def run_case(name, gpu, ref):
    st, ops = D.pinned_cases()[name]()
    o = D.run_oracle(st, ops)
    check_branches(name, o)
    if name.startswith("queue/"):
        check_queue(name.split("/")[1], o, D.queue_case(name.split("/")[1])[2])
    sections = D.sections_of(o)

    def gpu_after(i, ex, n):
        compare_exact(f"{name} decay {i}: engine", ex.state(), o.calls[i]["post"], n, o.calls[i]["decayed"])
    D.run(gpu, st, ops, after_decay=gpu_after)
    if ref is None:
        return
    got = {}

    def ref_after(i, ex, n):
        s = ex.state()
        compare_reference(f"{name} decay {i}: reference", s, o.calls[i]["post"], sections[:i + 1], n, o.calls[i]["decayed"])
        got["last"] = (s, n)
    D.run(ref, st, ops, before_decay=lambda i: D.check_reference_input(o.calls[i]), after_decay=ref_after)
    s, n = got["last"]
    refpins.check(D.pin_key(name), D.outcome_bytes(o.calls[-1]["post"], sections, o.calls[-1]["decayed"]),
                  D.outcome_bytes(s, sections, n))


@pytest.mark.gpu
@pytest.mark.parametrize("name", NAMES)
def test_decay_engine_and_reference_equal_oracle(name, gpu, request):
    ref = request.getfixturevalue("ref") if HL.decay_available() else None     # the engine leg runs in any case
    run_case(name, gpu, ref)


@pytest.mark.gpu
def test_reference_cases_are_run():
    """the three-way cases above ran the reference: its queue took the pushes and Decay freed blocks (skipped, and so
    reported, where oracle/_ref/libitmharness.so lacks the decay entry points)"""
    if not HL.decay_available():
        pytest.skip(NO_REF)
    r = RefRun()
    st, ops, _ = D.queue_case("depth")
    r.load(st)
    r.push(ops[0][1])
    r.push(ops[1][1])
    assert r.h.queue_size() == 2
    r.frame(10)
    assert r.decay(3, 1, False) == 1 and r.h.queue_size() == 1
    r.h.close()


def test_reference_guard_rejects_chain_mate_inputs():
    """check_reference_input refuses, before the reference runs, a snapshot with two positions in one bucket and a full
    decay that deletes a member of a multi-entry chain (CPU only: the reference stands in as an executor that must not be
    called)"""
    class MustNotRun:
        def load(self, st):
            pass

        def push(self, pos):
            pass

        def frame(self, f):
            pass

        def decay(self, *a):
            raise AssertionError("the reference ran on an input the guard must refuse")

    st, ops = D.crafted_case(3, 0)
    grp = D.colliding_positions(2, 1, 5)[0]
    bad_partial = [("push", np.concatenate([ops[0][1], grp])), ("frame", 20), ("decay", 3, 0, False)]
    bad_full = [("frame", 20), ("decay", 3, 0, True)]      # crafted_case(full=False) has empty-able chain members
    for bad in (bad_partial, bad_full):
        o = D.run_oracle(st, bad)
        with pytest.raises(AssertionError, match="race"):
            D.run(MustNotRun(), st, bad, before_decay=lambda i: D.check_reference_input(o.calls[i]))
    # and every pinned case passes it
    for name in ("crafted/partial/mw3_age2", "crafted/full/mw3_age2", "queue/reset"):
        o = D.run_oracle(*D.pinned_cases()[name]())
        for c in o.calls:
            D.check_reference_input(c)


# ---- oracle against engine on real sequences -------------------------------------------------------------------------

def _deleted(pair_state_before, pair_state_after):
    """bucket heads that lost their block and the VBA blocks freed between two oracle states"""
    hb, ha = pair_state_before["hash"], pair_state_after["hash"]
    n = hb.shape[0] - pair_state_before["excessList"].shape[0]
    heads = set(np.nonzero((hb["ptr"][:n] >= 0) & (ha["ptr"][:n] == -2))[0].tolist())
    a, b = pair_state_before["lastFreeBlockId"], pair_state_after["lastFreeBlockId"]
    return heads, set(pair_state_after["allocationList"][a + 1:b + 1].tolist())


@pytest.mark.gpu
def test_follow_on_allocation_reuses_freed_blocks():
    """After a decay deletes blocks, the next allocation takes freed VBA blocks from the top of the free list and re-fills
    bucket heads left at ptr == -2; the engine does both exactly as the oracle (Pair.step compares every stage)."""
    cfg = parity.Cfg(frames=7)            # Decay(3, 1) runs below, after each step
    pair = parity.Pair(cfg)
    L = pair.L
    seen, pending = dict(heads=0, blocks=0), {}

    def on_allocated(p, hv):
        if pending:
            hs = p.host.state()["hash"]
            seen["heads"] += sum(1 for i in pending["heads"] if hs["ptr"][i] >= 0)
            seen["blocks"] += len(pending["blocks"] & set(hs["ptr"][hs["ptr"] >= 0].tolist()))
    for i, (depth, rgb, M, proj) in enumerate(parity.frames_of(cfg)):
        pair.step(depth, rgb, M, proj, i, on_allocated=on_allocated)
        before = pair.host.state()
        pair.reco.Decay(pair.scene, pair.rs, 3, 1, False)
        L.oracle_decay(pair.host.engine, C.byref(pair.host.scene), C.byref(pair.host.rs), 3, 1, 0)
        pair.compare_scene(f"frame {i} decay")
        pending["heads"], pending["blocks"] = _deleted(before, pair.host.state())
    assert seen["blocks"] > 0 and seen["heads"] > 0, seen


@pytest.mark.gpu
def test_reset_scene_mid_sequence():
    """ResetScene between frames empties the decay queue and keeps the frame index running (Reco_CUDA.cu:145-172): the
    frames after it allocate with the continued allocatedTime and decay from the fresh queue, on the engine as on the oracle"""
    cfg = parity.Cfg(frames=7, decay=(3, 1))
    pair = parity.Pair(cfg)
    L = pair.L
    frames = list(parity.frames_of(cfg))
    for i, (depth, rgb, M, proj) in enumerate(frames[:3]):
        pair.step(depth, rgb, M, proj, i)
    assert L.oracle_queue_size(pair.host.engine) == 1
    pair.reco.ResetScene(pair.scene)
    L.oracle_reset_scene(pair.host.engine, C.byref(pair.host.scene))
    pair.compare_scene("after ResetScene")
    assert L.oracle_queue_size(pair.host.engine) == 0 and L.oracle_frame_index(pair.host.engine) == pair.eng.frameIdx == 3
    freed = 0
    for i, (depth, rgb, M, proj) in enumerate(frames[3:], start=3):
        pair.step(depth, rgb, M, proj, i)
        freed = L.oracle_decayed_block_count(pair.host.engine)
    hs = pair.host.state()["hash"]
    assert hs["allocatedTime"][hs["ptr"] >= 0].min() >= 3        # everything now in the map was allocated after the reset
    assert freed > 0 and pair.reco.GetDecayedBlockCount() == freed
