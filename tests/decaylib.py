"""Voxel-decay cases and the executors that run them (test infrastructure).

A case is a state S (hash table, voxel block array, allocation list, excess list, visibility bytes, the two free-list
cursors) and a list of operations on the decay queue: push a snapshot of block positions, set the frame index, reload S
(ResetScene + S, which empties the queue and keeps the frame index), Decay(maxWeight, minAge, forceAll). The same case runs
on the CPU oracle, on the engine (tests/test_gpu_decay.py) and on the reference's own CUDA Decay through
oracle/_ref/libitmharness.so, so the three start every call from identical inputs.

The reference's deleteBlock rewrites chain entries while other CTAs walk the same chain without a lock
(ITMSceneReconstructionEngine_CUDA.cu:1025-1111), so it is only run on inputs where no CTA can meet a chain another CTA
changes: `check_reference_input` enforces that before every reference call, from the oracle's outcome of the same call.
"""
import ctypes as C
import hashlib

import numpy as np

from dynslam_b200 import abi, synth
from tests import hostlib as H

# the reference's table sizes are compile-time constants (ITMLibDefines.h:42, :52)
NB, NE, NUM_BLOCKS = 0x100000, 0x80000, 32768
IMG = (8, 8)            # the render state's images are not used by Decay
PROJ = (5.0, 5.0, 4.0, 4.0)     # intrinsics of the harness's unused camera
STREET_FRAMES = 5


def hash_index(p):
    p = np.asarray(p, np.int64).reshape(-1, 3).astype(np.uint32)
    h = (p[:, 0] * np.uint32(73856093)) ^ (p[:, 1] * np.uint32(19349669)) ^ (p[:, 2] * np.uint32(83492791))
    return (h & np.uint32(NB - 1)).astype(np.int64)


def reset_state():
    """ResetScene's state (Reco_CUDA.cu:145-172)"""
    hs = np.zeros(NB + NE, abi.HASH_ENTRY_DTYPE)
    hs["ptr"] = -2
    vox = np.zeros(NUM_BLOCKS * 512, abi.VOXEL_DTYPE)
    vox["sdf"] = 32767
    return dict(hash=hs, voxels=vox, allocationList=np.arange(NUM_BLOCKS, dtype=np.int32), excessList=np.arange(NE, dtype=np.int32),
                visType=np.zeros(NB + NE, np.uint8), lastFreeBlockId=NUM_BLOCKS - 1, lastFreeExcessListId=NE - 1)


def copy_state(st):
    return {k: (v.copy() if isinstance(v, np.ndarray) else v) for k, v in st.items()}


def chains(hs):
    """bucket -> list of entry indices along its chain (allocated or not, as findVoxel walks it)"""
    out = {}
    for b in np.nonzero((hs["ptr"][:NB] >= 0) | (hs["offset"][:NB] >= 1))[0]:
        idx, c = int(b), []
        while True:
            c.append(idx)
            if hs["offset"][idx] < 1:
                break
            idx = NB + int(hs["offset"][idx]) - 1
        out[int(b)] = c
    return out


# ---- crafted states --------------------------------------------------------------------------------------------------

def colliding_positions(k, n, seed):
    """n groups of k block positions that share a hash bucket, every group in a bucket of its own"""
    rng = np.random.default_rng(seed)
    g = np.stack(np.meshgrid(*[np.arange(-48, 48)] * 3, indexing="ij"), -1).reshape(-1, 3)
    g = g[rng.permutation(len(g))]
    b = hash_index(g)
    order = np.argsort(b, kind="stable")
    bs = b[order]
    starts = np.r_[0, np.nonzero(np.diff(bs))[0] + 1]
    counts = np.diff(np.r_[starts, len(bs)])
    groups = [g[order[s:s + k]] for s, c in zip(starts, counts) if c >= k]
    return [groups[i] for i in rng.choice(len(groups), size=n, replace=False)]


def free_positions(n, used_buckets, seed):
    """n positions whose buckets are all different and not in used_buckets"""
    rng = np.random.default_rng(seed)
    out, used = [], set(used_buckets)
    while len(out) < n:
        p = rng.integers(-3000, 3000, size=3)
        b = int(hash_index(p)[0])
        if b not in used:
            used.add(b)
            out.append(p)
    return np.array(out, np.int32).reshape(-1, 3)


class Builder:
    """Allocates blocks in a ResetScene state the way allocateVoxelBlocksList_device does (free-list pointer from the top,
    excess slots from the top of the excess list, successors linked at the chain's end) and fills their voxels."""

    def __init__(self, seed=0):
        self.st = reset_state()
        self.rng = np.random.default_rng(seed)

    def add_chain(self, positions, times, vis):
        st, hs, ptrs = self.st, self.st["hash"], []
        prev = -1
        for k, p in enumerate(positions):
            ptr = int(st["allocationList"][st["lastFreeBlockId"]])
            st["lastFreeBlockId"] -= 1
            if k == 0:
                idx = int(hash_index(p)[0])
                assert hs["ptr"][idx] == -2 and hs["offset"][idx] == 0
            else:
                exl = int(st["excessList"][st["lastFreeExcessListId"]])
                st["lastFreeExcessListId"] -= 1
                idx = NB + exl
                hs["offset"][prev] = exl + 1
            hs["pos"][idx] = p
            hs["offset"][idx] = 0
            hs["ptr"][idx] = ptr
            hs["allocatedTime"][idx] = times[k]
            st["visType"][idx] = vis[k]
            prev = idx
            ptrs.append(ptr)
        return ptrs

    def fill(self, ptr, kind, maxWeight):
        """voxel contents of block ptr relative to the decay's maxWeight:
        confident: every w_depth above maxWeight (never reset); at_max: every w_depth == maxWeight; low: w_depth in
        [1, maxWeight]; zero_stale: w_depth 0 everywhere, sdf / colour / w_color left over; one_noisy: confident but one
        voxel at maxWeight. Colour and w_color are non-zero so that a reset that forgets them shows."""
        r = self.rng
        v = np.zeros(512, abi.VOXEL_DTYPE)
        v["sdf"] = r.integers(-32767, 32768, 512)
        v["clr"] = r.integers(1, 256, (512, 3))
        v["w_color"] = r.integers(1, 256, 512)
        hi = min(maxWeight + 1, 255)
        if kind == "confident":
            v["w_depth"] = r.integers(hi, 256, 512) if hi < 255 else 255
        elif kind == "at_max":
            v["w_depth"] = maxWeight
        elif kind == "low":
            v["w_depth"] = r.integers(1, maxWeight + 1, 512) if maxWeight >= 1 else 0
        elif kind == "zero_stale":
            v["w_depth"] = 0
        elif kind == "one_noisy":
            v["w_depth"] = r.integers(hi, 256, 512) if hi < 255 else 255
            v["w_depth"][int(r.integers(0, 512))] = maxWeight
        else:
            raise ValueError(kind)
        self.st["voxels"][ptr * 512:(ptr + 1) * 512] = v


def pad(minAge):
    """minAge empty snapshots after the one under test: Decay pops the oldest once more than minAge are queued (:526)"""
    return [("push", np.zeros((0, 3), np.int32))] * minAge


def crafted_case(maxWeight, minAge, full=False, seed=1):
    """Chains of length 2-4 with exactly one member in the snapshot and empty-able (a head with a successor, a middle and a
    tail entry), every member with its own visibility byte; single blocks with w_depth == maxWeight and maxWeight + 1, all
    w_depth 0 with stale contents, one noisy voxel among confident ones, allocatedTime == f - minAge and f - minAge + 1;
    a snapshot position that is not allocated. full=True: every chain member stays (Reap must not delete a chain member,
    see check_reference_input), the singles are as above."""
    f = 20
    old = f - minAge - 3
    b = Builder(seed)
    L = []
    groups = colliding_positions(4, 3, seed)
    empty_kind = "one_noisy" if full else None
    # (chain length, index of the member in the snapshot, its contents)
    layout = [(2, 0, empty_kind or "at_max"), (3, 1, empty_kind or "zero_stale"), (4, 3, empty_kind or "low")]
    vis_base = 10
    for (n, sel, kind), grp in zip(layout, groups):
        pos = grp[:n]
        ptrs = b.add_chain(pos, [old] * n, [vis_base + k for k in range(n)])
        vis_base += 10
        for k, ptr in enumerate(ptrs):
            b.fill(ptr, kind if k == sel else "confident", maxWeight)
        L.append(pos[sel])
    singles = [("at_max", old), ("confident", old), ("zero_stale", old), ("one_noisy", old), ("at_max", f - minAge),
               ("at_max", f - minAge + 1)]
    if maxWeight < 255:
        singles.append(("at_max_plus_one", old))
    sp = free_positions(len(singles) + 1, [int(hash_index(g[0])[0]) for g in groups], seed + 100)
    for (kind, t), p in zip(singles, sp):
        ptr = b.add_chain([p], [t], [3])[0]
        if kind == "at_max_plus_one":
            b.fill(ptr, "at_max", maxWeight)
            b.st["voxels"]["w_depth"][ptr * 512:(ptr + 1) * 512] = maxWeight + 1
        else:
            b.fill(ptr, kind, maxWeight)
        L.append(p)
    L.append(sp[-1])                                     # in the snapshot, not in the map
    L = np.array(L, np.int32)
    if full:
        ops = [("frame", f), ("decay", maxWeight, minAge, True)]
    else:
        ops = [("push", L)] + pad(minAge) + [("frame", f), ("decay", maxWeight, minAge, False)]
    return b.st, ops


def queue_case(kind, maxWeight=3):
    """Three single blocks X, Y, Z (each empty-able at maxWeight) in snapshots A, B, C; the queue operations decide which
    of them a Decay reaches.
      depth:  push A, B; Decay(minAge 2) with 2 snapshots queued does nothing; Decay(minAge 1) pops the OLDEST, A.
      empty:  push an empty snapshot and B; the first Decay(minAge 0) pops the empty one and changes nothing, the second B.
      catchup: push A, B, C; InfiniTamDriver::DecayCatchup's min_decay_age (3) calls with minAge 0 reach all three.
      reset:  push A; ResetScene + the state again; push B; Decay(minAge 0) reaches B only: ResetScene emptied the queue."""
    f = 10
    b = Builder(7)
    sp = free_positions(3, [], 77)
    for p in sp:
        b.fill(b.add_chain([p], [0], [1])[0], "at_max", maxWeight)
    A, B, Cc = sp[0:1], sp[1:2], sp[2:3]
    empty = np.zeros((0, 3), np.int32)
    ops = {"depth": [("push", A), ("push", B), ("frame", f), ("decay", maxWeight, 2, False), ("decay", maxWeight, 1, False)],
           "empty": [("push", empty), ("push", B), ("frame", f), ("decay", maxWeight, 0, False), ("decay", maxWeight, 0, False)],
           "catchup": [("push", A), ("push", B), ("push", Cc), ("frame", f)] + [("decay", maxWeight, 0, False)] * 3,
           "reset": [("push", A), ("frame", f), ("reload",), ("push", B), ("decay", maxWeight, 0, False)]}[kind]
    return b.st, ops, dict(X=sp[0], Y=sp[1], Z=sp[2])


# ---- street states -----------------------------------------------------------------------------------------------------

_street = None


def street_state():
    """The oracle's map after STREET_FRAMES frames of the seeded KITTI-shaped sequence (scale 0.25, 32768 blocks, no decay),
    its front (oldest) snapshot with every pair of same-bucket positions dropped, and its frame index."""
    global _street
    if _street is None:
        L = H.oracle()
        scene = synth.StreetScene(seed=6, length_m=80.0)
        frames = [synth.kitti_frame(scene, f * 2, scale=0.25) for f in range(STREET_FRAMES)]
        w, h = frames[0][0].shape[1], frames[0][0].shape[0]
        vol = H.HostVolume(NUM_BLOCKS, NB, NE, w, h)
        for depth, rgb, M, proj in frames:
            v = H.make_view(depth, rgb, M, proj)
            assert L.oracle_allocate_from_depth(vol.engine, C.byref(vol.scene), C.byref(vol.rs), C.byref(v), 0, 0) == 0
            L.oracle_integrate(vol.engine, C.byref(vol.scene), C.byref(vol.rs), C.byref(v), 0)
        n = L.oracle_peek_snapshot(vol.engine, None, 0)
        snap = np.zeros((max(n, 1), 3), np.int32)
        assert L.oracle_peek_snapshot(vol.engine, H.vptr(snap), n) == n > 1000
        snap = snap[:n]
        b = hash_index(snap)
        _, inv, cnt = np.unique(b, return_inverse=True, return_counts=True)
        keep = snap[cnt[inv] == 1]
        st = dict(hash=vol.hash.copy(), voxels=vol.voxels.copy(), allocationList=vol.allocationList.copy(),
                  excessList=vol.excessList.copy(), visType=vol.visType.copy(), lastFreeBlockId=vol.scene.lastFreeBlockId,
                  lastFreeExcessListId=vol.scene.lastFreeExcessListId)
        _street = (st, keep, int(L.oracle_frame_index(vol.engine)), len(snap) - len(keep))
    return _street


def street_case(maxWeight, minAge):
    st, L, f, _ = street_state()
    return copy_state(st), [("push", L)] + pad(minAge) + [("frame", f), ("decay", maxWeight, minAge, False)]


def without_chains(st):
    """st with every multi-entry chain cut back to its head: each excess entry is unlinked, its block returned to the free
    list, its slot cleared (and left out of the excess free list, as deleteBlock leaves it, :1075)"""
    st = copy_state(st)
    hs = st["hash"]
    for b, c in chains(hs).items():
        for idx in c[1:]:
            if hs["ptr"][idx] >= 0:
                st["lastFreeBlockId"] += 1
                st["allocationList"][st["lastFreeBlockId"]] = hs["ptr"][idx]
            hs[idx] = np.zeros(1, abi.HASH_ENTRY_DTYPE)[0]
            hs["ptr"][idx] = -2
            st["visType"][idx] = 0
        hs["offset"][b] = 0
    return st


def street_full_case(maxWeight, minAge):
    st, _, f, _ = street_state()
    return without_chains(st), [("frame", f), ("decay", maxWeight, minAge, True)]


# ---- executors ---------------------------------------------------------------------------------------------------------

class OracleRun:
    """The oracle on a case. Records, per Decay call, the state before it, the snapshot it pops (or None), what it freed
    and the oracle's branch counters."""

    def __init__(self):
        self.L = H.oracle()
        self.vol = H.HostVolume(NUM_BLOCKS, NB, NE, *IMG)
        self.calls = []

    def load(self, st):
        L, vol = self.L, self.vol
        L.oracle_reset_scene(vol.engine, C.byref(vol.scene))
        for k in ("hash", "voxels", "allocationList", "excessList", "visType"):
            getattr(vol, k)[...] = st[k]
        vol.scene.lastFreeBlockId, vol.scene.lastFreeExcessListId = st["lastFreeBlockId"], st["lastFreeExcessListId"]

    def push(self, pos):
        pos = np.ascontiguousarray(pos, np.int32).reshape(-1, 3)
        self.L.oracle_push_snapshot(self.vol.engine, H.vptr(pos) if len(pos) else None, len(pos))

    def frame(self, f):
        self.L.oracle_set_frame_index(self.vol.engine, f)

    def front(self):
        n = self.L.oracle_peek_snapshot(self.vol.engine, None, 0)
        if n < 0:
            return None
        out = np.zeros((max(n, 1), 3), np.int32)
        self.L.oracle_peek_snapshot(self.vol.engine, H.vptr(out), n)
        return out[:n]

    def decay(self, maxWeight, minAge, forceAll):
        L, vol = self.L, self.vol
        pops = not forceAll and L.oracle_queue_size(vol.engine) > minAge
        pre = dict(hash=vol.hash.copy(), visType=vol.visType.copy(), lastFreeBlockId=vol.scene.lastFreeBlockId)
        snap = self.front() if pops else None
        L.oracle_decay_branches((C.c_long * 5)())
        L.oracle_decay(vol.engine, C.byref(vol.scene), C.byref(vol.rs), maxWeight, minAge, int(forceAll))
        br = (C.c_long * 5)()
        L.oracle_decay_branches(br)
        post = self.state()
        freed = post["allocationList"][pre["lastFreeBlockId"] + 1:post["lastFreeBlockId"] + 1].copy()
        self.calls.append(dict(pre=pre, post=post, snapshot=snap, forceAll=forceAll, freed=freed,
                               branches=dict(zip(("age_skip", "voxel_reset", "head_with_successor", "head_alone", "excess_entry"), br)),
                               decayed=int(L.oracle_decayed_block_count(vol.engine)), popped=pops))
        return self.calls[-1]["decayed"]

    def state(self):
        vol = self.vol
        return dict(hash=vol.hash.copy(), voxels=vol.voxels.copy(), allocationList=vol.allocationList.copy(),
                    excessList=vol.excessList.copy(), visType=vol.visType.copy(), lastFreeBlockId=vol.scene.lastFreeBlockId,
                    lastFreeExcessListId=vol.scene.lastFreeExcessListId)


def run(ex, st, ops, after_decay=None, before_decay=None):
    """ops on executor ex (load / push / frame / decay / state); after_decay(i, ex, decayed) and before_decay(i) run
    around Decay call i"""
    ex.load(st)
    i = 0
    for op in ops:
        if op[0] == "push":
            ex.push(op[1])
        elif op[0] == "frame":
            ex.frame(op[1])
        elif op[0] == "reload":
            ex.load(st)
        elif op[0] == "decay":
            if before_decay is not None:
                before_decay(i)
            n = ex.decay(op[1], op[2], op[3])
            if after_decay is not None:
                after_decay(i, ex, n)
            i += 1
        else:
            raise ValueError(op)


def run_oracle(st, ops):
    o = OracleRun()
    run(o, st, ops)
    return o


def check_reference_input(call):
    """Raises unless the reference's Decay is deterministic and in bounds on this call (`call`: the oracle's record of the
    same call). Partial decay: no two snapshot positions share a hash bucket, found or not, so that every bucket chain is
    walked and changed by one CTA only. Full decay: no bucket chain with more than one entry holds a block the call
    deletes, so that no CTA walks a chain while another rewrites it."""
    if call["forceAll"]:
        hs = call["pre"]["hash"]
        freed = set(int(p) for p in call["freed"])
        for b, c in chains(hs).items():
            if len(c) > 1:
                hit = [i for i in c if int(hs["ptr"][i]) in freed]
                if hit:
                    raise AssertionError(f"full decay deletes entry {hit[0]} of the {len(c)}-entry chain of bucket {b}: the "
                                         f"reference's unlocked chain walks would race with it")
    elif call["snapshot"] is not None and len(call["snapshot"]):
        b = hash_index(call["snapshot"])
        u, cnt = np.unique(b, return_counts=True)
        if (cnt > 1).any():
            raise AssertionError(f"{int((cnt > 1).sum())} hash buckets hold two or more snapshot positions (first: bucket "
                                 f"{int(u[cnt > 1][0])}): the reference's unlocked chain walks would race")


def canonical(state, sections):
    """state with each freed section [a, b) of the allocation list sorted (the reference pushes freed blocks with atomicAdd)"""
    al = state["allocationList"].copy()
    for a, b in sections:
        al[a:b] = np.sort(al[a:b])
    return al


def outcome_bytes(state, sections, decayed):
    """order-free outcome of a case: hash table, visibility bytes, the allocation list with its freed sections sorted, the
    counters, and the SHA-256 of the voxel block array"""
    ctr = np.array([state["lastFreeBlockId"], state["lastFreeExcessListId"], decayed], np.int64)
    return (state["hash"].tobytes() + state["visType"].tobytes() + canonical(state, sections).tobytes() + ctr.tobytes() +
            hashlib.sha256(state["voxels"].tobytes()).digest())


def sections_of(oracle_run):
    return [(c["pre"]["lastFreeBlockId"] + 1, c["pre"]["lastFreeBlockId"] + 1 + len(c["freed"])) for c in oracle_run.calls]


def entry_of(state, pos):
    """entry index of block pos in state's table, or -1 (findBlock)"""
    hs, idx = state["hash"], int(hash_index(pos)[0])
    while True:
        if tuple(int(c) for c in hs["pos"][idx]) == tuple(int(c) for c in pos) and hs["ptr"][idx] >= 0:
            return idx
        if hs["offset"][idx] < 1:
            return -1
        idx = NB + int(hs["offset"][idx]) - 1


# cases pinned to the reference's outcomes (tests/golden/ref_pins.json) and run live on the three executors
CRAFTED_PARAMS = [(3, 2), (0, 1), (1, 0), (254, 3)]
STREET_PARAMS = [(1, 2), (3, 2), (50, 1), (0, 1), (255, 0)]
STREET_FULL_PARAMS = [(1, 2), (3, 0)]
QUEUE_KINDS = ["depth", "empty", "catchup", "reset"]


def pinned_cases():
    """name -> zero-argument builder of (state, ops)"""
    cases = {}
    for mw, ma in CRAFTED_PARAMS:
        cases[f"crafted/partial/mw{mw}_age{ma}"] = (lambda mw=mw, ma=ma: crafted_case(mw, ma))
        cases[f"crafted/full/mw{mw}_age{ma}"] = (lambda mw=mw, ma=ma: crafted_case(mw, ma, full=True))
    for mw, ma in STREET_PARAMS:
        cases[f"street/partial/mw{mw}_age{ma}"] = (lambda mw=mw, ma=ma: street_case(mw, ma))
    for mw, ma in STREET_FULL_PARAMS:
        cases[f"street/full/mw{mw}_age{ma}"] = (lambda mw=mw, ma=ma: street_full_case(mw, ma))
    for k in QUEUE_KINDS:
        cases[f"queue/{k}"] = (lambda k=k: queue_case(k)[:2])
    return cases


def pin_key(name):
    return f"oracle_vs_ref/decay/{name}"
