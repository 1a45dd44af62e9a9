"""ctypes binding of oracle/_ref/libitmharness.so (test / baseline infrastructure): the real ITMLib
objects driven through the abstract engine interfaces with either the UNMODIFIED reference CUDA
engines (impl 0) or the B200 shim classes (impl 1) behind them. See oracle/itm_harness.cpp."""
import ctypes as C
import os

import numpy as np

from dynslam_b200 import abi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "oracle", "_ref", "libitmharness.so")
REFERENCE_CUDA, B200_SHIM = 0, 1


def available():
    return os.path.exists(SO)


# Entry points that run the reference's own Decay on a supplied state. Where the reference's sources cannot be read at
# build time, oracle/build_ref.sh keeps an oracle/_ref built earlier, which may predate them: the other harness tests
# still run against such a library, and the decay tests run without the reference (its outcomes stay pinned in
# tests/golden/ref_pins.json).
DECAY_ENTRY_POINTS = ("harness_upload_state", "harness_push_snapshot", "harness_set_frame_index", "harness_queue_size",
                      "harness_decay", "harness_download_lists")


def decay_available():
    return available() and all(hasattr(lib(), n) for n in DECAY_ENTRY_POINTS)


_L = None


def lib():
    global _L
    if _L is None:
        abi.load_library()          # libb200fusion.so first (the harness links against it)
        L = C.CDLL(SO)
        vp = C.c_void_p
        L.harness_create.restype = vp
        L.harness_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float,
                                     C.c_int, C.c_long]
        L.harness_destroy.argtypes = [vp]
        L.harness_destroy.restype = None
        L.harness_error.argtypes = [vp]
        L.harness_error.restype = C.c_char_p
        L.harness_mute_stdout.argtypes = [vp, C.c_int]
        L.harness_mute_stdout.restype = None
        L.harness_process_frame.argtypes = [vp, vp, vp, C.POINTER(C.c_float), C.c_int, C.c_int, C.c_int, C.c_int]
        L.harness_process_frame_timed.argtypes = [vp, vp, vp, C.POINTER(C.c_float), C.c_int, C.c_int, C.c_int, C.POINTER(C.c_double)]
        L.harness_pin.argtypes = [vp, C.c_size_t]
        L.harness_unpin.argtypes = [vp]
        L.harness_sync.argtypes = [vp]
        L.harness_sync.restype = None
        L.harness_counters.argtypes = [vp, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_long)]
        L.harness_counters.restype = None
        L.harness_download.argtypes = [vp, vp, vp, vp, vp]
        L.harness_download.restype = None
        if all(hasattr(L, n) for n in DECAY_ENTRY_POINTS):
            L.harness_download_lists.argtypes = [vp, vp, vp, vp]
            L.harness_download_lists.restype = None
            L.harness_upload_state.argtypes = [vp, vp, vp, vp, vp, vp, C.c_int, C.c_int]
            L.harness_push_snapshot.argtypes = [vp, vp, C.c_long]
            L.harness_set_frame_index.argtypes = [vp, C.c_long]
            L.harness_queue_size.argtypes = [vp]
            L.harness_queue_size.restype = C.c_long
            L.harness_decay.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_long)]
        L.vbh_create.restype = vp
        L.vbh_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float]
        L.vbh_destroy.argtypes = [vp]
        L.vbh_destroy.restype = None
        L.vbh_update_view.argtypes = [vp, vp, vp, C.c_int, C.c_int]
        L.vbh_update_view.restype = None
        L.vbh_time_update_view.argtypes = [vp, C.c_int, C.c_int]
        L.vbh_time_update_view.restype = C.c_double
        L.vbh_time_device_only.argtypes = [vp, C.c_int]
        L.vbh_time_device_only.restype = C.c_double
        L.vbh_download.argtypes = [vp, vp]
        L.vbh_download.restype = None
        _L = L
    return _L


class ViewBuilderHarness:
    """ITMViewBuilder_CUDA (impl 0) or ITMViewBuilder_B200 (impl 1) behind the abstract ITMViewBuilder."""

    def __init__(self, impl, w, h, proj):
        self.L = lib()
        self.w, self.h = w, h
        self.h_ = self.L.vbh_create(impl, w, h, float(proj[0]), float(proj[1]), float(proj[2]), float(proj[3]))

    def update_view(self, raw, rgb, useBilateralFilter=True, modelSensorNoise=False):
        raw = np.ascontiguousarray(raw, dtype=np.int16)
        rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
        self.L.vbh_update_view(self.h_, raw.ctypes.data, rgb.ctypes.data, int(useBilateralFilter), int(modelSensorNoise))
        out = np.zeros((self.h, self.w), dtype=np.float32)
        self.L.vbh_download(self.h_, out.ctypes.data)
        return out

    def time_update_view(self, iters=50, useBilateralFilter=True):
        return self.L.vbh_time_update_view(self.h_, int(useBilateralFilter), iters)

    def time_device_only(self, iters=50):
        return self.L.vbh_time_device_only(self.h_, iters)

    def close(self):
        if self.h_:
            self.L.vbh_destroy(self.h_)
            self.h_ = None


class Harness:
    def __init__(self, impl, w, h, proj, voxelSize=0.05, mu=0.75, maxW=50, numBlocks=0x60000, mute=True):
        self.L = lib()
        self.w, self.h, self.numBlocks = w, h, numBlocks
        self.h_ = self.L.harness_create(impl, w, h, float(proj[0]), float(proj[1]), float(proj[2]), float(proj[3]), voxelSize, mu, maxW,
                                        numBlocks)
        self.noTotal = self.L.harness_table_entries()
        if mute:
            self.L.harness_mute_stdout(self.h_, 1)

    def process_frame(self, depth, rgb, M, decay=None, raycast=True):
        depth = np.ascontiguousarray(depth, dtype=np.float32)
        rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
        m = abi.mat_to_c(M)
        rc = self.L.harness_process_frame(self.h_, depth.ctypes.data, rgb.ctypes.data, m, decay[0] if decay else 0,
                                          decay[1] if decay else 0, int(decay is not None), int(raycast))
        if rc:
            raise RuntimeError(self.L.harness_error(self.h_).decode())

    def process_frame_timed(self, depth, rgb, M, stage_us, decay=None):
        """Same frame with a device synchronise + wall clock after every ITMLib call; stage_us (6 doubles) accumulates."""
        m = abi.mat_to_c(M)
        rc = self.L.harness_process_frame_timed(self.h_, depth.ctypes.data, rgb.ctypes.data, m, decay[0] if decay else 0,
                                                decay[1] if decay else 0, int(decay is not None), stage_us)
        if rc:
            raise RuntimeError(self.L.harness_error(self.h_).decode())

    def sync(self):
        self.L.harness_sync(self.h_)

    def counters(self):
        a, b, c, d = C.c_int(), C.c_int(), C.c_int(), C.c_long()
        self.L.harness_counters(self.h_, C.byref(a), C.byref(b), C.byref(c), C.byref(d))
        return dict(lastFreeBlockId=a.value, lastFreeExcessListId=b.value, noVisibleBlocks=c.value, decayed=d.value)

    def download(self):
        hash_ = np.zeros(self.noTotal, dtype=abi.HASH_ENTRY_DTYPE)
        vox = np.zeros(self.numBlocks * 512, dtype=abi.VOXEL_DTYPE)
        rays = np.zeros((self.h, self.w, 4), dtype=np.float32)
        img = np.zeros((self.h, self.w, 4), dtype=np.uint8)
        self.L.harness_download(self.h_, hash_.ctypes.data, vox.ctypes.data, rays.ctypes.data, img.ctypes.data)
        return dict(hash=hash_, voxels=vox, rays=rays, image=img)

    # ---- the reference's own Decay on a supplied state (REFERENCE_CUDA only) ----
    def _ok(self, rc):
        if rc:
            raise RuntimeError(self.L.harness_error(self.h_).decode())

    def upload_state(self, hash_, voxels, allocationList, excessList, visType, lastFreeBlockId, lastFreeExcessListId):
        """ResetScene (empties the decay queue, keeps the frame index), then the given state"""
        arrs = [np.ascontiguousarray(a) for a in (hash_, voxels, allocationList, excessList, visType)]
        assert arrs[0].nbytes == self.noTotal * 20 and arrs[1].nbytes == self.numBlocks * 512 * 8 and arrs[4].nbytes == self.noTotal
        self._ok(self.L.harness_upload_state(self.h_, *[a.ctypes.data for a in arrs], int(lastFreeBlockId), int(lastFreeExcessListId)))

    def push_snapshot(self, positions):
        p = np.ascontiguousarray(positions, dtype=np.int32).reshape(-1, 3)
        self._ok(self.L.harness_push_snapshot(self.h_, p.ctypes.data if len(p) else None, len(p)))

    def set_frame_index(self, f):
        self._ok(self.L.harness_set_frame_index(self.h_, int(f)))

    def queue_size(self):
        return self.L.harness_queue_size(self.h_)

    def decay(self, maxWeight, minAge, forceAll=False):
        """the reference's Decay; returns GetDecayedBlockCount() (blocks freed since the last upload_state)"""
        n = C.c_long()
        self._ok(self.L.harness_decay(self.h_, int(maxWeight), int(minAge), int(forceAll), C.byref(n)))
        return n.value

    def download_state(self, excessSize):
        d = self.download()
        alloc = np.zeros(self.numBlocks, np.int32)
        exl = np.zeros(excessSize, np.int32)
        vis = np.zeros(self.noTotal, np.uint8)
        self.L.harness_download_lists(self.h_, alloc.ctypes.data, exl.ctypes.data, vis.ctypes.data)
        c = self.counters()
        return dict(hash=d["hash"], voxels=d["voxels"], allocationList=alloc, excessList=exl, visType=vis,
                    lastFreeBlockId=c["lastFreeBlockId"], lastFreeExcessListId=c["lastFreeExcessListId"])

    def close(self):
        if self.h_:
            self.L.harness_mute_stdout(self.h_, 0)
            self.L.harness_destroy(self.h_)
            self.h_ = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


PATCHED_SO = os.path.join(ROOT, "oracle", "_ref", "libitmpatched.so")


def patched_available():
    return os.path.exists(PATCHED_SO)


class PatchedMainEngine:
    """The reference's ITMMainEngine built from the PATCHED ITMLib (integration/itmlib_b200.patch, integration/build_patched.sh):
    backend 0 = settings->engineBackend BACKEND_REFERENCE, 1 = BACKEND_B200. Frames go in as DynSLAM feeds them: raw int16
    depth (mm) + RGBA through ITMMainEngine::ProcessFrame, pose set externally."""
    _L = None

    def __init__(self, backend, w, h, proj, voxelSize=0.05, mu=0.75, numBlocks=0x60000):
        if PatchedMainEngine._L is None:
            abi.load_library()
            L = C.CDLL(PATCHED_SO)
            vp = C.c_void_p
            L.med_create.restype = vp
            L.med_create.argtypes = [C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_float, C.c_long]
            L.med_error.argtypes = [vp]; L.med_error.restype = C.c_char_p
            L.med_process_frame.argtypes = [vp, vp, vp, C.POINTER(C.c_float)]
            L.med_get_raycast_image.argtypes = [vp, vp]; L.med_get_raycast_image.restype = None
            L.med_counters.argtypes = [vp, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]; L.med_counters.restype = None
            L.med_destroy.argtypes = [vp]; L.med_destroy.restype = None
            PatchedMainEngine._L = L
        self.L, self.w, self.h = PatchedMainEngine._L, w, h
        self.h_ = self.L.med_create(backend, w, h, float(proj[0]), float(proj[1]), float(proj[2]), float(proj[3]), voxelSize, mu, numBlocks)
        err = self.L.med_error(self.h_).decode()
        if err:
            raise RuntimeError(err)

    def process_frame(self, raw, rgb, M):
        raw = np.ascontiguousarray(raw, dtype=np.int16)
        rgb = np.ascontiguousarray(rgb, dtype=np.uint8)
        rc = self.L.med_process_frame(self.h_, raw.ctypes.data, rgb.ctypes.data, abi.mat_to_c(M))
        if rc:
            raise RuntimeError(self.L.med_error(self.h_).decode())

    def raycast_image(self):
        out = np.zeros((self.h, self.w, 4), dtype=np.uint8)
        self.L.med_get_raycast_image(self.h_, out.ctypes.data)
        return out

    def counters(self):
        a, b, c = C.c_int(), C.c_int(), C.c_int()
        self.L.med_counters(self.h_, C.byref(a), C.byref(b), C.byref(c))
        return dict(lastFreeBlockId=a.value, allocatedEntries=c.value)

    def close(self):
        if self.h_:
            self.L.med_destroy(self.h_)
            self.h_ = None
