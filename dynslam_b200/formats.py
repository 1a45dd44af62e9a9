"""The on-disk formats either side of the path (SURVEY 8(f) rank 4) for hosts without OpenCV / pfmLib / ITMMesh: thin wrappers over
libb200host.so (csrc/hostio.c). They return exactly what the C-ABI consumes — int16 millimetre depth (PrecomputedDepthProvider),
byte masks of a bounding box (PrecomputedSegmentationProvider) — and write what it fills (ITMMesh::Triangle -> Wavefront OBJ)."""
import ctypes as C

import numpy as np

from . import abi

_ERR = {-1: "cannot open", -2: "malformed file", -3: "size mismatch", -4: "out of memory"}


def _check(rc, what, path):
    if rc:
        raise RuntimeError(f"{what} [{path}]: {_ERR.get(rc, rc)}")


def read_pfm(path):
    """ReadFilePFM (src/pfmLib/ImageIOpfm.cpp:49-156): float32 [h, w] ("Pf") or [h, w, 3] ("PF"), row 0 at the top."""
    h = abi.host_library()
    w_, h_, b_, data = C.c_int(), C.c_int(), C.c_int(), C.POINTER(C.c_float)()
    _check(h.b200h_read_pfm(str(path).encode(), C.byref(w_), C.byref(h_), C.byref(b_), C.byref(data)), "Could not read PFM image", path)
    n = w_.value * h_.value * b_.value
    out = np.ctypeslib.as_array(data, shape=(n,)).copy()
    h.b200h_free(data)
    return out.reshape(h_.value, w_.value) if b_.value == 1 else out.reshape(h_.value, w_.value, 3)


def read_depth_xml(path):
    """The OpenCV FileStorage XML dump of the CV_16SC1 matrix "depth-frame" (PrecomputedDepthProvider.cpp:32-42): int16 [h, w], millimetres."""
    h = abi.host_library()
    w_, h_, data = C.c_int(), C.c_int(), C.POINTER(C.c_int16)()
    _check(h.b200h_read_depth_xml(str(path).encode(), C.byref(w_), C.byref(h_), C.byref(data)), "Could not read precomputed depth map", path)
    out = np.ctypeslib.as_array(data, shape=(w_.value * h_.value,)).copy()
    h.b200h_free(data)
    return out.reshape(h_.value, w_.value)


def clamp_max_depth(depth, max_depth_m):
    """PrecomputedDepthProvider.cpp:53-72, in place: int16 or float32 millimetres beyond the provider's maximum become 0."""
    h = abi.host_library()
    assert depth.flags["C_CONTIGUOUS"]
    if depth.dtype == np.int16:
        h.b200h_clamp_max_depth_s16(depth.ctypes.data, depth.size, float(max_depth_m))
    elif depth.dtype == np.float32:
        h.b200h_clamp_max_depth_f32(depth.ctypes.data, depth.size, float(max_depth_m))
    else:
        raise TypeError("int16 or float32 depth expected")
    return depth


def read_mask_txt(path, width, height):
    """ReadMask (DS/InstRecLib/PrecomputedSegmentationProvider.cpp:24-71): the numpy text dump of an instance mask, uint8 [height, width]."""
    h = abi.host_library()
    out = np.zeros((height, width), np.uint8)
    _check(h.b200h_read_mask_txt(str(path).encode(), width, height, out.ctypes.data), "Could not read mask", path)
    return out


def checkpoint_header(buf):
    """The b200_checkpoint_header of a checkpoint (Engine.save_checkpoint, b200_checkpoint_save) as a dict, with "sections" mapping
    each section name to (offset, length) in bytes. Reads only the header; b200_checkpoint_load checks the rest."""
    b = np.frombuffer(memoryview(buf).cast("B"), dtype=np.uint8)
    if b.size < abi.CHECKPOINT_HEADER_BYTES:
        raise ValueError(f"{b.size} bytes: shorter than the {abi.CHECKPOINT_HEADER_BYTES}-byte checkpoint header")
    h = b[:abi.CHECKPOINT_HEADER_BYTES].view(abi.CHECKPOINT_HEADER_DTYPE)[0]
    if bytes(h["magic"]) != abi.CHECKPOINT_MAGIC:
        raise ValueError("not a checkpoint (bad magic)")
    out = {k: h[k].item() for k in abi.CHECKPOINT_HEADER_DTYPE.names if k not in ("magic", "section", "reserved")}
    out["sections"] = {n: (int(h["section"][i, 0]), int(h["section"][i, 1])) for i, n in enumerate(abi.CHECKPOINT_SECTIONS)}
    return out


def write_obj(path, triangles, noTotalTriangles=None, noMaxTriangles=None):
    """ITMMesh::WriteOBJ (ITMLib/Objects/ITMMesh.h:46-122) on an array of abi.TRIANGLE_DTYPE."""
    h = abi.host_library()
    t = np.ascontiguousarray(triangles)
    assert t.dtype == abi.TRIANGLE_DTYPE or (t.dtype == np.float32 and t.size % 18 == 0)
    n = int(noTotalTriangles if noTotalTriangles is not None else t.size // (1 if t.dtype == abi.TRIANGLE_DTYPE else 18))
    nmax = int(noMaxTriangles if noMaxTriangles is not None else n)
    rc = h.b200h_write_obj(str(path).encode(), t.ctypes.data, n, nmax)
    if rc == -3:
        raise RuntimeError(f"Unable to save mesh to file [{path}]. Too many triangles: {n} while the maximum is {nmax}.")
    if rc:
        raise RuntimeError("Could not open file for writing the mesh.\n")
