"""Shared inputs and bindings for the stereo-input tests: the oracle's restatement of DynSLAM's per-frame input conversions
(oracle/input_oracle.c -> oracle/libinputoracle.so), the reference's own functions where oracle/_ref/libinputref.so is built
(oracle/build_input_ref.sh), seeded disparity / depth / BGR inputs that reach every branch of DepthFromDisparityMap and of the XML
clamp, and the digests of the reference's outputs on those inputs (tests/golden/stereo_input_pins.json).

The digests are kept and checked as tests/refpins.py does for tests/golden/ref_pins.json. After a deliberate change of the inputs,
record them again where oracle/_ref is built:
    REFPINS_RECORD=1 python -m pytest tests/test_stereo_input_oracle.py
"""
import atexit
import ctypes as C
import json
import os

import numpy as np

from tests import hostlib as H
from tests import refpins

ORACLE_SO = os.path.join(H.ROOT, "oracle", "libinputoracle.so")
INPUTREF_SO = os.path.join(H.ROOT, "oracle", "_ref", "libinputref.so")
PINS = os.path.join(H.ROOT, "tests", "golden", "stereo_input_pins.json")

_recorded = {}


def _write_pins():
    if not _recorded:
        return
    try:
        with open(PINS) as f:
            old = json.load(f)["pins"]
    except FileNotFoundError:
        old = {}
    with open(PINS, "w") as f:
        json.dump({"what": "SHA-256, length and sampled 32-bit words (byte offset -> hex, little-endian) of the reference's own "
                           "stereo-input outputs on the seeded inputs of tests/test_stereo_input_oracle.py",
                   "pins": dict(sorted({**old, **_recorded}.items()))}, f, indent=1)
        f.write("\n")


if refpins.RECORD:
    atexit.register(_write_pins)


def check_pin(key, ours, ref=None):
    """ours: the oracle's bytes; ref: the reference's bytes, or None where oracle/_ref is not built. Asserts ours == ref when both
    exist, and that ours has the stored digest of the reference's output."""
    if ref is not None:
        assert ours == ref, f"{key}: differs from the reference's own code"
        if refpins.RECORD:
            _recorded[key] = refpins._pin(ref, key)
            return
    with open(PINS) as f:
        pin = json.load(f)["pins"].get(key)
    assert pin is not None, f"{key}: no stored digest in {PINS}"
    if refpins.digest(ours) != pin["sha256"]:
        where = refpins._where(pin, ours) or "outside the sampled words"
        raise AssertionError(f"{key}: differs from the stored digest of the reference's output; {where}")

# (name, baseline_m, focal_length_px, min_depth_m, max_depth_m). "kitti": the KITTI rig (f * b ~ 380 m px against 20 m);
# "short_rig": f * b = 5 m px < max_depth, where a disparity below 1 px maps inside the bounds, so only the reading of the
# reference's unqualified abs() decides it; "min0": no lower bound; "near_limit": the largest accepted maximum depth.
CALIBS = [("kitti", 0.5372, 707.0912, 0.5, 20.0), ("short_rig", 0.5, 10.0, 0.5, 20.0), ("min0", 0.5372, 707.0912, 0.0, 20.0),
          ("near_limit", 0.5372, 707.0912, 0.0, 32.766)]
# the reference's text for a maximum depth of 32.768 m (DS/DepthProvider.h:113-117)
MAX_DEPTH_ERROR = "Unsupported maximum depth of 32.768002 meters (32768 mm, larger than the 32767 limit)."
CLAMP_MAX = [20.0, 15.5, 0.0015, 32.766, 0.0]


def oracle():
    if not os.path.exists(ORACLE_SO):
        raise RuntimeError(f"{ORACLE_SO} is missing: run `python __graft_entry__.py`")
    L = C.CDLL(ORACLE_SO)
    L.oracle_depth_from_disparity.argtypes = [C.c_void_p, C.c_void_p, C.c_int] + [C.c_float] * 4
    L.oracle_depth_from_disparity.restype = None
    L.oracle_clamp_depth_mm.argtypes = [C.c_void_p, C.c_int, C.c_float]
    L.oracle_clamp_depth_mm.restype = None
    L.oracle_bgr_to_rgba.argtypes = [C.c_void_p, C.c_void_p, C.c_int]
    L.oracle_bgr_to_rgba.restype = None
    return L


def reference():
    if not os.path.exists(INPUTREF_SO):
        return None
    R = C.CDLL(INPUTREF_SO)
    R.ref_depth_from_disparity.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int] + [C.c_float] * 4
    R.ref_clamp_depth_mm.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_float]
    R.ref_clamp_depth_mm.restype = None
    R.ref_bgr_to_rgba.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int]
    R.ref_bgr_to_rgba.restype = None
    R.ref_input_last_error.restype = C.c_char_p
    return R


def _f32(x):
    return np.float32(x)


def disparities(calib, w, h, seed=0):
    """(h, w) float32: realistic disparities (0.5-250 px) with every edge case placed in the first rows."""
    _, b, f, dmin, dmax = calib
    rng = np.random.default_rng(seed)
    d = rng.uniform(0.5, 250.0, (h, w)).astype(np.float32)
    tiny = np.float32(np.finfo(np.float32).tiny)
    special = [0.0, -0.0, 1e-6, -1e-6, 1e-5, -1e-5, 0.5, -0.5, 0.999, -0.999, np.nextafter(_f32(1), _f32(0)), 1.0, -1.0,
               np.nextafter(_f32(1), _f32(2)), -3.0, -250.0, np.nan, -np.nan, np.inf, -np.inf, tiny, -tiny, tiny / 4, -tiny / 4,
               1e30, -1e30, 2147483648.0, -2147483648.0, 3e9, 65536.5]
    special += list(np.linspace(-1.0, 1.0, 41, dtype=np.float32))
    # disparities whose millimetre value lands one ulp either side of the bounds and of integer millimetres
    fb = _f32(f) * _f32(b)
    targets = [int(np.float32(dmin) * np.float32(1000.0)), int(np.float32(dmax) * np.float32(1000.0)), 1234, 5000, 15000]
    for t in targets:
        if t <= 0:
            continue
        d0 = np.float32(np.float64(fb) * 1000.0 / t)
        for k in range(-3, 4):
            x = d0
            for _ in range(abs(k)):
                x = np.nextafter(x, np.float32(np.inf if k > 0 else -np.inf))
            special.append(x)
    special = np.array(special, np.float32)
    flat = d.reshape(-1)
    n = min(flat.size, special.size)
    flat[:n] = special[:n]
    return d


def depth_mm(w, h, max_depth_m, seed=0):
    """(h, w) int16 millimetres over the whole int16 range, dense around max_depth_m * 1000 +- 1."""
    rng = np.random.default_rng(seed)
    d = rng.integers(-32768, 32768, (h, w)).astype(np.int16)
    m = int(round(float(np.float32(max_depth_m) * np.float32(1000.0))))
    special = [m - 2, m - 1, m, m + 1, m + 2, 0, -1, 1, -32768, 32767, 20000, 20001, 19999]
    special = np.clip(np.array(special), -32768, 32767).astype(np.int16)
    flat = d.reshape(-1)
    flat[:special.size] = special
    flat[special.size::7] = np.clip(m + rng.integers(-3, 4, flat[special.size::7].size), -32768, 32767)
    return d


def bgr_image(w, h, seed=0):
    return np.random.default_rng(seed).integers(0, 256, (h, w, 3)).astype(np.uint8)


def oracle_depth(L, disp, calib):
    _, b, f, dmin, dmax = calib
    out = np.zeros(disp.shape, np.int16)
    L.oracle_depth_from_disparity(H.vptr(out), H.vptr(disp), disp.size, b, f, dmin, dmax)
    return out


def oracle_clamp(L, depth, max_depth_m):
    out = depth.copy()
    L.oracle_clamp_depth_mm(H.vptr(out), out.size, max_depth_m)
    return out


def oracle_rgba(L, bgr):
    out = np.zeros(bgr.shape[:2] + (4,), np.uint8)
    L.oracle_bgr_to_rgba(H.vptr(out), H.vptr(bgr), bgr.shape[0] * bgr.shape[1])
    return out
