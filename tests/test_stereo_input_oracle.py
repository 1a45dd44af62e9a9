"""CPU: the oracle's restatement of DynSLAM's per-frame input conversions (oracle/input_oracle.c) against the reference's own
DepthProvider::DepthFromDisparityMap<float> + PrecomputedDepthProvider::DepthFromDisparity, the XML max-depth clamp of
PrecomputedDepthProvider::ReadPrecomputed and CvToItm(const cv::Mat3b &, ...), compiled from the reference tree into
oracle/_ref/libinputref.so (oracle/build_input_ref.sh, oracle/ref_input_driver.cpp): byte for byte, stored as digests
(tests/golden/stereo_input_pins.json, tests/stereolib.py; the reference also runs live where oracle/_ref is built)."""
import numpy as np
import pytest

from tests import hostlib as H
from tests import stereolib as S


@pytest.mark.parametrize("calib", S.CALIBS, ids=[c[0] for c in S.CALIBS])
def test_depth_from_disparity_pinned_to_reference(calib):
    L, R = S.oracle(), S.reference()
    disp = S.disparities(calib, 97, 61, seed=len(calib[0]))
    ours = S.oracle_depth(L, disp, calib)
    ref = None
    if R:
        ref = np.zeros_like(ours)
        _, b, f, dmin, dmax = calib
        assert R.ref_depth_from_disparity(H.vptr(ref), H.vptr(disp), 97, 61, b, f, dmin, dmax) == 0
    S.check_pin(f"stereo_input/disparity/{calib[0]}", ours.tobytes(), ref.tobytes() if R else None)
    if calib[0] != "short_rig":
        assert (ours != 0).sum() > 0.5 * ours.size             # the realistic part converts
    else:
        # 5 m px: a disparity of 0.5 px is 10 m, inside the bounds, yet the reference gives 0 (int abs(int) of 0)
        flat_d, flat_o = disp.reshape(-1), ours.reshape(-1)
        sub = (np.abs(flat_d) < 1) & (np.abs(flat_d) > 0.25)
        assert sub.any() and (flat_o[sub] == 0).all()


def test_max_depth_limit_is_the_references():
    """max_depth_mm >= 32767 throws in the reference; the engine rejects it with the same text (tests/test_gpu_stereo_input.py)."""
    R = S.reference()
    if R is None:
        pytest.skip("oracle/_ref/libinputref.so is not built")
    disp = np.ones((5, 5), np.float32)
    out = np.zeros((5, 5), np.int16)
    assert R.ref_depth_from_disparity(H.vptr(out), H.vptr(disp), 5, 5, 0.5, 700.0, 0.5, 32.768) == -1
    assert R.ref_input_last_error().decode() == S.MAX_DEPTH_ERROR
    assert R.ref_depth_from_disparity(H.vptr(out), H.vptr(disp), 5, 5, 0.5, 700.0, 0.5, 32.767) == 0   # 32766.998 mm truncates


@pytest.mark.parametrize("max_depth_m", S.CLAMP_MAX)
def test_clamp_depth_mm_pinned_to_reference(max_depth_m):
    L, R = S.oracle(), S.reference()
    depth = S.depth_mm(53, 37, max_depth_m, seed=int(max_depth_m * 10))
    ours = S.oracle_clamp(L, depth, max_depth_m)
    ref = None
    if R:
        ref = depth.copy()
        R.ref_clamp_depth_mm(H.vptr(ref), 53, 37, max_depth_m)
    S.check_pin(f"stereo_input/clamp/{max_depth_m}", ours.tobytes(), ref.tobytes() if R else None)
    m = int(round(float(np.float32(max_depth_m) * np.float32(1000.0))))
    assert ours.reshape(-1)[0] == m - 2 if m - 2 >= -32768 else True
    assert (ours[depth > m] == 0).all() and (ours[depth <= m] == depth[depth <= m]).all()


@pytest.mark.parametrize("shape", [(61, 97), (5, 7), (375, 1242)])
def test_bgr_to_rgba_pinned_to_reference(shape):
    L, R = S.oracle(), S.reference()
    h, w = shape
    bgr = S.bgr_image(w, h, seed=w)
    ours = S.oracle_rgba(L, bgr)
    assert (ours[..., 3] == 255).all() and np.array_equal(ours[..., :3], bgr[..., ::-1])
    ref = None
    if R:
        ref = np.zeros_like(ours)
        R.ref_bgr_to_rgba(H.vptr(ref), H.vptr(bgr), w, h)
    S.check_pin(f"stereo_input/bgr/{w}x{h}", ours.tobytes(), ref.tobytes() if R else None)
