"""CPU: the free-view preview's part of the C-ABI — the symbols libb200fusion.so exports, the argument lists the Python layer
declares for them, and the rejections the library makes before it touches CUDA (no engine)."""
import ctypes as C

from dynslam_b200 import abi, engine as E

CALLS = {"b200_render_view_async": 7, "b200_render_view_sync": 2, "b200_render_view_submit": 8, "b200_render_view_wait": 2,
         "b200_engine_wait_engine": 2}


def test_symbols_and_argument_lists():
    lib = abi.load_library()
    for name, nargs in CALLS.items():
        assert name in abi.EXPORTS
        f = getattr(lib, name)
        assert len(f.argtypes) == nargs and f.argtypes[0] is C.c_void_p, name
    for name in ("b200_render_view_async", "b200_render_view_submit"):
        a = getattr(lib, name).argtypes
        assert a[1:5] == [C.POINTER(abi.Scene), C.POINTER(abi.RenderState), C.POINTER(abi.Camera), C.c_int]
    for m in ("RenderFreeView", "RenderFreeViewSync", "RenderFreeViewSubmit", "RenderFreeViewWait"):
        assert callable(getattr(E.VisualisationEngine, m))
    assert callable(E.Engine.wait_engine)


def test_header_declares_them():
    import os
    hdr = open(os.path.join(os.path.dirname(abi.__file__), "..", "include", "b200fusion.h")).read()
    for name in CALLS:
        assert f"b200_status {name}(" in hdr, name


def test_null_engine_is_rejected_without_cuda():
    lib = abi.load_library()
    s, rs, cam = abi.Scene(), abi.RenderState(), abi.Camera()
    assert lib.b200_render_view_async(None, C.byref(s), C.byref(rs), C.byref(cam), 0, None, None) == abi.ERR_INVALID
    assert lib.b200_render_view_submit(None, C.byref(s), C.byref(rs), C.byref(cam), 0, None, None, 0) == abi.ERR_INVALID
    assert lib.b200_render_view_sync(None, C.byref(rs)) == abi.ERR_INVALID
    assert lib.b200_render_view_wait(None, 0) == abi.ERR_INVALID
    assert lib.b200_engine_wait_engine(None, None) == abi.ERR_INVALID
