"""CPU: the volume group's and the volume restart's part of the C-ABI — the symbols libb200fusion.so exports, the argument lists
the Python layer declares for them, the header's declarations and struct layouts, and the rejections the library makes before
it touches CUDA (no engine, no group)."""
import ctypes as C
import os
import subprocess

from dynslam_b200 import abi, engine as E, volumes as V

CALLS = {"b200_volume_restart_async": 3, "b200_group_create": 2, "b200_group_destroy": 1, "b200_group_last_error": 1,
         "b200_group_slot": 5, "b200_group_slot_images": 3, "b200_group_track_start": 2, "b200_group_frame_async": 9,
         "b200_group_sync": 1}


def test_symbols_and_argument_lists():
    lib = abi.load_library()
    for name, nargs in CALLS.items():
        assert name in abi.EXPORTS
        f = getattr(lib, name)
        assert len(f.argtypes) == nargs, name
    assert lib.b200_volume_restart_async.argtypes == [C.c_void_p, C.POINTER(abi.Scene), C.POINTER(abi.RenderState)]
    assert lib.b200_group_create.argtypes[0] == C.POINTER(abi.GroupConfig)
    a = lib.b200_group_frame_async.argtypes
    assert a[3] == C.POINTER(abi.View) and a[4] == C.POINTER(abi.GroupCar) and a[5] == C.c_int
    assert lib.b200_group_last_error.restype == C.c_char_p
    assert callable(E.Engine.restart_volume)
    for m in ("track_start", "frame", "sync", "close", "prepare"):
        assert callable(getattr(E.VolumeGroup, m))
    for m in ("step", "state", "upload", "synchronize", "track_start"):
        assert callable(getattr(V.GroupStreetVolumes, m))


def test_header_declares_them():
    hdr = open(os.path.join(os.path.dirname(abi.__file__), "..", "include", "b200fusion.h")).read()
    for name in CALLS:
        ret = "void " if name == "b200_group_destroy" else ("const char *" if name == "b200_group_last_error" else "b200_status ")
        assert f"{ret}{name}(" in hdr, name
    for t in ("b200_group_config", "b200_group_images", "b200_group_car"):
        assert f"}} {t};" in hdr, t
    shim = open(os.path.join(os.path.dirname(abi.__file__), "itm_shim", "ITMEngines_B200.h")).read()
    assert "void RestartScene(" in shim and "b200_volume_restart_async(" in shim


def test_struct_layouts(tmp_path):
    """the new PODs compiled by gcc: size and every field offset equal the ctypes mirror's"""
    pairs = [("b200_group_config", abi.GroupConfig), ("b200_group_images", abi.GroupImages), ("b200_group_car", abi.GroupCar)]
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "b200fusion.h"', 'int main(void) {']
    for cname, cls in pairs:
        lines.append(f'  printf("{cname} size %zu\\n", sizeof({cname}));')
        for fname, _ in cls._fields_:
            lines.append(f'  printf("{cname} {fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ['  return 0;', '}']
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines))
    subprocess.run(["/usr/bin/gcc", "-I", os.path.join(os.path.dirname(abi.__file__), "..", "include"), "-o", str(exe), str(src)],
                   check=True)
    got = {}
    for ln in subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.splitlines():
        a, b, c = ln.split()
        got[(a, b)] = int(c)
    for cname, cls in pairs:
        assert got[(cname, "size")] == C.sizeof(cls), cname
        for fname, _ in cls._fields_:
            assert got[(cname, fname)] == getattr(cls, fname).offset, (cname, fname)


def test_null_handles_are_rejected_without_cuda():
    lib = abi.load_library()
    s, rs, v = abi.Scene(), abi.RenderState(), abi.View()
    assert lib.b200_volume_restart_async(None, C.byref(s), C.byref(rs)) == abi.ERR_INVALID
    h = C.c_void_p()
    assert lib.b200_group_create(None, C.byref(h)) == abi.ERR_INVALID and not h.value
    assert b"null" in lib.b200_group_last_error(None)
    cfg = abi.GroupConfig()             # no static volume
    assert lib.b200_group_create(C.byref(cfg), C.byref(h)) == abi.ERR_INVALID and not h.value
    lib.b200_group_destroy(None)
    eng = C.c_void_p()
    assert lib.b200_group_slot(None, 0, C.byref(eng), None, None) == abi.ERR_INVALID
    assert lib.b200_group_slot_images(None, 0, None) == abi.ERR_INVALID
    assert lib.b200_group_track_start(None, 0) == abi.ERR_INVALID
    assert lib.b200_group_frame_async(None, None, None, C.byref(v), None, 0, None, None, None) == abi.ERR_INVALID
    assert lib.b200_group_sync(None) == abi.ERR_INVALID
