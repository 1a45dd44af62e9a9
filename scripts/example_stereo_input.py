"""DynSLAM's DispNet input, from the files to the fused frame, with no host conversion: each frame's disparity PFM is read with
formats.read_pfm and handed to b200_host_frame_submit_stereo with the BGR colour image, as OpenCV loads it.

    python scripts/example_stereo_input.py [DIR]

DIR holds NNNNNN.pfm disparity maps and NNNNNN.bgr raw BGR8 frames (KITTI's 1242x375). Without DIR, a few synthetic frames of
the KITTI-shaped street are written to a temporary directory first.
"""
import os
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from dynslam_b200 import abi, formats, synth  # noqa: E402
from dynslam_b200 import engine as E  # noqa: E402

W, H = synth.KITTI_W, synth.KITTI_H


def write_synthetic(d, n=6):
    street = synth.StreetScene(seed=6, length_m=100.0)
    for f in range(n):
        depth, rgb, _, _ = synth.kitti_frame(street, f)
        bgr, disp = synth.stereo_frame(depth, rgb)
        with open(os.path.join(d, f"{f:06d}.pfm"), "wb") as fh:   # little-endian "Pf", bottom row first
            fh.write(b"Pf\n%d %d\n-1.0\n" % (W, H))
            fh.write(np.ascontiguousarray(disp[::-1]).astype("<f4").tobytes())
        bgr.tofile(os.path.join(d, f"{f:06d}.bgr"))


def main():
    d = sys.argv[1] if len(sys.argv) > 1 else tempfile.mkdtemp()
    if len(sys.argv) <= 1:
        write_synthetic(d)
    names = sorted(n[:-4] for n in os.listdir(d) if n.endswith(".pfm"))
    dev = torch.device("cuda:0")
    scene = E.Scene(E.SceneParams(), 0x20000, 0x40000, 0x20000, device="cuda:0")
    eng = E.Engine(scene, (W, H))
    rs = E.VisualisationEngine(eng, scene).CreateRenderState((W, H))
    E.SceneReconstructionEngine(eng).ResetScene(scene)
    points = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)
    normals = torch.zeros_like(points)
    view = E.View(torch.zeros((H, W), dtype=torch.float32, device=dev), torch.zeros((H, W, 4), dtype=torch.uint8, device=dev),
                  synth.kitti_pose(0), synth.kitti_intrinsics())
    din = E.make_depth_input(abi.DEPTH_IN_DISPARITY_F32, synth.KITTI_BASELINE_M, synth.KITTI_FX, 0.5, 20.0)
    calib = E.make_view_calib()
    out = [torch.zeros(H * W * 4, dtype=torch.uint8).pin_memory() for _ in range(2)]
    depth_mm = [torch.zeros((H, W), dtype=torch.int16, device=dev) for _ in range(2)]
    keep = [None, None]
    for i, n in enumerate(names):
        slot = i & 1
        eng.host_frame_wait(slot)
        disp = torch.from_numpy(formats.read_pfm(os.path.join(d, n + ".pfm"))).pin_memory()
        bgr = torch.from_numpy(np.fromfile(os.path.join(d, n + ".bgr"), np.uint8).reshape(H, W, 3)).pin_memory()
        keep[slot] = (disp, bgr)                                       # host buffers live until the slot is waited for
        view.set_pose(synth.kitti_pose(i))
        eng.host_frame_submit_stereo(rs, view, bgr, disp, din, calib, points, normals, decay=(1, 200), h_out=out[slot],
                                     depth_mm_out=depth_mm[slot], slot=slot)
    eng.host_frame_wait(0)
    eng.host_frame_wait(1)
    eng.sync(rs)
    last = (len(names) - 1) & 1
    print(f"{len(names)} frames fused; visible blocks {rs.noVisibleBlocks}; "
          f"valid depth pixels in the last frame {int((depth_mm[last] > 0).sum())}")


if __name__ == "__main__":
    main()
