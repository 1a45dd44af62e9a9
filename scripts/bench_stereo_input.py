"""Measures DynSLAM's per-frame input path on the KITTI-sized synthetic stream (1242x375) and prints one JSON line:

  (a) the host conversion DynSLAM runs today (DepthFromDisparityMap + CvToItm, single-threaded C: the oracle's restatement,
      pinned to the reference) followed by b200_host_frame_submit_raw (int16 depth + RGBA8 up, 6 B/px), against
  (b) b200_host_frame_submit_stereo (float disparity + BGR8 up, 7 B/px; the conversion runs on the device's copy stream).

Both run the same frames, pipelined over the two staging slots with decay, after a warm-up, alternating (a) and (b) `--reps`
times; the final states of (a) and (b) are compared. The conversion kernel's time comes from the launch trace's event pairs over
`--kernel-frames` frames of a separate run. The card's name and power limit are read in the same run.

    python scripts/bench_stereo_input.py [--steps 200] [--warmup 40] [--reps 2] [--kernel-frames 1000]
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from dynslam_b200 import abi, synth  # noqa: E402
from dynslam_b200 import engine as E  # noqa: E402
from tests import stereolib as S  # noqa: E402

W, H = synth.KITTI_W, synth.KITTI_H
DECAY = (1, 200)
N_DISTINCT = 48


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                           timeout=30)
        power = q.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        power = None
    return name, power


def make_frames():
    street = synth.StreetScene(seed=6, length_m=200.0)
    out = []
    for f in range(N_DISTINCT):
        depth, rgb, M, proj = synth.kitti_frame(street, f)
        bgr, disp = synth.stereo_frame(depth, rgb)
        out.append((torch.from_numpy(bgr).pin_memory(), torch.from_numpy(disp).pin_memory(), M, proj))
    return out


class Run:
    def __init__(self):
        dev = torch.device("cuda:0")
        self.scene = E.Scene(E.SceneParams(), 0x60000, 0x100000, 0x80000, device="cuda:0")
        self.eng = E.Engine(self.scene, (W, H))
        E.SceneReconstructionEngine(self.eng).ResetScene(self.scene)
        self.rs = E.VisualisationEngine(self.eng, self.scene).CreateRenderState((W, H))
        self.points = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)
        self.normals = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)
        self.view = E.View(torch.zeros((H, W), dtype=torch.float32, device=dev), torch.zeros((H, W, 4), dtype=torch.uint8, device=dev),
                           np.eye(4, dtype=np.float32), synth.kitti_intrinsics())
        self.out = [torch.zeros(H * W * 4, dtype=torch.uint8).pin_memory() for _ in range(2)]
        self.raw = [torch.zeros((H, W), dtype=torch.int16).pin_memory() for _ in range(2)]
        self.rgba = [torch.zeros((H, W, 4), dtype=torch.uint8).pin_memory() for _ in range(2)]
        self.calib = E.make_view_calib()
        self.din = E.make_depth_input(abi.DEPTH_IN_DISPARITY_F32, synth.KITTI_BASELINE_M, synth.KITTI_FX, 0.5, 20.0)
        self.L = S.oracle()
        self.host_s = 0.0
        torch.cuda.synchronize()

    def frame(self, i, frames, stereo):
        slot = i & 1
        bgr, disp, M, _ = frames[i % len(frames)]
        self.eng.host_frame_wait(slot)
        self.view.set_pose(M)
        if stereo:
            self.eng.host_frame_submit_stereo(self.rs, self.view, bgr, disp, self.din, self.calib, self.points, self.normals, decay=DECAY,
                                              h_out=self.out[slot], slot=slot)
        else:
            t0 = time.perf_counter()
            self.L.oracle_depth_from_disparity(self.raw[slot].data_ptr(), disp.data_ptr(), W * H, self.din.baseline_m,
                                               self.din.focal_length_px, self.din.min_depth_m, self.din.max_depth_m)
            self.L.oracle_bgr_to_rgba(self.rgba[slot].data_ptr(), bgr.data_ptr(), W * H)
            self.host_s += time.perf_counter() - t0
            self.eng.host_frame_submit_raw(self.rs, self.view, self.raw[slot], self.rgba[slot], self.calib, self.points, self.normals,
                                           decay=DECAY, h_out=self.out[slot], slot=slot)

    def drain(self):
        self.eng.host_frame_wait(0)
        self.eng.host_frame_wait(1)
        self.eng.sync(self.rs)

    def digest(self):
        h = hashlib.sha256()
        for t in (self.scene.hash, self.scene.voxels, self.scene.allocationList, self.rs.raycastImage, self.points):
            h.update(t.cpu().numpy().tobytes())
        return h.hexdigest()


def timed(frames, stereo, warmup, steps):
    r = Run()
    for i in range(warmup):
        r.frame(i, frames, stereo)
    r.drain()
    r.host_s = 0.0
    t0 = time.perf_counter()
    for i in range(warmup, warmup + steps):
        r.frame(i, frames, stereo)
    r.drain()
    dt = time.perf_counter() - t0
    return steps / dt, r.host_s / steps, r.digest()


def kernel_time(frames, n_frames):
    r = Run()
    for i in range(8):
        r.frame(i, frames, True)
    r.drain()
    r.eng.set_timing(3)
    durs = []
    for i in range(8, 8 + n_frames):
        r.frame(i, frames, True)
        if i % 50 == 49:
            r.drain()
            durs += [b - a for name, a, b in r.eng.trace() if name == "k_stereo_input"]
    r.drain()
    durs += [b - a for name, a, b in r.eng.trace() if name == "k_stereo_input"]
    r.eng.set_timing(0)
    return durs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=40)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--kernel-frames", type=int, default=1000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_stereo_input needs a GPU")
    name, power = card()
    frames = make_frames()
    host_fps, dev_fps, host_ms, digests = [], [], [], set()
    for _ in range(a.reps):
        fps, hs, dg = timed(frames, False, a.warmup, a.steps)
        host_fps.append(fps); host_ms.append(hs * 1e3); digests.add(("host", dg))
        fps, _, dg2 = timed(frames, True, a.warmup, a.steps)
        dev_fps.append(fps); digests.add(("device", dg2))
    parity = len({d for _, d in digests}) == 1
    durs = kernel_time(frames, a.kernel_frames)
    print(json.dumps({
        "workload": f"KITTI-sized synthetic stream {W}x{H}, DispNet disparity + BGR8 in, decay {DECAY}, pipelined over two slots",
        "gpu": name, "power_limit": power,
        "steps": a.steps, "warmup": a.warmup, "reps": a.reps,
        "host_convert_then_submit_raw_fps": [round(x, 1) for x in host_fps],
        "submit_stereo_fps": [round(x, 1) for x in dev_fps],
        "host_conversion_ms_per_frame": [round(x, 3) for x in host_ms],
        "conversion_kernel_us": {"launches": len(durs), "mean": round(float(np.mean(durs)), 2) if durs else None,
                                 "median": round(float(np.median(durs)), 2) if durs else None},
        "h2d_bytes_per_frame": {"host_convert_then_submit_raw": W * H * 6, "submit_stereo": W * H * 7},
        "final_state_equal": parity,
    }))


if __name__ == "__main__":
    main()
