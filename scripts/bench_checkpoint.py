"""Measures b200_checkpoint_save / b200_checkpoint_load on two maps and prints one JSON line:

  kitti: the KITTI-sized synthetic stream (1242x375, 5 cm voxels, decay (1, 200)) after a 230-frame pre-roll;
  4mm:   the 4 mm stream of bench.py's configs[4] (voxels 4 mm, mu 16 mm, its frame generator) in a 0x100000-block
         (4 GiB) voxel block array, fused until the array is three quarters full or --frames-4mm frames, for a large map.

For each: payload bytes and block count; save and load times from a host clock around the synchronous calls (median of
--reps) and their effective GB/s over the checkpoint's bytes; the classify / gather / scatter kernels' device times from
torch.profiler in a separate pass; and the naive arm, a whole-buffer cudaMemcpy of voxel block array, hash table, lists and
images to pinned host memory and back. Each load is checked by saving again (identical bytes). The card's name and power
limit are read in the same run.

    python scripts/bench_checkpoint.py [--preroll 230] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from dynslam_b200 import formats, synth  # noqa: E402
from dynslam_b200 import engine as E  # noqa: E402

W, H = synth.KITTI_W, synth.KITTI_H
DECAY = (1, 200)
NUM_BLOCKS, NUM_BUCKETS, EXCESS = 0x60000, 0x100000, 0x80000


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True,
                           timeout=30)
        power = q.stdout.strip() or None
    except (OSError, subprocess.SubprocessError):
        power = None
    return name, power


class Volume:
    def __init__(self, params, geometry=(NUM_BLOCKS, NUM_BUCKETS, EXCESS)):
        dev = torch.device("cuda:0")
        self.scene = E.Scene(params, *geometry, device="cuda:0")
        self.eng = E.Engine(self.scene, (W, H))
        E.SceneReconstructionEngine(self.eng).ResetScene(self.scene)
        self.rs = E.VisualisationEngine(self.eng, self.scene).CreateRenderState((W, H))
        self.points = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)
        self.normals = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)

    def fuse(self, frames, stop_below=None):
        n = 0
        for depth, rgb, M, proj in frames:
            v = E.View(torch.from_numpy(depth).cuda(), torch.from_numpy(rgb).cuda(), M, proj)
            self.eng.process_frame_async(self.rs, v, self.points, self.normals, decay=DECAY)
            self.eng.sync(self.rs)
            n += 1
            if stop_below is not None and self.scene.lastFreeBlockId < stop_below:
                break
        return n


def timed(fn, reps):
    ts = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), out


def naive_arm(vol, reps):
    """whole-buffer copies of everything a checkpoint covers (VBA, table, lists, images) to pinned memory and back"""
    s, r = vol.scene, vol.rs
    bufs = [s.voxels, s.hash, s.allocationList, s.excessList, r.visibleBlockPositions, r.entriesVisibleType, r.renderingRangeImage,
            r.raycastResult, r.raycastImage]
    host = [torch.empty(b.numel(), dtype=b.dtype).pin_memory() for b in bufs]
    nbytes = sum(b.numel() * b.element_size() for b in bufs)

    def down():
        for h, b in zip(host, bufs):
            h.copy_(b, non_blocking=True)

    def up():
        for h, b in zip(host, bufs):
            b.copy_(h, non_blocking=True)
    td, _ = timed(down, reps)
    tu, _ = timed(up, reps)
    return dict(bytes=nbytes, d2h_s=td, h2d_s=tu, d2h_GBps=nbytes / td / 1e9, h2d_GBps=nbytes / tu / 1e9)


def kernel_times(vol, buf):
    """device time per checkpoint kernel (sum over its launches) for one save and one load, from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        vol.eng.load_checkpoint(vol.scene, vol.rs, buf)   # (a load discards the kept classification: the save classifies again)
        vol.eng.save_checkpoint(vol.scene, vol.rs)
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        if ev.key.startswith("k_ck_"):
            name = ev.key.split("(")[0]
            out[name] = out.get(name, 0.0) + ev.device_time_total / 1e3   # us -> ms
    return {k: round(v, 3) for k, v in out.items()}


def measure(name, vol, reps):
    buf = vol.eng.save_checkpoint(vol.scene, vol.rs)
    hdr = formats.checkpoint_header(buf)
    t_save, _ = timed(lambda: vol.eng.save_checkpoint(vol.scene, vol.rs), reps)
    t_load, _ = timed(lambda: vol.eng.load_checkpoint(vol.scene, vol.rs, buf), reps)
    again = vol.eng.save_checkpoint(vol.scene, vol.rs)
    assert again.tobytes() == buf.tobytes(), "save -> load -> save differs"
    return dict(workload=name, bytes=int(buf.size), blocks=int(hdr["noBlocks"]), payload_bytes=int(hdr["noBlocks"]) * 4096,
                hash_entries=int(hdr["noEntries"]), queue_snapshots=int(hdr["noSnapshots"]),
                save_s=round(t_save, 5), load_s=round(t_load, 5), save_GBps=round(buf.size / t_save / 1e9, 3),
                load_GBps=round(buf.size / t_load / 1e9, 3), kernels_ms=kernel_times(vol, buf),
                naive={k: (round(v, 5) if isinstance(v, float) else v) for k, v in naive_arm(vol, reps).items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preroll", type=int, default=230)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--frames-4mm", type=int, default=24, help="at most this many frames for the 4 mm map")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_checkpoint.py measures on a GPU; none is visible")
    name, power = card()
    street = synth.StreetScene(seed=6, length_m=400.0)
    results = []
    v = Volume(E.SceneParams())
    v.fuse((synth.kitti_frame(street, f) for f in range(args.preroll)))
    results.append(measure(f"kitti 5 cm after {args.preroll} frames", v, args.reps))
    del v
    torch.cuda.empty_cache()
    import bench
    nb4 = 0x100000
    v = Volume(E.SceneParams(voxelSize=0.004, mu=0.016, maxW=50), (nb4, 0x400000, 0x100000))
    n = v.fuse(bench.gen_frames_hires(5, args.frames_4mm), stop_below=nb4 // 4)
    results.append(measure(f"kitti 4 mm after {n} frames", v, args.reps))
    print(json.dumps(dict(metric="checkpoint", device=name, power_limit=power, results=results)))


if __name__ == "__main__":
    main()
