"""Measures the free-view preview (colour + depth images of a volume from a novel pose, landed on the host) and prints one
JSON line. Two maps: the KITTI-sized synthetic stream (1242x375, 5 cm voxels, decay (1, 200)) after a 230-frame pre-roll, and
the 4 mm stream of bench.py's configs[4] after 24 frames. A fixed, seeded set of 64 novel poses. Arms, alternated round by round
in one process, each warmed up and timed with a host clock around work that ends in a synchronise, for at least --seconds each:

  reference_shape     per preview, colour then depth as DynSLAM asks for them: 2 x (b200_find_visible_blocks,
                      b200_expected_depths, b200_render_image), each image copied to pageable host memory
  fused               b200_render_view_submit / b200_render_view_wait over the two slots, pinned host images
  fused_under_fusion  (KITTI map) the fused frame loop alone, and with a preview submitted after every frame: frames/s of both
  three_volumes       (KITTI map) static volume + two instance-sized volumes on engines of their own, composited:
                      reference shape per volume + b200_composite_instances, against b200_render_view_async per engine +
                      b200_engine_wait_engine + b200_composite_instances

Also: device time per kernel and preview from the engine's launch trace (CUDA events around every launch), launches per
preview from b200_frame_stats.launches, and the host synchronisations per preview AS READ FROM THE CODE (engine.cu,
preview.cu), not counted at run time. The last pose's images of both arms are compared, byte for byte, before anything is
printed. The card's name and power limit are read in the same run.

    python scripts/bench_free_view.py [--preroll 230] [--seconds 1.5]
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

from dynslam_b200 import abi, synth  # noqa: E402
from dynslam_b200 import engine as E  # noqa: E402

W, H = synth.KITTI_W, synth.KITTI_H
DECAY = (1, 200)
GEOMETRY = (0x60000, 0x100000, 0x80000)
COLOUR = abi.RENDER_COLOUR_FROM_VOLUME
# host synchronisations per preview, read from the code: each of the three synchronous calls ends in one stream synchronise,
# and each pageable cudaMemcpy blocks: 2 x (3 + 1);
# the fused arm blocks once, in b200_render_view_wait
HOST_SYNCS_READ_FROM_CODE = dict(reference_shape=8, fused=1)


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
    def __init__(self, params, geometry=GEOMETRY):
        dev = torch.device("cuda:0")
        self.scene = E.Scene(params, *geometry, device="cuda:0")
        self.eng = E.Engine(self.scene, (W, H))
        E.SceneReconstructionEngine(self.eng).ResetScene(self.scene)
        self.vis = E.VisualisationEngine(self.eng, self.scene)
        self.rs = self.vis.CreateRenderState((W, H))
        self.fv = [self.vis.CreateRenderState((W, H)) for _ in range(2)]
        self.points = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)
        self.normals = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)
        self.col = torch.zeros(H * W * 4, dtype=torch.uint8, device=dev)
        self.dep = torch.zeros(H * W, dtype=torch.float32, device=dev)
        self.h_col = [torch.zeros(H * W * 4, dtype=torch.uint8).pin_memory() for _ in range(2)]
        self.h_dep = [torch.zeros(H * W, dtype=torch.float32).pin_memory() for _ in range(2)]
        self.p_col, self.p_dep = torch.zeros(H * W * 4, dtype=torch.uint8), torch.zeros(H * W, dtype=torch.float32)   # pageable

    def fuse(self, frames):
        for depth, rgb, M, proj in frames:
            v = E.View(torch.from_numpy(depth).cuda(), torch.from_numpy(rgb).cuda(), M, proj)
            self.eng.process_frame_async(self.rs, v, self.points, self.normals, decay=DECAY)
            self.eng.sync(self.rs)

    def reference_shape(self, cam, to_host=True):
        """GetImage then GetFloatImage from one pose: everything twice"""
        for t, out in ((COLOUR, self.p_col), (abi.RENDER_DEPTH_MAP, self.p_dep)):
            self.vis.FindVisibleBlocks(cam, self.fv[0])
            self.vis.CreateExpectedDepths(cam, self.fv[0])
            self.vis.RenderImage(cam, self.fv[0], self.col, self.dep, t)
            if to_host:
                out.copy_(self.col if t == COLOUR else self.dep)


def novel_poses(frames, n=64, seed=3):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        M = synth.kitti_pose(int(rng.integers(0, frames))).astype(np.float64)
        yaw = np.deg2rad(rng.uniform(-30.0, 30.0))
        R = np.eye(4)
        R[0, 0], R[0, 2], R[2, 0], R[2, 2] = np.cos(yaw), np.sin(yaw), -np.sin(yaw), np.cos(yaw)
        M = R @ M
        M[0, 3] += rng.uniform(-1.0, 1.0)
        M[1, 3] += rng.uniform(0.0, 0.5)
        out.append(E.make_camera(M.astype(np.float32), synth.kitti_intrinsics()))
    return out


def run_fused(vol, cams):
    for k, cam in enumerate(cams):
        s = k & 1
        vol.vis.RenderFreeViewWait(s)
        vol.vis.RenderFreeViewSubmit(cam, vol.fv[s], vol.h_col[s], vol.h_dep[s], COLOUR, s)
    vol.vis.RenderFreeViewWait(0)
    vol.vis.RenderFreeViewWait(1)


def alternate(arms, seconds):
    """arms: name -> (callable, previews per call). Rounds alternate the arms until each has run for `seconds`."""
    for fn, _ in arms.values():
        fn()                                       # warm-up: every shape the timed window uses
    spent, done = {k: 0.0 for k in arms}, {k: 0 for k in arms}
    while min(spent.values()) < seconds:
        for name, (fn, n) in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            spent[name] += time.perf_counter() - t0
            done[name] += n
    return {k: dict(previews=done[k], seconds=round(spent[k], 4), previews_per_s=round(done[k] / spent[k], 1),
                    ms_per_preview=round(1e3 * spent[k] / done[k], 4)) for k in arms}


def kernel_times(vol, cams, fn):
    """device time per kernel name, per preview, from the launch trace (an event pair around every traced launch)"""
    vol.eng.set_timing(3)
    fn(cams)
    rows = vol.eng.trace()
    vol.eng.set_timing(0)
    out = {}
    for name, a, b in rows:
        out[name] = out.get(name, 0.0) + (b - a)
    return {k: round(v / len(cams), 2) for k, v in sorted(out.items())}


def launches(vol, cams, fn):
    before = vol.eng.stats().launches
    fn(cams)
    return (vol.eng.stats().launches - before) / len(cams)


def check_equal(vol, cam):
    vol.reference_shape(cam)
    run_fused(vol, [cam])
    assert vol.p_col.numpy().tobytes() == vol.h_col[0].numpy().tobytes(), "colour images of the two arms differ"
    assert vol.p_dep.numpy().tobytes() == vol.h_dep[0].numpy().tobytes(), "depth images of the two arms differ"
    return bool((vol.p_dep.numpy() > 0).any())


def measure_single(name, vol, cams, seconds):
    ref = lambda cs=cams: [vol.reference_shape(c) for c in cs]
    fused = lambda cs=cams: run_fused(vol, cs)
    res = alternate(dict(reference_shape=(ref, len(cams)), fused=(fused, len(cams))), seconds)
    for arm, fn in (("reference_shape", ref), ("fused", fused)):
        res[arm]["kernel_us_per_preview"] = kernel_times(vol, cams[:16], fn)
        res[arm]["launches_per_preview"] = launches(vol, cams[:16], fn)
        res[arm]["host_syncs_per_preview_read_from_code"] = HOST_SYNCS_READ_FROM_CODE[arm]
    return dict(workload=name, outputs_equal=True, last_pose_sees_surface=check_equal(vol, cams[-1]), **res)


def measure_under_fusion(vol, street, first, cams, seconds):
    views = []
    for f in range(first, first + 8):
        depth, rgb, M, proj = synth.kitti_frame(street, f)
        views.append(E.View(torch.from_numpy(depth).cuda(), torch.from_numpy(rgb).cuda(), M, proj))
    torch.cuda.synchronize()
    n = 64

    def loop(previews):
        for i in range(n):
            vol.eng.process_frame_async(vol.rs, views[i % 8], vol.points, vol.normals, decay=DECAY)
            if previews:
                s = i & 1
                vol.vis.RenderFreeViewWait(s)
                vol.vis.RenderFreeViewSubmit(cams[i % len(cams)], vol.fv[s], vol.h_col[s], vol.h_dep[s], COLOUR, s)
        vol.vis.RenderFreeViewWait(0)
        vol.vis.RenderFreeViewWait(1)
        vol.eng.sync(vol.rs)
    res = alternate(dict(fusion_alone=(lambda: loop(False), n), fusion_with_previews=(lambda: loop(True), n)), seconds)
    return {k: dict(frames=v["previews"], seconds=v["seconds"], frames_per_s=v["previews_per_s"], ms_per_frame=v["ms_per_preview"])
            for k, v in res.items()}


def measure_three_volumes(static, cams, seconds):
    cars = []
    for seed in (11, 12):
        v = Volume(E.SceneParams(voxelSize=0.035, mu=1.0), (7142, GEOMETRY[1], GEOMETRY[2]))
        sc = synth.StreetScene(seed=seed, length_m=60.0)
        v.fuse(synth.kitti_frame(sc, 2 * f, zmax=8.0) for f in range(3))
        cars.append(v)
    vols = [static] + cars
    fr = E.InstanceFrames(static.eng)
    tints = E.MATPLOTLIB2_PALETTE[:2]
    out = {}

    def finish(tag):
        fr.CompositeInstances(static.col, static.dep, [(c.col, c.dep, t) for c, t in zip(cars, tints)], wait_inputs=False)
        static.p_col.copy_(static.col)
        static.p_dep.copy_(static.dep)
        out[tag] = (static.p_col.numpy().tobytes(), static.p_dep.numpy().tobytes())

    def old(cs=cams):
        for cam in cs:
            for v in vols:       # colour last, so that col and dep both hold this pose's render
                v.vis.FindVisibleBlocks(cam, v.fv[0]); v.vis.CreateExpectedDepths(cam, v.fv[0])
                v.vis.RenderImage(cam, v.fv[0], v.col, v.dep, abi.RENDER_DEPTH_MAP)
                v.vis.FindVisibleBlocks(cam, v.fv[0]); v.vis.CreateExpectedDepths(cam, v.fv[0])
                v.vis.RenderImage(cam, v.fv[0], v.col, v.dep, COLOUR)
            finish("old")

    def new(cs=cams):
        for cam in cs:
            for v in vols:
                v.vis.RenderFreeView(cam, v.fv[0], v.col, v.dep, COLOUR, sync=False)
            for c in cars:
                static.eng.wait_engine(c.eng)
            finish("new")
    res = alternate(dict(reference_shape=(old, len(cams)), fused=(new, len(cams))), seconds)
    old(cams[-1:])
    new(cams[-1:])
    assert out["old"] == out["new"], "composites of the two arms differ"
    return dict(volumes=3, outputs_equal=True, **res)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--preroll", type=int, default=230)
    ap.add_argument("--frames-4mm", type=int, default=24)
    ap.add_argument("--seconds", type=float, default=1.5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_free_view.py measures on a GPU; none is visible")
    name, power = card()
    street = synth.StreetScene(seed=6, length_m=400.0)
    v = Volume(E.SceneParams())
    v.fuse(synth.kitti_frame(street, f) for f in range(args.preroll))
    cams = novel_poses(args.preroll)
    results = [measure_single(f"kitti 5 cm after {args.preroll} frames", v, cams, args.seconds)]
    results[0]["three_volumes"] = measure_three_volumes(v, cams, args.seconds)
    results[0]["fused_under_fusion"] = measure_under_fusion(v, street, args.preroll, cams, args.seconds)
    del v
    torch.cuda.empty_cache()
    import bench
    v = Volume(E.SceneParams(voxelSize=0.004, mu=0.016, maxW=50), (0x100000, 0x400000, 0x100000))
    v.fuse(bench.gen_frames_hires(5, args.frames_4mm))
    results.append(measure_single(f"kitti 4 mm after {args.frames_4mm} frames", v, novel_poses(args.frames_4mm), args.seconds))
    print(json.dumps(dict(metric="free_view_preview", device=name, power_limit=power, image=[W, H], poses=len(cams), results=results)))


if __name__ == "__main__":
    main()
