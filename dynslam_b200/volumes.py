"""The static map and K car volumes on one GPU: DynSLAM's per-frame sequence (InstanceReconstructor::ProcessFrame + FuseFrame,
DS/InstRecLib/InstanceReconstructor.cpp:363-389, :569-699) over the C-ABI, with no host synchronisation inside a frame.

One engine per volume. With shared_stream=True every engine runs on one stream (the volumes one after another); otherwise each
engine has a stream of its own and the frame forks and joins through b200_engine_wait_engine, so the volumes fuse concurrently
(include/b200fusion.h, at the engine handle; INTEGRATION.md, "Static map and car volumes on one GPU"). Both forms compute the
same bytes.

StreetVolumes makes each call of that sequence from Python; GroupStreetVolumes enqueues the same frame as one call of a volume
group (b200_group_frame_async), whose car volumes are slots created up front and restarted on the device for a new track.
"""
import numpy as np
import torch

from . import engine as E
from . import synth

# configs[2] of bench.py: the static map at ITMLibSettings' sizes, a car volume as InstanceReconstructor.cpp:365-389 makes it
# (voxel 0.035 m, mu 1.0, 5 x 5 x 10 m / 0.035 m -> 7142 blocks) with the full-size table
STATIC_BLOCKS, NUM_BUCKETS, EXCESS = 0x60000, 0x100000, 0x80000
CAR_BLOCKS = 7142
DECAY = (1, 200)                 # --max_decay_weight=1 --min_decay_age=200 (DynSLAMGUI.cpp:38-40)
TINTS = [(0x1f, 0x77, 0xb4, 255), (0xff, 0x7f, 0x0e, 255), (0x2c, 0xa0, 0x2c, 255), (0xd6, 0x27, 0x28, 255),
         (0x94, 0x67, 0xbd, 255), (0x8c, 0x56, 0x4b, 255), (0xe3, 0x77, 0xc2, 255), (0x7f, 0x7f, 0x7f, 255)]


def street_frames(first, count, ncars, w=synth.KITTI_W, h=synth.KITTI_H, seed=6, length_m=1200.0):
    """(depth, rgb, M, proj, [silhouette mask or None per car]) of the street of `seed` with `ncars` followed cars, at w x h
    (the KITTI intrinsics scaled to the size)"""
    scene = synth.StreetScene(seed=seed, length_m=length_m)
    cars = [synth.FollowedCar(i, seed=3) for i in range(ncars)]
    proj = synth.kitti_intrinsics() * np.float32(w / synth.KITTI_W)
    out = []
    for f in range(first, first + count):
        M = synth.kitti_pose(f)
        depth, rgb, ident = scene.render(M, w, h, float(proj[0]), float(proj[1]), float(proj[2]), float(proj[3]),
                                         extra_boxes=[c.box(f) for c in cars], want_ids=True)
        out.append((depth, rgb, M, proj, [synth.silhouette_mask(ident, i) for i in range(ncars)]))
    return out


class DeviceFrame:
    """One input frame resident on the device: depth, colour, and the silhouette ops that cut each car out of it"""

    def __init__(self, frame, index, cars, inst_rgb, inst_depth, device):
        depth, rgb, M, proj, masks = frame
        self.depth = torch.from_numpy(depth).to(device)
        self.rgb = torch.from_numpy(rgb).to(device)
        self.M, self.proj, self.index = M, proj, index
        self.car_poses = [car.object_pose(index, M) for car in cars]
        self.keep, ops = [], []
        self.masks = [None] * len(masks)          # per car: its b200_mask, or None when it is not in the frame
        for k, m in enumerate(masks):
            if m is None:
                continue
            t = torch.from_numpy(m[1]).to(device)
            self.keep.append(t)
            mk = E.make_mask(m[0], t)
            self.masks[k] = mk
            ops.append((E.EXTRACT, mk, mk, inst_rgb[k], inst_depth[k]))
        self.ops = E.InstanceFrames.prepare_ops(ops) if ops else None


class StreetVolumes:
    """The static map and `ncars` car volumes of one GPU, fed frame by frame (step) in DynSLAM's order:
    silhouettes on the static engine's stream -> every car waits for it and fuses its instance frame (colour and depth renders
    for the composite) -> the static map fuses the rest -> the static engine waits for every car and composites."""

    def __init__(self, ncars, w, h, shared_stream, device="cuda:0", decay=DECAY, static_blocks=STATIC_BLOCKS,
                 car_blocks=CAR_BLOCKS, num_buckets=NUM_BUCKETS, excess=EXCESS):
        dev = torch.device(device)
        self.dev, self.w, self.h, self.decay, self.ncars = dev, w, h, decay, ncars
        n = 1 + ncars
        first = torch.cuda.Stream(device=dev)
        self.streams = [first] * n if shared_stream else [first] + [torch.cuda.Stream(device=dev) for _ in range(ncars)]
        self.scenes, self.engines, self.rs, self.points, self.normals = [], [], [], [], []
        for i in range(n):
            with torch.cuda.stream(self.streams[i]):
                if i == 0:
                    sc = E.Scene(E.SceneParams(), static_blocks, num_buckets, excess, device=device)
                else:
                    sc = E.Scene(E.SceneParams(voxelSize=0.035, mu=1.0, maxW=50), car_blocks, num_buckets, excess, device=device)
                eng = E.Engine(sc, (w, h), stream=self.streams[i].cuda_stream)
                E.SceneReconstructionEngine(eng).ResetScene(sc)
                self.scenes.append(sc)
                self.engines.append(eng)
                self.rs.append(E.VisualisationEngine(eng, sc).CreateRenderState((w, h)))
                self.points.append(torch.zeros(h * w * 4, dtype=torch.float32, device=dev))
                self.normals.append(torch.zeros(h * w * 4, dtype=torch.float32, device=dev))
        with torch.cuda.stream(first):
            self.frame_rgb = torch.zeros((h, w, 4), dtype=torch.uint8, device=dev)
            self.frame_depth = torch.zeros((h, w), dtype=torch.float32, device=dev)
            self.inst_rgb = [torch.zeros((h, w, 4), dtype=torch.uint8, device=dev) for _ in range(ncars)]
            self.inst_depth = [torch.zeros((h, w), dtype=torch.float32, device=dev) for _ in range(ncars)]
            self.car_colour = [torch.zeros((h, w, 4), dtype=torch.uint8, device=dev) for _ in range(ncars)]
            self.car_depth = [torch.zeros((h, w), dtype=torch.float32, device=dev) for _ in range(ncars)]
            self.static_depth = torch.zeros((h, w), dtype=torch.float32, device=dev)
            self.out_color = torch.zeros((h, w, 4), dtype=torch.uint8, device=dev)
            self.out_depth = torch.zeros((h, w), dtype=torch.float32, device=dev)
        torch.cuda.synchronize(dev)
        self.frames_api = E.InstanceFrames(self.engines[0])
        self._cars = [synth.FollowedCar(i, seed=3) for i in range(ncars)]

    def upload(self, frames, first=0):
        """device-resident copies of host frames (street_frames), frame indices first, first + 1, ..."""
        return [DeviceFrame(fr, first + i, self._cars, self.inst_rgb, self.inst_depth, self.dev) for i, fr in enumerate(frames)]

    def step(self, fr, between=None):
        """enqueue one frame of every volume; no host synchronisation. between(self) is called after the cars' frames are
        enqueued and before the static map's (free-view renders, stand-alone calls of the tests)"""
        static, s0 = self.engines[0], self.streams[0]
        with torch.cuda.stream(s0):
            self.frame_depth.copy_(fr.depth)
            self.frame_rgb.copy_(fr.rgb)
            for k in range(self.ncars):     # an instance frame holds its car's pixels only (ProcessSilhouette_CPU, :91-127)
                self.inst_depth[k].zero_()
                self.inst_rgb[k].fill_(255)
            if fr.ops is not None:
                self.frames_api.ProcessSilhouettes(self.frame_rgb, self.frame_depth, fr.ops, sync=False, wait_inputs=False)
        for k in range(self.ncars):
            car = self.engines[1 + k]
            with torch.cuda.stream(self.streams[1 + k]):
                car.wait_engine(static)
                view = E.View(self.inst_depth[k], self.inst_rgb[k], fr.car_poses[k], fr.proj)
                car.process_frame_async(self.rs[1 + k], view, self.points[1 + k], self.normals[1 + k], decay=self.decay,
                                        colour_out=self.car_colour[k], depth_out=self.car_depth[k])
        if between is not None:
            between(self)
        with torch.cuda.stream(s0):
            view = E.View(self.frame_depth, self.frame_rgb, fr.M, fr.proj)
            static.process_frame_async(self.rs[0], view, self.points[0], self.normals[0], decay=self.decay, depth_out=self.static_depth)
            for k in range(self.ncars):
                static.wait_engine(self.engines[1 + k])
            # the static map's layer is its shaded raycast image (the ICP pass writes it), the cars go on top
            self.out_color.copy_(self._raycast_image(0))
            self.out_depth.copy_(self.static_depth)
            layers = [(self.car_colour[k], self.car_depth[k], TINTS[k % len(TINTS)]) for k in range(self.ncars)]
            self.frames_api.CompositeInstances(self.out_color, self.out_depth, layers, wait_inputs=False)

    def _raycast_image(self, i):
        return self.rs[i].raycastImage.view(self.h, self.w, 4)

    def synchronize(self):
        for s in set(self.streams):
            s.synchronize()
        for i, eng in enumerate(self.engines):
            eng.sync(self.rs[i])

    def state(self, i):
        """the bytes of volume i: its checkpoint (b200_checkpoint_save), ray points, raycast image and ICP maps"""
        ck = self.engines[i].save_checkpoint(self.scenes[i], self.rs[i])
        rs = self.rs[i]
        return {"checkpoint": ck, "rays": rs.raycastResult.cpu().numpy().tobytes(), "image": self._raycast_image(i).cpu().numpy().tobytes(),
                "points": self.points[i].cpu().numpy().tobytes(), "normals": self.normals[i].cpu().numpy().tobytes()}

    def close(self):
        for eng in self.engines:
            eng.close()


class GroupStreetVolumes:
    """StreetVolumes' volumes and frames through a volume group (E.VolumeGroup): the static map is an engine of its own, the
    `ncars` car volumes are slots 0 .. ncars-1 of the group, started at construction. step(fr) is one b200_group_frame_async
    after the two copies of the input frame; state(i) gives the same bytes as StreetVolumes.state(i) for the same frames."""

    def __init__(self, ncars, w, h, shared_stream, device="cuda:0", decay=DECAY, static_blocks=STATIC_BLOCKS,
                 car_blocks=CAR_BLOCKS, num_buckets=NUM_BUCKETS, excess=EXCESS, max_cars=None):
        dev = torch.device(device)
        self.dev, self.w, self.h, self.decay, self.ncars = dev, w, h, decay, ncars
        self.stream = torch.cuda.Stream(device=dev)
        with torch.cuda.stream(self.stream):
            self.static_scene = E.Scene(E.SceneParams(), static_blocks, num_buckets, excess, device=device)
            self.static = E.Engine(self.static_scene, (w, h), stream=self.stream.cuda_stream)
            E.SceneReconstructionEngine(self.static).ResetScene(self.static_scene)
            self.static_rs = E.VisualisationEngine(self.static, self.static_scene).CreateRenderState((w, h))
            self.static_points = torch.zeros(h * w * 4, dtype=torch.float32, device=dev)
            self.static_normals = torch.zeros(h * w * 4, dtype=torch.float32, device=dev)
            self.frame_rgb = torch.zeros((h, w, 4), dtype=torch.uint8, device=dev)
            self.frame_depth = torch.zeros((h, w), dtype=torch.float32, device=dev)
            self.out_color = torch.zeros((h, w, 4), dtype=torch.uint8, device=dev)
            self.out_depth = torch.zeros((h, w), dtype=torch.float32, device=dev)
        torch.cuda.synchronize(dev)
        self.group = E.VolumeGroup(self.static, self.static_rs, self.static_points, self.static_normals,
                                   ncars if max_cars is None else max_cars, shared_stream=shared_stream, numBlocks=car_blocks,
                                   numBuckets=num_buckets, excessSize=excess, voxelSize=0.035, mu=1.0, maxW=50)
        for k in range(ncars):
            self.group.track_start(k)
        self.static_view = E.View(self.frame_depth, self.frame_rgb, np.eye(4, dtype=np.float32), synth.kitti_intrinsics())
        self._cars = [synth.FollowedCar(i, seed=3) for i in range(ncars)]

    def upload(self, frames, first=0):
        """device-resident copies of host frames (street_frames), as StreetVolumes.upload makes them"""
        return [DeviceFrame(fr, first + i, self._cars, [None] * self.ncars, [None] * self.ncars, self.dev)
                for i, fr in enumerate(frames)]

    def cars(self, fr, plan=None):
        """the GroupCar list of frame fr: car k in slot k, extracted when it is in the frame, fused, with TINTS[k]. plan (optional):
        per car, (action, fuse) replacing that default, or None to leave the car out of the frame"""
        out = []
        for k in range(self.ncars):
            action, fuse = (E.EXTRACT if fr.masks[k] is not None else E.KEEP), True
            if plan is not None:
                if plan[k] is None:
                    continue
                action, fuse = plan[k]
            m = fr.masks[k] if action != E.KEEP else None
            out.append(E.GroupCar(k, action, m, m, fr.car_poses[k], fr.proj, fuse=fuse, tint=TINTS[k % len(TINTS)]))
        return out

    def prepare(self, fr, plan=None):
        """(fr, the prepared b200_group_car array): enqueued by step without building the array again"""
        return fr, E.VolumeGroup.prepare(self.cars(fr, plan))

    def step(self, fr, plan=None):
        """enqueue one frame of every volume: the two copies of the input frame and one b200_group_frame_async; no host
        synchronisation. fr: a DeviceFrame or prepare()'s result"""
        fr, cars = fr if isinstance(fr, tuple) else self.prepare(fr, plan)
        with torch.cuda.stream(self.stream):
            self.frame_depth.copy_(fr.depth)
            self.frame_rgb.copy_(fr.rgb)
            self.static_view.set_pose(fr.M)
            self.static_view.c.proj_d = self.static_view.c.proj_rgb = E.abi.f4(*[float(x) for x in fr.proj])
            self.group.frame(self.frame_rgb, self.frame_depth, self.static_view, cars, self.out_color, self.out_depth, decay=self.decay,
                             wait_inputs=False)

    def track_start(self, slot):
        with torch.cuda.stream(self.stream):
            self.group.track_start(slot)

    def synchronize(self):
        self.stream.synchronize()
        self.group.sync()

    def volume(self, i):
        """(engine, scene, render state, points, normals) of volume i: 0 the static map, 1 + k car k's slot"""
        if i == 0:
            return self.static, self.static_scene, self.static_rs, self.static_points, self.static_normals
        sl = self.group.slots[i - 1]
        return sl.engine, sl.scene, sl.rs, sl.points, sl.normals

    def state(self, i):
        """the bytes of volume i, as StreetVolumes.state(i) gives them"""
        eng, sc, rs, points, normals = self.volume(i)
        ck = eng.save_checkpoint(sc, rs)
        return {"checkpoint": ck, "rays": rs.raycastResult.cpu().numpy().tobytes(),
                "image": rs.raycastImage.view(self.h, self.w, 4).cpu().numpy().tobytes(),
                "points": points.cpu().numpy().tobytes(), "normals": normals.cpu().numpy().tobytes()}

    def close(self):
        self.group.close()
        self.static.close()
