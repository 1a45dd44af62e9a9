"""Seeded synthetic depth+RGB streams shaped like the BASELINE.json configs (SURVEY.md 8d).

No dataset is available offline, so every workload is rendered analytically with numpy:
  * config 1  "plane": 640x480, fronto-parallel plane at 1.5 m with a sine ripple, 2% holes.
  * config 2  "kitti": 1242x375 street (ground plane, two facades, parked-car boxes), camera
              moving +0.8 m/frame along z with a +-0.5 deg yaw sinusoid, depth clamped to
              [0.5, 20] m and quantised to integer millimetres (DS/Input.h:71-72,
              DS/InfiniTamDriver.cpp:52,77).
  * config 3  per-instance frames: the same frame masked to one car's silhouette (depth 0 / RGB
              255 outside, DS/InstRecLib/InstanceReconstructor.cpp:91-127).
Camera convention is KITTI's: x right, y down, z forward. Poses are world->camera (pose_d->GetM()).
"""
import numpy as np

KITTI_W, KITTI_H = 1242, 375
# itm-sample-calib-from-kitti-odometry-sequence-06.txt:1-3 rescaled from 1226x370 (SURVEY 8a)
KITTI_FX = KITTI_FY = 707.0912
KITTI_CX = 601.8873 * 1242.0 / 1226.0
KITTI_CY = 183.1104 * 375.0 / 370.0
KITTI_BASELINE_M = 0.5372   # the KITTI stereo rig's colour-camera baseline (DS/Input.h's StereoCalibration for the odometry sequences)


def _rot_y(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, 0, s], [0, 1, 0], [-s, 0, c]], dtype=np.float64)


class StreetScene:
    """Ground plane y=1.65, facades x=+-8, axis-aligned boxes ("parked cars")."""

    def __init__(self, seed=6, length_m=1200.0, n_boxes=None, facade_x=8.0):
        rng = np.random.RandomState(seed)
        self.seed = seed
        self.ground_y = 1.65
        self.facade_x = facade_x
        n = n_boxes if n_boxes is not None else int(length_m / 12.0)
        boxes = []
        for i in range(n):
            side = -1.0 if rng.rand() < 0.5 else 1.0
            cx = side * rng.uniform(2.6, 4.2)
            cz = 6.0 + i * (length_m / max(n, 1)) + rng.uniform(-2.0, 2.0)
            hw, hh, hl = rng.uniform(0.8, 0.95), rng.uniform(0.7, 0.85), rng.uniform(1.9, 2.4)
            boxes.append((cx - hw, self.ground_y - 2 * hh, cz - hl, cx + hw, self.ground_y, cz + hl))
        self.boxes = np.array(boxes, dtype=np.float64).reshape(-1, 6)

    def render(self, M_world_to_cam, w, h, fx, fy, cx, cy, zmin=0.5, zmax=20.0, extra_boxes=None,
               want_ids=False):
        """Returns depth (float32 metres, int-mm quantised, 0 = invalid), rgb (uint8 h,w,4) and
        optionally an id map (0 ground, 1/2 facades, 10+i box i, 1000+j extra box j)."""
        M = np.asarray(M_world_to_cam, dtype=np.float64)
        R, t = M[:3, :3], M[:3, 3]
        o = -R.T @ t
        xs = (np.arange(w, dtype=np.float64) - cx) / fx
        ys = (np.arange(h, dtype=np.float64) - cy) / fy
        dxc, dyc = np.meshgrid(xs, ys)
        dc = np.stack([dxc, dyc, np.ones_like(dxc)], axis=-1)  # camera-frame ray, z component 1
        d = dc @ R  # == (R^T dc)
        best = np.full((h, w), np.inf)
        ident = np.zeros((h, w), dtype=np.int32)

        def take(tt, valid, idv):
            nonlocal best, ident
            ok = valid & (tt > 1e-6) & (tt < best)
            best = np.where(ok, tt, best)
            ident = np.where(ok, idv, ident)

        with np.errstate(divide="ignore", invalid="ignore"):
            tg = (self.ground_y - o[1]) / d[..., 1]
            take(tg, d[..., 1] > 1e-9, 0)
            for k, sx in enumerate((-self.facade_x, self.facade_x)):
                tf = (sx - o[0]) / d[..., 0]
                yy = o[1] + tf * d[..., 1]
                take(tf, np.isfinite(tf) & (yy > -6.0) & (yy < self.ground_y), 1 + k)
            allb = [(10 + i, b) for i, b in enumerate(self.boxes)]
            if extra_boxes is not None:
                allb += [(1000 + j, b) for j, b in enumerate(np.asarray(extra_boxes, dtype=np.float64))]
            for idv, b in allb:
                # cheap cull: box centre must be within zmax+5 m of the camera
                c = 0.5 * (b[:3] + b[3:])
                if np.linalg.norm(c - o) > zmax + 6.0:
                    continue
                t0 = (b[:3] - o) / d
                t1 = (b[3:] - o) / d
                tn = np.minimum(t0, t1).max(axis=-1)
                tf_ = np.maximum(t0, t1).min(axis=-1)
                take(tn, (tn <= tf_) & np.isfinite(tn), idv)
        depth = np.where(np.isfinite(best), best, 0.0)  # camera z == t because dc.z == 1
        depth = np.where((depth >= zmin) & (depth <= zmax), depth, 0.0)
        mm = np.floor(depth * 1000.0 + 0.5).astype(np.int32)
        depth32 = (mm.astype(np.float32) * np.float32(0.001)).astype(np.float32)
        # colour: world-space checker tinted by surface id
        pw = o[None, None, :] + np.where(np.isfinite(best), best, 0.0)[..., None] * d
        chk = (np.floor(pw[..., 0] * 2.0) + np.floor(pw[..., 1] * 2.0) + np.floor(pw[..., 2] * 2.0)).astype(np.int64)
        base = np.where((chk & 1) == 0, 200, 90).astype(np.int32)
        tint = ((ident * 37 + self.seed * 11) % 97).astype(np.int32)
        rgb = np.zeros((h, w, 4), dtype=np.uint8)
        rgb[..., 0] = np.clip(base + tint - 40, 0, 255)
        rgb[..., 1] = np.clip(base - tint // 2, 0, 255)
        rgb[..., 2] = np.clip(base // 2 + tint, 0, 255)
        rgb[..., 3] = 255
        if want_ids:
            return depth32, rgb, ident
        return depth32, rgb


def kitti_pose(frame, step_m=0.8, yaw_amp_deg=0.5, yaw_period=60.0):
    """world->camera 4x4 (float32) of frame `frame` of the config-2 trajectory."""
    yaw = np.deg2rad(yaw_amp_deg) * np.sin(2.0 * np.pi * frame / yaw_period)
    Rcw = _rot_y(yaw)  # camera->world rotation
    pos = np.array([0.15 * np.sin(frame / 35.0), 0.0, step_m * frame])
    M = np.eye(4)
    M[:3, :3] = Rcw.T
    M[:3, 3] = -Rcw.T @ pos
    return M.astype(np.float32)


def kitti_intrinsics():
    return np.array([KITTI_FX, KITTI_FY, KITTI_CX, KITTI_CY], dtype=np.float32)


def kitti_frame(scene, frame, w=KITTI_W, h=KITTI_H, zmax=20.0, scale=1.0, **kw):
    """(depth, rgb, M_d, proj) for frame `frame` of config 2; `scale` shrinks the image for tests."""
    proj = kitti_intrinsics() * np.float32(scale)
    ww, hh = int(round(w * scale)), int(round(h * scale))
    M = kitti_pose(frame)
    out = scene.render(M, ww, hh, float(proj[0]), float(proj[1]), float(proj[2]), float(proj[3]), zmax=zmax, **kw)
    return out + (M, proj)


def stereo_frame(depth, rgb, focal_length_px=KITTI_FX, baseline_m=KITTI_BASELINE_M):
    """DynSLAM's stored stereo input for a rendered frame: OpenCV's BGR8 image (h, w, 3) of `rgb` and the float32 disparity
    f * b / depth a DispNet PFM holds (0 where there is no depth)."""
    bgr = np.ascontiguousarray(rgb[..., 2::-1])
    fb = np.float32(focal_length_px) * np.float32(baseline_m)
    with np.errstate(divide="ignore"):
        disp = np.where(depth > 0, fb / np.maximum(depth, np.float32(1e-30)), np.float32(0.0)).astype(np.float32)
    return bgr, disp


def plane_frame(seed=1, w=640, h=480, z0=1.5, ripple=0.1, holes=0.02):
    """config 1: plane at 1.5 m + 0.1*sin ripple, 2% holes, 8x8 checkerboard colour; identity pose,
    ITMIntrinsics defaults (580,580,320,240; Objects/ITMIntrinsics.h:50-55)."""
    rng = np.random.RandomState(seed)
    xs, ys = np.meshgrid(np.arange(w, dtype=np.float64), np.arange(h, dtype=np.float64))
    depth = z0 + ripple * np.sin(xs / 37.0) * np.cos(ys / 29.0)
    hole = rng.rand(h, w) < holes
    depth = np.where(hole, 0.0, depth).astype(np.float32)
    chk = ((xs.astype(np.int64) // 8 + ys.astype(np.int64) // 8) & 1).astype(np.int32)
    noise = rng.randint(0, 32, size=(h, w))
    rgb = np.zeros((h, w, 4), dtype=np.uint8)
    rgb[..., 0] = np.clip(80 + 120 * chk + noise, 0, 255)
    rgb[..., 1] = np.clip(200 - 100 * chk + noise // 2, 0, 255)
    rgb[..., 2] = np.clip(40 + noise * 3, 0, 255)
    rgb[..., 3] = 255
    M = np.eye(4, dtype=np.float32)
    proj = np.array([580.0, 580.0, 320.0, 240.0], dtype=np.float32)
    return depth, rgb, M, proj


class MovingCar:
    """One rigidly moving box for config 3 (its own trajectory; static in its own object frame)."""

    def __init__(self, idx, seed=3):
        rng = np.random.RandomState(seed * 101 + idx)
        self.idx = idx
        self.lane_x = (-1.0 if idx % 2 else 1.0) * rng.uniform(1.2, 2.4)
        self.z0 = 8.0 + 5.0 * idx + rng.uniform(0, 2.0)
        self.speed = rng.uniform(0.6, 1.0)  # m/frame, roughly follows the ego car
        self.half = np.array([rng.uniform(0.8, 0.95), rng.uniform(0.7, 0.8), rng.uniform(1.9, 2.3)])

    def centre(self, frame, ground_y=1.65):
        return np.array([self.lane_x, ground_y - self.half[1], self.z0 + self.speed * frame])

    def box(self, frame):
        c = self.centre(frame)
        return np.concatenate([c - self.half, c + self.half])

    def object_pose(self, frame, M_world_to_cam):
        """object->camera transform used as pose_d of the instance volume (object frame = box centre
        at frame 0, axis aligned): M_cam<-world * T_world<-object(frame)."""
        T = np.eye(4)
        T[:3, 3] = self.centre(frame) - self.centre(0)
        return (np.asarray(M_world_to_cam, dtype=np.float64) @ T).astype(np.float32)


def instance_frame(depth, rgb, ident, car_index):
    """Masked copy of the frame for one instance: depth 0 and RGB 255 outside the silhouette
    (ProcessSilhouette_CPU, DS/InstRecLib/InstanceReconstructor.cpp:91-127)."""
    m = ident == (1000 + car_index)
    d = np.where(m, depth, np.float32(0.0)).astype(np.float32)
    c = np.where(m[..., None], rgb, np.uint8(255)).astype(np.uint8)
    return d, c


def hash_index(pos, mask):
    """hashIndex of DA/ITMRepresentationAccess.h:10-12 on (n,3) int block positions (uint32 wrap-around arithmetic)."""
    p = np.asarray(pos).astype(np.int64) & 0xffffffff
    h = ((p[:, 0] * 73856093) & 0xffffffff) ^ ((p[:, 1] * 19349669) & 0xffffffff) ^ ((p[:, 2] * 83492791) & 0xffffffff)
    return (h & mask).astype(np.int64)


def prefilled_hash(n_blocks, num_buckets, excess_size, seed=4, allocated_time=0):
    """configs[3] (SURVEY 8d config 4): a valid ITMVoxelBlockHash state with `n_blocks` allocated blocks, built directly
    instead of through thousands of frames: block i (seeded random distinct positions) owns VBA slot i;
    the first block of every bucket sits in the ordered part, the others are chained through the excess list in order of
    arrival, exactly as serial allocation would leave them. Returns (entries[num_buckets+excess_size] with the HASH_ENTRY
    dtype, allocationList, excessList, lastFreeBlockId, lastFreeExcessListId) for a scene with numBlocks == n_blocks."""
    from . import abi
    rng = np.random.RandomState(seed)
    # distinct positions scattered over a (2 * half)^3 box of blocks, about 2% occupancy (surfaces are sparse in block space)
    half = max(8, int(np.ceil((n_blocks / 0.02) ** (1.0 / 3.0) / 2.0)))
    codes = np.unique(rng.randint(0, (2 * half) ** 3, size=int(n_blocks * 1.1) + 64, dtype=np.int64))
    while codes.size < n_blocks:
        codes = np.unique(np.concatenate([codes, rng.randint(0, (2 * half) ** 3, size=n_blocks, dtype=np.int64)]))
    codes = codes[rng.permutation(codes.size)[:n_blocks]]
    pos = np.stack([codes % (2 * half), (codes // (2 * half)) % (2 * half), codes // (2 * half) ** 2], axis=-1).astype(np.int64) - half
    pos = pos.astype(np.int16)
    bucket = hash_index(pos, num_buckets - 1)
    order = np.argsort(bucket, kind="stable")                  # arrival order inside a bucket = block id order
    b_sorted = bucket[order]
    first = np.ones(n_blocks, dtype=bool)
    first[1:] = b_sorted[1:] != b_sorted[:-1]
    ent = np.zeros(num_buckets + excess_size, dtype=abi.HASH_ENTRY_DTYPE)
    ent["ptr"] = -2
    heads = order[first]
    ent["pos"][bucket[heads]] = pos[heads]
    ent["ptr"][bucket[heads]] = heads
    ent["allocatedTime"][bucket[heads]] = allocated_time
    nf = np.nonzero(~first)[0]
    rest = order[nf]
    n_ex = rest.size
    if n_ex > excess_size:
        raise ValueError(f"{n_ex} chained blocks do not fit the excess list of {excess_size}")
    # excess slots are popped from the top of the free stack (excessList[i] = i), in block-id order
    slot_of = np.full(n_blocks, -1, dtype=np.int64)
    slot_of[np.sort(rest)] = excess_size - 1 - np.arange(n_ex)
    eidx = num_buckets + slot_of[rest]
    ent["pos"][eidx] = pos[rest]
    ent["ptr"][eidx] = rest
    ent["allocatedTime"][eidx] = allocated_time
    prev = order[nf - 1]                                       # predecessor in the same bucket's chain
    prev_idx = np.where(first[nf - 1], bucket[prev], num_buckets + slot_of[prev])
    ent["offset"][prev_idx] = slot_of[rest] + 1
    alloc_list = np.arange(n_blocks, dtype=np.int32)
    excess_list = np.arange(excess_size, dtype=np.int32)
    return ent, alloc_list, excess_list, -1, excess_size - 1 - n_ex


class FollowedCar(MovingCar):
    """A car that stays in the ego camera's view for the whole stream (configs[2] bench): it drives at the ego speed with a
    slow longitudinal oscillation, car `idx` further ahead than car `idx - 1`, alternating lanes."""

    def __init__(self, idx, seed=3, step_m=0.8):
        super().__init__(idx, seed)
        self.step_m = step_m
        self.z_rel = 5.5 + 1.7 * idx
        self.phase = 0.9 * idx

    def centre(self, frame, ground_y=1.65):
        z = self.step_m * frame + self.z_rel + 1.2 * np.sin(frame / 23.0 + self.phase)
        return np.array([self.lane_x, ground_y - self.half[1], z])


def silhouette_mask(ident, car_index):
    """(inclusive bbox, box-sized uint8 mask) of car `car_index` in an id map, or None when it is not visible — the form
    DynSLAM's segmentation provider hands to InstanceReconstructor (Utils/Mask.h, Utils/BoundingBox.h)."""
    m = ident == (1000 + car_index)
    if not m.any():
        return None
    ys, xs = np.nonzero(m)
    x0, x1, y0, y1 = int(xs.min()), int(xs.max()), int(ys.min()), int(ys.max())
    return (x0, y0, x1, y1), np.ascontiguousarray(m[y0:y1 + 1, x0:x1 + 1]).astype(np.uint8)
