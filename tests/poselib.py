"""General-pose trajectories for the fusion tests: cameras that reverse, turn in place, pitch, roll, turn upside down, look
down at the ground from 1 m, or sit kilometres from the origin, with fx != fy, principal points off the image centre (one
outside the image) and image sizes that are not multiples of the kernels' tiles. Seeded and deterministic.

Every frame is rendered in street coordinates (synth.StreetScene: ground y = 1.65, facades x = +-8, boxes), and the fusion
path is given M_world = M_street @ T(offset): a world point p sits at p + offset in the street. The offset moves the map's
block coordinates anywhere, negative included, while the scene stays analytic, so a fused surface can also be checked
against the geometry it was built from (`surface_distance`, float64)."""
import numpy as np

from dynslam_b200 import synth

SCENE_SEED, SCENE_LENGTH = 6, 80.0
VOXEL = 0.05


def _rx(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[1, 0, 0], [0, c, -s], [0, s, c]], dtype=np.float64)


def _rz(a):
    c, s = np.cos(a), np.sin(a)
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1]], dtype=np.float64)


def street_pose(centre, yaw=0.0, pitch=0.0, roll=0.0):
    """world->camera 4x4 (float64) of a camera at `centre` (street coordinates, KITTI axes: x right, y down, z forward).
    Angles in degrees: yaw turns right about the vertical, pitch < 0 looks down, roll turns the image clockwise."""
    R = synth._rot_y(np.deg2rad(yaw)) @ _rx(np.deg2rad(pitch)) @ _rz(np.deg2rad(roll))   # camera -> street
    M = np.eye(4)
    M[:3, :3] = R.T
    M[:3, 3] = -R.T @ np.asarray(centre, np.float64)
    return M


def translate(offset):
    T = np.eye(4)
    T[:3, 3] = offset
    return T


class Trajectory:
    """Frames of one named camera path. `poses` are street poses (float64); `proj` = (fx, fy, cx, cy); `size` = (w, h)."""

    def __init__(self, name, poses, size, proj, offset, zmax=20.0, mu=0.3, table=(16384, 0x4000, 0x2000)):
        self.name, self.street_poses, self.size = name, poses, size
        self.proj = np.asarray(proj, np.float32)
        self.offset = np.asarray(offset, np.float64)
        self.zmax, self.mu = zmax, mu
        self.table = table            # (numBlocks, numBuckets, excessSize) of the GPU runs

    @property
    def w(self):
        return self.size[0]

    @property
    def h(self):
        return self.size[1]

    def world_pose(self, M_street):
        """the fusion path's world->camera matrix (float32) of a street pose"""
        return (np.asarray(M_street, np.float64) @ translate(self.offset)).astype(np.float32)

    def frames(self):
        """(depth, rgb, M_world, proj) of every frame"""
        scene = synth.StreetScene(seed=SCENE_SEED, length_m=SCENE_LENGTH)
        fx, fy, cx, cy = (float(v) for v in self.proj)
        out = []
        for Ms in self.street_poses:
            depth, rgb = scene.render(Ms, self.w, self.h, fx, fy, cx, cy, zmax=self.zmax)
            out.append((depth, rgb, self.world_pose(Ms), self.proj.copy()))
        return out

    def turned(self, degrees):
        """world pose of the last frame's camera turned by `degrees` about its own vertical axis"""
        R = np.eye(4)
        R[:3, :3] = synth._rot_y(np.deg2rad(degrees)).T
        return self.world_pose(R @ self.street_poses[-1])

    def cfg_kw(self):
        """parity.Cfg arguments that run this trajectory"""
        return dict(size=self.size, frames=len(self.street_poses), source=self.frames, zmax=self.zmax, mu=self.mu, voxelSize=VOXEL,
                    numBlocks=self.table[0], numBuckets=self.table[1], excessSize=self.table[2])


def _reverse():
    # driving backwards (towards -z), slight weave; world = street - offset puts x, y and z of every block below zero
    poses = [street_pose((0.12 * np.sin(f), 0.0, 45.0 - 0.8 * f), yaw=180.0 + 2.0 * np.sin(0.7 * f)) for f in range(6)]
    return Trajectory("reverse", poses, (301, 117), (252.0, 231.0, 170.3, 50.6), (10.3, 2.1, 66.7))


def _turn_in_place():
    # a full turn in 45 degree steps (the field of view is about 62 degrees, so consecutive frames overlap), camera next to the
    # world origin: rays march in every x / z sign combination and cross the zero planes
    poses = [street_pose((0.05 * f, 0.0, 20.0), yaw=45.0 * f) for f in range(8)]
    return Trajectory("turn_in_place", poses, (97, 61), (80.0, 95.0, 40.2, 35.7), (0.13, 0.4, 20.07))


def _pitch_roll():
    # four frames looking 45 degrees down with a 30 degree roll, then one rolled 90 degrees and one upside down
    poses = [street_pose((0.3 * f - 0.5, -0.4, 10.0 + 0.6 * f), yaw=12.0 * f, pitch=-45.0, roll=30.0) for f in range(4)]
    poses.append(street_pose((0.8, -0.3, 12.5), yaw=35.0, pitch=-15.0, roll=90.0))
    poses.append(street_pose((0.6, -0.2, 13.0), yaw=-10.0, pitch=-5.0, roll=180.0))
    return Trajectory("pitch_roll", poses, (301, 117), (262.0, 244.0, 121.7, 71.9), (-3.1, 1.2, 14.6))


def _ground_close():
    # 1 m above the ground looking 60 degrees down at the full KITTI size: blocks next to the camera cover hundreds of
    # 1/8-resolution cells. mu = 1 m widens the band to some 100 listed blocks, 64-87 of them with such boxes; the table is one
    # list-kernel tile (8192 entries), so the list kernel runs in one CTA and its AL_BIG overflow is reached
    poses = [street_pose((1.0 + 0.15 * f, 0.65, 15.0 + 0.25 * f), yaw=20.0 * f, pitch=-60.0, roll=4.0 * f) for f in range(4)]
    return Trajectory("ground_close", poses, (synth.KITTI_W, synth.KITTI_H), (707.0912, 690.5, 640.3, 170.2), (7.7, -0.35, 9.1),
                      zmax=8.0, mu=1.0, table=(8192, 0x1000, 0x1000))


def _far():
    # kilometres from the origin on every axis: block coordinates in the thousands (inside int16), of both signs. The principal
    # point lies outside the image (cx > w, cy < 0), so every pixel looks left of and below the optical axis.
    poses = [street_pose((0.2 * f, -0.3, 5.0 + 0.7 * f), yaw=30.0 + 3.0 * f, pitch=10.0) for f in range(5)]
    return Trajectory("far", poses, (97, 61), (70.0, 64.0, 104.5, -7.5), (2650.3, -1830.7, 3120.9))


TRAJECTORIES = {t.name: t for t in (_reverse(), _turn_in_place(), _pitch_roll(), _ground_close(), _far())}
NAMES = list(TRAJECTORIES)


def get(name):
    return TRAJECTORIES[name]


# ---- the analytic scene in float64 -------------------------------------------------------------------------------------
def _box_distance(p, b):
    """distance of points p (n, 3) to the surface of the solid box b = (x0, y0, z0, x1, y1, z1)"""
    lo, hi = b[:3], b[3:]
    outside = np.linalg.norm(np.maximum(np.maximum(lo - p, p - hi), 0.0), axis=1)
    inside = np.minimum(p - lo, hi - p).min(axis=1)
    return np.where(outside > 0.0, outside, np.maximum(inside, 0.0))


def surface_distance(p_street):
    """float64 distance of street points (n, 3) to the nearest surface of the scene the trajectories render"""
    scene = synth.StreetScene(seed=SCENE_SEED, length_m=SCENE_LENGTH)
    p = np.asarray(p_street, np.float64)
    d = np.abs(p[:, 1] - scene.ground_y)
    for sx in (-scene.facade_x, scene.facade_x):                 # facade rectangles, y in [-6, ground_y], unbounded in z
        dy = np.maximum(np.maximum(-6.0 - p[:, 1], p[:, 1] - scene.ground_y), 0.0)
        d = np.minimum(d, np.hypot(p[:, 0] - sx, dy))
    for b in scene.boxes:
        d = np.minimum(d, _box_distance(p, b))
    return d


def found_points_street(rays, voxelSize, offset):
    """street coordinates (float64) of the found raycast points (raycastResult: world voxel units, w > 0 where found) and the
    found fraction of the image"""
    r = np.asarray(rays, np.float32).reshape(-1, 4)
    hit = r[:, 3] > 0
    return r[hit, :3].astype(np.float64) * np.float64(np.float32(voxelSize)) + offset, float(hit.mean())


def distance_stats(rays, voxelSize, offset):
    """(median, p99, found fraction) of the found points' distances to the scene, in voxels"""
    p, frac = found_points_street(rays, voxelSize, offset)
    d = surface_distance(p) / voxelSize
    return float(np.median(d)), float(np.percentile(d, 99)), frac


# ---- which list items carry a box of more than 512 live cells (float32 ProjectSingleBlock) --------------------------------
SUB = 8


def block_boxes(pos, M, proj, w, h, voxelSize):
    """ProjectSingleBlock (DA/ITMVisualisationEngine.h:29-71) of the blocks at `pos`, restated in float32 in the reference's
    operation order, vectorised: (ulx, uly, lrx, lry, drawn) in 1/8-resolution cells, clamped to the full-resolution bounds"""
    f = np.float32
    M, proj, vs = np.asarray(M, f), np.asarray(proj, f), f(voxelSize)
    pos = np.asarray(pos, np.int64).reshape(-1, 3)
    n = len(pos)
    ulx, uly = np.full(n, w // SUB, np.int64), np.full(n, h // SUB, np.int64)
    lrx, lry = np.full(n, -1, np.int64), np.full(n, -1, np.int64)
    zmax = np.full(n, f(0.05), f)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        for corner in range(8):
            c = [((pos[:, k] + ((corner >> k) & 1)).astype(f) * f(8)).astype(f) * vs for k in range(3)]
            q = [((M[r, 0] * c[0] + M[r, 1] * c[1]).astype(f) + M[r, 2] * c[2]).astype(f) + M[r, 3] for r in range(3)]
            q = [x.astype(f) for x in q]
            ok = q[2] >= f(1e-6)
            px = (((proj[0] * q[0]).astype(f) / q[2]).astype(f) + proj[2]).astype(f) / f(SUB)
            py = (((proj[1] * q[1]).astype(f) / q[2]).astype(f) + proj[3]).astype(f) / f(SUB)
            fpx, cpx = np.floor(np.where(ok, px, 0)).astype(np.int64), np.ceil(np.where(ok, px, 0)).astype(np.int64)
            fpy, cpy = np.floor(np.where(ok, py, 0)).astype(np.int64), np.ceil(np.where(ok, py, 0)).astype(np.int64)
            ulx, lrx = np.where(ok, np.minimum(ulx, fpx), ulx), np.where(ok, np.maximum(lrx, cpx), lrx)
            uly, lry = np.where(ok, np.minimum(uly, fpy), uly), np.where(ok, np.maximum(lry, cpy), lry)
            zmax = np.where(ok, np.maximum(zmax, q[2]), zmax)
    ulx, uly, lrx, lry = np.maximum(ulx, 0), np.maximum(uly, 0), np.minimum(lrx, w - 1), np.minimum(lry, h - 1)
    drawn = (ulx <= lrx) & (uly <= lry) & (zmax >= f(0.05))
    return ulx, uly, lrx, lry, drawn


def big_live_boxes(pos, M, proj, w, h, voxelSize):
    """mask of the blocks whose box has more than 512 cells inside the live 1/8-resolution corner (the cells the fused frame's
    list kernel rasterises; alloc.cu hands such boxes to the whole CTA, at most AL_BIG = 64 of them per CTA)"""
    ulx, uly, lrx, lry, drawn = block_boxes(pos, M, proj, w, h, voxelSize)
    liveX, liveY = (w - 1) // SUB, (h - 1) // SUB
    live = drawn & (ulx <= liveX) & (uly <= liveY)
    cells = (np.minimum(lrx, liveX) - ulx + 1) * (np.minimum(lry, liveY) - uly + 1)
    return live & (cells > 512)


def list_kernel_shares(n_items, grid):
    """CTA of every list item in the list kernel's grid-stride loop over groups of 32 items"""
    return (np.arange(n_items) // 32) % grid
