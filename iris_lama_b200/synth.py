"""Seeded synthetic 2-D lidar worlds shared by the tests, the oracle harness and bench.py.

SURVEY.md section 8(d): axis-aligned wall segments, exact ray/segment intersection, range noise
N(0, 0.01 m) from PCG64(1234), odometry = truth composed with per-step noise N(0, 0.01 m),
N(0, 0.005 rad) from PCG64(4321) and accumulated (so it drifts).  Points are expressed in the
sensor frame as (r cos a, r sin a, 0); the sensor sits at the base origin with identity
orientation (the layout of lama::PointCloudXYZ, include/lama/types.h:111-120).
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np


def _rect(x0, y0, x1, y1):
    return [(x0, y0, x1, y0), (x1, y0, x1, y1), (x1, y1, x0, y1), (x0, y1, x0, y0)]


def make_room(size: float = 20.0, pillars: bool = True) -> np.ndarray:
    """Square room centred on the origin, optionally with four 2 m x 2 m pillars at (+-0.2 size, +-0.2 size)."""
    h = size / 2.0
    segs = _rect(-h, -h, h, h)
    if pillars:
        q = size * 0.2
        for cx in (-q, q):
            for cy in (-q, q):
                segs += _rect(cx - 1.0, cy - 1.0, cx + 1.0, cy + 1.0)
    return np.asarray(segs, dtype=np.float64)


def make_corridor(length: float = 60.0, width: float = 2.0, alcove_every: float = 5.0, alcove_depth: float = 0.5) -> np.ndarray:
    """Corridor along +x starting at x = -2 with alcoves on both sides so x is observable."""
    x0, x1 = -2.0, length - 2.0
    hw = width / 2.0
    segs = [(x0, -hw, x0, hw), (x1, -hw, x1, hw)]
    for side in (-1.0, 1.0):
        y = side * hw
        x = x0
        k = 0
        while x < x1 - 1e-9:
            xn = min(x + alcove_every, x1)
            # wall piece then a 1 m wide alcove
            xa = min(x + alcove_every - 1.0, x1)
            segs.append((x, y, xa, y))
            if xa < xn:
                yd = side * (hw + alcove_depth)
                segs += [(xa, y, xa, yd), (xa, yd, xn, yd), (xn, yd, xn, y)]
            x = xn
            k += 1
    return np.asarray(segs, dtype=np.float64)


def cast(segments: np.ndarray, pose, angles: np.ndarray, max_range: float = 30.0) -> np.ndarray:
    """Exact ranges of rays from pose=(x,y,theta) at sensor-frame `angles` against wall segments."""
    x, y, th = pose
    a = angles + th
    dx = np.cos(a)[:, None]
    dy = np.sin(a)[:, None]
    x1, y1, x2, y2 = (segments[:, i][None, :] for i in range(4))
    ex, ey = x2 - x1, y2 - y1
    den = dx * ey - dy * ex
    with np.errstate(divide="ignore", invalid="ignore"):
        t = ((x1 - x) * ey - (y1 - y) * ex) / den
        u = ((x1 - x) * dy - (y1 - y) * dx) / den
    ok = (np.abs(den) > 1e-12) & (t > 1e-9) & (u >= 0.0) & (u <= 1.0)
    t = np.where(ok, t, np.inf)
    r = t.min(axis=1)
    return np.minimum(r, max_range)


def scan_points(ranges: np.ndarray, angles: np.ndarray) -> np.ndarray:
    pts = np.zeros((ranges.shape[0], 3), dtype=np.float64)
    pts[:, 0] = ranges * np.cos(angles)
    pts[:, 1] = ranges * np.sin(angles)
    return pts


def beam_angles(n_beams: int, fov_deg: float) -> np.ndarray:
    fov = math.radians(fov_deg)
    if fov_deg >= 360.0:
        return -math.pi + np.arange(n_beams, dtype=np.float64) * (2 * math.pi / n_beams)
    return np.linspace(-fov / 2.0, fov / 2.0, n_beams, dtype=np.float64)


def loop_trajectory(n: int, radius: float = 6.0, step: float = 0.1, max_turn: float = 0.05) -> np.ndarray:
    """Rounded square of half side `radius` centred on the origin, driven counter-clockwise: starts at
    (radius, 0) heading +y, straight legs joined by quarter turns of at most max_turn rad per step (corner radius
    step / max_turn).  Returns n poses (x, y, theta); laps repeat for as long as n asks."""
    rt = step / max_turn
    quarter = int(round((math.pi / 2.0) / max_turn))
    poses = np.zeros((n, 3), dtype=np.float64)
    x, y, th = radius, 0.0, math.pi / 2.0
    leg_steps = int(round((radius - rt) / step))        # first leg: from the middle of the right side
    full_leg = int(round(2.0 * (radius - rt) / step))
    left, turning = leg_steps, 0
    for i in range(n):
        poses[i] = (x, y, th)
        if turning > 0:
            th += (math.pi / 2.0) / quarter
            turning -= 1
            if turning == 0:
                left = full_leg
        else:
            left -= 1
            if left == 0:
                turning = quarter
        x += step * math.cos(th)
        y += step * math.sin(th)
    poses[:, 2] = (poses[:, 2] + math.pi) % (2 * math.pi) - math.pi
    return poses


def line_trajectory(n: int, step: float = 0.1, x0: float = 0.0, wobble: float = 0.0) -> np.ndarray:
    poses = np.zeros((n, 3), dtype=np.float64)
    poses[:, 0] = x0 + step * np.arange(n)
    if wobble:
        poses[:, 2] = wobble * np.sin(np.arange(n) * 0.05)
    return poses


def _compose(a, b):
    ca, sa = math.cos(a[2]), math.sin(a[2])
    return (a[0] + ca * b[0] - sa * b[1], a[1] + sa * b[0] + ca * b[1], a[2] + b[2])


def _between(a, b):
    ca, sa = math.cos(a[2]), math.sin(a[2])
    dx, dy = b[0] - a[0], b[1] - a[1]
    return (ca * dx + sa * dy, -sa * dx + ca * dy, b[2] - a[2])


@dataclass
class Dataset:
    name: str
    segments: np.ndarray
    truth: np.ndarray      # (T,3)
    odom: np.ndarray       # (T,3) drifting odometry
    scans: np.ndarray      # (T,N,3) float64 points in the sensor frame
    angles: np.ndarray
    max_range: float

    @property
    def n_scans(self):
        return self.scans.shape[0]

    @property
    def n_beams(self):
        return self.scans.shape[1]


def make_dataset(name: str, n_scans: int, n_beams: int | None = None, range_seed: int = 1234, odom_seed: int = 4321,
                 range_sigma: float = 0.01, odom_sigma_xy: float = 0.01, odom_sigma_th: float = 0.005) -> Dataset:
    """name in {"loc_room", "corridor", "room", "loop"} -- configs 1-4 of BASELINE.json."""
    max_range = 30.0
    if name == "loc_room":
        segs = make_room(20.0, pillars=False)
        nb, fov = n_beams or 360, 360.0
        truth = np.zeros((n_scans, 3))
        truth[:, 0] = 1.5 + 0.1 * np.arange(n_scans)
        truth[:, 1] = -2.0
        truth[:, 2] = 0.3
    elif name == "corridor":
        segs = make_corridor()
        nb, fov = n_beams or 720, 360.0
        truth = line_trajectory(n_scans, 0.05 if n_scans > 1000 else 0.1, 0.0, wobble=0.05)
        truth[:, 0] = np.minimum(truth[:, 0], 55.0)
    elif name == "room":
        segs = make_room(20.0, pillars=True)
        nb, fov = n_beams or 1080, 270.0
        truth = loop_trajectory(n_scans, radius=7.0, step=0.1)
    elif name == "loop":
        segs = make_room(30.0, pillars=True)
        nb, fov = n_beams or 1080, 270.0
        truth = loop_trajectory(n_scans, radius=10.0, step=0.1)
    else:
        raise ValueError(name)
    angles = beam_angles(nb, fov)
    rng_r = np.random.Generator(np.random.PCG64(range_seed))
    rng_o = np.random.Generator(np.random.PCG64(odom_seed))
    scans = np.zeros((n_scans, nb, 3), dtype=np.float64)
    odom = np.zeros((n_scans, 3), dtype=np.float64)
    cur = tuple(truth[0])
    for t in range(n_scans):
        r = cast(segs, truth[t], angles, max_range)
        r = r + rng_r.normal(0.0, range_sigma, size=nb)
        scans[t] = scan_points(r, angles)
        if t == 0:
            odom[0] = truth[0]
        else:
            d = _between(tuple(truth[t - 1]), tuple(truth[t]))
            d = (d[0] + rng_o.normal(0.0, odom_sigma_xy), d[1] + rng_o.normal(0.0, odom_sigma_xy), d[2] + rng_o.normal(0.0, odom_sigma_th))
            cur = _compose(cur, d)
            odom[t] = cur
    return Dataset(name, segs, truth, odom, scans, angles, max_range)


def make_pose_graph(n_nodes, n_loops, seed=7, step=0.1, odom_sigma=(0.02, 0.02, 0.004), loop_sigma=(0.01, 0.01, 0.002), radius=2.0):
    """Synthetic input of SimplePGO (BASELINE.json configs[4]): a robot driving laps of a rounded figure whose size drifts slowly, so that it
    keeps revisiting places.  Returns (truth n x 3, node_list n x 3 = odometry-integrated poses with drift, edge_list [(from, to, xyr)]):
    the loop edges connect poses that are close in space (< radius) but far apart in time, measured with a little noise."""
    rng = np.random.default_rng(seed)
    t = np.arange(n_nodes) * step
    lap = 40.0                                     # metres per lap
    ang = 2 * np.pi * t / lap
    r = 5.0 + 1.5 * np.sin(0.37 * ang)             # the laps do not coincide exactly
    x, y = r * np.cos(ang), r * np.sin(ang) * 0.8
    th = np.arctan2(np.gradient(y), np.gradient(x))
    truth = np.stack([x, y, th], 1)

    def se2(p):
        c, s = np.cos(p[2]), np.sin(p[2])
        return np.array([[c, -s, p[0]], [s, c, p[1]], [0, 0, 1.0]])

    def xyr(m):
        return np.array([m[0, 2], m[1, 2], np.arctan2(m[1, 0], m[0, 0])])

    T = [se2(p) for p in truth]
    nodes = [truth[0].copy()]
    cur = T[0]
    for i in range(n_nodes - 1):
        d = xyr(np.linalg.inv(T[i]) @ T[i + 1]) + rng.normal(0, odom_sigma)
        cur = cur @ se2(d)
        nodes.append(xyr(cur))
    # loop closures: spatial neighbours that are not temporal neighbours
    from scipy.spatial import cKDTree
    tree = cKDTree(truth[:, :2])
    pairs = [(a, b) for a, b in tree.query_pairs(radius) if abs(a - b) > 50]
    rng.shuffle(pairs)
    edges = []
    for a, b in pairs[:n_loops]:
        a, b = (a, b) if a < b else (b, a)
        edges.append((int(a), int(b), xyr(np.linalg.inv(T[a]) @ T[b]) + rng.normal(0, loop_sigma)))
    return truth, np.array(nodes), edges


# ---- 3-D scenes for the truncated signed distance map ----------------------------------------------------------------------------
def make_scene_3d():
    """A 10 x 10 x 3 m room (the inside of an axis-aligned box) with a box standing on the floor and a sphere in the air."""
    return dict(room=(np.array([-5.0, -5.0, 0.0]), np.array([5.0, 5.0, 3.0])),
                boxes=[(np.array([1.0, -2.0, 0.0]), np.array([2.0, -1.0, 1.2]))],
                spheres=[(np.array([-1.5, 1.5, 1.0]), 0.6)])


def cast_3d(scene, origin, dirs, max_range=30.0):
    """Ranges along unit world directions (n, 3) from `origin`: the nearest of the room's walls (exit of its box), the obstacle boxes
    (slab entry) and the spheres."""
    o = np.asarray(origin, np.float64)
    d = np.asarray(dirs, np.float64)
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / d
        lo, hi = scene["room"]
        t_exit = np.maximum((lo - o) * inv, (hi - o) * inv)
        t = np.minimum(np.nanmin(np.where(np.isfinite(t_exit), t_exit, np.inf), axis=1), max_range)
        for blo, bhi in scene["boxes"]:
            t1, t2 = (blo - o) * inv, (bhi - o) * inv
            tmin = np.nanmax(np.minimum(t1, t2), axis=1)
            tmax = np.nanmin(np.maximum(t1, t2), axis=1)
            hit = (tmax >= tmin) & (tmin > 0)
            t = np.where(hit, np.minimum(t, tmin), t)
    for c, r in scene["spheres"]:
        oc = o - c
        b = d @ oc
        disc = b * b - (oc @ oc - r * r)
        ts = -b - np.sqrt(np.maximum(disc, 0.0))
        t = np.where((disc >= 0) & (ts > 0), np.minimum(t, ts), t)
    return t


def ring_lidar_dirs(n_rings=32, n_az=900, fov_down_deg=-15.0, fov_up_deg=15.0):
    """Unit beam directions (n_rings * n_az, 3) of a spinning ring lidar in its own frame, ring-major."""
    el = np.deg2rad(np.linspace(fov_down_deg, fov_up_deg, n_rings))
    az = np.arange(n_az) * (2 * np.pi / n_az)
    e, a = np.meshgrid(el, az, indexing="ij")
    return np.stack([np.cos(e) * np.cos(a), np.cos(e) * np.sin(a), np.sin(e)], axis=-1).reshape(-1, 3)


def quat_xyzw(yaw, pitch=0.0, roll=0.0):
    """Quaternion (x, y, z, w) of Rz(yaw) Ry(pitch) Rx(roll)."""
    cy, sy, cp, sp, cr, sr = np.cos(yaw / 2), np.sin(yaw / 2), np.cos(pitch / 2), np.sin(pitch / 2), np.cos(roll / 2), np.sin(roll / 2)
    return np.array([sr * cp * cy - cr * sp * sy, cr * sp * cy + sr * cp * sy, cr * cp * sy - sr * sp * cy, cr * cp * cy + sr * sp * sy])


def quat_matrix(q):
    x, y, z, w = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)],
                     [2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)],
                     [2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)]])


def make_clouds_3d(n_clouds, n_rings=32, n_az=900, seed=5, range_sigma=0.005, max_range=30.0):
    """Seeded 3-D lidar sequence in make_scene_3d(): a sensor 1 m above the floor on a 2.5 m circle, slightly pitched.
    Returns (clouds: list of (n, 3) points in the sensor frame, origins (S, 3), quats (S, 4) xyzw) -- world sensor poses."""
    scene = make_scene_3d()
    dirs = ring_lidar_dirs(n_rings, n_az)
    rng = np.random.Generator(np.random.PCG64(seed))
    clouds, origins, quats = [], np.zeros((n_clouds, 3)), np.zeros((n_clouds, 4))
    for k in range(n_clouds):
        a = 2 * np.pi * k / max(1, n_clouds)
        origins[k] = (2.5 * np.cos(a), 2.5 * np.sin(a), 1.0)
        quats[k] = quat_xyzw(a + np.pi / 2, 0.05 * np.sin(3 * a))
        r = cast_3d(scene, origins[k], dirs @ quat_matrix(quats[k]).T, max_range)
        r = r + rng.normal(0.0, range_sigma, size=r.shape)
        clouds.append(dirs * r[:, None])
    return clouds, origins, quats
