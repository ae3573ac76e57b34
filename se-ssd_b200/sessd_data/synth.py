"""Seeded synthetic inputs of KITTI shape (SURVEY.md §8d).  No dataset is available offline.

* ``uniform_cloud``  -- "uniform-20k": x~U(0,70.4), y~U(-40,40), z~U(-3,1), r~U(0,1), float32, NOT shuffled
  (point order is part of the voxeliser's semantics).
* ``ring_cloud``     -- "ring-20k": a 64-beam spinning-LiDAR-like scan of a ground plane plus random car-sized
  cuboids; gives KITTI-like surface clustering (active sites grow far less through strided convs).
* ``random_boxes``   -- car-sized rotated boxes + scores for the IoU / NMS stage.
"""
import numpy as np

PC_RANGE = (0.0, -40.0, -3.0, 70.4, 40.0, 1.0)
VOXEL_SIZE = (0.05, 0.05, 0.1)


def uniform_cloud(seed, n=20000):
    rng = np.random.default_rng(seed)
    x = rng.uniform(0.0, 70.4, n)
    y = rng.uniform(-40.0, 40.0, n)
    z = rng.uniform(-3.0, 1.0, n)
    r = rng.uniform(0.0, 1.0, n)
    return np.stack([x, y, z, r], 1).astype(np.float32)


def ring_cloud(seed, n=20000, n_cars=30):
    rng = np.random.default_rng(seed)
    elev = np.deg2rad(np.linspace(-24.8, 2.0, 64))
    azim = np.deg2rad(np.arange(-45.0, 45.0, 0.18))
    el, az = np.meshgrid(elev, azim, indexing="ij")
    el, az = el.ravel(), az.ravel()
    dx, dy, dz = np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)
    ground_z = -1.73
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.where(dz < -1e-6, ground_z / dz, np.inf)
    t = np.minimum(t, 70.0)
    # cars: axis-aligned-in-own-frame slabs test, ray from origin
    cx = rng.uniform(5.0, 65.0, n_cars)
    cy = rng.uniform(-35.0, 35.0, n_cars)
    yaw = rng.uniform(-np.pi, np.pi, n_cars)
    half = np.array([3.9 / 2, 1.6 / 2, 1.56 / 2])
    cz = ground_z + half[2]
    for k in range(n_cars):
        c, s = np.cos(yaw[k]), np.sin(yaw[k])
        ox, oy, oz = -cx[k], -cy[k], -cz
        # rotate ray into the box frame
        rdx, rdy = dx * c + dy * s, -dx * s + dy * c
        rox, roy = ox * c + oy * s, -ox * s + oy * c
        tmin = np.full_like(t, -np.inf)
        tmax = np.full_like(t, np.inf)
        for o, d, h in ((rox, rdx, half[0]), (roy, rdy, half[1]), (oz, dz, half[2])):
            with np.errstate(divide="ignore", invalid="ignore"):
                t1 = (-h - o) / d
                t2 = (h - o) / d
            lo, hi = np.minimum(t1, t2), np.maximum(t1, t2)
            tmin = np.maximum(tmin, lo)
            tmax = np.minimum(tmax, hi)
        hit = (tmax >= tmin) & (tmin > 0)
        t = np.where(hit & (tmin < t), tmin, t)
    t = t + rng.normal(0.0, 0.02, t.shape)
    pts = np.stack([dx * t, dy * t, dz * t, rng.uniform(0, 1, t.shape)], 1)
    lo = np.array(PC_RANGE[:3])
    hi = np.array(PC_RANGE[3:])
    ok = np.all((pts[:, :3] >= lo) & (pts[:, :3] < hi), 1) & np.isfinite(t)
    pts = pts[ok]
    if len(pts) >= n:
        sel = np.sort(rng.choice(len(pts), n, replace=False))
        pts = pts[sel]
    else:
        pad = pts[rng.integers(0, len(pts), n - len(pts))] + rng.normal(0, 0.01, (n - len(pts), 4))
        pts = np.concatenate([pts, pad], 0)
    return pts.astype(np.float32)


def random_boxes(seed, n=1000, spread=1.0):
    """[n,7] = x,y,z,w,l,h,r car-sized boxes and [n] scores in (0.3,1)."""
    rng = np.random.default_rng(seed)
    x = rng.uniform(0.0, 70.4 * spread, n)
    y = rng.uniform(-40.0 * spread, 40.0 * spread, n)
    z = rng.uniform(-2.0, 0.0, n)
    w = rng.normal(1.6, 0.1, n)
    l = rng.normal(3.9, 0.3, n)
    h = rng.normal(1.56, 0.1, n)
    r = rng.uniform(-np.pi, np.pi, n)
    boxes = np.stack([x, y, z, w, l, h, r], 1).astype(np.float32)
    scores = rng.uniform(0.3, 1.0, n).astype(np.float32)
    return boxes, scores


def ring_boxes(seed, n_cars=30):
    """the [n_cars, 7] lidar boxes (x y z w l h r) of the cars ring_cloud(seed, n, n_cars) places: the first draws of its generator
    (centres, yaw); the car's 3.9 m side lies along its own x axis, which is the box's l (along its y) turned by pi / 2"""
    rng = np.random.default_rng(seed)
    cx = rng.uniform(5.0, 65.0, n_cars)
    cy = rng.uniform(-35.0, 35.0, n_cars)
    yaw = rng.uniform(-np.pi, np.pi, n_cars)
    z = np.full(n_cars, -1.73 + 1.56 / 2)
    return np.stack([cx, cy, z, np.full(n_cars, 1.6), np.full(n_cars, 3.9), np.full(n_cars, 1.56), yaw - np.pi / 2], 1).astype(np.float32)
