"""Planted inputs of the TEASER++ refiner tests: a rendered depth patch (a tilted, bumped surface inside a box) and a
measured depth that is the same patch moved by a small rigid motion, with outliers and holes; every frame has its own K."""
import numpy as np


def intrinsics(H, W, f=None, seed=0):
    rng = np.random.default_rng(seed)
    f = f or 1.2 * max(H, W)
    return np.array([[f * (1 + 0.02 * rng.standard_normal()), 0, W / 2 + rng.uniform(-2, 2)],
                     [0, f * (1 + 0.02 * rng.standard_normal()), H / 2 + rng.uniform(-2, 2)], [0, 0, 1]], np.float32)


def patch(H, W, box, z0=700.0, seed=0):
    """Rendered depth f32 [H,W]: positive inside box (x0, y0, x1, y1), with a few background holes."""
    rng = np.random.default_rng(seed)
    x0, y0, x1, y1 = box
    v, u = np.mgrid[0:H, 0:W].astype(np.float64)
    z = z0 + 0.08 * (u - W / 2) - 0.05 * (v - H / 2) + 12 * np.sin(u / max(W, 1) * 9) * np.cos(v / max(H, 1) * 7)
    d = np.zeros((H, W), np.float32)
    d[y0:y1, x0:x1] = z[y0:y1, x0:x1]
    d[(rng.random((H, W)) < 0.03)] = 0
    return d


def measured(rendered, K, dR_deg=1.5, dt=(3.0, -2.0, 4.0), outliers=0.1, holes=0.05, noise=0.5, seed=1):
    """The rendered patch moved by a rigid motion (re-projected per pixel along the viewing ray so that pixel-aligned
    correspondences are offset, as a pose error gives), plus outlier depths and missing pixels."""
    rng = np.random.default_rng(seed)
    H, W = rendered.shape
    a = np.deg2rad(dR_deg)
    R = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
    v, u = np.mgrid[0:H, 0:W].astype(np.float64)
    z = rendered.astype(np.float64)
    x = (u - K[0, 2]) * z / K[0, 0]
    y = (v - K[1, 2]) * z / K[1, 1]
    P = np.stack([x, y, z], -1) @ R.T + np.asarray(dt)
    m = P[..., 2] + noise * rng.standard_normal((H, W))
    m = np.where(rendered > 0, m, 0.0)
    out = rng.random((H, W)) < outliers
    m = np.where(out & (rendered > 0), m + rng.uniform(60, 300, (H, W)), m)
    m[rng.random((H, W)) < holes] = 0
    background = rng.random((H, W)) < 0.5
    m = np.where((rendered <= 0) & background, z.max() + 150.0, m)
    return m.astype(np.float32)


def pose(seed=0):
    rng = np.random.default_rng(seed)
    q = rng.standard_normal(4)
    q /= np.linalg.norm(q)
    w, x, y, z = q
    T = np.eye(4, dtype=np.float32)
    T[:3, :3] = [[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                 [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                 [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]]
    T[:3, 3] = rng.uniform(-50, 50, 3) + [0, 0, 700]
    return T
