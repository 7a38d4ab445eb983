"""Scenes of the depth-refiner tests (tests/test_gpu_icp.py, tests/test_gpu_icp_solver.py): meshes in mm, poses, and
measured depth rendered with the project's own rasteriser at 640 x 480."""
import numpy as np
import torch

from gigapose_b200 import render
from oracle import icp_port

DEV = "cuda:0"
H, W = 480, 640
K = np.array([[572.4114, 0.0, 325.2611], [0.0, 573.57043, 242.04899], [0.0, 0.0, 1.0]], np.float32)


def ellipsoid(radii=(80.0, 50.0, 30.0), n_lat=48, n_lon=96):
    """A bumpy, asymmetric ellipsoid (mm)."""
    th = np.linspace(0, np.pi, n_lat)[:, None]
    ph = np.linspace(0, 2 * np.pi, n_lon, endpoint=False)[None]
    bump = 1 + 0.08 * np.sin(3 * th) * np.cos(2 * ph) + 0.05 * np.cos(5 * ph + 1.0) * np.sin(th) ** 2
    x = radii[0] * np.sin(th) * np.cos(ph) * bump
    y = radii[1] * np.sin(th) * np.sin(ph) * bump
    z = radii[2] * np.cos(th) * bump + 0 * ph + 8.0 * (np.sin(th) * np.cos(ph)) ** 2
    V = np.stack([x, y, z], -1).reshape(-1, 3).astype(np.float32)
    F = []
    for i in range(n_lat - 1):
        for j in range(n_lon):
            a, b = i * n_lon + j, i * n_lon + (j + 1) % n_lon
            F += [[a, a + n_lon, b], [b, a + n_lon, b + n_lon]]
    return dict(vertices=V, faces=np.array(F, np.int32))


def box(c, s):
    v = np.array([[x, y, z] for x in (-1, 1) for y in (-1, 1) for z in (-1, 1)], np.float32) * np.float32(s) / 2 + c
    f = [[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1], [2, 3, 7], [2, 7, 6], [0, 2, 6], [0, 6, 4],
         [1, 5, 7], [1, 7, 3]]
    return v, np.array(f, np.int32)


def assembly():
    """A box with a cylinder standing off one corner (mm)."""
    bv, bf = box(np.zeros(3, np.float32), (70, 45, 30))
    n = 48
    a = np.linspace(0, 2 * np.pi, n, endpoint=False)
    ring = np.stack([18 + 14 * np.cos(a), 10 + 14 * np.sin(a)], -1)
    cv = np.concatenate([np.c_[ring, np.full(n, 15.0)], np.c_[ring, np.full(n, 60.0)], [[18, 10, 15], [18, 10, 60]]])
    cf = []
    for j in range(n):
        k = (j + 1) % n
        cf += [[j, k, n + k], [j, n + k, n + j], [2 * n, k, j], [2 * n + 1, n + j, n + k]]
    V = np.concatenate([bv, cv.astype(np.float32)])
    F = np.concatenate([bf, np.array(cf, np.int32) + len(bv)])
    return dict(vertices=V.astype(np.float32), faces=F)


def plate():
    """A flat 120 x 90 mm square: a degenerate object for point-to-plane ICP."""
    v = np.array([[-60, -45, 0], [60, -45, 0], [60, 45, 0], [-60, 45, 0]], np.float32)
    return dict(vertices=v, faces=np.array([[0, 1, 2], [0, 2, 3]], np.int32))


def rot(axis, deg):
    axis = np.asarray(axis, np.float64) / np.linalg.norm(axis)
    return icp_port.rodrigues(axis * np.deg2rad(deg))


def pose(R, t):
    T = np.eye(4)
    T[:3, :3], T[:3, 3] = R, t
    return T.astype(np.float32)


def perturb(T, axis, deg, dt):
    return pose(rot(axis, deg) @ T[:3, :3].astype(np.float64), T[:3, 3] + np.asarray(dt))


def render_depth(mesh, T, Km=K):
    r = render.render_templates(mesh, torch.as_tensor(T)[None], Km, size=(H, W), device=DEV)
    return r["depth"][0]


def scene(mesh, T_true, background=150.0, Km=K):
    """Measured depth: the object at T_true in front of a plane `background` mm behind it; mask = the object's pixels."""
    d = render_depth(mesh, T_true, Km)
    mask = d > 0
    if background is not None:
        z = float(T_true[2, 3]) + background
        bg = dict(vertices=np.array([[-2e3, -2e3, z], [2e3, -2e3, z], [2e3, 2e3, z], [-2e3, 2e3, z]], np.float32),
                  faces=np.array([[0, 1, 2], [0, 2, 3]], np.int32))
        d = torch.where(mask, d, render_depth(bg, np.eye(4, dtype=np.float32), Km))
    return d, mask


def noisy_occluded_scene(mesh, T_true):
    """scene() with sigma = 1 mm noise, 10 % missing pixels and a box occluder 120 mm in front over 30 % of the mask;
    the mask leaves the occluded pixels out."""
    d, mask = scene(mesh, T_true)
    g = torch.Generator(device=DEV).manual_seed(3)
    d = d + torch.randn(d.shape, generator=g, device=DEV)
    d = torch.where(torch.rand(d.shape, generator=g, device=DEV) < 0.1, torch.zeros_like(d), d)
    ys, xs = torch.nonzero(mask, as_tuple=True)
    y0, y1, x0 = int(ys.min()), int(ys.max()), int(xs.min())
    cols = torch.sort(xs).values
    x_cut = int(cols[int(0.3 * len(cols))])
    d[y0:y1 + 1, x0:x_cut] = float(T_true[2, 3]) - 120.0
    m = mask.clone()
    m[y0:y1 + 1, x0:x_cut] = False
    return d, m


T_ELL = pose(rot([0.3, 1.0, 0.2], 35), [30.0, -20.0, 700.0])
T_ASM = pose(rot([1.0, -0.4, 0.5], 50), [-40.0, 25.0, 800.0])
