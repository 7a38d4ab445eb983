"""Template poses of the reference's test configuration, generated in fp64 rather than read from its predefined .npy
files (src/lib3d/create_template_poses.py, template_transform.py:39-70, render_bop_templates.py:69-70).

The views are the vertices of Blender's icosphere.  Level 0 is the 42-vertex sphere Blender adds by default: its
icosahedron with every edge split once and the new vertices pushed onto the unit sphere, then every vertex on the unit
sphere.  Each further level splits every edge at its midpoint and re-projects the new vertices onto the sphere (42, 162
and 642 views).  A camera sits at 1000 mm x the vertex looking at the origin (`look_at`), the views are ordered by
(elevation, azimuth), and the object pose is the inverse of the camera pose.  Blender computed in fp32, so the
reference's poses differ from these in the last fp32 bits (DESIGN.md, row f15).

    template_poses(level=1, distribution="all", zoom=0.4) -> float64 [T,4,4]
"""
from __future__ import annotations

import numpy as np

LEVELS = (0, 1, 2)
DISTRIBUTIONS = ("all", "upper")


# Blender's icosahedron (bmo_primitive's icovert table, radius 200): its coordinates have five significant digits, so
# the vertices lie up to 1e-5 off the sphere and the views are not exactly symmetric; the reference's poses keep that
ICOSAHEDRON = np.array([
    [0.0, 0.0, -200.0], [144.72, -105.144, -89.443], [-55.277, -170.128, -89.443], [-178.885, 0.0, -89.443],
    [-55.277, 170.128, -89.443], [144.72, 105.144, -89.443], [55.277, -170.128, 89.443], [-144.72, -105.144, 89.443],
    [-144.72, 105.144, 89.443], [55.277, 170.128, 89.443], [178.885, 0.0, 89.443], [0.0, 0.0, 200.0]]) / 200.0


def icosahedron():
    """-> (V f64 [12,3], F i64 [20,3]): Blender's icosahedron at radius 1 (not normalised) and its faces."""
    F = []
    for k in range(5):              # lower ring 1..5, upper ring 6..10, each ring's neighbours adjacent
        l0, l1, u0, u1 = 1 + k, 1 + (k + 1) % 5, 6 + k, 6 + (k + 1) % 5
        F += [[0, l1, l0], [l0, l1, u0], [u0, l1, u1], [u0, u1, 11]]
    return ICOSAHEDRON.copy(), np.array(F, np.int64)


def subdivide(V, F):
    """Splits every edge at its midpoint, re-projected onto the unit sphere; each triangle becomes four."""
    V, mid, out = list(V), {}, []

    def m(a, b):
        key = (min(a, b), max(a, b))
        if key not in mid:
            p = (V[a] + V[b]) / 2
            mid[key] = len(V)
            V.append(p / np.linalg.norm(p))
        return mid[key]

    for a, b, c in F:
        ab, bc, ca = m(a, b), m(b, c), m(c, a)
        out += [[a, ab, ca], [ab, b, bc], [ca, bc, c], [ab, bc, ca]]
    return np.array(V), np.array(out, np.int64)


def icosphere(level):
    """-> f64 [T,3] unit vertices of the level's icosphere, ordered by (elevation, azimuth) as the reference sorts them;
    azimuth is atan2(x, y).  The sort is in fp64: where the reference's fp32 elevations differ by noise alone (below
    1e-7 rad), its order within the ring follows that noise, and this one the fp64 elevation, then the azimuth."""
    if level not in LEVELS:
        raise ValueError(f"template level {level!r} is not one of {LEVELS}")
    V, F = subdivide(*icosahedron())
    V /= np.linalg.norm(V, axis=1, keepdims=True)
    for _ in range(level):
        V, F = subdivide(V, F)
    el = np.arctan2(V[:, 2], np.hypot(V[:, 0], V[:, 1]))
    az = np.arctan2(V[:, 0], V[:, 1])
    return V[np.lexsort((az, el))]


def look_at(cam):
    """Camera -> world pose of a camera at `cam` [3] looking at the origin (+z forward), with the reference's up
    hint: -z, or -y when the camera lies on the z axis."""
    fwd = -cam / np.linalg.norm(cam)
    tmp = np.array([0.0, 0.0, -1.0])
    if min(np.linalg.norm(cam - tmp), np.linalg.norm(cam + tmp)) < 1e-3:
        tmp = np.array([0.0, -1.0, 0.0])
    right = np.cross(tmp, fwd)
    right /= np.linalg.norm(right)
    up = np.cross(fwd, right)
    up /= np.linalg.norm(up)
    M = np.eye(4)
    M[:3, :3] = np.stack([right, up, fwd], 1)
    M[:3, 3] = cam
    return M


def camera_poses(level):
    """f64 [T,4,4] camera -> object poses in mm (the reference's cam_poses_level{level}.npy)."""
    out = np.stack([look_at(v) for v in icosphere(level)])
    out[:, :3, 3] *= 1000.0
    return out


def template_poses(level=1, distribution="all", zoom=0.4):
    """f64 [T,4,4] object -> camera poses in mm of the level's icosphere views: the inverse of `camera_poses`
    (obj_poses_level{level}.npy), only the views whose camera has z >= 0 for distribution "upper", the translation
    scaled by `zoom`.  Level 1, "all" and zoom 0.4 are the reference's test templates (162 views)."""
    if distribution not in DISTRIBUTIONS:
        raise ValueError(f"pose distribution {distribution!r} is not one of {DISTRIBUTIONS}")
    cam = camera_poses(level)
    R = cam[:, :3, :3].transpose(0, 2, 1)
    obj = np.zeros_like(cam)
    obj[:, :3, :3] = R
    obj[:, :3, 3] = -np.einsum("nij,nj->ni", R, cam[:, :3, 3]) * zoom
    obj[:, 3, 3] = 1.0
    return obj[cam[:, 2, 3] >= 0] if distribution == "upper" else obj
