"""An independent fp64 restatement of row f17's contract (the header comment of gigapose_b200/csrc/reconstruct.cu), for
tests/test_gpu_reconstruct.py and tests/test_reconstruct_cpu.py.  It imports nothing of gigapose_b200.reconstruct.

`fuse` applies the frames to a grid in fp64 and flags every voxel whose update sequence an fp32 rounding could change:
a projection within `eps_px` of a half pixel, or a comparison (z <= 0, sdf >= -mu, z < D - mu) within `eps_len` of its
threshold.  `extract` runs marching tetrahedra on a given grid: the sign and weight decisions read the grid's own f32
values, so they are exact, and the vertex positions are computed in fp64."""
import itertools

import numpy as np

PERMS = [(0, 1, 2), (0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)]


def centres(dims, origin, voxel):
    """Voxel centres f64 [nz,ny,nx,3] (x, y, z) of a grid of `dims` (nx, ny, nz)."""
    nx, ny, nz = dims
    o = np.asarray(origin, np.float32).astype(np.float64)
    s = float(np.float32(voxel))
    z, y, x = np.meshgrid(np.arange(nz), np.arange(ny), np.arange(nx), indexing="ij")
    return np.stack([o[0] + (x + 0.5) * s, o[1] + (y + 0.5) * s, o[2] + (z + 0.5) * s], -1)


def fuse(dims, origin, voxel, trunc, frames, eps_px=2e-4, eps_len=None):
    """frames: [(depth f32 [H,W], mask [H,W], K [3,3], pose [4,4])], K and pose taken as f32 values.  -> (tsdf f64,
    weight f64, near_tie bool), each [nz,ny,nx].  The default margins hold the fp32 error about ten times over for
    poses a few hundred mm away and images up to a few thousand px: u carries a few ulp of K02 z / z (~1e-5 px), the
    lengths a few ulp of |x_c| (eps_len = 1e-5 |x_c|max)."""
    c = centres(dims, origin, voxel).reshape(-1, 3)
    mu = float(np.float32(trunc))
    tsdf, w = np.zeros(len(c)), np.zeros(len(c))
    near = np.zeros(len(c), bool)
    for depth, mask, K, pose in frames:
        K = np.asarray(K, np.float32).astype(np.float64)
        P = np.asarray(pose, np.float32).astype(np.float64)
        H, W = depth.shape
        xc = c @ P[:3, :3].T + P[:3, 3]
        z = xc[:, 2]
        eps = eps_len if eps_len is not None else 1e-5 * max(1.0, float(np.abs(xc).max()))
        near |= np.abs(z) < eps
        front = z > 0
        zs = np.where(front, z, 1.0)
        u = (K[0, 0] * xc[:, 0] + K[0, 1] * xc[:, 1] + K[0, 2] * z) / zs
        v = (K[1, 1] * xc[:, 1] + K[1, 2] * z) / zs
        for a in (u, v):
            near |= front & (np.abs(a - np.floor(a) - 0.5) < eps_px)
        ru, rv = np.rint(u), np.rint(v)
        inside = front & (ru >= 0) & (ru < W) & (rv >= 0) & (rv < H)
        iu, iv = np.where(inside, ru, 0).astype(np.int64), np.where(inside, rv, 0).astype(np.int64)
        D = np.asarray(depth, np.float32)[iv, iu].astype(np.float64)
        m = np.asarray(mask)[iv, iu] != 0
        has = inside & (D > 0)
        sdf = D - z
        upd_in = has & m & (sdf >= -mu)
        upd_out = has & ~m & (z < D - mu)
        near |= has & m & (np.abs(sdf + mu) < eps)
        near |= has & ~m & (np.abs(z - (D - mu)) < eps)
        value = np.where(upd_in, np.minimum(1.0, sdf / mu), 1.0)
        upd = upd_in | upd_out
        tsdf = np.where(upd, (tsdf * w + value) / (w + 1.0), tsdf)
        w = w + upd
    shape = (dims[2], dims[1], dims[0])
    return tsdf.reshape(shape), w.reshape(shape), near.reshape(shape)


def _corner(code):
    return np.array([code & 1, code >> 1 & 1, code >> 2 & 1], np.float64)


def _tet_codes(k):
    a, b, _ = PERMS[k]
    return [0, 1 << a, (1 << a) | (1 << b), 7]


def _case_triangles(k, inside):
    """Triangles of tetrahedron k for the inside bits (tuple of 4 bools), as lists of 3 (corner i, corner j) edges,
    wound outward: orientation decided geometrically from the edge midpoints."""
    n_in = sum(inside)
    if n_in in (0, 4):
        return []
    codes = _tet_codes(k)
    pos = [_corner(c) for c in codes]
    out_dir = (np.mean([pos[i] for i in range(4) if not inside[i]], 0) - np.mean([pos[i] for i in range(4) if inside[i]], 0))

    def wind(tri):
        p = [(pos[i] + pos[j]) / 2 for i, j in tri]
        if np.dot(np.cross(p[1] - p[0], p[2] - p[0]), out_dir) < 0:
            tri = [tri[0], tri[2], tri[1]]
        return tri

    if n_in in (1, 3):
        lone = [i for i in range(4) if inside[i] == (n_in == 1)][0]
        others = [i for i in range(4) if i != lone]
        return [wind([(lone, o) for o in others])]
    a, b = [i for i in range(4) if inside[i]]
    c, d = [i for i in range(4) if not inside[i]]
    return [wind([(a, c), (a, d), (b, d)]), wind([(a, c), (b, d), (b, c)])]


def extract(grid, origin, voxel):
    """Marching tetrahedra on grid [nz,ny,nx,2] (f32 tsdf, weight) -> dict(vertices f64 [V,3], faces i64 [F,3],
    edges i64 [V,2] (grid point linear index, direction code) of each vertex)."""
    g = np.asarray(grid, np.float32)
    nz, ny, nx, _ = g.shape
    tsdf, w = g[..., 0], g[..., 1]
    cz, cy, cx = np.meshgrid(np.arange(nz - 1), np.arange(ny - 1), np.arange(nx - 1), indexing="ij")
    cx, cy, cz = cx.reshape(-1), cy.reshape(-1), cz.reshape(-1)
    n_cubes = len(cx)
    point = lambda code: ((cz + (code >> 2 & 1)) * ny + (cy + (code >> 1 & 1))) * nx + (cx + (code & 1))
    flat_t, flat_w = tsdf.reshape(-1), w.reshape(-1)
    keys = np.full((n_cubes, 6, 2, 3), -1, np.int64)
    for k in range(6):
        codes = _tet_codes(k)
        idx = [point(c) for c in codes]
        val = [flat_t[i] for i in idx]
        ok = np.all([flat_w[i] > 0 for i in idx], 0)
        for i, j in itertools.combinations(range(4), 2):
            ok &= ~(((val[i] == 1) & (val[j] == -1)) | ((val[i] == -1) & (val[j] == 1)))
        bits = sum((val[i] < 0).astype(np.int64) << i for i in range(4))
        for case in range(16):
            sel = ok & (bits == case)
            if not sel.any():
                continue
            tris = _case_triangles(k, tuple(bool(case >> i & 1) for i in range(4)))
            for t, tri in enumerate(tris):
                for e, (i, j) in enumerate(tri):
                    lo, hi = (i, j) if i < j else (j, i)
                    keys[sel, k, t, e] = idx[lo][sel] * 8 + (codes[lo] ^ codes[hi])
    keys = keys.reshape(-1, 3)
    keys = keys[keys[:, 0] >= 0]
    uniq = np.unique(keys)
    faces = np.searchsorted(uniq, keys)
    p, d = uniq // 8, uniq % 8
    o = np.asarray(origin, np.float32).astype(np.float64)
    s = float(np.float32(voxel))
    px, py, pz = p % nx, (p // nx) % ny, p // (nx * ny)
    q = ((pz + (d >> 2 & 1)) * ny + (py + (d >> 1 & 1))) * nx + (px + (d & 1))
    v0, v1 = flat_t[p].astype(np.float64), flat_t[q].astype(np.float64)
    t = v0 / (v0 - v1)
    V = np.stack([o[a] + (np.stack([px, py, pz])[a] + 0.5 + t * (d >> a & 1)) * s for a in range(3)], 1)
    return dict(vertices=V, faces=faces, edges=np.stack([p, d], 1))


def topology(faces, n_vertices=None):
    """-> dict(manifold: every undirected edge in exactly two faces, oriented: every directed edge once, euler:
    V - E + F over the referenced vertices)."""
    F = np.asarray(faces, np.int64)
    directed = np.concatenate([F[:, [0, 1]], F[:, [1, 2]], F[:, [2, 0]]])
    und = np.sort(directed, 1)
    _, und_counts = np.unique(und, axis=0, return_counts=True)
    _, dir_counts = np.unique(directed, axis=0, return_counts=True)
    V = len(np.unique(F)) if n_vertices is None else n_vertices
    return dict(manifold=bool(np.all(und_counts == 2)), oriented=bool(np.all(dir_counts == 1)),
                euler=int(V - len(und_counts) + len(F)))


def signed_volume(vertices, faces):
    V = np.asarray(vertices, np.float64)
    a, b, c = (V[np.asarray(faces)[:, i]] for i in range(3))
    return float(np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6.0)
