"""An fp64 ray caster for the rasteriser (csrc/render.cu), the scenes it is compared on, and the comparison with its
bars.  Shared by tests/test_gpu_render_fp64.py (the kernels) and tests/test_render_fp64_cpu.py (oracle/render_port.py).

The caster restates the renderer's definition, not its arithmetic: it imports nothing from oracle/ and works in camera
space from the caller's float32 inputs promoted to float64.

  Samples    pixel (i, j) = (column, row) is centred at (i, j); gp_render_templates takes 4 samples at (-1/8, -3/8),
             (3/8, -1/8), (-3/8, 1/8), (1/8, 3/8) px from the centre, gp_render_depth one at the centre.
  Ray, hit   the ray of sample (u, v) has direction d = K^-1 (u, v, 1) with the full K (K01 included), so d_z = 1 and
             the ray parameter of a hit is its camera-space z.  Against a triangle P0 P1 P2 (either winding) the hit
             has z = [P0 P1 P2] / (d . n), n = (P1 - P0) x (P2 - P0), and 3-D barycentrics
             mu_i = d . (P_j x P_k) / (d . n) (Cramer's rule, i.e. the Moller-Trumbore solution written out); the
             sample is inside iff every mu_i >= 0.  A face with a vertex at z <= z_near, a vertex index outside [0, V)
             or a vertex projected 2^22 px or more from the origin is dropped (stated departures of the contract).
  Visibility the nearest hit wins.
  Attributes colour and UV are sum_i mu_i a_i at the 3-D hit point: perspective-correct by construction.
  Texture    bilinear at level 0 with repeat wrap; texel (c, r) of a texture whose row 0 is on top has its centre at
             u = (c + 1/2) / tw, v = (th - 1 - r + 1/2) / th.
  Resolve    RGB = 255 x the mean of the 4 samples (background 0), unquantised; alpha = any sample covered; the
             templates' depth = the smallest covered sample z; boxes [x0, y0, x1, y1) with exclusive max,
             (0, 0, W, H) for an empty view.

Bars.  The kernel differs from this definition in two ways only, both bounded per sample:
  (1) snapping: it moves each projected vertex k to the 1/256 px grid, by at most eps_k = 1/512 px plus the float32
      error of its projection (bounded in `_camera` from the operation count).  For a sample inside a triangle, with
      screen barycentrics lambda_k, any quantity q interpolated over the triangle (depth, colour, UV) obeys
      dq/du_k = -lambda_k dq/du (the vertex moves, the sample does not), so its snap sensitivity is
      S_q = sum_k |lambda_k| (eps_u,k |dq/du| + eps_v,k |dq/dv|).  dq/du and dq/dv are analytic here: z and mu_i are
      ratios of linear functions of (u, v), so the derivatives are exact formulas evaluated in float64 (relative
      error ~1e-15, nothing next to the bars).  The terms second order in eps are smaller than S_q by a further
      factor of about eps / (the triangle's smallest altitude): under 1 % except on sub-pixel faces, whose samples
      mostly lie within delta of an edge and are excluded.
  (2) float32 arithmetic: counted per operation, each rounding contributing at most one unit u = 2^-24 relative.
      Depth (sample_weights, sample_depth): float(w_i), float(2A), the division, the product with 1/z_i and the
      rounding of that reciprocal give 5u per term; the two additions of three positive terms 2u; the final
      reciprocal u: 8u, plus the relative float32 error r of the camera-space z_i (gamma_4 x sum |terms| / z).  So
      c_z = 8 + r / u, and the depth bar is S_z + c_z ulp(z) (ulp(z) >= u z).
  Coverage: the edge function E_k of the unsnapped projection (in px^2, positive inside) moves under the snap by at
      most dE_k = eps_u,a |b_y - p_y| + eps_v,a |p_x - b_x| + eps_u,b |p_y - a_y| + eps_v,b |p_x - a_x|
      + 2 eps_a eps_b (exact: E is bilinear in the vertices).  dE_k / |b - a| is delta, the distance in px within
      which the kernel may decide either way; about 1/256 px near the middle of an edge.  A face covers a sample
      robustly iff every E_k > dE_k, misses it robustly iff some E_k < -dE_k; `score` = min_k E_k / dE_k is > 1 or
      < -1 accordingly.  A sample's coverage is unambiguous iff its best score over all faces is outside [-1, 1]."""
from __future__ import annotations

import numpy as np

U = 2.0 ** -24                    # unit roundoff of float32
SNAP = 1.0 / 512                  # largest move of a vertex snapped to 1/256 px
GUARD = 2.0 ** 22
SAMPLES4 = np.array([[-1 / 8, -3 / 8], [3 / 8, -1 / 8], [-3 / 8, 1 / 8], [1 / 8, 3 / 8]])
SAMPLES1 = np.zeros((1, 2))
RESOLVE_Q = 1e-4                  # resolve arithmetic in q units: 3 additions of <= 4 and x255, < 4 x 4u x 63.75 + 255u
MUTATIONS = ("pixel_centre_half", "mirrored_pattern", "affine", "flip_v", "cull_back", "ignore_k01")


def _ulp32(z):
    return np.spacing(np.abs(z).astype(np.float32)).astype(np.float64)


def _camera(V, pose, K, ignore_k01):
    """Per vertex: camera coordinates, projection (u, v), the float32 error bounds of the kernel's z and of its
    projection.  The kernel's camera coordinate is a sum of 4 rounded terms: error <= 4u sum|terms| (gamma_4)."""
    P = np.asarray(pose, np.float32).astype(np.float64).reshape(4, 4)
    terms = V[:, None, :] * P[None, :3, :3]
    cam = terms.sum(-1) + P[:3, 3]
    err = 4 * U * (np.abs(terms).sum(-1) + np.abs(P[:3, 3]))
    x, y, z = cam.T
    ex, ey, ez = err.T
    k00, k01, k02, k11, k12 = K[0, 0], 0.0 if ignore_k01 else K[0, 1], K[0, 2], K[1, 1], K[1, 2]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        a, b = k00 * x + k01 * y, k11 * y
        u, v = a / z + k02, b / z + k12
        # products, sum and division of the numerator (4u over its magnitude), the camera errors, the final addition
        au, bv = np.abs(k00 * x) + np.abs(k01 * y), np.abs(b)
        eu = (abs(k00) * ex + abs(k01) * ey + 4 * U * au) / z + np.abs(a) / z * (ez / z) + U * np.abs(u)
        ev = (abs(k11) * ey + 3 * U * bv) / z + bv / z * (ez / z) + U * np.abs(v)
    return cam, u, v, ez / np.abs(z), SNAP + eu, SNAP + ev


class Cast:
    """The per-sample result of `cast` for one view, flattened over (pixel row, column, sample)."""


def _faces_setup(mesh, pose, K, z_near, cull_back, ignore_k01):
    V = np.asarray(mesh["vertices"], np.float32).astype(np.float64).reshape(-1, 3)
    Fi = np.asarray(mesh["faces"], np.int64).reshape(-1, 3)
    Kd = np.asarray(K, np.float32).astype(np.float64).reshape(3, 3)
    if ignore_k01:
        Kd = Kd.copy()
        Kd[0, 1] = 0.0
    cam, u, v, rz, eu, ev = _camera(V, pose, Kd, ignore_k01)
    inb = ((Fi >= 0) & (Fi < len(V))).all(1)
    fi = np.where(inb[:, None], Fi, 0)
    with np.errstate(invalid="ignore"):
        ok_v = (cam[:, 2] > z_near) & (np.abs(u) < GUARD) & (np.abs(v) < GUARD)
    valid = inb & ok_v[fi].all(1)
    P = cam[fi]                                                   # [F,3 corners,3]
    q = np.stack([u[fi], v[fi]], -1)                              # [F,3,2] projected, px
    area2 = ((q[:, 1, 0] - q[:, 0, 0]) * (q[:, 2, 1] - q[:, 0, 1]) - (q[:, 1, 1] - q[:, 0, 1]) * (q[:, 2, 0] - q[:, 0, 0]))
    valid &= np.isfinite(area2) & (area2 != 0)
    if cull_back:
        valid &= area2 > 0
    n = np.cross(P[:, 1] - P[:, 0], P[:, 2] - P[:, 0])
    c = np.stack([np.cross(P[:, 1], P[:, 2]), np.cross(P[:, 2], P[:, 0]), np.cross(P[:, 0], P[:, 1])], 1)
    Kinv_T = np.linalg.inv(Kd).T
    return dict(valid=valid, P=P, q=q, orient=np.sign(area2), A=np.einsum("fi,fi->f", n, P[:, 0]),
                n=n @ Kinv_T.T, c=c @ Kinv_T.T, z=P[:, :, 2], eu=eu[fi], ev=ev[fi], cz=8 + rz[fi].max(1) / U,
                r=rz[fi].max(1), faces=fi)


def _edges(f, sx, sy):
    """Edge functions E [n,3] (positive inside) and their snap bounds dE [n,3] of faces f at samples (sx, sy)."""
    q, o = f["q"], f["orient"]
    E, dE = [], []
    for k in range(3):
        a, b = (k + 1) % 3, (k + 2) % 3
        ax, ay, bx, by = q[:, a, 0], q[:, a, 1], q[:, b, 0], q[:, b, 1]
        E.append(o * ((bx - ax) * (sy - ay) - (by - ay) * (sx - ax)))
        ea, eb = np.maximum(f["eu"][:, a], f["ev"][:, a]), np.maximum(f["eu"][:, b], f["ev"][:, b])
        dE.append(f["eu"][:, a] * np.abs(by - sy) + f["ev"][:, a] * np.abs(sx - bx) + f["eu"][:, b] * np.abs(sy - ay)
                  + f["ev"][:, b] * np.abs(sx - ax) + 2 * ea * eb)
    return np.stack(E, 1), np.stack(dE, 1)


def _hit(f, sx, sy):
    """z, 3-D barycentrics mu [n,3] and their derivatives in u and v, screen barycentrics lambda [n,3]."""
    D = f["n"][:, 0] * sx + f["n"][:, 1] * sy + f["n"][:, 2]
    N = f["c"][:, :, 0] * sx[:, None] + f["c"][:, :, 1] * sy[:, None] + f["c"][:, :, 2]
    with np.errstate(divide="ignore", invalid="ignore"):
        z = f["A"] / D
        mu = N / D[:, None]
        z_u, z_v = -f["A"] * f["n"][:, 0] / D ** 2, -f["A"] * f["n"][:, 1] / D ** 2
        mu_u = (f["c"][:, :, 0] * D[:, None] - N * f["n"][:, 0:1]) / D[:, None] ** 2
        mu_v = (f["c"][:, :, 1] * D[:, None] - N * f["n"][:, 1:2]) / D[:, None] ** 2
        lam = mu * f["z"] / z[:, None]
    return z, mu, mu_u, mu_v, lam, z_u, z_v


def _sens(f, lam, q_u, q_v):
    """Snap sensitivity sum_k |lambda_k| (eps_u,k |dq/du| + eps_v,k |dq/dv|); q_u, q_v [n] or [n,c]."""
    wu, wv = (np.abs(lam) * f["eu"]).sum(1), (np.abs(lam) * f["ev"]).sum(1)
    if q_u.ndim == 2:
        wu, wv = wu[:, None], wv[:, None]
    return wu * np.abs(q_u) + wv * np.abs(q_v)


def _take(f, idx):
    return {k: v[idx] for k, v in f.items()}


def bilinear(tex, U_, V_, flip_v=False):
    """Bilinear level-0 lookup with repeat wrap -> rgb [n,3], and the local Lipschitz constants (largest difference of
    adjacent texels, wrap included) in x and y over the 4 x 4 texels around the footprint, per texel [n,3] each."""
    th, tw = tex.shape[:2]
    fx, fy = U_ * tw - 0.5, V_ * th - 0.5
    x0, y0 = np.floor(fx), np.floor(fy)
    ax, ay = (fx - x0)[:, None], (fy - y0)[:, None]
    cols = np.mod(x0[:, None].astype(np.int64) + np.arange(-1, 3), tw)              # [n,4]
    rows_b = np.mod(y0[:, None].astype(np.int64) + np.arange(-1, 3), th)            # counted from the bottom
    rows = rows_b if flip_v else th - 1 - rows_b
    blk = tex[rows[:, :, None], cols[:, None, :]]                                   # [n,4 rows,4 cols,3]
    top = (1 - ax) * blk[:, 1, 1] + ax * blk[:, 1, 2]
    bot = (1 - ax) * blk[:, 2, 1] + ax * blk[:, 2, 2]
    rgb = (1 - ay) * top + ay * bot
    lx = np.abs(np.diff(blk, axis=2)).max((1, 2))
    ly = np.abs(np.diff(blk, axis=1)).max((1, 2))
    return rgb, lx, ly


def _texture_global_lipschitz(tex):
    wx = np.concatenate([tex, tex[:, :1]], 1)
    wy = np.concatenate([tex, tex[:1]], 0)
    return np.abs(np.diff(wx, axis=1)).max((0, 1)), np.abs(np.diff(wy, axis=0)).max((0, 1))


def cast(mesh, pose, K, H, W, z_near, n_samples=4, mutation=None, chunk=1 << 20):
    """Casts every sample of one view.  `mutation` (one of MUTATIONS) changes the definition, to show that the bars
    catch a renderer that differs in that way.  -> Cast (see the attributes set below)."""
    shift, mirror = (0.5 if mutation == "pixel_centre_half" else 0.0), mutation == "mirrored_pattern"
    affine, flip_v = mutation == "affine", mutation == "flip_v"
    offs = (SAMPLES4 if n_samples == 4 else SAMPLES1).copy()
    if mirror:
        offs[:, 0] = -offs[:, 0]
    offs += shift
    NS = len(offs)
    f = _faces_setup(mesh, pose, K, z_near, mutation == "cull_back", mutation == "ignore_k01")
    nsamp = H * W * NS
    score = np.full(nsamp, -np.inf)
    recs = []
    fid = np.nonzero(f["valid"])[0]
    reach = np.abs(offs).max() + 1.0
    q = f["q"][fid]
    x0 = np.maximum(np.ceil(q[:, :, 0].min(1) - reach), 0).astype(np.int64)
    x1 = np.minimum(np.floor(q[:, :, 0].max(1) + reach), W - 1).astype(np.int64)
    y0 = np.maximum(np.ceil(q[:, :, 1].min(1) - reach), 0).astype(np.int64)
    y1 = np.minimum(np.floor(q[:, :, 1].max(1) + reach), H - 1).astype(np.int64)
    keep = (x1 >= x0) & (y1 >= y0)
    fid, x0, y0, bw, bh = fid[keep], x0[keep], y0[keep], (x1 - x0 + 1)[keep], (y1 - y0 + 1)[keep]
    starts = np.concatenate([[0], np.cumsum(bw * bh)])
    for lo in range(0, int(starts[-1]), chunk):
        idx = np.arange(lo, min(lo + chunk, int(starts[-1])))
        k = np.searchsorted(starts, idx, side="right") - 1
        p = idx - starts[k]
        px, py, face = x0[k] + p % bw[k], y0[k] + p // bw[k], fid[k]
        fk = _take(f, face)
        for s in range(NS):
            sx, sy = px + offs[s, 0], py + offs[s, 1]
            E, dE = _edges(fk, sx, sy)
            sc = (E / dE).min(1)
            sid = (py * W + px) * NS + s
            np.maximum.at(score, sid, sc)
            z, mu, _, _, lam, z_u, z_v = _hit(fk, sx, sy)
            inside = (mu >= 0).all(1)
            m = sc >= -1                                            # the face may cover the sample
            zb = _sens(fk, lam, z_u, z_v) + fk["cz"] * _ulp32(z)
            if affine:                                              # depth affine in screen space instead of 1/z
                lam2 = E / E.sum(1, keepdims=True)
                z = (lam2 * fk["z"]).sum(1)
            recs.append(np.rec.fromarrays([sid[m], face[m], z[m], zb[m], inside[m], sc[m]],
                                          names="sid,face,z,zbar,inside,score"))
    r = np.concatenate(recs).view(np.recarray) if recs else np.rec.fromarrays(
        [np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0), np.zeros(0), np.zeros(0, bool), np.zeros(0)],
        names="sid,face,z,zbar,inside,score")
    c = Cast()
    c.H, c.W, c.NS, c.offsets, c.faces, c.records = H, W, NS, offs, f, r
    c.score = score
    c.covered = np.zeros(nsamp, bool)
    c.face = np.full(nsamp, -1, np.int64)
    c.z = np.zeros(nsamp)
    c.zbar = np.zeros(nsamp)
    c.gap = np.full(nsamp, np.inf)
    ins = r[r.inside]
    order = np.lexsort((ins.z, ins.sid))
    ins = ins[order]
    first = np.ones(len(ins), bool)
    first[1:] = ins.sid[1:] != ins.sid[:-1]
    win = ins[first]
    c.covered[win.sid] = True
    c.face[win.sid], c.z[win.sid], c.zbar[win.sid] = win.face, win.z, win.zbar
    second = np.nonzero(~first & np.concatenate([[False], first[:-1]]))[0]
    c.gap[ins.sid[second]] = ins.z[second] - c.z[ins.sid[second]]
    # the winner is unambiguous when it covers robustly and its depth interval lies before every other face that may
    # cover the sample
    other = np.full(nsamp, np.inf)
    rest = r.face != c.face[r.sid]
    np.minimum.at(other, r.sid[rest], r.z[rest] - r.zbar[rest])
    robust_win = np.zeros(nsamp, bool)
    np.logical_or.at(robust_win, r.sid[(r.face == c.face[r.sid]) & (r.score > 1)], True)
    c.cov_clear = np.abs(score) > 1
    c.win_clear = c.covered & robust_win & (c.z + c.zbar < other)
    c.clean = c.cov_clear & (~c.covered | c.win_clear)
    c.mesh, c.mutation = mesh, mutation
    c.px = (np.arange(nsamp) // NS) % W + offs[np.arange(nsamp) % NS, 0]
    c.py = (np.arange(nsamp) // NS) // W + offs[np.arange(nsamp) % NS, 1]
    _snapped_depth(c)
    return c


def _snapped_depth(c):
    """The arithmetic-only reference: 1 / z of the plane through the SNAPPED screen vertices, affine in screen space,
    at the covered samples; NaN where a vertex of the winning face is within its projection error of a rounding tie
    (the kernel might snap it to the other neighbour)."""
    c.zsnap = np.full(len(c.z), np.nan)
    s = np.nonzero(c.covered)[0]
    if c.mutation is not None or not len(s):
        return
    f = _take(c.faces, c.face[s])
    t = f["q"] * 256
    tie = (np.abs(t - np.rint(t)) > 0.5 - 256 * (np.stack([f["eu"], f["ev"]], -1) - SNAP)).any((1, 2))
    g = np.rint(t) / 256
    sx, sy = c.px[s], c.py[s]
    e = []
    for k in range(3):
        a, b = g[:, (k + 1) % 3], g[:, (k + 2) % 3]
        e.append((b[:, 0] - a[:, 0]) * (sy - a[:, 1]) - (b[:, 1] - a[:, 1]) * (sx - a[:, 0]))
    e = np.stack(e, 1)
    with np.errstate(divide="ignore", invalid="ignore"):
        lam = e / e.sum(1, keepdims=True)
        zs = 1 / (lam / f["z"]).sum(1)
    c.zsnap[s] = np.where(tie, np.nan, zs)


def shade(c, mutation=None):
    """Colour and its bar (both in [0, 1] units) at the covered samples of Cast c -> (rgb [n,3], bar [n,3]); the bar is
    the snap sensitivity plus the float32 arithmetic: (20u + 2r) sum_i mu_i |a_i| for an interpolated attribute
    (weights 5u + r, product u, two additions 2u, times z 8u + r + u: 17u + 2r, rounded up), then for a texture the
    lookup's x = U tw - 1/2 (2 roundings) through the local Lipschitz constant per texel, plus 6u for its lerps."""
    mesh, nsamp = c.mesh, len(c.z)
    rgb, bar = np.zeros((nsamp, 3)), np.zeros((nsamp, 3))
    s = np.nonzero(c.covered)[0]
    if not len(s):
        return rgb, bar
    f = _take(c.faces, c.face[s])
    z, mu, mu_u, mu_v, lam, _, _ = _hit(f, c.px[s], c.py[s])
    if mutation == "affine":
        E, _ = _edges(f, c.px[s], c.py[s])
        mu = E / E.sum(1, keepdims=True)
    ar = 20 * U + 2 * f["r"]

    def interp(a):                                                  # a [n,3 corners] -> value, bar
        val = (mu * a).sum(1)
        return val, _sens(f, lam, (mu_u * a).sum(1), (mu_v * a).sum(1)) + ar * (mu * np.abs(a)).sum(1)
    if mesh.get("texture") is not None:
        tex = np.asarray(mesh["texture"], np.float32).astype(np.float64)
        th, tw = tex.shape[:2]
        uv = np.asarray(mesh["face_uv"], np.float32).astype(np.float64).reshape(-1, 3, 2)[c.face[s]]
        Uv, Ub = interp(uv[..., 0])
        Vv, Vb = interp(uv[..., 1])
        col, lx, ly = bilinear(tex, Uv, Vv, flip_v=mutation == "flip_v")
        dfx = tw * Ub + U * (2 * np.abs(Uv * tw) + 1)
        dfy = th * Vb + U * (2 * np.abs(Vv * th) + 1)
        gx, gy = _texture_global_lipschitz(tex)
        lx = np.where((dfx < 1)[:, None], lx, gx)
        ly = np.where((dfy < 1)[:, None], ly, gy)
        b = lx * dfx[:, None] + ly * dfy[:, None] + 6 * U
    elif mesh.get("vertex_color") is not None:
        vc = np.asarray(mesh["vertex_color"], np.float32).astype(np.float64)[f["faces"]]      # [n,3 corners,3]
        out = [interp(vc[..., ch]) for ch in range(3)]
        col, b = np.stack([o[0] for o in out], 1), np.stack([o[1] for o in out], 1)
    else:
        cc = mesh.get("constant_color")
        col = np.broadcast_to(np.ones(3) if cc is None else np.asarray(cc, np.float32).astype(np.float64), (len(s), 3))
        b = np.zeros((len(s), 3))
    rgb[s], bar[s] = col, b
    return rgb, bar


# ------------------------------------------------------------------------------------------------------ comparison
def _worst(err, bar):
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(bar > 0, err / bar, np.where(err > 0, np.inf, 0.0))
    return float(r.max()) if r.size else 0.0


def compare(c, keys=None, depth=None, box=None, rgba=None):
    """Compares one view of a renderer's output with Cast c.  keys uint64 [H,W,NS] (the per-sample key buffer), depth
    f32 [H,W], box [4], rgba f32 [4,H,W] (templates).  Without keys (the CPU port of gp_render_depth) the sample is
    the pixel and its z is the depth map.  -> dict of comparisons, each with n (checked), fail, worst (largest
    error / bar; for coverage the largest |score| of a mismatch) and where applicable excl (excluded fraction)."""
    H, W, NS = c.H, c.W, c.NS
    rep = {}
    if keys is not None:
        kf = np.asarray(keys).reshape(-1)
        got_cov = kf != np.uint64(0xFFFFFFFFFFFFFFFF)
        got_face = (kf & np.uint64(0xFFFFFFFF)).astype(np.int64)
        got_z = (kf >> np.uint64(32)).astype(np.uint32).view(np.float32).astype(np.float64)
    else:
        dflat = np.asarray(depth, np.float32).reshape(-1).astype(np.float64)
        got_cov, got_face, got_z = dflat > 0, None, dflat
    cand = np.isfinite(c.score)                                     # samples some face's box reaches
    mis = c.cov_clear & (got_cov != c.covered)
    rep["coverage"] = dict(n=int(c.cov_clear.sum()), fail=int(mis.sum()),
                           worst=float(np.abs(c.score[mis]).max()) if mis.any() else 0.0,
                           excl=float((cand & ~c.cov_clear).sum() / max(cand.sum(), 1)))
    both = c.win_clear & got_cov
    if got_face is not None:
        bad = both & (got_face != c.face)
        rep["face"] = dict(n=int(both.sum()), fail=int(bad.sum()), worst=float(bad.any()) * np.inf,
                           excl=float((c.covered & c.cov_clear & ~c.win_clear).sum() / max(c.covered.sum(), 1)))
    err = np.abs(got_z - c.z)[both]
    rep["depth"] = dict(n=int(both.sum()), fail=int((err > c.zbar[both]).sum()), worst=_worst(err, c.zbar[both]))
    ok = both & np.isfinite(c.zsnap)
    if c.mutation is None:
        bar = c.faces["cz"][c.face[ok]] * _ulp32(c.z[ok])
        e2 = np.abs(got_z[ok] - c.zsnap[ok])
        rep["depth_arith"] = dict(n=int(ok.sum()), fail=int((e2 > bar).sum()), worst=_worst(e2, bar),
                                  ulps=float((e2 / _ulp32(c.z[ok])).max()) if ok.any() else 0.0)
    pix_clean = c.clean.reshape(-1, NS).all(1)
    cov_clear_pix = c.cov_clear.reshape(-1, NS).all(1)
    if depth is not None:
        d = np.asarray(depth, np.float32).reshape(-1).astype(np.float64)
        cov = c.covered.reshape(-1, NS)
        zref = np.where(cov, c.z.reshape(-1, NS), np.inf).min(1)
        zbar = np.where(cov, c.zbar.reshape(-1, NS), 0).max(1)
        bg = cov_clear_pix & ~cov.any(1)
        chk = pix_clean & cov.any(1)
        e = np.abs(d - zref)[chk]
        rep["depth_map"] = dict(n=int(chk.sum() + bg.sum()), fail=int((e > zbar[chk]).sum() + (d[bg] != 0).sum()),
                                worst=_worst(e, zbar[chk]) if not (d[bg] != 0).any() else np.inf)
        if keys is not None:                                        # the map is the smallest covered key
            kz = np.where(got_cov, got_z, np.inf).reshape(-1, NS).min(1)
            rep["depth_map"]["fail"] += int((np.where(np.isfinite(kz), kz, 0) != d).sum())
    if rgba is not None:
        q = np.rint(np.asarray(rgba, np.float32)[:3].reshape(3, -1).T.astype(np.float64) * 255)
        col, bar = shade(c, c.mutation)
        cov = c.covered.reshape(-1, NS, 1)
        ref = 255 * np.where(cov, col.reshape(-1, NS, 3), 0).mean(1)
        e = 255 * np.where(cov, bar.reshape(-1, NS, 3), 0).mean(1) + RESOLVE_Q
        m = pix_clean
        if c.mesh.get("texture") is None and c.mesh.get("vertex_color") is None:
            m = cov_clear_pix                                       # constant colour: exact wherever coverage is clear
            exact = np.rint(255 * np.where(cov, col.reshape(-1, NS, 3), 0).sum(1) / 4)
            bad = (q != exact)[m]
            rep["rgb"] = dict(n=int(m.sum()), fail=int(bad.sum()), worst=float(np.abs(q - exact)[m].max(initial=0)),
                              excl=float(1 - m.mean()))
        else:
            d_ = np.abs(q - ref)[m]
            rep["rgb"] = dict(n=int(m.sum()), fail=int((d_ > 0.5 + e[m]).sum()), worst=_worst(d_, 0.5 + e[m]),
                              excl=float(((~m) & cov.any((1, 2))).sum() / max(cov.any((1, 2)).sum(), 1)),
                              e_max=float(e[m].max(initial=0)))
        alpha = np.asarray(rgba, np.float32)[3].reshape(-1)
        aref = c.covered.reshape(-1, NS).any(1)
        am = (c.covered & c.cov_clear).reshape(-1, NS).any(1) | (~c.covered & c.cov_clear).reshape(-1, NS).all(1)
        rep["alpha"] = dict(n=int(am.sum()), fail=int(((alpha > 0) != aref)[am].sum()), worst=0.0)
    if box is not None:
        cs = c.covered & c.cov_clear
        lo_pix = cs.reshape(-1, NS).any(1).reshape(H, W)                        # certainly covered
        hi_pix = (cs | ~c.cov_clear).reshape(-1, NS).any(1).reshape(H, W)      # possibly covered
        ref = c.covered.reshape(-1, NS).any(1).reshape(H, W)

        def bb(m):
            ys, xs = np.nonzero(m)
            return np.array([xs.min(), ys.min(), xs.max() + 1, ys.max() + 1] if len(xs) else [0, 0, W, H])
        b, lo, hi, rb = np.asarray(box).astype(np.int64), bb(lo_pix), bb(hi_pix), bb(ref)
        if not lo_pix.any():
            ok_box = (not hi_pix.any() and b.tolist() == [0, 0, W, H]) or hi_pix.any()
        else:
            ok_box = (hi[:2] <= b[:2]).all() and (b[:2] <= lo[:2]).all() and (lo[2:] <= b[2:]).all() and \
                (b[2:] <= hi[2:]).all()
        ok_box = ok_box and np.abs(b - rb).max() <= 1
        rep["box"] = dict(n=1, fail=int(not ok_box), worst=float(np.abs(b - rb).max()), exact=bool((lo == hi).all()))
    return rep


def failures(rep):
    return {k: v for k, v in rep.items() if v["fail"]}


def merge(reports):
    """Per comparison over many views: n summed, fail summed, worst and excl the largest."""
    out = {}
    for rep in reports:
        for k, v in rep.items():
            o = out.setdefault(k, dict(n=0, fail=0, worst=0.0))
            o["n"] += v["n"]
            o["fail"] += v["fail"]
            o["worst"] = max(o["worst"], v["worst"])
            for extra in ("excl", "ulps", "e_max"):
                if extra in v:
                    o[extra] = max(o.get(extra, 0.0), v[extra])
    return out


def mutation_margin(rep, which):
    """How clearly a mutated definition fails: the number of failures and the worst ratio over the comparisons
    `which` (the ones the mutation is meant to break)."""
    return sum(rep[w]["fail"] for w in which if w in rep), max((rep[w]["worst"] for w in which if w in rep), default=0.0)


# ------------------------------------------------------------------------------------------------------------ scenes
TEMPLATE_K = np.array([[572.4114, 0.0, 320.0], [0.0, 573.57043, 240.0], [0.0, 0.0, 1.0]], np.float32)
HOPE_K = np.array([[1390.53, 0.0, 964.957], [0.0, 1386.99, 522.212], [0.0, 0.0, 1.0]], np.float32)


def icosphere(subdiv, radius, rng, bumps=0.15):
    t = (1 + 5 ** 0.5) / 2
    V = [[-1, t, 0], [1, t, 0], [-1, -t, 0], [1, -t, 0], [0, -1, t], [0, 1, t], [0, -1, -t], [0, 1, -t],
         [t, 0, -1], [t, 0, 1], [-t, 0, -1], [-t, 0, 1]]
    Fc = [[0, 11, 5], [0, 5, 1], [0, 1, 7], [0, 7, 10], [0, 10, 11], [1, 5, 9], [5, 11, 4], [11, 10, 2], [10, 7, 6],
          [7, 1, 8], [3, 9, 4], [3, 4, 2], [3, 2, 6], [3, 6, 8], [3, 8, 9], [4, 9, 5], [2, 4, 11], [6, 2, 10],
          [8, 6, 7], [9, 8, 1]]
    V = [np.array(v, float) / np.linalg.norm(v) for v in V]
    for _ in range(subdiv):
        mid, out = {}, []

        def m(a, b):
            key = (min(a, b), max(a, b))
            if key not in mid:
                p = V[a] + V[b]
                V.append(p / np.linalg.norm(p))
                mid[key] = len(V) - 1
            return mid[key]
        for a, b, c in Fc:
            ab, bc, ca = m(a, b), m(b, c), m(c, a)
            out += [[a, ab, ca], [b, bc, ab], [c, ca, bc], [ab, bc, ca]]
        Fc = out
    V = np.array(V)
    V *= radius * (1 + bumps * rng.uniform(-1, 1, (len(V), 1)))
    return V.astype(np.float32), np.array(Fc, np.int32)


def uv_sphere(V, Fc, scale):
    """Per-corner UVs from longitude / latitude, scaled past [0, 1] so that the repeat wrap is exercised."""
    d = V / np.linalg.norm(V, axis=1, keepdims=True)
    uv = np.stack([np.arctan2(d[:, 1], d[:, 0]) / (2 * np.pi) + 0.5, np.arccos(np.clip(d[:, 2], -1, 1)) / np.pi], 1)
    return (uv[Fc] * scale).astype(np.float32)


def ramp_texture(th=37, tw=53):
    """Non-square; R ramps along the columns and G down the rows, so that both wrap seams (texel tw - 1 next to
    texel 0, and the top row next to the bottom one) are full-scale jumps and a flipped v is obvious; B is smooth."""
    r, cc = np.meshgrid(np.arange(th), np.arange(tw), indexing="ij")
    return np.stack([cc / (tw - 1), r / (th - 1), 0.5 + 0.3 * np.sin(2 * np.pi * cc / tw) * np.cos(2 * np.pi * r / th)],
                    -1).astype(np.float32)


def _shuffle_windings(Fc, rng):
    flip = rng.random(len(Fc)) < 0.5
    Fc = Fc.copy()
    Fc[flip] = Fc[flip][:, ::-1]
    return Fc


def grid(nx, ny, sx, sy, rng):
    """A flat nx x ny cell grid of side sx x sy centred on the origin in the z = 0 plane, random diagonals and
    windings."""
    gx, gy = np.meshgrid(np.linspace(-sx / 2, sx / 2, nx + 1), np.linspace(-sy / 2, sy / 2, ny + 1))
    V = np.stack([gx, gy, np.zeros_like(gx)], -1).reshape(-1, 3)
    F = []
    for j in range(ny):
        for i in range(nx):
            a, b, c, d = j * (nx + 1) + i, j * (nx + 1) + i + 1, (j + 1) * (nx + 1) + i + 1, (j + 1) * (nx + 1) + i
            F += [[a, b, c], [a, c, d]] if rng.random() < 0.5 else [[a, b, d], [b, c, d]]
    uv = np.stack([(gx + sx / 2) / sx, (gy + sy / 2) / sy], -1).reshape(-1, 2)
    return V.astype(np.float32), _shuffle_windings(np.array(F, np.int32), rng), uv


def rot(axis, deg):
    a = np.asarray(axis, float) / np.linalg.norm(axis)
    t = np.radians(deg)
    Kx = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(t) * Kx + (1 - np.cos(t)) * Kx @ Kx


def pose(R, t):
    P = np.eye(4)
    P[:3, :3], P[:3, 3] = R, t
    return P.astype(np.float32)


def scaled_K(K, s, H=None, W=None):
    K = np.array(K, np.float64)
    K[:2] *= s
    if H is not None:
        K[0, 2], K[1, 2] = (W - 1) / 2, (H - 1) / 2
    return K.astype(np.float32)


def scenes(full):
    """Seeded procedural scenes: dict name -> dict(mesh, poses [n,4,4], K, H, W, z_near, mode, mutations).  `full`:
    the kernel's sizes (480 x 640 templates, 1080 x 1920 depth); otherwise small images for the CPU port.  Sizes
    37 x 53 are used by both."""
    rng = np.random.default_rng(20)
    out = {}
    Ht, Wt, Kt = (480, 640, TEMPLATE_K) if full else (60, 80, scaled_K(TEMPLATE_K, 1 / 8, 60, 80))
    Hd, Wd, Kd = (1080, 1920, HOPE_K) if full else (54, 96, scaled_K(HOPE_K, 1 / 20, 54, 96))
    K_odd = np.array([[64.0, 0.0, 26.0], [0.0, 66.0, 18.0], [0.0, 0.0, 1.0]], np.float32)
    tex = ramp_texture()
    # oblique planes: 2 x 2 cells of 200 mm tilted about x, centred at z = 400; depth spans ~300 .. 500 at 85 deg
    for deg in (60, 75, 85):
        V, F, uv = grid(2, 2, 200.0, 200.0, rng)
        P = pose(rot([1, 0, 0], deg) @ rot([0, 0, 1], 10), [8.0, -5.0, 400.0])
        col = rng.uniform(0, 1, (len(V), 3)).astype(np.float32)
        out[f"oblique{deg}_colour"] = dict(mesh=dict(vertices=V, faces=F, vertex_color=col), poses=P[None], K=Kt,
                                           H=Ht, W=Wt)
        fuv = (uv[F] * np.array([3.1, 2.3]) - np.array([0.7, 0.4])).astype(np.float32)   # past [0, 1], both signs
        out[f"oblique{deg}_texture"] = dict(mesh=dict(vertices=V, faces=F, face_uv=fuv, texture=tex), poses=P[None],
                                            K=Kt, H=Ht, W=Wt)
    # a closed bumpy icosphere, both windings, two views in one call
    V, F = icosphere(3 if full else 2, 60.0, rng)
    F = _shuffle_windings(F, rng)
    two = np.stack([pose(rot([0.3, 1, 0.2], 25), [10.0, -6.0, 420.0]), pose(rot([1, -0.4, 0.5], 140), [-15.0, 9.0, 380.0])])
    out["sphere_colour"] = dict(mesh=dict(vertices=V, faces=F, vertex_color=rng.uniform(0, 1, (len(V), 3)).astype(np.float32)),
                                poses=two, K=Kt, H=Ht, W=Wt)
    out["sphere_texture"] = dict(mesh=dict(vertices=V, faces=F, face_uv=uv_sphere(V, F, 3.0), texture=tex), poses=two,
                                 K=Kt, H=Ht, W=Wt)
    # two planes that cut each other: visibility flips along the intersection line
    Va, Fa, _ = grid(4, 4, 180.0, 180.0, rng)
    Va1 = (Va @ rot([0, 1, 0], 35).T).astype(np.float32)
    Va2 = (Va @ (rot([0, 1, 0], -30) @ rot([1, 0, 0], 20)).T).astype(np.float32)
    inter = dict(vertices=np.concatenate([Va1, Va2]), faces=np.concatenate([Fa, Fa + len(Va)]),
                 vertex_color=rng.uniform(0, 1, (2 * len(Va), 3)).astype(np.float32))
    out["intersecting"] = dict(mesh=inter, poses=pose(np.eye(3), [0.0, 0.0, 450.0])[None], K=Kt, H=Ht, W=Wt)
    # screen-filling faces (CTA path) behind sub-pixel ones (per-thread path)
    n_tiny = 20000 if full else 600
    big = np.array([[-3000, -3000, 300], [3000, -3000, 300], [0, 3000, 300],
                    [-3000, 3000, 310], [0, -3000, 310], [3000, 3000, 310]], np.float32)
    ctr = np.stack([rng.uniform(-60, 60, n_tiny), rng.uniform(-45, 45, n_tiny), rng.uniform(200, 280, n_tiny)], 1)
    tiny = (ctr[:, None] + rng.uniform(-0.12, 0.12, (n_tiny, 3, 3)) * ctr[:, None, 2:] / 250).reshape(-1, 3)
    Vb = np.concatenate([big, tiny]).astype(np.float32)
    Fb = _shuffle_windings(np.arange(len(Vb), dtype=np.int32).reshape(-1, 3), rng)
    out["big_and_tiny"] = dict(mesh=dict(vertices=Vb, faces=Fb, vertex_color=rng.uniform(0, 1, (len(Vb), 3)).astype(np.float32)),
                               poses=pose(np.eye(3), [0.0, 0.0, 0.0])[None], K=Kt, H=Ht, W=Wt)
    # clipping and exclusions, identity pose so that camera coordinates are the vertices themselves
    out["clipped"] = dict(mesh=_clipped_mesh(Kt, Ht, Wt, rng), poses=np.eye(4, dtype=np.float32)[None], K=Kt, H=Ht, W=Wt)
    out["clipped_odd"] = dict(mesh=_clipped_mesh(K_odd, 37, 53, rng), poses=np.eye(4, dtype=np.float32)[None], K=K_odd,
                              H=37, W=53)
    # cameras: skew K01 and an off-centre principal point, 37 x 53
    Ks = np.array([[64.0, 9.0, 15.0], [0.0, 66.0, 25.0], [0.0, 0.0, 1.0]], np.float32)
    Vs, Fs = icosphere(2, 60.0, rng)
    sk = dict(vertices=Vs, faces=_shuffle_windings(Fs, rng), vertex_color=rng.uniform(0, 1, (len(Vs), 3)).astype(np.float32))
    two_s = np.stack([pose(rot([0, 1, 0], 15), [50.0, -40.0, 420.0]), pose(rot([1, 0, 1], 70), [-60.0, 30.0, 400.0])])
    out["skew_offcentre"] = dict(mesh=sk, poses=two_s, K=Ks, H=37, W=53)
    Kw = np.array(Kt, np.float32).copy()
    Kw[0, 1], Kw[0, 2], Kw[1, 2] = 0.06 * Kw[0, 0], 0.3 * Wt, 0.62 * Ht
    out["skew_template"] = dict(mesh=sk, poses=two_s, K=Kw, H=Ht, W=Wt)
    # depth only (gp_render_depth): the HOPE frame size, and 37 x 53 with skew
    out["depth_sphere"] = dict(mesh=dict(vertices=V, faces=F), poses=two, K=Kd, H=Hd, W=Wd, mode="depth")
    out["depth_intersecting"] = dict(mesh=dict(vertices=inter["vertices"], faces=inter["faces"]),
                                     poses=pose(rot([0, 0, 1], 20), [30.0, 10.0, 500.0])[None], K=Kd, H=Hd, W=Wd,
                                     mode="depth")
    out["depth_skew_odd"] = dict(mesh=dict(vertices=Vs, faces=sk["faces"]), poses=two_s, K=Ks, H=37, W=53, mode="depth")
    out["depth_clipped_odd"] = dict(mesh=dict(vertices=out["clipped_odd"]["mesh"]["vertices"],
                                              faces=out["clipped_odd"]["mesh"]["faces"]),
                                    poses=np.eye(4, dtype=np.float32)[None], K=K_odd, H=37, W=53, mode="depth")
    for s in out.values():
        s.setdefault("mode", "templates")
        s.setdefault("z_near", 100.0)
    return out


def _clipped_mesh(K, H, W, rng):
    """A constant-colour scene in camera coordinates (identity pose):
      - a 6 x 6 cell wall at z = 500 reaching past every side of the image (negative pixel coordinates included);
      - a sliver with one vertex at 0.8 x 2^22 px (kept: its samples in the image are checked) and one with a vertex at
        1.2 x 2^22 px (dropped: the wall shows through);
      - a triangle crossing z_near = 100 (dropped: the wall shows through), and one whose vertices are one float32 ulp
        beyond z_near (kept)."""
    fx, fy, cx, cy = float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2])

    def at(u, v, z):                                              # camera point projecting to (u, v) px at depth z
        return [(u - cx - K[0, 1] * (v - cy) / fy) * z / fx, (v - cy) * z / fy, z]
    Vg, Fg, _ = grid(6, 6, 1.0, 1.0, rng)
    corners = np.array(at(-0.3 * W, -0.4 * H, 500.0))
    span = np.array(at(1.35 * W, 1.3 * H, 500.0)) - corners
    Vw = np.stack([corners[0] + (Vg[:, 0] + 0.5) * span[0], corners[1] + (Vg[:, 1] + 0.5) * span[1],
                   np.full(len(Vg), 500.0)], 1)
    z1 = float(np.nextafter(np.float32(100.0), np.float32(np.inf)))
    extra = [at(0.8 * GUARD, 0.3 * H, 300.0), at(0.2 * W, 0.25 * H, 300.0), at(0.25 * W, 0.7 * H, 300.0),
             at(-1.2 * GUARD, 0.5 * H, 300.0), at(0.7 * W, 0.35 * H, 300.0), at(0.8 * W, 0.8 * H, 300.0),
             at(0.35 * W, 0.1 * H, 90.0), at(0.6 * W, 0.15 * H, 150.0), at(0.5 * W, 0.45 * H, 150.0),
             at(0.15 * W, 0.55 * H, z1), at(0.45 * W, 0.6 * H, z1), at(0.3 * W, 0.92 * H, z1)]
    ex = np.array(extra, np.float64)
    ex[9:, 2] = z1
    V = np.concatenate([Vw, ex]).astype(np.float32)
    assert (V[-3:, 2] == np.float32(z1)).all()
    n = len(Vw)
    F = np.concatenate([Fg, n + np.array([[0, 1, 2], [3, 5, 4], [6, 7, 8], [9, 11, 10]], np.int32)])
    return dict(vertices=V, faces=F, constant_color=np.float32([0.25, 0.625, 0.875]))


# which comparisons each mutated definition must break, and on which scene
MUTATION_CASES = [("pixel_centre_half", "sphere_colour", ("coverage",)),
                  ("mirrored_pattern", "sphere_colour", ("coverage",)),
                  ("affine", "oblique85_colour", ("depth", "rgb")),
                  ("affine", "oblique85_texture", ("rgb",)),
                  ("flip_v", "oblique75_texture", ("rgb",)),
                  ("cull_back", "oblique75_colour", ("coverage",)),
                  ("ignore_k01", "skew_template", ("coverage",))]


# every scene must keep these comparisons non-vacuous: the largest excluded fraction (of the samples some face's box
# reaches, of the covered samples, of the covered pixels) and the fewest checked samples
MAX_EXCLUDED = dict(coverage=0.01, face=0.05, rgb=0.1)
MIN_CHECKED = dict(depth=400, depth_map=1000)


def cast_views(scene, mutation=None, cache=None):
    """One Cast per view of `scene`; scenes that share geometry, camera and size (colour / texture variants) share
    them through `cache`."""
    ns = 4 if scene["mode"] == "templates" else 1
    out = []
    for P in scene["poses"]:
        key = (id(scene["mesh"]["vertices"]), id(scene["mesh"]["faces"]), P.tobytes(), np.asarray(scene["K"]).tobytes(),
               scene["H"], scene["W"], ns, mutation)
        c = cache.get(key) if cache is not None else None
        if c is None:
            c = cast(scene["mesh"], P, scene["K"], scene["H"], scene["W"], scene["z_near"], ns, mutation)
            if cache is not None:
                cache[key] = c
        c.mesh = scene["mesh"]
        out.append(c)
    return out


def check_scene(scene, outputs, mutation=None, cache=None):
    """Casts every view of `scene` (with `mutation`) and compares it with `outputs`, the renderer's per-view dicts
    (keys / depth / box / rgba) -> (merged report, per-view Casts)."""
    casts = cast_views(scene, mutation, cache)
    return merge([compare(c, **out) for c, out in zip(casts, outputs)]), casts


def assert_within_bars(name, rep):
    """Every comparison passes, and none is vacuous."""
    bad = failures(rep)
    assert not bad, f"{name}: outside the bars: {bad}"
    for k, lim in MAX_EXCLUDED.items():
        if k in rep:
            assert rep[k]["excl"] <= lim, f"{name}: {k} excludes {rep[k]['excl']:.4f} > {lim}"
    for k, lim in MIN_CHECKED.items():
        assert rep[k]["n"] >= lim, f"{name}: only {rep[k]['n']} {k} checks"


def assert_mutation_fails(name, mutation, rep, which):
    """A mutated definition must fail the comparisons it targets clearly: at least 20 failures, and a worst
    error-to-bar ratio (for coverage: the worst |score|, the edge distance over delta) of at least 10."""
    n, worst = mutation_margin(rep, which)
    assert n >= 20 and worst >= 10, f"{name} / {mutation}: only {n} failures, worst ratio {worst:.3g}"
    return n, worst


def clipped_scene_is_exercised(scene, casts):
    """The clipped scene's reference must contain what it is there for: the sliver near the 2^22 px guard and the
    face one ulp beyond z_near are kept and win clean samples; the face past the guard and the face crossing z_near
    are dropped, and the samples inside their projections are covered by what lies behind them."""
    c = casts[0]
    nf = len(scene["mesh"]["faces"])
    kept, ulp_face, dropped = nf - 4, nf - 1, (nf - 3, nf - 2)
    f = c.faces
    assert f["valid"][kept] and f["valid"][ulp_face] and not f["valid"][dropped[0]] and not f["valid"][dropped[1]]
    for w in (kept, ulp_face):
        assert (c.win_clear & (c.face == w)).sum() >= 5, f"face {w} wins no clean sample"
    for d in dropped:
        q = f["q"][d]
        E = [(q[(k + 2) % 3, 0] - q[(k + 1) % 3, 0]) * (c.py - q[(k + 1) % 3, 1])
             - (q[(k + 2) % 3, 1] - q[(k + 1) % 3, 1]) * (c.px - q[(k + 1) % 3, 0]) for k in range(3)]
        E = np.stack(E) * f["orient"][d]
        behind = (E > 0).all(0)
        assert behind.sum() >= 5 and c.covered[behind].all() and (c.face[behind] != d).all()
