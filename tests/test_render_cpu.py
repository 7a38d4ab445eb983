"""Row f5 without a GPU: the PLY reader on hand-written files of each BOP model variant, its refusals, and analytic
cases for the CPU restatement of the renderer (oracle/render_port.py) that tests/test_gpu_render.py compares the
kernel against bit for bit."""
import struct

import numpy as np
import pytest

from gigapose_b200.render import PlyError, _device_mesh, read_ply
from oracle import render_port as rp

V3 = np.array([[0, 0, 0], [10.5, 0, 0], [0, 20.25, 0], [1, 2, 3]], np.float32)
F2 = np.array([[0, 1, 2], [1, 3, 2]], np.int32)


def _write_ply(path, fmt, vprops, vrows, fprops, frows, comments=()):
    """vprops [(name, type)], vrows list of tuples; fprops [(name, count_type, item_type)], frows list of lists of
    sequences (one per list property)."""
    head = ["ply", f"format {fmt} 1.0", *[f"comment {c}" for c in comments], f"element vertex {len(vrows)}"]
    head += [f"property {t} {n}" for n, t in vprops]
    head += [f"element face {len(frows)}"] + [f"property list {ct} {it} {n}" for n, ct, it in fprops] + ["end_header"]
    code = {"float": "f", "uchar": "B", "int": "i", "uint": "I", "double": "d", "ushort": "H"}
    with open(path, "wb") as f:
        f.write(("\n".join(head) + "\n").encode())
        for r in vrows:
            if fmt == "ascii":
                f.write((" ".join(str(x) for x in r) + "\n").encode())
            else:
                f.write(b"".join(struct.pack("<" + code[t], x) for x, (_, t) in zip(r, vprops)))
        for r in frows:
            if fmt == "ascii":
                f.write((" ".join(f"{len(lst)} " + " ".join(str(x) for x in lst) for lst in r) + "\n").encode())
            else:
                for lst, (_, ct, it) in zip(r, fprops):
                    f.write(struct.pack("<" + code[ct], len(lst)) + b"".join(struct.pack("<" + code[it], x) for x in lst))


@pytest.mark.parametrize("fmt", ["binary_little_endian", "ascii"])
def test_ply_with_uchar_vertex_colours_lm_style(tmp_path, fmt):
    """LM / LM-O / TUD-L / IC-BIN / HB: x y z nx ny nz red green blue [alpha] (uchar), vertex_indices."""
    rgb = np.array([[255, 0, 10], [0, 128, 20], [7, 8, 9], [1, 2, 255]])
    vp = [("x", "float"), ("y", "float"), ("z", "float"), ("nx", "float"), ("ny", "float"), ("nz", "float"),
          ("red", "uchar"), ("green", "uchar"), ("blue", "uchar"), ("alpha", "uchar")]
    rows = [tuple(V3[i].tolist()) + (0.0, 0.0, 1.0) + tuple(rgb[i].tolist()) + (255,) for i in range(4)]
    _write_ply(tmp_path / "m.ply", fmt, vp, rows, [("vertex_indices", "uchar", "int")], [[f.tolist()] for f in F2])
    m = read_ply(tmp_path / "m.ply")
    assert np.array_equal(m["vertices"], V3) and m["vertices"].dtype == np.float32
    assert np.array_equal(m["faces"], F2) and m["faces"].dtype == np.int32
    assert np.array_equal(m["vertex_color"], (rgb / np.float32(255)).astype(np.float32))
    assert m["texture"] is None and m["face_uv"] is None


@pytest.mark.parametrize("fmt", ["binary_little_endian", "ascii"])
def test_ply_cad_without_colour_tless_style(tmp_path, fmt):
    """T-LESS / ITODD CAD models: geometry (and normals) only; float colours, when present, are taken as is."""
    vp = [("x", "float"), ("y", "float"), ("z", "float"), ("nx", "float"), ("ny", "float"), ("nz", "float")]
    _write_ply(tmp_path / "m.ply", fmt, vp, [tuple(v.tolist()) + (1.0, 0.0, 0.0) for v in V3],
               [("vertex_indices", "uchar", "uint")], [[f.tolist()] for f in F2])
    m = read_ply(tmp_path / "m.ply")
    assert np.array_equal(m["vertices"], V3) and np.array_equal(m["faces"], F2)
    assert m["vertex_color"] is None and m["texture"] is None
    vp = [("x", "float"), ("y", "float"), ("z", "float"), ("red", "float"), ("green", "float"), ("blue", "float")]
    _write_ply(tmp_path / "c.ply", fmt, vp, [tuple(v.tolist()) + (0.25, 0.5, 1.0) for v in V3],
               [("vertex_indices", "uchar", "int")], [[f.tolist()] for f in F2])
    assert np.array_equal(read_ply(tmp_path / "c.ply")["vertex_color"], np.tile(np.float32([0.25, 0.5, 1.0]), (4, 1)))


def _texture_png(path):
    from PIL import Image
    tex = (np.arange(4 * 5 * 3).reshape(4, 5, 3) * 4).astype(np.uint8)
    Image.fromarray(tex).save(path)
    return tex.astype(np.float32) / np.float32(255)


@pytest.mark.parametrize("fmt", ["binary_little_endian", "ascii"])
def test_ply_textured_per_vertex_uv_ycbv_style(tmp_path, fmt):
    """YCB-V: texture_u / texture_v per vertex and `comment TextureFile`; the UVs are expanded to face corners."""
    tex = _texture_png(tmp_path / "obj_000001.png")
    uv = np.array([[0, 0], [1, 0], [0, 1], [0.5, 0.25]], np.float32)
    vp = [("x", "float"), ("y", "float"), ("z", "float"), ("texture_u", "float"), ("texture_v", "float")]
    _write_ply(tmp_path / "m.ply", fmt, vp, [tuple(V3[i].tolist()) + tuple(uv[i].tolist()) for i in range(4)],
               [("vertex_indices", "uchar", "int")], [[f.tolist()] for f in F2], comments=["TextureFile obj_000001.png"])
    m = read_ply(tmp_path / "m.ply")
    assert np.array_equal(m["texture"], tex)
    assert np.array_equal(m["face_uv"], uv[F2])


@pytest.mark.parametrize("fmt", ["binary_little_endian", "ascii"])
def test_ply_textured_per_face_texcoord_hope_style(tmp_path, fmt):
    """Per-face `texcoord` lists (6 floats per triangle) and s / t names are read as well."""
    tex = _texture_png(tmp_path / "t.png")
    tc = [[0.0, 0.0, 1.0, 0.0, 0.0, 1.0], [0.5, 0.5, 0.25, 0.75, 1.0, 1.0]]
    _write_ply(tmp_path / "m.ply", fmt, [("x", "float"), ("y", "float"), ("z", "float")], [tuple(v.tolist()) for v in V3],
               [("vertex_indices", "uchar", "int"), ("texcoord", "uchar", "float")],
               [[F2[i].tolist(), tc[i]] for i in range(2)], comments=["TextureFile t.png"])
    m = read_ply(tmp_path / "m.ply")
    assert np.array_equal(m["face_uv"], np.float32(tc).reshape(2, 3, 2)) and np.array_equal(m["texture"], tex)
    _write_ply(tmp_path / "st.ply", fmt, [("x", "float"), ("y", "float"), ("z", "float"), ("s", "float"), ("t", "float")],
               [tuple(v.tolist()) + (0.125, 0.5) for v in V3], [("vertex_indices", "uchar", "int")],
               [[f.tolist()] for f in F2], comments=["TextureFile t.png"])
    assert np.array_equal(read_ply(tmp_path / "st.ply")["face_uv"], np.tile(np.float32([0.125, 0.5]), (2, 3, 1)))


def test_malformed_ply_files_raise(tmp_path):
    vp = [("x", "float"), ("y", "float"), ("z", "float")]
    good = lambda fmt="binary_little_endian", faces=None, **kw: _write_ply(
        tmp_path / "m.ply", fmt, vp, [tuple(v.tolist()) for v in V3], kw.get("fprops", [("vertex_indices", "uchar", "int")]),
        faces if faces is not None else [[f.tolist()] for f in F2], **{k: v for k, v in kw.items() if k != "fprops"})
    (tmp_path / "m.ply").write_bytes(b"plx\nformat ascii 1.0\nend_header\n")
    with pytest.raises(PlyError, match="magic"):
        read_ply(tmp_path / "m.ply")
    (tmp_path / "m.ply").write_bytes(b"ply\nformat binary_big_endian 1.0\nelement vertex 0\nend_header\n")
    with pytest.raises(PlyError, match="unsupported PLY format"):
        read_ply(tmp_path / "m.ply")
    (tmp_path / "m.ply").write_bytes(b"ply\nformat ascii 1.0\nelement vertex 1\nproperty float x\n")
    with pytest.raises(PlyError, match="end_header"):
        read_ply(tmp_path / "m.ply")
    good()
    data = (tmp_path / "m.ply").read_bytes()
    (tmp_path / "m.ply").write_bytes(data[:-5])
    with pytest.raises(PlyError, match="truncated"):
        read_ply(tmp_path / "m.ply")
    for fmt in ("binary_little_endian", "ascii"):
        good(fmt, faces=[[[0, 1, 2, 3]]])                                         # a quad
        with pytest.raises(PlyError, match="triangle"):
            read_ply(tmp_path / "m.ply")
        for bad in ([0, 1, 4], [0, -1, 2]):
            good(fmt, faces=[[bad]])
            with pytest.raises(PlyError, match="outside"):
                read_ply(tmp_path / "m.ply")
    good(comments=["TextureFile missing.png"])
    with pytest.raises(PlyError, match="not found"):
        read_ply(tmp_path / "m.ply")
    (tmp_path / "m.ply").write_bytes(b"ply\nformat ascii 1.0\nelement vertex 1\nproperty float x\nproperty float y\n"
                                     b"property float z\nend_header\n0 0 0\n")
    with pytest.raises(PlyError, match="face element"):
        read_ply(tmp_path / "m.ply")


def test_meshes_given_as_arrays_are_validated_before_upload():
    with pytest.raises(ValueError, match="outside"):
        _device_mesh(dict(vertices=V3, faces=np.array([[0, 1, 4]])), "cpu")


# ------------------------------------------------------------------------------------------------ oracle, analytic
K512 = np.array([[512, 0, 0], [0, 512, 0], [0, 0, 1]], np.float32)


def _quad(u0, v0, side, z, flip=False):
    """Camera-frame square whose projection under K512 is [u0, u0 + side] x [v0, v0 + side] px."""
    s = np.float32(z / 512)
    c = np.array([[u0, v0], [u0 + side, v0], [u0 + side, v0 + side], [u0, v0 + side]], np.float32) * s
    V = np.concatenate([c, np.full((4, 1), z, np.float32)], 1)
    Fc = np.array([[0, 1, 2], [0, 2, 3]]) if not flip else np.array([[0, 2, 1], [0, 3, 2]])
    return V, Fc


@pytest.mark.parametrize("flip", [False, True])
def test_axis_aligned_quad_covers_exactly_the_expected_samples(flip):
    """An 8 x 8 px square at z = 1024 whose left / top edges pass exactly through samples (top-left rule: included)
    and whose right / bottom edges too (excluded).  Its doubled area is 2^22 in 1/256 px units, so every barycentric
    weight is exact: depth is exactly 1024 and a constant 0.5 albedo stays exactly 0.5."""
    H, W = 24, 32
    u0, v0 = 10.125, 5.375
    V, Fc = _quad(u0, v0, 8.0, 1024.0, flip)
    col = np.full((4, 3), 0.5, np.float32)
    out = rp.render(V, Fc, np.eye(4), K512, H, W, 100.0, vertex_color=col)
    sx = np.arange(W)[None, :, None] + rp.SAMPLE_DX[None, None, :] / 256
    sy = np.arange(H)[:, None, None] + rp.SAMPLE_DY[None, None, :] / 256
    want = (sx >= u0) & (sx < u0 + 8) & (sy >= v0) & (sy < v0 + 8)
    got = out["keys"] != rp.EMPTY
    assert np.array_equal(got, want)
    assert ((sx == u0) & want).any() and ((sy == v0) & want).any()     # samples on the included edges exist
    z = (out["keys"][got] >> np.uint64(32)).astype(np.uint32).view(np.float32)
    assert np.all(z == 1024.0)
    n = want.sum(-1)
    assert np.array_equal(out["depth"], np.where(n > 0, 1024.0, 0.0).astype(np.float32))
    expect = (np.rint(np.float32(0.5) * n / 4 * 255) / np.float32(255)).astype(np.float32)
    assert np.array_equal(out["rgba"][:3], np.broadcast_to(expect, (3, H, W)))
    assert np.array_equal(out["rgba"][3], (n > 0).astype(np.float32))
    ys, xs = np.nonzero(n)
    assert out["box"].tolist() == [xs.min(), ys.min(), xs.max() + 1, ys.max() + 1] == [10, 5, 19, 14]


def test_tessellated_plane_is_watertight():
    """A jittered grid of triangles with random diagonals, windings and vertex depths: every sample inside the
    outline is owned by exactly one face, every sample outside by none."""
    g = np.random.default_rng(3)
    n, x0, x1, y0, y1 = 9, 3.125, 37.125, 2.375, 27.375
    gx, gy = np.meshgrid(np.linspace(x0, x1, n + 1), np.linspace(y0, y1, n + 1))
    inner = (slice(1, -1), slice(1, -1))
    gx[inner] += g.uniform(-0.7, 0.7, gx[inner].shape)          # a fifth of the spacing: no folds
    gy[inner] += g.uniform(-0.5, 0.5, gy[inner].shape)
    z = np.full(gx.shape, 1000.0)
    z[inner] = g.uniform(800, 1200, z[inner].shape)
    V = np.stack([gx * z / 1000, gy * z / 1000, z], -1).reshape(-1, 3).astype(np.float32)
    faces = []
    for i in range(n):
        for j in range(n):
            a, b, c, d = i * (n + 1) + j, i * (n + 1) + j + 1, (i + 1) * (n + 1) + j + 1, (i + 1) * (n + 1) + j
            tris = [[a, b, c], [a, c, d]] if g.random() < 0.5 else [[a, b, d], [b, c, d]]
            faces += [t[::-1] if g.random() < 0.5 else t for t in tris]
    faces = np.array(faces)
    K = np.array([[1000, 0, 0], [0, 1000, 0], [0, 0, 1]], np.float32)
    H, W = 32, 42
    t = rp._setup(V, faces, np.eye(4), K, 100.0)
    assert t["valid"].all()
    py, px, s = [a.ravel() for a in np.meshgrid(np.arange(H), np.arange(W), np.arange(4), indexing="ij")]
    sx, sy = px * 256 + rp.SAMPLE_DX[s], py * 256 + rp.SAMPLE_DY[s]
    count = np.zeros(len(sx), np.int64)
    for f in range(len(faces)):
        count += rp._weights(t, np.full(len(sx), f), sx, sy)[1]
    inside = (sx >= x0 * 256) & (sx < x1 * 256) & (sy >= y0 * 256) & (sy < y1 * 256)
    assert np.array_equal(count, inside.astype(np.int64))
    assert (sx == x0 * 256).any() and (sy == y0 * 256).any()
    keys = rp.rasterize(V, faces, np.eye(4), K, H, W, 100.0)[0].ravel()
    assert np.array_equal(keys != rp.EMPTY, inside)


def test_coplanar_duplicate_faces_resolve_to_the_lowest_id():
    """Exact depth ties are broken by face id whatever the winding or the order in the file."""
    V, Fc = _quad(4.0, 4.0, 8.0, 1000.0)
    far, _ = _quad(2.0, 2.0, 12.0, 2000.0)
    V = np.concatenate([V, far])
    faces = np.array([[4, 5, 6], Fc[0][::-1], Fc[0], Fc[1], [4, 6, 7], Fc[1][::-1]])
    keys = rp.rasterize(V, faces, np.eye(4), K512, 20, 20, 100.0)[0]
    ids = (keys & np.uint64(0xFFFFFFFF))[keys != rp.EMPTY]
    assert set(ids.tolist()) == {0, 1, 3, 4}                 # far quad around the edge; 1 beats 2, 3 beats 5


def test_near_plane_drops_the_whole_triangle_and_an_empty_view_has_the_full_box():
    V, Fc = _quad(4.0, 4.0, 8.0, 1000.0)
    V[1, 2] = 100.0                                           # a vertex of face 0 only, on the near plane
    keys = rp.rasterize(V, Fc, np.eye(4), K512, 20, 20, 100.0)[0]
    alone = rp.rasterize(V, Fc[1:], np.eye(4), K512, 20, 20, 100.0)[0]
    assert np.array_equal(keys != rp.EMPTY, alone != rp.EMPTY) and (keys != rp.EMPTY).sum() == 128   # half of 8 x 8 px, 4 samples each
    assert np.all((keys[keys != rp.EMPTY] & np.uint64(0xFFFFFFFF)) == 1)
    out = rp.render(V[:0], Fc[:0], np.eye(4), K512, 20, 30, 100.0)
    assert out["box"].tolist() == [0, 0, 30, 20] and not out["rgba"].any() and not out["depth"].any()


def test_render_entry_points_reject_bad_arguments_without_a_gpu():
    """gp_render_query_sizes sizes the key buffer (8 B x 4 samples per pixel); gp_render_templates checks its
    arguments before it touches a device."""
    import ctypes as C

    from gigapose_b200 import _lib, build
    build.build()
    lib = _lib.load()
    ws = C.c_size_t()
    assert lib.gp_render_query_sizes(3, 480, 640, C.byref(ws)) == 0 and ws.value == 3 * 480 * 640 * 4 * 8
    assert lib.gp_render_query_sizes(3, 0, 640, C.byref(ws)) == -1 and b"image size" in lib.gp_last_error()
    assert lib.gp_render_query_sizes(-1, 480, 640, C.byref(ws)) == -1
    assert lib.gp_render_query_sizes(1, 480, 640, None) == -1
    fake = 1 << 20                                   # never dereferenced: every call below fails validation first

    def call(**kw):
        a = dict(n=2, H=48, W=64, nv=4, v=fake, nf=2, f=fake, vc=None, uv=None, tex=None, th=0, tw=0, cc=None, poses=fake,
                 K=fake, z_near=100.0, ws=fake, rgba=fake, depth=None, boxes=fake)
        a.update(kw)
        rc = lib.gp_render_templates(*a.values(), None)
        return rc, lib.gp_last_error()
    for kw, word in [(dict(n=70000), b"n_views"), (dict(W=9000), b"image size"), (dict(nf=-1), b"negative"),
                     (dict(z_near=0.0), b"z_near"), (dict(z_near=float("inf")), b"z_near"), (dict(poses=None), b"null"),
                     (dict(ws=None), b"null"), (dict(boxes=None), b"null"), (dict(f=None), b"mesh"),
                     (dict(vc=fake, tex=fake, uv=fake, th=2, tw=2), b"not both"), (dict(tex=fake, th=2, tw=2), b"face_uv"),
                     (dict(tex=fake, uv=fake, th=0, tw=2), b"tex_h"), (dict(uv=fake), b"face_uv without texture")]:
        rc, msg = call(**kw)
        assert rc == -1 and word in msg, (kw, rc, msg)
