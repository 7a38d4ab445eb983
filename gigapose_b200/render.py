"""Template renders from CAD meshes on the GPU (row f5): `read_ply` loads a BOP model file, `render_templates` renders
its template views with `gp_render_templates` (csrc/render.cu, whose header comment states the full contract).  The
reference renders with Panda3D at 640 x 480 under one white ambient light (src/custom_megapose/call_panda3d.py:45-59),
so a template is the surface albedo with a 4x multisampled edge, a mask and a bounding box."""
from __future__ import annotations

import ctypes as C
import os
import re

import numpy as np
import torch

from . import _lib
from ._lib import check

# the template camera of the reference (call_panda3d.py:45-47): the LINEMOD focal lengths with the principal point at
# the image centre of 640 x 480
TEMPLATE_K = ((572.4114, 0.0, 320.0), (0.0, 573.57043, 240.0), (0.0, 0.0, 1.0))
TEMPLATE_SIZE = (480, 640)
WORKSPACE_BYTES = 512 << 20        # key buffer per chunk of views: 9.8 MB per 640 x 480 view -> 54 views

_PLY_TYPES = {"char": "i1", "int8": "i1", "uchar": "u1", "uint8": "u1", "short": "i2", "int16": "i2", "ushort": "u2",
              "uint16": "u2", "int": "i4", "int32": "i4", "uint": "u4", "uint32": "u4", "float": "f4", "float32": "f4",
              "double": "f8", "float64": "f8"}


class PlyError(ValueError):
    pass


def _parse_header(f):
    if f.readline().strip() != b"ply":
        raise PlyError("not a PLY file (no 'ply' magic)")
    fmt, texture, elements = None, None, []
    while True:
        line = f.readline()
        if not line:
            raise PlyError("header has no end_header")
        words = line.decode("ascii", "replace").split()
        if not words:
            continue
        if words[0] == "end_header":
            break
        if words[0] == "format":
            if len(words) < 2 or words[1] not in ("ascii", "binary_little_endian"):
                raise PlyError(f"unsupported PLY format {' '.join(words[1:])!r} (ascii and binary_little_endian are read)")
            fmt = words[1]
        elif words[0] == "comment" and len(words) >= 3 and words[1] == "TextureFile":
            texture = line.decode("ascii", "replace").split(None, 2)[2].strip()
        elif words[0] == "element":
            if len(words) != 3 or not re.fullmatch(r"\d+", words[2]):
                raise PlyError(f"bad element line {line!r}")
            elements.append((words[1], int(words[2]), []))
        elif words[0] == "property":
            if not elements:
                raise PlyError("property before any element")
            if words[1] == "list":
                if len(words) != 5 or words[2] not in _PLY_TYPES or words[3] not in _PLY_TYPES:
                    raise PlyError(f"bad list property {line!r}")
                elements[-1][2].append((words[4], words[2], words[3]))
            else:
                if len(words) != 3 or words[1] not in _PLY_TYPES:
                    raise PlyError(f"bad property {line!r}")
                elements[-1][2].append((words[2], None, words[1]))
    if fmt is None:
        raise PlyError("header has no format line")
    return fmt, texture, elements


def _list_len(name):
    return 3 if name in ("vertex_indices", "vertex_index") else 6 if name == "texcoord" else None


def _row_dtype(props, ascii_mode):
    """Structured dtype of one element row; list properties must have the triangle length (3 indices, 6 texcoords)."""
    fields = []
    for name, count_t, item_t in props:
        if count_t is None:
            fields.append((name, "f8" if ascii_mode else "<" + _PLY_TYPES[item_t]))
        else:
            n = _list_len(name)
            if n is None:
                raise PlyError(f"unsupported list property {name!r}")
            fields.append((name + "#n", "f8" if ascii_mode else "<" + _PLY_TYPES[count_t]))
            fields.append((name, ("f8" if ascii_mode else "<" + _PLY_TYPES[item_t], (n,))))
    return np.dtype(fields)


def read_ply(path):
    """Reads a triangle mesh in the PLY variants of the BOP models (ascii or binary_little_endian):
    vertex x y z, optional red green blue [alpha] (uchar 0..255 or float 0..1), optional texture_u / texture_v (or s / t);
    face vertex_indices and an optional per-face texcoord list; `comment TextureFile <png>` relative to the file.
    -> dict(vertices f32 [V,3], faces i32 [F,3], vertex_color f32 [V,3] or None, face_uv f32 [F,3,2] or None,
    texture f32 [Ht,Wt,3] in [0,1] (row 0 on top) or None).  Raises PlyError on anything malformed, including a face
    index outside [0, V)."""
    with open(path, "rb") as f:
        fmt, texture_name, elements = _parse_header(f)
        body = f.read()
    ascii_mode = fmt == "ascii"
    tokens = np.array(body.split(), dtype=np.float64) if ascii_mode else None
    data, off = {}, 0
    for name, count, props in elements:
        dt = _row_dtype(props, ascii_mode)
        if ascii_mode:
            width = dt.itemsize // 8
            if off + count * width > len(tokens):
                raise PlyError(f"element {name!r} truncated")
            rows = tokens[off:off + count * width].copy().view(dt)
            off += count * width
        else:
            if off + count * dt.itemsize > len(body):
                raise PlyError(f"element {name!r} truncated")
            rows = np.frombuffer(body, dtype=dt, count=count, offset=off)
            off += count * dt.itemsize
        for pname, count_t, _ in props:
            if count_t is not None and count and np.any(rows[pname + "#n"] != _list_len(pname)):
                raise PlyError(f"element {name!r}: every {pname} list must have {_list_len(pname)} entries "
                               "(triangle meshes only)")
        data[name] = rows
    if ascii_mode and off != len(tokens):
        raise PlyError(f"{len(tokens) - off} values after the last element")
    if "vertex" not in data or "face" not in data:
        raise PlyError("need a vertex and a face element")
    vx = data["vertex"]
    names = vx.dtype.names
    if not all(c in names for c in "xyz"):
        raise PlyError("vertex element lacks x y z")
    V = np.stack([vx["x"], vx["y"], vx["z"]], 1).astype(np.float32)
    if not np.isfinite(V).all():
        raise PlyError("non-finite vertex coordinates")
    fc = data["face"]
    idx_name = "vertex_indices" if "vertex_indices" in fc.dtype.names else "vertex_index" if "vertex_index" in fc.dtype.names else None
    if idx_name is None:
        raise PlyError("face element lacks vertex_indices")
    faces = np.asarray(fc[idx_name])
    if faces.size and (faces.min() < 0 or faces.max() >= len(V) or np.any(faces != np.round(faces))):
        raise PlyError(f"face indices outside [0, {len(V)})")
    faces = faces.astype(np.int32).reshape(-1, 3)
    color = None
    if all(c in names for c in ("red", "green", "blue")):
        ply_types = {n: t for n, _, t in next(e[2] for e in elements if e[0] == "vertex")}
        color = np.stack([vx["red"], vx["green"], vx["blue"]], 1).astype(np.float32)
        if _PLY_TYPES[ply_types["red"]][0] in "iu":            # 8-bit colours; float colours are already in [0, 1]
            color = color / np.float32(255)
    uv = None
    for un, vn in (("texture_u", "texture_v"), ("s", "t")):
        if un in names and vn in names:
            uv = np.stack([vx[un], vx[vn]], 1).astype(np.float32)[faces.astype(np.int64)]       # per vertex -> per corner
    if "texcoord" in fc.dtype.names:
        uv = np.asarray(fc["texcoord"], np.float32).reshape(-1, 3, 2)
    texture = None
    if texture_name is not None:
        from PIL import Image
        tex_path = os.path.join(os.path.dirname(os.path.abspath(path)), texture_name)
        if not os.path.exists(tex_path):
            raise PlyError(f"texture file {texture_name!r} not found next to {path}")
        with Image.open(tex_path) as im:
            texture = np.asarray(im.convert("RGB"), dtype=np.float32) / np.float32(255)
        if uv is None:
            raise PlyError("a TextureFile without texture coordinates")
    return dict(vertices=V, faces=faces, vertex_color=color, face_uv=uv if texture is not None else None, texture=texture)


def _device_mesh(mesh, device):
    """Mesh dict -> contiguous device tensors; a texture takes precedence over vertex colours."""
    def t(x, dtype):
        return None if x is None else torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x).to(
            device=device, dtype=dtype).contiguous()
    V = t(mesh["vertices"], torch.float32).reshape(-1, 3)
    Fc = t(mesh["faces"], torch.int64).reshape(-1, 3)
    if Fc.numel() and (int(Fc.min()) < 0 or int(Fc.max()) >= V.shape[0]):
        raise ValueError(f"face indices outside [0, {V.shape[0]})")
    out = dict(vertices=V, faces=Fc.to(torch.int32), vertex_color=None, face_uv=None, texture=None,
               constant_color=t(mesh.get("constant_color"), torch.float32))
    if mesh.get("texture") is not None:
        out["texture"] = t(mesh["texture"], torch.float32)
        out["face_uv"] = t(mesh["face_uv"], torch.float32).reshape(-1, 3, 2)
        assert out["texture"].dim() == 3 and out["texture"].shape[2] == 3, "texture must be [Ht,Wt,3]"
        assert out["face_uv"].shape[0] == Fc.shape[0], "face_uv must be [F,3,2]"
    elif mesh.get("vertex_color") is not None:
        out["vertex_color"] = t(mesh["vertex_color"], torch.float32).reshape(-1, 3)
        assert out["vertex_color"].shape[0] == V.shape[0], "vertex_color must be [V,3]"
    return out


def _ptr(x):
    return x.data_ptr() if x is not None else None


def render_chunk(dm, poses, K, H, W, z_near, workspace, rgba, depth, boxes):
    """One gp_render_templates call on device tensors (dm from _device_mesh); enqueued on the current stream."""
    lib = _lib.load()
    tex = dm["texture"]
    check(lib.gp_render_templates(poses.shape[0], H, W, dm["vertices"].shape[0], _ptr(dm["vertices"]), dm["faces"].shape[0],
                                  _ptr(dm["faces"]), _ptr(dm["vertex_color"]), _ptr(dm["face_uv"]), _ptr(tex),
                                  tex.shape[0] if tex is not None else 0, tex.shape[1] if tex is not None else 0,
                                  _ptr(dm["constant_color"]), poses.data_ptr(), K.data_ptr(), float(z_near),
                                  workspace.data_ptr(), rgba.data_ptr(), _ptr(depth), boxes.data_ptr(),
                                  torch.cuda.current_stream(poses.device).cuda_stream))


@torch.no_grad()
def render_templates(mesh, poses, K=TEMPLATE_K, size=TEMPLATE_SIZE, z_near=100.0, device=None):
    """Renders the views `poses` [n,4,4] (object -> camera, in the mesh's length unit; mm for BOP) of `mesh` (a
    `read_ply` dict or a path) with intrinsics K [3,3] at size (H, W) -> dict(rgba [n,4,H,W] f32, depth [n,H,W] f32,
    boxes [n,4] i64 xyxy, exclusive max) on the GPU.  z_near is in the mesh unit (Panda3D's 0.1 m = 100 mm).  A mesh
    with neither texture nor vertex colours is drawn in mesh["constant_color"] (RGB in [0, 1]), white when absent."""
    if isinstance(mesh, (str, os.PathLike)):
        mesh = read_ply(mesh)
    device = torch.device(device if device is not None else
                          poses.device if torch.is_tensor(poses) and poses.is_cuda else torch.cuda.current_device())
    if device.type != "cuda":
        raise _lib.GigaPoseNativeError("render_templates runs on CUDA devices only (no CPU fallback)")
    H, W = int(size[0]), int(size[1])
    dm = _device_mesh(mesh, device)
    poses = torch.as_tensor(poses, dtype=torch.float32).to(device).reshape(-1, 4, 4).contiguous()
    K = torch.as_tensor(K, dtype=torch.float32).to(device).reshape(3, 3).contiguous()
    n = poses.shape[0]
    per_view = C.c_size_t()
    check(_lib.load().gp_render_query_sizes(1, H, W, C.byref(per_view)))
    per_view = per_view.value
    chunk = max(1, min(n, WORKSPACE_BYTES // per_view))
    rgba = torch.empty(n, 4, H, W, device=device)
    depth = torch.empty(n, H, W, device=device)
    boxes = torch.empty(n, 4, dtype=torch.int64, device=device)
    with torch.cuda.device(device):
        workspace = torch.empty(chunk * per_view, dtype=torch.uint8, device=device)
        for v0 in range(0, n, chunk):
            v1 = min(n, v0 + chunk)
            render_chunk(dm, poses[v0:v1], K, H, W, z_near, workspace, rgba[v0:v1], depth[v0:v1], boxes[v0:v1])
    return dict(rgba=rgba, depth=depth, boxes=boxes)
