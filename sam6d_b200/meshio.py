"""CAD input of the CLIs: PLY reading and area-weighted surface sampling -- what the reference gets from
`trimesh.load_mesh(cad_path).sample(n)` (PEM/run_inference_custom.py:182-183; trimesh is not a dependency here).
Host-side numpy; ASCII and binary_little_endian PLY with `vertex` (x, y, z first) and `face` (vertex_indices list) elements.
load_ply_mesh() also reads per-vertex texture coordinates and the `comment TextureFile` image of BOP's textured models."""
import os
from dataclasses import dataclass
from typing import Optional

import numpy as np

_PLY_TYPES = {"char": "i1", "uchar": "u1", "short": "i2", "ushort": "u2", "int": "i4", "uint": "u4", "float": "f4", "double": "f8",
              "int8": "i1", "uint8": "u1", "int16": "i2", "uint16": "u2", "int32": "i4", "uint32": "u4", "float32": "f4", "float64": "f8"}


def _read_ply(path):
    """-> (vertex columns {name: array}, faces (F,3) int64 or empty, header comments)"""
    with open(path, "rb") as fh:
        fmt, elements, comments = None, [], []
        while True:
            line = fh.readline()
            if not line:
                raise ValueError("PLY header not terminated")
            tok = line.decode("ascii", "replace").strip().split()
            if not tok:
                continue
            if tok[0] == "format":
                fmt = tok[1]
            elif tok[0] == "comment":
                comments.append(tok[1:])
            elif tok[0] == "element":
                elements.append(dict(name=tok[1], count=int(tok[2]), props=[]))
            elif tok[0] == "property":
                elements[-1]["props"].append(tok[1:])
            elif tok[0] == "end_header":
                break
        vcols, faces = None, np.zeros((0, 3), np.int64)
        for el in elements:
            names = [p[-1] for p in el["props"]]
            if el["name"] == "vertex":
                if fmt == "ascii":
                    data = np.loadtxt(fh, max_rows=el["count"], dtype=np.float64, ndmin=2)
                    cols = {n: data[:, i] for i, n in enumerate(names)}
                else:
                    dt = np.dtype([(p[-1], ("<" if fmt == "binary_little_endian" else ">") + _PLY_TYPES[p[0]]) for p in el["props"]])
                    rec = np.frombuffer(fh.read(dt.itemsize * el["count"]), dtype=dt)
                    cols = {n: rec[n] for n in names}
                vcols = cols
            elif el["name"] == "face":
                if fmt == "ascii":
                    rows = [fh.readline().split() for _ in range(el["count"])]
                    tris = []
                    for r in rows:
                        n = int(r[0])
                        idx = [int(v) for v in r[1:1 + n]]
                        tris += [[idx[0], idx[k], idx[k + 1]] for k in range(1, n - 1)]       # fan triangulation
                    faces = np.asarray(tris, dtype=np.int64).reshape(-1, 3)
                else:
                    end = "<" if fmt == "binary_little_endian" else ">"
                    ct, it = _PLY_TYPES[el["props"][0][1]], _PLY_TYPES[el["props"][0][2]]
                    tris = []
                    for _ in range(el["count"]):
                        n = int(np.frombuffer(fh.read(np.dtype(ct).itemsize), dtype=end + ct)[0])
                        idx = np.frombuffer(fh.read(np.dtype(it).itemsize * n), dtype=end + it).astype(np.int64)
                        tris += [[idx[0], idx[k], idx[k + 1]] for k in range(1, n - 1)]
                    faces = np.asarray(tris, dtype=np.int64).reshape(-1, 3)
            else:
                if fmt == "ascii":
                    for _ in range(el["count"]):
                        fh.readline()
                else:
                    raise ValueError(f"binary PLY element {el['name']} is not supported")
    if vcols is None:
        raise ValueError("PLY without a vertex element")
    return vcols, faces, comments


def _colors(cols):
    if all(c in cols for c in ("red", "green", "blue")):
        return np.stack([cols["red"], cols["green"], cols["blue"]], axis=1).astype(np.uint8)
    return None


def load_ply(path):
    """-> (vertices (V,3) float32, faces (F,3) int64 or empty, vertex colours (V,3) uint8 or None)"""
    cols, faces, _ = _read_ply(path)
    return np.stack([cols["x"], cols["y"], cols["z"]], axis=1).astype(np.float32), faces, _colors(cols)


@dataclass
class Mesh:
    """A triangle mesh with its appearance: numpy arrays from load_ply_mesh, CUDA tensors after sam6d_b200.render.upload.
    vertices (V,3) float32 in model units, faces (F,3) int, colors (V,3) uint8, uv (V,2) float32 (v = 0 is the bottom row
    of the texture), texture (Ht,Wt,3) uint8 RGB; any of the last three may be None."""
    vertices: object
    faces: object
    colors: Optional[object] = None
    uv: Optional[object] = None
    texture: Optional[object] = None
    texture_file: Optional[str] = None


def load_ply_mesh(path, read_texture: bool = True) -> Mesh:
    """load_ply plus texture coordinates (vertex properties texture_u/texture_v or s/t) and the image named by
    `comment TextureFile <png>` (relative to the PLY's folder), as in BOP's YCB-V models"""
    cols, faces, comments = _read_ply(path)
    verts = np.stack([cols["x"], cols["y"], cols["z"]], axis=1).astype(np.float32)
    uv = None
    for u, v in (("texture_u", "texture_v"), ("s", "t")):
        if u in cols and v in cols:
            uv = np.stack([cols[u], cols[v]], axis=1).astype(np.float32)
            break
    tex_file = next((" ".join(c[1:]) for c in comments if len(c) > 1 and c[0] == "TextureFile"), None)
    if tex_file is not None:
        tex_file = os.path.join(os.path.dirname(os.path.abspath(path)), tex_file)
    texture = None
    if read_texture and uv is not None and tex_file is not None:
        import cv2
        img = cv2.imread(tex_file, cv2.IMREAD_COLOR)
        if img is None:
            raise FileNotFoundError(f"texture {tex_file} named by {path} cannot be read")
        texture = np.ascontiguousarray(img[:, :, ::-1])
    return Mesh(verts, faces, _colors(cols), uv, texture, tex_file)


def sample_surface(verts, faces, n, rng=None, return_normals: bool = False):
    """area-weighted random points on the triangles (trimesh.sample.sample_surface semantics); vertices when there are no faces.
    rng: numpy's global RNG (default), a RandomState or a Generator.  return_normals: also the unit normal of each point's
    face, (b - a) x (c - a) normalised (float32), from the same draws; a mesh without faces has none (ValueError)."""
    rng = rng if rng is not None else np.random
    uniform = rng.random if isinstance(rng, np.random.Generator) else rng.random_sample
    if len(faces) == 0:
        if return_normals:
            raise ValueError("sample_surface: a mesh without faces has no normals")
        return verts[rng.choice(len(verts), n, replace=len(verts) < n)].astype(np.float32)
    a, b, c = verts[faces[:, 0]].astype(np.float64), verts[faces[:, 1]].astype(np.float64), verts[faces[:, 2]].astype(np.float64)
    cross = np.cross(b - a, c - a)
    area = 0.5 * np.linalg.norm(cross, axis=1)
    f = np.searchsorted(np.cumsum(area), uniform(n) * area.sum())
    f = np.minimum(f, len(faces) - 1)
    u = uniform((n, 2))
    flip = u.sum(axis=1) > 1.0
    u[flip] = 1.0 - u[flip]
    pts = (a[f] + u[:, :1] * (b[f] - a[f]) + u[:, 1:] * (c[f] - a[f])).astype(np.float32)
    if not return_normals:
        return pts
    nrm = cross[f] / np.maximum(2.0 * area[f], np.finfo(np.float64).tiny)[:, None]
    return pts, nrm.astype(np.float32)


def save_ply(path, mesh: Mesh) -> None:
    """write a numpy Mesh as binary little-endian PLY: vertex x, y, z float (+ red, green, blue uchar when it has colours) and
    face `list uchar int vertex_indices`, the layout BOP's models use.  load_ply_mesh reads it back exactly."""
    v = np.asarray(mesh.vertices)
    f = np.asarray(mesh.faces)
    if v.ndim != 2 or v.shape[1] != 3 or f.ndim != 2 or f.shape[1] != 3:
        raise ValueError(f"save_ply: vertices (V,3) and faces (F,3), got {v.shape} and {f.shape}")
    if len(f) and (f.min() < 0 or f.max() >= len(v) or f.max() > np.iinfo(np.int32).max):
        raise ValueError(f"save_ply: face indices outside [0, {len(v)})")
    props = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")]
    if mesh.colors is not None:
        c = np.asarray(mesh.colors)
        if c.shape != v.shape or c.dtype != np.uint8:
            raise ValueError(f"save_ply: colors (V,3) uint8, got {c.shape} {c.dtype}")
        props += [("red", "u1"), ("green", "u1"), ("blue", "u1")]
    vrec = np.empty(len(v), dtype=np.dtype(props))
    for k, name in enumerate("xyz"):
        vrec[name] = v[:, k]
    if mesh.colors is not None:
        for k, name in enumerate(("red", "green", "blue")):
            vrec[name] = c[:, k]
    frec = np.empty(len(f), dtype=np.dtype([("n", "u1"), ("i", "<i4", (3,))]))
    frec["n"] = 3
    frec["i"] = f
    head = ["ply", "format binary_little_endian 1.0", f"element vertex {len(v)}"]
    head += [f"property {'float' if t == '<f4' else 'uchar'} {n}" for n, t in props]
    head += [f"element face {len(f)}", "property list uchar int vertex_indices", "end_header"]
    with open(path, "wb") as fh:
        fh.write(("\n".join(head) + "\n").encode("ascii"))
        fh.write(vrec.tobytes())
        fh.write(frec.tobytes())
