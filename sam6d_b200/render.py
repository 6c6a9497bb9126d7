"""CAD template rendering on the GPU: the stage SAM-6D/Render/render_{custom,bop}_templates.py runs in BlenderProc.

    level0_template_poses()  the 42 object -> camera poses of the CNOS level-0 view set (ISM/utils/poses/create_template_poses.py)
    template_K(size)         the template camera: f = 560, c = 256 at 512 x 512, scaled with the size
    render(meshes, poses, K, height, width)  every view of every mesh in one batched rasteriser call (csrc/render.cu)

The rasteriser's visibility is exact (fixed-point edge functions, top-left rule, one 64-bit atomicMin per pixel on depth and
face id), so oracle/render_oracle.py reproduces it bit for bit.  Shading is a documented stand-in for Cycles: albedo (vertex
colour, bilinear texture or base colour) x (ambient + (1 - ambient) max(0, n.l)) with a point light at 2.5x the camera
position (render_custom_templates.py:68-72), no shadows, no BSDF."""
import math
from typing import Sequence

import numpy as np
import torch

from . import _lib
from .meshio import Mesh

# the (O*T*H*W) u64 visibility buffer of one rasteriser call stays within this many bytes; more objects are rendered in chunks
VIS_BUDGET_BYTES = 1 << 30
BIG_LIST_CAP = 1 << 20


def _icosphere_level0():
    """the 42 vertices of Blender's subdivision-2 icosphere: poles on +-z, the upper ring of the icosahedron at azimuths
    18 + 72 k degrees (az = atan2(x, y)), the lower ring 36 degrees further, plus the 30 normalised edge midpoints"""
    el = math.atan(0.5)
    pts = [(0.0, 0.0, 1.0), (0.0, 0.0, -1.0)]
    for k in range(5):
        for ring_el, az_deg in ((el, 18.0 + 72.0 * k), (-el, 54.0 + 72.0 * k)):
            az = math.radians(az_deg)
            pts.append((math.cos(ring_el) * math.sin(az), math.cos(ring_el) * math.cos(az), math.sin(ring_el)))
    v = np.asarray(pts, dtype=np.float64)
    d = np.linalg.norm(v[:, None] - v[None], axis=2)
    edge = d[d > 1e-9].min()
    mids = [v[i] + v[j] for i in range(12) for j in range(i + 1, 12) if d[i, j] < edge * 1.001]
    m = np.asarray(mids)
    m /= np.linalg.norm(m, axis=1, keepdims=True)
    out = np.concatenate([v, m])
    assert out.shape == (42, 3)
    return out


def _look_at(loc):
    """camera -> world of a camera at loc looking at the origin (create_template_poses.py:75-104): up hint (0,0,-1), (0,-1,0)
    at the poles; columns right, up, forward"""
    forward = -loc / np.linalg.norm(loc)
    tmp = np.array([0.0, 0.0, -1.0])
    if min(np.linalg.norm(loc - tmp), np.linalg.norm(loc + tmp)) < 1e-3:
        tmp = np.array([0.0, -1.0, 0.0])
    right = np.cross(tmp, forward)
    right /= np.linalg.norm(right)
    up = np.cross(forward, right)
    up /= np.linalg.norm(up)
    return np.stack([right, up, forward], axis=1)


def level0_template_poses(distance: float = 1.0) -> np.ndarray:
    """-> (42,4,4) float64 object -> camera poses (OpenCV camera: x right, y down, z forward), camera `distance` from the
    origin, ordered by elevation ascending, then azimuth ascending.  The reference's obj_poses_level0.npy holds the same
    rotations with distance 1000 (mm), in an order decided by float32 rounding inside Blender; pass that file to the
    template CLIs with --poses to render in its order."""
    pos = _icosphere_level0()
    el = np.arctan2(pos[:, 2], np.hypot(pos[:, 0], pos[:, 1]))
    az = np.arctan2(pos[:, 0], pos[:, 1])
    order = np.lexsort((np.round(az, 9), np.round(el, 9)))
    poses = np.zeros((42, 4, 4))
    for i, k in enumerate(order):
        R = _look_at(pos[k]).T                                       # world -> camera
        poses[i, :3, :3] = R
        poses[i, :3, 3] = -R @ (pos[k] * distance)
        poses[i, 3, 3] = 1.0
    return poses


VIEW_COUNTS = {0: 42, 1: 162, 2: 642}          # onboarding_config.level_templates -> views of the CNOS view set
POSE_DISTRIBUTIONS = ("all", "upper")


def _icosphere_points(level: int) -> np.ndarray:
    """camera directions of the level-`level` view set: the level-0 vertices (_icosphere_level0) refined `level` times by 1-to-4
    midpoint subdivision with re-normalisation, as Blender's icosphere of subdivision level + 2 -> (VIEW_COUNTS[level], 3)"""
    pts = _icosphere_level0()
    d = np.linalg.norm(pts[:12, None] - pts[None, :12], axis=2)
    edge = d[d > 1e-9].min()
    adj = d < edge * 1.001
    # the icosahedron's 20 faces, each cut into 4 with its three edge midpoints (rows 12.. of _icosphere_level0, in its order)
    mid = {}
    k = 12
    for i in range(12):
        for j in range(i + 1, 12):
            if adj[i, j]:
                mid[(i, j)] = mid[(j, i)] = k
                k += 1
    faces = []
    for a in range(12):
        for b in range(a + 1, 12):
            for c in range(b + 1, 12):
                if adj[a, b] and adj[b, c] and adj[a, c]:
                    ab, bc, ca = mid[(a, b)], mid[(b, c)], mid[(c, a)]
                    faces += [(a, ab, ca), (ab, b, bc), (ca, bc, c), (ab, bc, ca)]
    for _ in range(level):
        pts, faces = _subdivide(pts, faces)
    assert pts.shape == (VIEW_COUNTS[level], 3)
    return pts


def _subdivide(pts, faces):
    """one 1-to-4 split of every triangle; each edge's midpoint is added once, normalised onto the unit sphere"""
    pts = list(pts)
    mid = {}

    def m(i, j):
        key = (min(i, j), max(i, j))
        if key not in mid:
            v = pts[i] + pts[j]
            pts.append(v / np.linalg.norm(v))
            mid[key] = len(pts) - 1
        return mid[key]
    out = []
    for a, b, c in faces:
        ab, bc, ca = m(a, b), m(b, c), m(c, a)
        out += [(a, ab, ca), (ab, b, bc), (ca, bc, c), (ab, bc, ca)]
    return np.asarray(pts), out


def _poses_at(pos: np.ndarray, distance: float) -> np.ndarray:
    """unit camera positions -> (n,4,4) object -> camera poses, ordered by elevation ascending, then azimuth ascending"""
    el = np.arctan2(pos[:, 2], np.hypot(pos[:, 0], pos[:, 1]))
    az = np.arctan2(pos[:, 0], pos[:, 1])
    order = np.lexsort((np.round(az, 9), np.round(el, 9)))
    poses = np.zeros((len(pos), 4, 4))
    for i, k in enumerate(order):
        R = _look_at(pos[k]).T                                       # world -> camera
        poses[i, :3, :3] = R
        poses[i, :3, 3] = -R @ (pos[k] * distance)
        poses[i, 3, 3] = 1.0
    return poses


def camera_centres(poses: np.ndarray) -> np.ndarray:
    """(n,4,4) object -> camera poses -> (n,3) camera centres in the object frame, -R^T t"""
    return -np.einsum("tji,tj->ti", poses[:, :3, :3], poses[:, :3, 3])


def template_poses(level: int = 0, pose_distribution: str = "all", distance: float = 1.0) -> np.ndarray:
    """-> (T,4,4) float64 object -> camera poses of the CNOS view set onboarding_config.level_templates = level (0 / 1 / 2 =
    42 / 162 / 642 views, ISM/utils/poses/pose_utils.py:70-100) with the camera `distance` from the origin, ordered by
    elevation, then azimuth, ascending.  pose_distribution "upper" keeps the cameras with z >= 0, the equator included
    (26 / 91 / 341 views): an object resting on a table is never seen from below.  Level 0 "all" is level0_template_poses()."""
    if level not in VIEW_COUNTS:
        raise ValueError(f"level_templates must be one of {sorted(VIEW_COUNTS)}, got {level!r}")
    if pose_distribution not in POSE_DISTRIBUTIONS:
        raise ValueError(f"pose_distribution must be one of {POSE_DISTRIBUTIONS}, got {pose_distribution!r}")
    poses = level0_template_poses(distance) if level == 0 else _poses_at(_icosphere_points(level), distance)
    if pose_distribution == "upper":
        # equator cameras are sums of mirror-image pairs, so their z is 0 exactly; the margin only absorbs -R^T t's rounding
        poses = poses[camera_centres(poses)[:, 2] >= -1e-9 * max(distance, 1.0)]
    return poses


def template_view_set(level: int = 0, pose_distribution: str = "all", distance: float = 1.0):
    """the template directory's view layout -> (poses (N,4,4) float64, ism_index (T,) int64).  The 42 level-0 views come first,
    in level0_template_poses()'s order (so rgb_0..41, which the PEM reads, are always those views), then the views of
    template_poses(level, pose_distribution) that are not level-0 views, in that set's order.  ism_index lists, in the set's
    own order, where each of its T views sits among the N: the ISM scores against poses[ism_index]."""
    base = level0_template_poses(distance)
    chosen = template_poses(level, pose_distribution, distance)
    cb, cc = camera_centres(base), camera_centres(chosen)
    d = np.linalg.norm(cc[:, None] - cb[None], axis=2)
    tol = 1e-6 * max(distance, 1.0)
    in_base = d.min(axis=1) < tol
    extra = chosen[~in_base]
    index = np.where(in_base, d.argmin(axis=1), 0)
    index[~in_base] = len(base) + np.arange(len(extra))
    return np.concatenate([base, extra]), index.astype(np.int64)


def template_K(size: int = 512) -> np.ndarray:
    """the template camera: f = 560 px, principal point at the centre of a 512 x 512 image, scaled to size x size"""
    s = size / 512.0
    return np.array([[560.0 * s, 0.0, size / 2.0], [0.0, 560.0 * s, size / 2.0], [0.0, 0.0, 1.0]])


def upload(mesh: Mesh, device="cuda") -> Mesh:
    """numpy Mesh (meshio.load_ply_mesh) -> the same Mesh with CUDA tensors of the dtypes render() takes"""
    def t(a, dt):
        return None if a is None else torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(device)
    return Mesh(t(mesh.vertices, np.float32), t(mesh.faces, np.int32), t(mesh.colors, np.uint8), t(mesh.uv, np.float32),
                t(mesh.texture, np.uint8), mesh.texture_file)


def _check(t, dtype, name, shape_tail):
    if not isinstance(t, torch.Tensor) or not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor (CPU not supported)")
    if t.dtype != dtype:
        raise RuntimeError(f"{name} must be {dtype}, got {t.dtype}")
    if t.dim() != 1 + len(shape_tail) or tuple(t.shape[1:]) != tuple(shape_tail):
        raise RuntimeError(f"{name} must have shape (n, {', '.join(map(str, shape_tail))}), got {tuple(t.shape)}")


def render(meshes: Sequence[Mesh], poses: torch.Tensor, K, height: int, width: int, ambient: float = 0.3, base_color=0.8,
           znear: float = 1e-3):
    """Render T views of each of O meshes on the current stream.

    meshes   O Mesh records of CUDA tensors (upload()): vertices (V,3) f32, faces (F,3) i32, and optionally colors (V,3) u8 or
             uv (V,2) f32 + texture (Ht,Wt,3) u8; a texture wins over colours, a mesh with neither gets base_color
    poses    (O,T,4,4) f32 CUDA, object -> camera (OpenCV axes), translation in model units
    K        (3,3) pinhole intrinsics (host values); base_color: grey level, (3,) or (O,3) in [0, 1]
    -> dict of device tensors: rgb (O,T,H,W,3) u8, mask (O,T,H,W) u8 (255 = object), xyz (O,T,H,W,3) f16 object coordinates
       (0 off the mask), tri (O,T,H,W) i32 face index (-1 = empty), depth (O,T,H,W) f32 camera z (0 = empty), dropped (O,) i32
       triangle-view pairs skipped because a vertex lies at z <= znear or beyond the +-2^14 px guard band (no clipping)"""
    O = len(meshes)
    if O == 0:
        raise ValueError("render: no meshes")
    if not isinstance(poses, torch.Tensor) or not poses.is_cuda:
        raise RuntimeError("poses must be a CUDA tensor (CPU not supported)")
    if poses.dtype != torch.float32 or poses.dim() != 4 or poses.shape[0] != O or tuple(poses.shape[2:]) != (4, 4):
        raise RuntimeError(f"poses must be float32 (O={O}, T, 4, 4), got {poses.dtype} {tuple(poses.shape)}")
    poses = poses.contiguous()
    dev = poses.device
    T, H, W = poses.shape[1], int(height), int(width)
    K = np.asarray(K.cpu() if isinstance(K, torch.Tensor) else K, dtype=np.float64).reshape(3, 3)
    base = np.broadcast_to(np.asarray(base_color, dtype=np.float32), (O, 3)) if np.ndim(base_color) < 2 else np.asarray(base_color, np.float32)
    for i, m in enumerate(meshes):
        _check(m.vertices, torch.float32, f"meshes[{i}].vertices", (3,))
        _check(m.faces, torch.int32, f"meshes[{i}].faces", (3,))
        if m.vertices.shape[0] == 0 or m.faces.shape[0] == 0:
            raise ValueError(f"meshes[{i}] has no vertices or no faces")
        if m.colors is not None:
            _check(m.colors, torch.uint8, f"meshes[{i}].colors", (3,))
        if m.uv is not None and m.texture is not None:
            _check(m.uv, torch.float32, f"meshes[{i}].uv", (2,))
            if not m.texture.is_cuda or m.texture.dtype != torch.uint8 or m.texture.dim() != 3 or m.texture.shape[2] != 3:
                raise RuntimeError(f"meshes[{i}].texture must be a CUDA uint8 (Ht,Wt,3) tensor")
        for a in (m.colors, m.uv):
            if a is not None and a.shape[0] != m.vertices.shape[0]:
                raise ValueError(f"meshes[{i}]: per-vertex attributes must have one row per vertex")
        lo, hi = int(m.faces.min()), int(m.faces.max())
        if lo < 0 or hi >= m.vertices.shape[0]:
            raise ValueError(f"meshes[{i}].faces index outside [0, {m.vertices.shape[0]})")

    out = dict(rgb=torch.empty(O, T, H, W, 3, dtype=torch.uint8, device=dev),
               mask=torch.empty(O, T, H, W, dtype=torch.uint8, device=dev),
               xyz=torch.empty(O, T, H, W, 3, dtype=torch.float16, device=dev),
               tri=torch.empty(O, T, H, W, dtype=torch.int32, device=dev),
               depth=torch.empty(O, T, H, W, dtype=torch.float32, device=dev),
               dropped=torch.empty(O, dtype=torch.int32, device=dev))
    per_obj = T * H * W * 8
    step = max(1, VIS_BUDGET_BYTES // per_obj)
    for o0 in range(0, O, step):
        o1 = min(O, o0 + step)
        _render_chunk(meshes[o0:o1], poses[o0:o1], K, H, W, ambient, base[o0:o1], znear, {k: v[o0:o1] for k, v in out.items()})
    return out


def _render_chunk(meshes, poses, K, H, W, ambient, base, znear, out):
    dev = poses.device
    O, T = poses.shape[:2]
    info = np.zeros((O, 8), np.int32)
    v0 = f0 = tex_total = 0
    tex_off = np.zeros(O, np.int64)
    any_col = any(m.colors is not None for m in meshes)
    any_tex = any(m.uv is not None and m.texture is not None for m in meshes)
    verts, faces, cols, uvs, texs = [], [], [], [], []
    for i, m in enumerate(meshes):
        nv, nf = m.vertices.shape[0], m.faces.shape[0]
        textured = m.uv is not None and m.texture is not None
        mode = 2 if textured else (1 if m.colors is not None else 0)
        th, tw = (m.texture.shape[0], m.texture.shape[1]) if textured else (0, 0)
        info[i] = (v0, nv, f0, nf, mode, th, tw, 0)
        verts.append(m.vertices)
        faces.append(m.faces)
        if any_col:
            cols.append(m.colors if m.colors is not None else torch.zeros(nv, 3, dtype=torch.uint8, device=dev))
        if any_tex:
            uvs.append(m.uv if textured else torch.zeros(nv, 2, dtype=torch.float32, device=dev))
            if textured:
                tex_off[i] = tex_total
                texs.append(m.texture.reshape(-1))
                tex_total += m.texture.numel()
        v0 += nv
        f0 += nf
    verts = torch.cat(verts).contiguous()
    faces = torch.cat(faces).contiguous()
    cols = torch.cat(cols).contiguous() if any_col else None
    uvs = torch.cat(uvs).contiguous() if any_tex else None
    texs = torch.cat(texs).contiguous() if any_tex else None
    tex_off_d = torch.from_numpy(tex_off).to(dev) if any_tex else None
    info_d = torch.from_numpy(info).to(dev)
    base_d = torch.from_numpy(np.ascontiguousarray(base, dtype=np.float32)).to(dev)
    vrec = torch.empty(T * v0, 4, dtype=torch.int32, device=dev)
    vis = torch.empty(O * T * H * W, dtype=torch.int64, device=dev)
    big_cap = min(T * f0, BIG_LIST_CAP)
    big = torch.empty(max(big_cap, 1), 2, dtype=torch.int32, device=dev)
    counters = torch.empty(O + 1, dtype=torch.int32, device=dev)
    _lib.call("sam6d_render_meshes", verts, faces, info_d, O, v0, f0, cols, uvs, texs, tex_off_d, base_d, poses, T, float(K[0, 0]),
              float(K[1, 1]), float(K[0, 2]), float(K[1, 2]), H, W, float(znear), float(ambient), vrec, vis, big, big_cap, counters,
              out["rgb"], out["mask"], out["xyz"], out["tri"], out["depth"])
    out["dropped"].copy_(counters[1:])
