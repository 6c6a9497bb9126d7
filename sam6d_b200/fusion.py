"""Object models from posed RGB-D views (not in the reference): truncated-signed-distance fusion into a voxel volume, then
marching tetrahedra, both on sm_90a (csrc/fusion.cu; the exact rules are in include/sam6d_b200.h).

The result is a coloured triangle mesh in mm, the input every CAD path of the project takes (SAM6D.onboard, run_sam6d
--cad_path, track_sam6d, make_models_info), so an object without a CAD model can go through the whole pipeline.  The views'
object -> camera poses are an input: estimating them (SfM or SLAM on an onboarding video) is not done here.

    vol = TsdfVolume(*view_bounds(depth, masks, K, poses, depth_scale)[:3])
    vol.integrate(rgb, depth, masks, K, poses, depth_scale)
    mesh = vol.mesh()                      # meshio.Mesh: vertices f32 mm, faces int64, colours u8

or fuse(...) for both steps.  Conventions: pixel (c, r) is the ray through u = c, v = r (inputs.py's); poses are BOP's
cam_R_m2c / cam_t_m2c with t in mm; depth_raw * depth_scale is depth in mm (BOP's scene_camera depth_scale)."""
import math
from typing import Optional

import numpy as np
import torch

from . import meshio, ops

FUSION_BUDGET_BYTES = 1 << 30    # device bytes of view images uploaded per integration launch (views are chunked to fit)
DEFAULT_RESOLUTION = 128         # voxels along the longest side of the views' box
DEFAULT_TRUNC_VOXELS = 4.0       # truncation distance in voxels
ZNEAR_MM = 1.0                   # voxels closer to a camera than this are not projected into its view
MAX_DIM = ops.TSDF_MAX_DIM

_DEPTH_DTYPES = (np.uint16, np.int32, np.float32)


def _np(x, name):
    """numpy array or torch tensor (any device) -> numpy, for host-side checks and small host arrays"""
    if isinstance(x, torch.Tensor):
        return x.detach().cpu().numpy()
    if isinstance(x, np.ndarray):
        return x
    raise TypeError(f"{name} must be a numpy array or a torch tensor, got {type(x).__name__}")


def _meta(x, name):
    """(shape, numpy dtype) of a numpy array or torch tensor, without copying it"""
    if isinstance(x, torch.Tensor):
        return tuple(x.shape), torch.empty(0, dtype=x.dtype).numpy().dtype
    if isinstance(x, np.ndarray):
        return x.shape, x.dtype
    raise TypeError(f"{name} must be a numpy array or a torch tensor, got {type(x).__name__}")


def _positive(x, name):
    try:
        x = float(x)
    except (TypeError, ValueError):
        raise ValueError(f"{name} must be a number, got {x!r}") from None
    if not (math.isfinite(x) and x > 0):
        raise ValueError(f"{name} must be finite and > 0, got {x}")
    return x


def pack_views(cam_K, poses_m2c, T: int):
    """cam_K (3,3) or (T,3,3), poses_m2c (T,4,4) (numpy or torch) -> (K (T,4) float32 fx, fy, cx, cy; pose (T,12) float32 R
    row-major, then t), the per-view arrays sam6d_tsdf_integrate reads"""
    K = np.asarray(_np(cam_K, "cam_K"), np.float64)
    P = np.asarray(_np(poses_m2c, "poses_m2c"), np.float64)
    if K.shape == (3, 3):
        K = np.broadcast_to(K, (T, 3, 3))
    if K.shape != (T, 3, 3):
        raise ValueError(f"cam_K must be (3,3) or (T,3,3) with T = {T}, got {K.shape}")
    if P.shape != (T, 4, 4):
        raise ValueError(f"poses_m2c must be (T,4,4) with T = {T}, got {P.shape}")
    if not np.isfinite(K).all():
        raise ValueError("cam_K must be finite")
    if not np.isfinite(P).all():
        raise ValueError("poses_m2c must be finite")
    if not ((K[:, 0, 0] > 0).all() and (K[:, 1, 1] > 0).all()):
        raise ValueError("cam_K: fx and fy must be > 0")
    k4 = np.stack([K[:, 0, 0], K[:, 1, 1], K[:, 0, 2], K[:, 1, 2]], axis=1).astype(np.float32)
    p12 = np.concatenate([P[:, :3, :3].reshape(T, 9), P[:, :3, 3]], axis=1).astype(np.float32)
    return k4, p12


def check_views(rgb_u8, depth_raw, masks, cam_K, poses_m2c, depth_scale):
    """the integration inputs' shapes, dtypes and values, checked on the host -> (T, H, W, K (T,4) f32, pose (T,12) f32,
    depth_scale as float32).  Raises ValueError / TypeError before anything reaches the device."""
    ds, dd = _meta(depth_raw, "depth_raw")
    rs, rd = _meta(rgb_u8, "rgb_u8")
    if len(ds) != 3:
        raise ValueError(f"depth_raw must be (T,H,W), got {ds}")
    T, H, W = ds
    if T < 1 or H < 1 or W < 1:
        raise ValueError(f"depth_raw must be (T,H,W) with T, H, W >= 1, got {ds}")
    if dd not in [np.dtype(d) for d in _DEPTH_DTYPES]:
        raise ValueError(f"depth_raw must be uint16, int32 or float32, got {dd}")
    if rs != (T, H, W, 3) or rd != np.uint8:
        raise ValueError(f"rgb_u8 must be uint8 (T,H,W,3) = {(T, H, W, 3)}, got {rd} {rs}")
    if masks is not None:
        ms, md = _meta(masks, "masks")
        if ms != (T, H, W) or md != np.uint8:
            raise ValueError(f"masks must be uint8 (T,H,W) = {(T, H, W)} or None, got {md} {ms}")
    for name, x in (("rgb_u8", rgb_u8), ("depth_raw", depth_raw), ("masks", masks)):
        if isinstance(x, torch.Tensor) and not x.is_cuda:
            raise ValueError(f"{name}: a torch tensor must be on the GPU (or pass a numpy array)")
    scale = _positive(depth_scale, "depth_scale")
    with np.errstate(over="ignore"):
        scale32 = np.float32(scale)
    if not (np.isfinite(scale32) and scale32 > 0):
        raise ValueError(f"depth_scale {scale} is not a positive float32")
    K, P = pack_views(cam_K, poses_m2c, T)
    return T, H, W, K, P, scale32


def view_bounds(depth_raw, masks, cam_K, poses_m2c, depth_scale, resolution: int = DEFAULT_RESOLUTION,
                voxel_size_mm: Optional[float] = None, trunc_voxels: float = DEFAULT_TRUNC_VOXELS):
    """the object-frame box of every view's back-projected depth (only the masked depth when masks are given), padded by
    trunc + 2 voxels on every side -> (bbox_min (3,), bbox_max (3,), voxel_size_mm, trunc_mm).  The voxel size is
    voxel_size_mm, or the box's longest side / resolution; trunc = trunc_voxels voxels.  These defaults were chosen on
    rendered views of procedural meshes and are not tuned on real data."""
    T = _meta(depth_raw, "depth_raw")[0][0]
    d_all = _np(depth_raw, "depth_raw")
    m_all = None if masks is None else _np(masks, "masks")
    K, P = pack_views(cam_K, poses_m2c, T)
    scale = _positive(depth_scale, "depth_scale")
    trunc_voxels = _positive(trunc_voxels, "trunc_voxels")
    lo, hi = np.full(3, np.inf), np.full(3, -np.inf)
    for k in range(T):
        d = d_all[k].astype(np.float64) * scale
        sel = d > 0 if m_all is None else (d > 0) & (m_all[k] != 0)
        r, c = np.nonzero(sel)
        if len(r) == 0:
            continue
        z = d[r, c]
        fx, fy, cx, cy = K[k].astype(np.float64)
        X = np.stack([(c - cx) * z / fx, (r - cy) * z / fy, z], axis=1)
        R, t = P[k, :9].astype(np.float64).reshape(3, 3), P[k, 9:].astype(np.float64)
        p = (X - t) @ R                                             # R^T (X - t), row-wise
        lo, hi = np.minimum(lo, p.min(axis=0)), np.maximum(hi, p.max(axis=0))
    if not np.isfinite(lo).all():
        raise ValueError("view_bounds: no view has valid (masked) depth")
    longest = float((hi - lo).max())
    if voxel_size_mm is None:
        resolution = int(resolution)
        if resolution < 1:
            raise ValueError(f"resolution must be >= 1, got {resolution}")
        if not longest > 0:
            raise ValueError("view_bounds: the depth spans no volume; give voxel_size_mm")
        voxel = longest / resolution
    else:
        voxel = _positive(voxel_size_mm, "voxel_size_mm")
    trunc = trunc_voxels * voxel
    pad = trunc + 2.0 * voxel
    return lo - pad, hi + pad, voxel, trunc


class TsdfVolume:
    """A TSDF volume over the object-frame box [bbox_min_mm, bbox_max_mm] (mm) with cubic voxels of voxel_size_mm: ceil(extent /
    voxel) voxels per side, each side in [2, 512], voxel (i, j, k)'s centre at bbox_min + (i + 0.5, j + 0.5, k + 0.5) voxel.
    trunc_mm defaults to 4 voxels.  Fields on the device, (nz, ny, nx) with x fastest: tsdf f32 (starts at 1), weight i32,
    csum (.., 3) colour sums (u32 bits in an int32 tensor), ccount i32."""

    def __init__(self, bbox_min_mm, bbox_max_mm, voxel_size_mm, trunc_mm=None, device=None):
        lo = np.asarray(_np(np.asarray(bbox_min_mm, np.float64), "bbox_min_mm"), np.float64).reshape(-1)
        hi = np.asarray(_np(np.asarray(bbox_max_mm, np.float64), "bbox_max_mm"), np.float64).reshape(-1)
        if lo.shape != (3,) or hi.shape != (3,) or not (np.isfinite(lo).all() and np.isfinite(hi).all()):
            raise ValueError(f"bbox_min_mm and bbox_max_mm must be 3 finite numbers each, got {bbox_min_mm}, {bbox_max_mm}")
        if not (hi > lo).all():
            raise ValueError(f"empty box: bbox_max_mm {hi.tolist()} must exceed bbox_min_mm {lo.tolist()} on every axis")
        self.voxel = _positive(voxel_size_mm, "voxel_size_mm")
        self.trunc = DEFAULT_TRUNC_VOXELS * self.voxel if trunc_mm is None else _positive(trunc_mm, "trunc_mm")
        dims = [int(math.ceil(e / self.voxel)) for e in (hi - lo)]
        if max(dims) > MAX_DIM:
            raise ValueError(f"the box needs {dims} voxels per side (x, y, z); at most {MAX_DIM}: use a larger voxel")
        self.nx, self.ny, self.nz = (max(2, n) for n in dims)
        self.bbox_min = lo.astype(np.float32)
        if not (np.isfinite(self.bbox_min).all() and np.isfinite(np.float32(self.voxel)) and np.isfinite(np.float32(self.trunc))):
            raise ValueError("the box, voxel and trunc must be finite in float32")
        self.device = torch.device("cuda" if device is None else device)
        shape = (self.nz, self.ny, self.nx)
        self.tsdf = torch.ones(shape, dtype=torch.float32, device=self.device)
        self.weight = torch.zeros(shape, dtype=torch.int32, device=self.device)
        self.csum = torch.zeros(shape + (3,), dtype=torch.int32, device=self.device)
        self.ccount = torch.zeros(shape, dtype=torch.int32, device=self.device)

    @property
    def dims(self):
        """(nx, ny, nz)"""
        return self.nx, self.ny, self.nz

    def integrate(self, rgb_u8, depth_raw, masks, cam_K, poses_m2c, depth_scale) -> "TsdfVolume":
        """fuse T views: rgb_u8 (T,H,W,3) uint8, depth_raw (T,H,W) uint16 / int32 / float32 (x depth_scale = mm, 0 = missing),
        masks (T,H,W) uint8 (non-zero = object) or None, cam_K (3,3) or (T,3,3), poses_m2c (T,4,4) object -> camera with t in
        mm.  numpy arrays or CUDA tensors; the views go to the device in chunks of at most FUSION_BUDGET_BYTES"""
        T, H, W, K, P, scale = check_views(rgb_u8, depth_raw, masks, cam_K, poses_m2c, depth_scale)
        dev = self.device
        raw_bytes = _meta(depth_raw, "depth_raw")[1].itemsize
        per_view = H * W * (3 + 4 + raw_bytes + (1 if masks is not None else 0))
        step = max(1, FUSION_BUDGET_BYTES // per_view)
        Kd = torch.from_numpy(K).to(dev)
        Pd = torch.from_numpy(P).to(dev)

        def up(x, k0, k1):
            x = x[k0:k1]
            x = x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x))
            return x.to(dev).contiguous()

        for k0 in range(0, T, step):
            k1 = min(T, k0 + step)
            raw = up(depth_raw, k0, k1)
            if raw.dtype == torch.uint16:       # widened through int16, whose device kernels every torch build has
                raw = raw.view(torch.int16).to(torch.int32).bitwise_and_(0xFFFF)
            # out of place: up() returns the caller's own tensor when it is already a contiguous CUDA float32 one
            depth_mm = torch.mul(raw.to(torch.float32), float(scale))     # one float32 product per pixel
            mask = None if masks is None else up(masks, k0, k1)
            ops.tsdf_integrate(up(rgb_u8, k0, k1), depth_mm, mask, Kd[k0:k1], Pd[k0:k1], self.tsdf, self.weight, self.csum,
                               self.ccount, self.bbox_min, float(np.float32(self.voxel)), float(np.float32(self.trunc)),
                               ZNEAR_MM)
        return self

    def mesh_tensors(self, min_weight: int = 1):
        """the extraction on the device -> (vertices (V,3) f32 mm, colours (V,3) u8, faces (F,3) i32) CUDA tensors"""
        return ops.tsdf_mesh(self.tsdf, self.weight, self.csum, self.ccount, self.bbox_min, float(np.float32(self.voxel)),
                             int(min_weight))

    def mesh(self, min_weight: int = 1) -> meshio.Mesh:
        """marching tetrahedra over the corners with weight >= min_weight -> numpy meshio.Mesh (vertices f32 mm, faces int64,
        colours u8), outward-facing, which SAM6D.onboard takes as is"""
        min_weight = int(min_weight)
        if min_weight < 1:
            raise ValueError(f"min_weight must be >= 1 (a corner no view saw has no distance), got {min_weight}")
        v, c, f = self.mesh_tensors(min_weight)
        return meshio.Mesh(vertices=v.cpu().numpy(), faces=f.cpu().numpy().astype(np.int64), colors=c.cpu().numpy())

    def state(self):
        """the volume's fields as numpy arrays: tsdf f32, weight i32, csum u32 (nz,ny,nx,3), ccount i32"""
        return dict(tsdf=self.tsdf.cpu().numpy(), weight=self.weight.cpu().numpy(), csum=self.csum.cpu().numpy().view(np.uint32),
                    ccount=self.ccount.cpu().numpy())


def fuse(rgb_u8, depth_raw, masks, cam_K, poses_m2c, depth_scale, resolution: int = DEFAULT_RESOLUTION,
         voxel_size_mm: Optional[float] = None, trunc_voxels: float = DEFAULT_TRUNC_VOXELS, min_weight: int = 1,
         device=None) -> meshio.Mesh:
    """view_bounds -> TsdfVolume -> integrate -> mesh in one call (the defaults are not tuned on real data)"""
    check_views(rgb_u8, depth_raw, masks, cam_K, poses_m2c, depth_scale)
    lo, hi, voxel, trunc = view_bounds(depth_raw, masks, cam_K, poses_m2c, depth_scale, resolution, voxel_size_mm, trunc_voxels)
    vol = TsdfVolume(lo, hi, voxel, trunc, device=device)
    vol.integrate(rgb_u8, depth_raw, masks, cam_K, poses_m2c, depth_scale)
    return vol.mesh(min_weight)
