"""oracle/pn2.py -- TEST INFRASTRUCTURE ONLY.

ctypes front-end of oracle/pn2_oracle.c (the CPU restatement of the reference's
CUDA-only PointNet++ ops).  Signatures mirror the reference pybind module
`pointnet2._ext` (PEM/model/pointnet2/_ext_src/src/bindings.cpp:11-24) so the
oracle can be dropped under the reference's Python wrappers
(PEM/model/pointnet2/pointnet2_utils.py:71,107,232,282).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
reference legs may import this module.
"""
import ctypes
import os
import subprocess

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "libpn2_oracle.so")
_lib = None


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "pn2_oracle.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.check_call(["make", "-s", "-C", _HERE, "all"])
    return _SO


def lib():
    global _lib
    if _lib is None:
        build()
        _lib = ctypes.CDLL(_SO)
        _lib.pn2_oracle_block_size.restype = ctypes.c_int
    return _lib


_ref_mod = None


def _ref():
    """CUDA tensors go to the REFERENCE's own kernels (oracle/_ref/pointnet2_ref_ext.so, built from the reference sources by
    oracle/build_ref_ext.py): the oracle port then runs on the GPU exactly as the reference would (the same-box reference
    line of bench.py)."""
    global _ref_mod
    if _ref_mod is None:
        from . import build_ref_ext
        _ref_mod = build_ref_ext.load_module()
        if _ref_mod is None:
            raise RuntimeError("oracle/_ref/pointnet2_ref_ext.so not present: CUDA inputs need the reference extension")
    return _ref_mod


def _f32(t: torch.Tensor) -> np.ndarray:
    return np.ascontiguousarray(t.detach().cpu().to(torch.float32).numpy())


def _i32(t: torch.Tensor) -> np.ndarray:
    return np.ascontiguousarray(t.detach().cpu().to(torch.int32).numpy())


def _p(a: np.ndarray):
    return a.ctypes.data_as(ctypes.c_void_p)


def furthest_point_sampling(points: torch.Tensor, nsamples: int) -> torch.Tensor:
    """points (B,N,3) f32 -> (B,nsamples) i32.  sampling_gpu.cu:75-178."""
    if points.is_cuda:
        return _ref().furthest_point_sampling(points.contiguous(), int(nsamples))
    x = _f32(points)
    b, n, _ = x.shape
    out = np.zeros((b, nsamples), dtype=np.int32)
    lib().pn2_oracle_fps(_p(x), b, n, int(nsamples), _p(out))
    return torch.from_numpy(out)


def gather_points(points: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    """points (B,C,N) f32, idx (B,M) i32 -> (B,C,M).  sampling_gpu.cu:13-25."""
    if points.is_cuda:
        return _ref().gather_points(points.contiguous(), idx.contiguous())
    x, i = _f32(points), _i32(idx)
    b, c, n = x.shape
    m = i.shape[1]
    out = np.zeros((b, c, m), dtype=np.float32)
    lib().pn2_oracle_gather(_p(x), _p(i), b, c, n, m, _p(out))
    return torch.from_numpy(out)


def ball_query(new_xyz: torch.Tensor, xyz: torch.Tensor, radius: float, nsample: int) -> torch.Tensor:
    """new_xyz (B,M,3), xyz (B,N,3) -> (B,M,nsample) i32.  ball_query_gpu.cu:14-49."""
    if new_xyz.is_cuda:
        return _ref().ball_query(new_xyz.contiguous(), xyz.contiguous(), float(radius), int(nsample))
    q, x = _f32(new_xyz), _f32(xyz)
    b, m, _ = q.shape
    n = x.shape[1]
    out = np.zeros((b, m, nsample), dtype=np.int32)
    lib().pn2_oracle_ball_query(_p(q), _p(x), b, n, m, ctypes.c_float(radius), int(nsample), _p(out))
    return torch.from_numpy(out)


def group_points(points: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    """points (B,C,N), idx (B,np,ns) i32 -> (B,C,np,ns).  group_points_gpu.cu:13-33."""
    if points.is_cuda:
        return _ref().group_points(points.contiguous(), idx.contiguous())
    x, i = _f32(points), _i32(idx)
    b, c, n = x.shape
    _, npnt, ns = i.shape
    out = np.zeros((b, c, npnt, ns), dtype=np.float32)
    lib().pn2_oracle_group(_p(x), _p(i), b, c, n, npnt, ns, _p(out))
    return torch.from_numpy(out)
