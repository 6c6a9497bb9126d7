"""Tensor-level wrappers over the C ABI (include/sam6d_b200.h).

PyTorch is used here only as the owner of device memory and of the current CUDA stream; every function validates its
arguments the way the reference's native layer does (CUDA, contiguous, dtype -- PEM/model/pointnet2/_ext_src/include/utils.h:10-30
raise through TORCH_CHECK -> RuntimeError) and then hands the tensors to libsam6d_b200.so through _lib.call.

A "row view" is a 2-D (rows, C) or 3-D (batch, rows, C) tensor whose last stride is 1, such as a column slice of a fused
projection or the rows behind a sequence's first token; its row and batch strides are read from .stride(), and a batch
stride of 0 (expand) shares one matrix across the batch.
"""
import math
from typing import Optional, Tuple

import numpy as np
import torch

from . import _lib

Tensor = torch.Tensor


def _check(t: Tensor, dtype, name: str, ndim: Optional[int] = None):
    if not isinstance(t, torch.Tensor):
        raise RuntimeError(f"{name} must be a torch.Tensor")
    if not t.is_cuda:
        raise RuntimeError(f"{name} must be a CUDA tensor (CPU not supported)")
    if t.dtype != dtype:
        raise RuntimeError(f"{name} must be {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise RuntimeError(f"{name} must be contiguous")
    if ndim is not None and t.dim() != ndim:
        raise RuntimeError(f"{name} must have {ndim} dims, got {t.dim()}")


def _rows(t: Tensor) -> Tuple[int, int, int]:
    """row view -> the (rows per batch, batch stride, row stride) triple of the header's row-op convention"""
    if t.dim() not in (2, 3) or t.stride(-1) != 1:
        raise RuntimeError(f"a row view is a 2-D or 3-D tensor with unit last stride, got shape {tuple(t.shape)} "
                           f"strides {t.stride()}")
    if t.dim() == 2:
        return t.shape[0], 0, t.stride(0)
    return t.shape[1], t.stride(0), t.stride(1)


# ---------------------------------------------------------------------------------------------- point-cloud ops
def furthest_point_sampling(xyz: Tensor, m: int) -> Tensor:
    """_ext.furthest_point_sampling: (B,N,3) f32 -> (B,m) i32."""
    _check(xyz, torch.float32, "points", 3)
    b, n, c = xyz.shape
    if c != 3:
        raise RuntimeError("points must be (B,N,3)")
    idx = torch.zeros(b, m, dtype=torch.int32, device=xyz.device)
    temp = torch.empty(b, n, dtype=torch.float32, device=xyz.device) if n > 4096 else None
    _lib.call("sam6d_fps", xyz, b, n, int(m), temp, idx)
    return idx


def furthest_point_sampling_single_cta(xyz: Tensor, m: int) -> Tensor:
    """the one-CTA general-n kernel (comparator of the cluster kernel that furthest_point_sampling uses for large clouds)"""
    _check(xyz, torch.float32, "points", 3)
    b, n, _ = xyz.shape
    idx = torch.zeros(b, m, dtype=torch.int32, device=xyz.device)
    temp = torch.empty(b, n, dtype=torch.float32, device=xyz.device)
    _lib.call("sam6d_fps_single_cta", xyz, b, n, int(m), temp, idx)
    return idx


def gather_points(points: Tensor, idx: Tensor) -> Tensor:
    """_ext.gather_points: (B,C,N) f32, (B,M) i32 -> (B,C,M)."""
    _check(points, torch.float32, "points", 3)
    _check(idx, torch.int32, "idx", 2)
    b, c, n = points.shape
    m = idx.shape[1]
    out = torch.zeros(b, c, m, dtype=torch.float32, device=points.device)
    _lib.call("sam6d_gather_points", points, idx, b, c, n, m, out)
    return out


def gather_rows(src: Tensor, idx: Tensor, n_rows: Optional[int] = None) -> Tensor:
    """channel-last gather: src (B,N,C) f32, idx (B,M) i32 -> (B,M,C)."""
    _check(src, torch.float32, "src", 3)
    _check(idx, torch.int32, "idx", 2)
    b, n, c = src.shape
    m = idx.shape[1]
    out = torch.empty(b, m, c, dtype=torch.float32, device=src.device)
    _lib.call("sam6d_gather_rows", src, idx, b, n, m, c, n * c, out)
    return out


def ball_query(new_xyz: Tensor, xyz: Tensor, radius: float, nsample: int, return_count: bool = False):
    """_ext.ball_query: new_xyz (B,M,3), xyz (B,N,3) -> (B,M,nsample) i32 [, count (B,M) i32]."""
    _check(new_xyz, torch.float32, "new_xyz", 3)
    _check(xyz, torch.float32, "xyz", 3)
    b, m, _ = new_xyz.shape
    n = xyz.shape[1]
    idx = torch.zeros(b, m, nsample, dtype=torch.int32, device=xyz.device)
    cnt = torch.zeros(b, m, dtype=torch.int32, device=xyz.device) if return_count else None
    _lib.call("sam6d_ball_query", new_xyz, xyz, b, n, m, radius, int(nsample), idx, cnt)
    return (idx, cnt) if return_count else idx


def ball_query_pair(new_xyz: Tensor, xyz: Tensor, ra: float, nsa: int, rb: float, nsb: int):
    """two concentric ball queries (ra <= rb) in one sweep -> (idx_a, cnt_a, idx_b, cnt_b)"""
    _check(new_xyz, torch.float32, "new_xyz", 3)
    _check(xyz, torch.float32, "xyz", 3)
    b, m, _ = new_xyz.shape
    n = xyz.shape[1]
    dev = xyz.device
    ia = torch.empty(b, m, nsa, dtype=torch.int32, device=dev)
    ib = torch.empty(b, m, nsb, dtype=torch.int32, device=dev)
    ca = torch.empty(b, m, dtype=torch.int32, device=dev)
    cb = torch.empty(b, m, dtype=torch.int32, device=dev)
    _lib.call("sam6d_ball_query_pair", new_xyz, xyz, b, n, m, ra, int(nsa), rb, int(nsb), ia, ib, ca, cb)
    return ia, ca, ib, cb


def group_points(points: Tensor, idx: Tensor) -> Tensor:
    """_ext.group_points: (B,C,N) f32, (B,np,ns) i32 -> (B,C,np,ns)."""
    _check(points, torch.float32, "points", 3)
    _check(idx, torch.int32, "idx", 3)
    b, c, n = points.shape
    _, npnt, ns = idx.shape
    out = torch.zeros(b, c, npnt, ns, dtype=torch.float32, device=points.device)
    _lib.call("sam6d_group_points", points, idx, b, c, n, npnt, ns, out)
    return out


# ---------------------------------------------------------------------------------------------- dense algebra
def _gemm_dims(A: Tensor, W: Tensor, residual: Optional[Tensor], out: Tensor):
    """(M, N, K, lda, ldw, ldc, ldr, batch, sA, sW, sC, sR) of the strided / batched GEMM contract: A, residual, out row views,
    W (N,K) shared by every problem or (batch, N, K)"""
    M, sA, lda = _rows(A)
    K, N = A.shape[-1], W.shape[-2]
    if W.shape[-1] != K or W.stride(-1) != 1 or W.dim() not in (2, 3):
        raise RuntimeError("gemm: W must be (N,K) or (batch,N,K) with A's inner dimension and unit last stride")
    _, sC, ldc = _rows(out)
    _, sR, ldr = (0, 0, 0) if residual is None else _rows(residual)
    return (M, N, K, lda, W.stride(-2), ldc, ldr, A.shape[0] if A.dim() == 3 else 1, sA, W.stride(0) if W.dim() == 3 else 0,
            sC, sR)


def gemm(A: Tensor, W: Tensor, bias: Optional[Tensor] = None, residual: Optional[Tensor] = None,
         out: Optional[Tensor] = None, relu=False, alpha: float = 1.0) -> Tensor:
    """out = alpha * A @ W^T (+bias) (act) (+residual), f32: A, residual, out row views (M,K), (M,N) or batched (batch,M,K),
    (batch,M,N); W (N,K) shared or (batch,N,K).  relu: False/True or the activation code (0 none, 1 ReLU, 2 GELU)."""
    if A.dtype != torch.float32 or W.dtype != torch.float32:
        raise RuntimeError("gemm: A and W must be float32")
    if out is None:
        out = torch.empty(*A.shape[:-1], W.shape[-2], dtype=torch.float32, device=A.device)
    _lib.call("sam6d_gemm_f32", A, W, bias, residual, out, *_gemm_dims(A, W, residual, out), alpha, relu)
    return out


_DT = {torch.float32: 0, torch.bfloat16: 1}


def gemm_tc(A: Tensor, W: Tensor, bias: Optional[Tensor] = None, residual: Optional[Tensor] = None, out: Optional[Tensor] = None,
            relu: bool = False, alpha: float = 1.0, out_dtype=torch.float32) -> Tensor:
    """tensor-core form of gemm(): A, W fp32|bf16 -> out fp32|bf16, fp32 accumulate"""
    if A.dtype not in _DT or W.dtype not in _DT:
        raise RuntimeError("gemm_tc: A and W must be float32 or bfloat16")
    if out is None:
        out = torch.empty(*A.shape[:-1], W.shape[-2], dtype=out_dtype, device=A.device)
    _lib.call("sam6d_gemm_bf16", A, _DT[A.dtype], W, _DT[W.dtype], bias, residual, out, _DT[out.dtype], *_gemm_dims(A, W, residual, out),
              alpha, relu)
    return out


def gemm_tma(A: Tensor, W: Tensor, bias: Optional[Tensor] = None, residual: Optional[Tensor] = None, out: Optional[Tensor] = None,
             act: int = 0, alpha: float = 1.0, out_dtype=torch.float32) -> Tensor:
    """persistent TMA-fed wgmma GEMM: A (M,K) bf16, W (N,K) bf16 -> (M,N) fp32|bf16.
    act=3 (SwiGLU): W and bias are a w12 packed by pack_swiglu_rows -> (M, N/2) bf16 silu(x w1^T + b1) * (x w2^T + b2)"""
    _check(A, torch.bfloat16, "A", 2)
    _check(W, torch.bfloat16, "W", 2)
    M, K = A.shape
    N = W.shape[0]
    if W.shape[1] != K:
        raise RuntimeError("gemm: inner dimensions differ")
    Nout = N // 2 if act == ACT_SWIGLU else N
    if out is None:
        out = torch.empty(M, Nout, dtype=torch.bfloat16 if act == ACT_SWIGLU else out_dtype, device=A.device)
    if residual is not None:
        _check(residual, out.dtype, "residual", 2)          # the residual stream has the element type of the output
    _lib.call("sam6d_gemm_tma", A, W, bias, residual, out, _DT[out.dtype], M, N, K, K, K, Nout, N, alpha, int(act))
    return out


ACT_GELU = 2
ACT_SWIGLU = 3


def pack_swiglu_rows(t: Tensor, block: int = 128) -> Tensor:
    """w12 (2H, K) or its bias (2H,) in the reference's order (rows [0, H) gate, [H, 2H) up) -> the order gemm_tma(act=3)
    reads: gate rows [128t, 128t + 128) followed by up rows [128t, 128t + 128), for t = 0 .. H/128 - 1.  H % 128 == 0."""
    H = t.shape[0] // 2
    if t.shape[0] != 2 * H or H % block:
        raise ValueError(f"SwiGLU w12 needs 2H rows with H % {block} == 0, got {t.shape[0]}")
    rest = t.shape[1:]
    return t.reshape(2, H // block, block, *rest).transpose(0, 1).reshape(2 * H, *rest).contiguous()


_VT_CACHE = {}


def _vt_buffer(rows: int, n1: int, device, slot: int) -> Tensor:
    """V^T operand buffers are reused across layers (stream order keeps producer and consumer apart); they are zeroed once so
    the key-padding columns, which the GEMM epilogue never writes, stay finite"""
    key = (rows, n1, str(device), slot, torch.cuda.current_stream(device).cuda_stream)   # one buffer per stream: no cross-stream reuse
    buf = _VT_CACHE.get(key)
    if buf is None:
        if len(_VT_CACHE) > 64:
            _VT_CACHE.clear()
        buf = torch.zeros(rows, n1, dtype=torch.bfloat16, device=device)
        _VT_CACHE[key] = buf
    return buf


def gemm_tma_vt(A: Tensor, W: Tensor, bias: Tensor, vt_col0: int, S: int, slot: int = 0) -> Tuple[Tensor, Tensor]:
    """fused QKV / KV projection: A (M,K) bf16, W (N,K) bf16 -> (QK (M, vt_col0) bf16, Vt) where the value columns
    [vt_col0, N) are written transposed per cloud of S token rows: Vt (M/S * (N - vt_col0), ceil16(S)) = the operand
    transpose_tokens would produce"""
    _check(A, torch.bfloat16, "A", 2)
    _check(W, torch.bfloat16, "W", 2)
    M, K = A.shape
    N = W.shape[0]
    if W.shape[1] != K or M % S or not (0 < vt_col0 < N):
        raise RuntimeError("gemm_tma_vt: shape mismatch")
    n1 = (S + 15) // 16 * 16
    out = torch.empty(M, vt_col0, dtype=torch.bfloat16, device=A.device)
    vt = _vt_buffer((M // S) * (N - vt_col0), n1, A.device, slot)
    _lib.call("sam6d_gemm_tma_vt", A, W, bias, out, M, N, K, K, K, vt_col0, vt, int(vt_col0), int(S), int(n1))
    return out, vt


def gemm_tma_vt2(A: Tensor, W: Tensor, bias: Tensor, vt_col0: int, vt_col1: int, S: int, slot: int = 0) -> Tuple[Tensor, Tensor, Tensor]:
    """gemm_tma_vt with a third column range: -> (C (M, vt_col0), Vt of columns [vt_col0, vt_col1), C2 (M, N - vt_col1)), all bf16"""
    _check(A, torch.bfloat16, "A", 2)
    _check(W, torch.bfloat16, "W", 2)
    M, K = A.shape
    N = W.shape[0]
    if W.shape[1] != K or M % S or not (0 < vt_col0 < vt_col1 < N):
        raise RuntimeError("gemm_tma_vt2: shape mismatch")
    n1 = (S + 15) // 16 * 16
    out = torch.empty(M, vt_col0, dtype=torch.bfloat16, device=A.device)
    out2 = torch.empty(M, N - vt_col1, dtype=torch.bfloat16, device=A.device)
    vt = _vt_buffer((M // S) * (vt_col1 - vt_col0), n1, A.device, slot)
    _lib.call("sam6d_gemm_tma_vt2", A, W, bias, out, M, N, K, K, K, vt_col0, vt, int(vt_col0), int(vt_col1), int(S), int(n1), out2,
              N - vt_col1)
    return out, vt, out2


def layernorm(x: Tensor, gamma: Tensor, beta: Tensor, eps: float = 1e-5, out: Optional[Tensor] = None) -> Tensor:
    """LayerNorm over the last dim of f32 rows: x and out contiguous (any rank) or row views"""
    if x.dtype != torch.float32:
        raise RuntimeError(f"x must be torch.float32, got {x.dtype}")
    C = x.shape[-1]
    if out is None:
        out = torch.empty_like(x)
    xv = x.view(-1, C) if x.is_contiguous() else x
    yv = out.view(-1, C) if out.is_contiguous() else out
    _lib.call("sam6d_layernorm", xv, *_rows(xv), yv, *_rows(yv), gamma, beta, x.numel() // C, C, eps)
    return out


def layernorm_bf16(x: Tensor, gamma: Tensor, beta: Tensor, eps: float = 1e-5) -> Tensor:
    """LayerNorm with bf16 output rows (feeds the TMA GEMM directly)"""
    _check(x, torch.float32, "x")
    C = x.shape[-1]
    rows = x.numel() // C
    out = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    _lib.call("sam6d_layernorm_bf16", x, rows, 0, C, out, rows, 0, C, gamma, beta, rows, int(C), eps)
    return out


def layernorm_bf16io(x: Tensor, gamma: Tensor, beta: Tensor, eps: float = 1e-5, out: Optional[Tensor] = None) -> Tensor:
    """LayerNorm over the last dim of contiguous bf16 rows, bf16 result (statistics in fp32)"""
    _check(x, torch.bfloat16, "x")
    C = x.shape[-1]
    rows = x.numel() // C
    if out is None:
        out = torch.empty_like(x)
    _lib.call("sam6d_layernorm_bf16io", x, max(rows, 1), 0, C, out, max(rows, 1), 0, C, gamma, beta, rows, int(C), eps)
    return out


def transformer_tail_bf16(hid: Tensor, x: Tensor, wo: Tensor, bo: Tensor, g1: Tensor, b1: Tensor, we: Tensor, be: Tensor, ws: Tensor,
                          bs: Tensor, g2: Tensor, b2: Tensor, out: Optional[Tensor] = None, eps: float = 1e-5) -> Tensor:
    """LN2(y + relu(y We^T + be) Ws^T + bs) with y = LN1(hid Wo^T + bo + x): the attention-layer tail + AttentionOutput of
    transformer.py:176-197 as one persistent TMA / wgmma kernel (csrc/tail_tc.cu).  hid, x (M,256) bf16 -> (M,256) bf16."""
    _check(hid, torch.bfloat16, "hid", 2)
    _check(x, torch.bfloat16, "x", 2)
    M = hid.shape[0]
    if hid.shape[1] != 256 or x.shape != hid.shape or wo.shape != (256, 256) or we.shape != (512, 256) or ws.shape != (256, 512):
        raise RuntimeError("transformer_tail_bf16: d_model 256, hidden 512")
    for w in (wo, we, ws):
        _check(w, torch.bfloat16, "weight", 2)
    if out is None:
        out = torch.empty_like(hid)
    _check(out, torch.bfloat16, "out", 2)
    _lib.call("sam6d_transformer_tail_bf16", hid, 256, x, 256, wo, bo, g1, b1, we, be, ws, bs, g2, b2, out, 256, int(M), eps)
    return out


def gather_rows_bf16_f32(src: Tensor, idx: Tensor) -> Tensor:
    """out[b,j,:] = float(src[b, idx[b,j], :]) for a bf16 (b,n,c) token matrix; negative index -> zero row"""
    _check(src, torch.bfloat16, "src", 3)
    _check(idx, torch.int32, "idx", 2)
    b, n, c = src.shape
    m = idx.shape[1]
    out = torch.empty(b, m, c, dtype=torch.float32, device=src.device)
    _lib.call("sam6d_gather_rows_bf16_f32", src, idx, b, n, m, c, n * c, out)
    return out


def gather_rows_bf16(src: Tensor, idx: Tensor) -> Tensor:
    """channel-last gather of bf16 rows (C even): moved as C/2 32-bit words by the fp32 gather kernel"""
    _check(src, torch.bfloat16, "src", 3)
    _check(idx, torch.int32, "idx", 2)
    b, n, c = src.shape
    m = idx.shape[1]
    out = torch.empty(b, m, c, dtype=torch.bfloat16, device=src.device)
    _lib.call("sam6d_gather_rows", src, idx, b, n, m, c // 2, n * c // 2, out)
    return out


def l2norm_rows(x: Tensor) -> Tensor:
    _check(x, torch.float32, "x")
    C = x.shape[-1]
    rows = x.numel() // C
    out = torch.empty_like(x)
    _lib.call("sam6d_l2norm_rows", x, rows, 0, C, out, rows, 0, C, rows, C)
    return out


def l2norm_rows_bf16(x: Tensor) -> Tensor:
    """F.normalize(x, dim=-1) with a bf16 result (operand of the tensor-core score GEMM)"""
    _check(x, torch.float32, "x")
    C = x.shape[-1]
    rows = x.numel() // C
    out = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    _lib.call("sam6d_l2norm_rows_bf16", x, max(rows, 1), 0, C, out, max(rows, 1), 0, C, rows, C)
    return out


def gemm_tma_batched(A: Tensor, W: Tensor, out: Tensor, alpha: float = 1.0, bias: Optional[Tensor] = None,
                     residual: Optional[Tensor] = None) -> Tensor:
    """A (batch, a_rows, K) bf16; W (batch, w_rows, K) bf16 or one shared (N, K) matrix; out a (batch, M, N) row view (fp32 or
    bf16, M <= a_rows, N <= w_rows) -> out[z] = alpha * A[z,:M] @ W[z,:N]^T (+ bias) (+ residual[z]) for every z; the residual
    is a row view with out's shape and element type (batch stride 0 shares one matrix)"""
    _check(A, torch.bfloat16, "A", 3)
    _check(W, torch.bfloat16, "W")
    batch, a_rows, K = A.shape
    M, c_bs, ldc = _rows(out)
    N = out.shape[-1]
    shared = W.dim() == 2
    if (W.shape[-1] != K or a_rows < M or out.dim() != 3 or out.shape[0] != batch
            or (not shared and (W.shape[0] != batch or W.shape[1] < N)) or (shared and W.shape[0] != N)):
        raise RuntimeError("gemm_tma_batched: shape mismatch")
    if residual is not None and residual.dtype != out.dtype:
        raise RuntimeError("gemm_tma_batched: the residual must have the output's element type")
    _, r_bs, ldr = (0, 0, 0) if residual is None else _rows(residual)
    _lib.call("sam6d_gemm_tma_batched", A, W, bias, residual, out, _DT[out.dtype], M, N, K, K, K, ldc, ldr, batch, a_rows,
              0 if shared else W.shape[1], c_bs, r_bs, alpha, 0)
    return out


def focus_rows(x: Tensor, sp_scale: Tensor, out: Optional[Tensor] = None) -> Tensor:
    """focused-linear-attention feature map of f32 row views; out may be x itself"""
    if out is None:
        out = torch.empty(x.shape, dtype=torch.float32, device=x.device)
    _lib.call("sam6d_focus_rows", x, *_rows(x), out, *_rows(out), sp_scale, x.numel() // x.shape[-1], x.shape[-1])
    return out


def rigid_warp(p: Tensor, R: Tensor, t: Tensor) -> Tensor:
    _check(p, torch.float32, "p", 3)
    _check(R, torch.float32, "R", 3)
    _check(t, torch.float32, "t", 2)
    out = torch.empty_like(p)
    _lib.call("sam6d_rigid_warp", p, R, t, p.shape[0], p.shape[1], out)
    return out


def cloud_radius(po: Tensor) -> Tensor:
    _check(po, torch.float32, "dense_po", 3)
    r = torch.empty(po.shape[0], dtype=torch.float32, device=po.device)
    _lib.call("sam6d_cloud_radius", po, po.shape[0], po.shape[1], r)
    return r


def scale_by_radius(x: Tensor, radius: Tensor) -> Tensor:
    _check(x, torch.float32, "x")
    _check(radius, torch.float32, "radius", 1)
    out = torch.empty_like(x)
    b = x.shape[0]
    _lib.call("sam6d_scale_by_radius", x, radius, b, x.numel() // max(b, 1), out)
    return out


# ---------------------------------------------------------------------------------------------- geometric embedding
def geo_indices(pts: Tensor, sigma_d: float, factor_a: float) -> Tensor:
    _check(pts, torch.float32, "points", 3)
    b, s, _ = pts.shape
    T = torch.empty(b, s, s, 4, dtype=torch.float32, device=pts.device)
    _lib.call("sam6d_geo_indices", pts, b, s, sigma_d, factor_a, T)
    return T


def geo_embed_f32(T: Tensor, div_term: Tensor, WaT: Tensor, WdT: Tensor, bias: Tensor) -> Tensor:
    _check(T, torch.float32, "T", 4)
    b, s, _, _ = T.shape
    E = torch.empty(b, s, s, 256, dtype=torch.float32, device=T.device)
    _lib.call("sam6d_geo_embed_f32", T, b * s * s, div_term, WaT, WdT, bias, E)
    return E


def geo_embed_tc(T: Tensor, div_term: Tensor, Wa_bf16: Tensor, Wd_bf16: Tensor, bias: Tensor, out_dtype=torch.bfloat16) -> Tensor:
    """wgmma version: weights (out,in) bf16, E (B,S,S,256) fp32 or bf16"""
    _check(T, torch.float32, "T", 4)
    _check(Wa_bf16, torch.bfloat16, "Wa", 2)
    _check(Wd_bf16, torch.bfloat16, "Wd", 2)
    b, s, _, _ = T.shape
    E = torch.empty(b, s, s, 256, dtype=out_dtype, device=T.device)
    _lib.call("sam6d_geo_embed_tc", T, b * s * s, div_term, Wa_bf16, Wd_bf16, bias, E, int(out_dtype == torch.bfloat16))
    return E


def geo_embed_dist_tc(T: Tensor, div_term: Tensor, Wd_bf16: Tensor, bias: Tensor) -> Tensor:
    """distance projection only: T (..., 4) f32 -> (..., 256) bf16 = proj_d(emb(T[..., 3])) + bias (wgmma)"""
    if T.dtype != torch.float32 or not T.is_cuda or not T.is_contiguous() or T.shape[-1] != 4:
        raise RuntimeError("T must be a contiguous CUDA float32 tensor (..., 4)")
    _check(Wd_bf16, torch.bfloat16, "Wd", 2)
    n = T.numel() // 4
    E = torch.empty(*T.shape[:-1], 256, dtype=torch.bfloat16, device=T.device)
    _lib.call("sam6d_geo_embed_dist_tc", T, n, div_term, Wd_bf16, bias, E)
    return E


def geo_embed_lut(T: Tensor, tabA: Tensor, inv_ha: float, tabD: Tensor, inv_hd: float, far: Tensor, div_term: Tensor, WdT_bf16: Tensor,
                  bias: Tensor) -> Tensor:
    """table-interpolation geometric embedding (csrc/geo_lut.cu): T (B,S,S,4) f32, tabA (na,256) / tabD (nd,256) bf16,
    far (B,2,S,256) bf16 -> E (B,S,S,256) bf16"""
    _check(T, torch.float32, "T", 4)
    _check(tabA, torch.bfloat16, "tabA", 2)
    _check(tabD, torch.bfloat16, "tabD", 2)
    _check(far, torch.bfloat16, "far", 4)
    _check(WdT_bf16, torch.bfloat16, "WdT", 2)
    b, s, _, _ = T.shape
    if far.shape != (b, 2, s, 256) or tabA.shape[1] != 256 or tabD.shape[1] != 256 or T.shape[3] != 4:
        raise RuntimeError("geo_embed_lut: shape mismatch")
    E = torch.empty(b, s, s, 256, dtype=torch.bfloat16, device=T.device)
    _lib.call("sam6d_geo_embed_lut", T, b, s, tabA, tabA.shape[0], inv_ha, tabD, tabD.shape[0], inv_hd, far, div_term, WdT_bf16, bias, E)
    return E


# ---------------------------------------------------------------------------------------------- attention
def rpe_scores(E: Tensor, U: Tensor) -> Tensor:
    """E (B,S,S,256) f32|bf16, U (B,S,4,256) f32 contiguous or a (B*S, 4*256) f32 row view (e.g. the u columns of a fused
    projection; 16-byte aligned, with a row stride that is a multiple of 4) -> (B,4,S,S) f32."""
    if E.dtype not in (torch.float32, torch.bfloat16):
        raise RuntimeError("E must be float32 or bfloat16")
    _check(E, E.dtype, "E", 4)
    B, S = E.shape[0], E.shape[1]
    if U.dim() == 4:
        U = U.view(B * S, -1)
    if U.dtype != torch.float32 or U.dim() != 2 or U.shape != (B * S, 1024) or U.stride(1) != 1:
        raise RuntimeError("rpe_scores: U must be a (B*S, 1024) float32 row view")
    SP = torch.empty(B, 4, S, S, dtype=torch.float32, device=E.device)
    _lib.call("sam6d_rpe_scores", E, int(E.dtype == torch.bfloat16), U, U.stride(0), B, S, SP)
    return SP


def rpe_scores_tc(E: Tensor, U: Tensor, ld: Optional[int] = None) -> Tensor:
    """E (B,S,S,256) bf16, U (B*S, 1024) bf16 = the four folded per-head queries of every token -> (B,4,S,ld) f32 score
    planes with row stride ld >= S (default S; columns [S, ld) are not written).  TMA + wgmma stream over E (csrc/rpe_tc.cu);
    S <= 200."""
    _check(E, torch.bfloat16, "E", 4)
    _check(U, torch.bfloat16, "U", 2)
    B, S = E.shape[0], E.shape[1]
    if U.shape != (B * S, 1024) or E.shape[3] != 256 or E.shape[2] != S:
        raise RuntimeError("rpe_scores_tc: E (B,S,S,256), U (B*S,1024)")
    ld = S if ld is None else ld
    SP = torch.empty(B, 4, S, ld, dtype=torch.float32, device=E.device)
    _lib.call("sam6d_rpe_scores_tc_ld", E, U, B, S, SP, int(ld))
    return SP


def rpe_scores_tc_padded(E: Tensor, U: Tensor) -> Tensor:
    """rpe_scores_tc into planes whose rows are padded to a multiple of 16 keys; attn_tc_padded_bias consumes them with
    16-byte copies"""
    return rpe_scores_tc(E, U, ld=(E.shape[1] + 15) // 16 * 16)


def attn_tc_padded_bias(Q: Tensor, q_col0: int, K: Tensor, k_col0: int, Vt: Tensor, B: int, H: int, Sq: int, Sk: int, D: int,
                        scale: float, bias: Tensor, out_dtype=torch.bfloat16) -> Tensor:
    """attn_tc with the dense bias in padded planes (B,H,Sq,ld) f32 (from rpe_scores_tc_padded); head dim 64"""
    _check(Q, torch.bfloat16, "Q", 2)
    _check(K, torch.bfloat16, "K", 2)
    _check(Vt, torch.bfloat16, "Vt", 2)
    _check(bias, torch.float32, "bias", 4)
    if bias.shape[:3] != (B, H, Sq) or bias.shape[3] < Sk or bias.shape[3] % 4:
        raise RuntimeError("attn_tc_padded_bias: bias (B,H,Sq,ld), ld >= Sk, ld % 4 == 0")
    out = torch.empty(B * Sq, H * D, dtype=out_dtype, device=Q.device)
    _lib.call("sam6d_attn_tc_bias_ld", Q, Q.shape[1], int(q_col0), K, K.shape[1], int(k_col0), Vt, Vt.shape[1], int(B), int(H), int(Sq),
              int(Sk), int(D), bias, bias.shape[3], scale, out, int(out_dtype == torch.bfloat16), H * D)
    return out


def mha(q: Tensor, k: Tensor, v: Tensor, bias: Optional[Tensor], scale: float, out: Tensor) -> Tensor:
    """softmax((q k^T + bias) * scale) v per head of 64 channels: q, out (B,Sq,H*64), k, v (B,Sk,H*64) f32 row views (e.g.
    column slices of a fused qkv projection); bias (B,H,Sq,Sk) f32 contiguous or None"""
    for t, name in ((q, "q"), (k, "k"), (v, "v"), (out, "out")):
        if t.dtype != torch.float32 or t.dim() != 3:
            raise RuntimeError(f"mha: {name} must be a 3-D float32 row view, got {t.dtype} with shape {tuple(t.shape)}")
    B, Sq, HD = q.shape
    Sk = k.shape[1]
    if HD % 64 or k.shape != (B, Sk, HD) or v.shape != (B, Sk, HD) or out.shape != (B, Sq, HD):
        raise RuntimeError(f"mha: q, out (B,Sq,H*64) and k, v (B,Sk,H*64), got q {tuple(q.shape)} k {tuple(k.shape)} "
                           f"v {tuple(v.shape)} out {tuple(out.shape)}")
    H = HD // 64
    if bias is not None:
        _check(bias, torch.float32, "bias", 4)
        if bias.shape != (B, H, Sq, Sk):
            raise RuntimeError(f"mha: bias must be (B,H,Sq,Sk) = {(B, H, Sq, Sk)}, got {tuple(bias.shape)}")
    _, q_bs, q_ld = _rows(q)
    _, k_bs, k_ld = _rows(k)
    _, v_bs, v_ld = _rows(v)
    _, o_bs, o_ld = _rows(out)
    _lib.call("sam6d_mha", q, q_ld, q_bs, k, k_ld, k_bs, v, v_ld, v_bs, bias, B, H, Sq, Sk, scale, out, o_ld, o_bs)
    return out


def pack_rel_pos(rel_h: Tensor, rel_w: Tensor, slab_rows: int = 32) -> Tensor:
    """rel_pos_h / rel_pos_w ((2S-1, D) fp32) -> the bf16 image the attention kernels bulk-copy into shared memory: for each
    table ceil(D/64) slabs of [slab_rows rows][64 channels], K-major with the 128-byte swizzle (16-byte chunk index XOR
    (row % 8)).  slab_rows = 32 for the 14 x 14 windows, 128 for the 64 x 64 global grid."""
    D = rel_h.shape[1]
    DS = (D + 63) // 64
    if rel_h.shape[0] > slab_rows or rel_w.shape[0] > slab_rows:
        raise RuntimeError("pack_rel_pos: table has more rows than the slab")
    blob = torch.zeros(2 * DS * slab_rows * 64, dtype=torch.bfloat16, device=rel_h.device)
    j = torch.arange(slab_rows, device=rel_h.device).view(slab_rows, 1)
    c = torch.arange(D, device=rel_h.device).view(1, D)
    off = j * 64 + ((((c % 64) // 8) ^ (j % 8)) * 8) + (c % 8)                     # element offset inside a slab
    for t, tab in enumerate((rel_h, rel_w)):
        n = tab.shape[0]
        idx = ((t * DS + c // 64) * slab_rows * 64 + off)[:n]
        blob[idx.reshape(-1)] = tab.to(torch.bfloat16).reshape(-1)
    return blob


def attn_global_tc(qkv: Tensor, vt: Tensor, rel_blob: Tensor, B: int, H: int, grid: int, scale: float, out_dtype=torch.bfloat16,
                   D: int = 80) -> Tensor:
    """SAM global attention (grid x grid = 4096 tokens, head_dim D = 80 for ViT-H or 64 for ViT-L / ViT-B) on wgmma: qkv
    (B*L, >= 2*H*D) bf16 rows [q|k(|v)], vt from transpose_tokens, rel_blob from pack_rel_pos(rel_h, rel_w, slab_rows=128)
    -> (B*L, H*D)"""
    _check(qkv, torch.bfloat16, "qkv", 2)
    _check(vt, torch.bfloat16, "vt", 2)
    _check(rel_blob, torch.bfloat16, "rel_blob", 1)
    L = grid * grid
    out = torch.empty(B * L, H * D, dtype=out_dtype, device=qkv.device)
    _lib.call("sam6d_attn_global_tc_ex", qkv, qkv.shape[1], vt, vt.shape[1], rel_blob, int(B), int(H), int(grid), int(D), scale, out,
              int(out_dtype == torch.bfloat16), H * D)
    return out


def attn_tc(Q: Tensor, q_col0: int, K: Tensor, k_col0: int, Vt: Tensor, B: int, H: int, Sq: int, Sk: int, D: int, scale: float,
            bias: Optional[Tensor] = None, rel: Optional[tuple] = None, bv: Optional[Tensor] = None,
            out_dtype=torch.float32) -> Tensor:
    """tensor-core attention (<= 256 keys).  Q, K: bf16 2-D matrices (rows = batch*tokens); Vt: bf16 (B*H*D, >= ceil16(Sk));
    bias: dense fp32 (B,H,Sq,Sk); rel = (rel_h, rel_w, Hs, Ws) for the decomposed rel-pos bias.  -> (B*Sq, H*D) fp32"""
    _check(Q, torch.bfloat16, "Q", 2)
    _check(K, torch.bfloat16, "K", 2)
    _check(Vt, torch.bfloat16, "Vt", 2)
    mode, rh, rw, Hs, Ws = 0, None, None, 0, 0
    if bias is not None:
        _check(bias, torch.float32, "bias", 4)
        mode = 1
    elif rel is not None:
        rh, Hs, Ws = rel                     # rh: pack_rel_pos(rel_pos_h, rel_pos_w)
        mode = 2
    out = torch.empty(B * Sq, H * D, dtype=out_dtype, device=Q.device)
    _lib.call("sam6d_attn_tc", Q, Q.shape[1], int(q_col0), K, K.shape[1], int(k_col0), Vt, Vt.shape[1], int(B), int(H), int(Sq), int(Sk),
              int(D), mode, bias, rh, rw, int(Hs), int(Ws), bv, scale, out, int(out_dtype == torch.bfloat16), H * D)
    return out


def attn_tc_ex(Q: Tensor, q_col0: int, K: Tensor, k_col0: int, Vt: Tensor, B: int, H: int, Sq: int, Sk: int, D: int, scale: float,
               k_brows: int, k_row0: int = 0, v_col0: int = 0, want_lse: bool = False, out_dtype=torch.bfloat16):
    """attn_tc (no bias) over a window of keys: batch b's keys are rows [b*k_brows + k_row0, +Sk) of K and columns [v_col0, +Sk) of
    its V^T rows.  -> (out (B*Sq, H*D), lse (B,H,Sq) f32 or None)"""
    _check(Q, torch.bfloat16, "Q", 2)
    _check(K, torch.bfloat16, "K", 2)
    _check(Vt, torch.bfloat16, "Vt", 2)
    out = torch.empty(B * Sq, H * D, dtype=out_dtype, device=Q.device)
    lse = torch.empty(B, H, Sq, dtype=torch.float32, device=Q.device) if want_lse else None
    _lib.call("sam6d_attn_tc_ex", Q, Q.shape[1], int(q_col0), K, K.shape[1], int(k_col0), Vt, Vt.shape[1], int(B), int(H), int(Sq), int(Sk),
              int(D), scale, int(k_brows), int(k_row0), int(v_col0), lse, out, int(out_dtype == torch.bfloat16), H * D)
    return out, lse


def attn_merge_key(Q: Tensor, q_col0: int, K: Tensor, k_col0: int, k_brows: int, key_row: int, Vt: Tensor, key_col: int, lse: Tensor,
                   B: int, H: int, Sq: int, scale: float, out: Tensor) -> Tensor:
    """folds one more key (row key_row of every batch's K rows, column key_col of its V^T rows) into the bf16 result `out` of
    attn_tc_ex (head dim 64), in place"""
    _check(out, torch.bfloat16, "out", 2)
    _check(lse, torch.float32, "lse", 3)
    _lib.call("sam6d_attn_merge_key", Q, Q.shape[1], int(q_col0), K, K.shape[1], int(k_col0), int(k_brows), int(key_row), Vt, Vt.shape[1],
              int(key_col), lse, int(B), int(H), int(Sq), scale, out, out.shape[1])
    return out


def transpose_tokens(src: Tensor, col0: int, C: int, nB: int, L: int) -> Tensor:
    """V^T for attn_tc: src bf16 (nB*L, ld) -> (nB*C, ceil16(L)) bf16, zero padded keys"""
    _check(src, torch.bfloat16, "src", 2)
    N1 = (L + 15) // 16 * 16
    out = torch.empty(nB * C, N1, dtype=torch.bfloat16, device=src.device)
    _lib.call("sam6d_transpose_tokens_bf16", src, src.shape[1], int(col0), int(C), int(nB), int(L), int(N1), out)
    return out


def linattn_kv(k: Tensor, v: Tensor, KV: Tensor, KS: Tensor):
    """kv-first branch of LinearAttention: focused keys k and values v ((B,J,H*64) f32 row views) -> KV (B,H,64,64), KS (B,H,64)"""
    B, J, _ = k.shape
    _, k_bs, k_ld = _rows(k)
    _, v_bs, v_ld = _rows(v)
    _lib.call("sam6d_linattn_kv", k, k_ld, k_bs, v, v_ld, v_bs, B, KV.shape[1], J, KV, KS)


def linattn_apply(q: Tensor, KV: Tensor, KS: Tensor, out: Tensor):
    """out[b,i,h] = (q'_h KV_h) / (q'_h . KS_h + 1e-6) for focused queries q and out (B,N,H*64) f32 row views"""
    _, x_bs, x_ld = _rows(out)
    _lib.call("sam6d_linattn_apply", q, *_rows(q), KV, KS, q.shape[0], KV.shape[1], out, x_bs, x_ld)


def linattn_kv_pack(k: Tensor, v: Tensor) -> Tuple[Tensor, Tensor]:
    """focused keys / values ((B,J,256) fp32 row views) -> (blob: B x 32 KB bf16 wgmma image of KV_h^T, KS (B,4,64) fp32)"""
    B, J, _ = k.shape
    _, k_bs, k_ld = _rows(k)
    _, v_bs, v_ld = _rows(v)
    blob = torch.empty(B, 4 * 64 * 64, dtype=torch.bfloat16, device=k.device)
    KS = torch.empty(B, 4, 64, dtype=torch.float32, device=k.device)
    _lib.call("sam6d_linattn_kv_pack", k, k_ld, k_bs, v, v_ld, v_bs, B, J, blob, KS)
    return blob, KS


def linattn_tc(q: Tensor, blob: Tensor, KS: Tensor, sp_scale: Tensor, out: Tensor):
    """dense tokens (bf16 row views q, out (B,rows,256)): focusing feature map + per-head (q' KV) / (q' . ksum) on wgmma"""
    B, rpb, _ = q.shape
    _, q_bs, q_ld = _rows(q)
    _, x_bs, x_ld = _rows(out)
    _lib.call("sam6d_linattn_tc", q, q_ld, q_bs, blob, KS, sp_scale, B, rpb, out, x_ld, x_bs)


# ---------------------------------------------------------------------------------------------- coarse pose
def coarse_assign(A: Tensor) -> Tuple[Tensor, Tensor]:
    _check(A, torch.float32, "atten", 3)
    B, S, _ = A.shape
    n = S - 1
    W = torch.empty(B, n * n, dtype=torch.float32, device=A.device)
    w1 = torch.empty(B, n, dtype=torch.float32, device=A.device)
    _lib.call("sam6d_coarse_assign", A, B, S, W, w1)
    return W, w1


def coarse_sample(W: Tensor, rand: Tensor) -> Tensor:
    _check(W, torch.float32, "W", 2)
    _check(rand, torch.float32, "rand", 2)
    B, L = W.shape
    nr = rand.shape[1]
    idx = torch.empty(B, nr, dtype=torch.int32, device=W.device)
    _lib.call("sam6d_coarse_sample", W, B, L, rand, nr, idx)
    return idx


def coarse_hypotheses(idx: Tensor, pts1: Tensor, pts2: Tensor) -> Tuple[Tensor, Tensor]:
    _check(idx, torch.int32, "idx", 2)
    _check(pts1, torch.float32, "pts1", 3)
    _check(pts2, torch.float32, "pts2", 3)
    B, n, _ = pts1.shape
    n1 = idx.shape[1] // 3
    Rt = torch.empty(B, n1, 12, dtype=torch.float32, device=idx.device)
    resid = torch.empty(B, n1, dtype=torch.float32, device=idx.device)
    _lib.call("sam6d_coarse_hypotheses", idx, pts1, pts2, B, n, n1, Rt, resid)
    return Rt, resid


def topk_smallest(v: Tensor, k: int) -> Tensor:
    _check(v, torch.float32, "v", 2)
    B, n = v.shape
    out = torch.empty(B, k, dtype=torch.int32, device=v.device)
    _lib.call("sam6d_topk_smallest", v, B, n, int(k), out)
    return out


def coarse_select(Rt: Tensor, top: Tensor, pts1: Tensor, w1: Tensor, model: Tensor):
    _check(Rt, torch.float32, "Rt", 3)
    _check(top, torch.int32, "top", 2)
    _check(model, torch.float32, "model", 3)
    B, n1, _ = Rt.shape
    n2 = top.shape[1]
    n = pts1.shape[1]
    scores = torch.empty(B, n2, dtype=torch.float32, device=Rt.device)
    R = torch.empty(B, 3, 3, dtype=torch.float32, device=Rt.device)
    t = torch.empty(B, 3, dtype=torch.float32, device=Rt.device)
    _lib.call("sam6d_coarse_select", Rt, top, B, n1, n2, pts1, w1, n, model, model.shape[1], scores, R, t)
    return R, t, scores


def hypothesis_thresholds(min_angle: float, min_dist: float) -> Tuple[float, float]:
    """min_angle (degrees), min_dist (radius-normalised) -> (cos_thr, d2_min) as sam6d_coarse_pick_distinct receives them: 1 + 2
    cos(min_angle) and min_dist^2, each evaluated in float64 and rounded to fp32"""
    return (float(np.float32(1.0 + 2.0 * np.cos(np.radians(float(min_angle))))),
            float(np.float32(float(min_dist) * float(min_dist))))


def coarse_pick_distinct(Rt: Tensor, top: Tensor, scores: Tensor, K: int, min_angle: float, min_dist: float):
    """K mutually distinct hypotheses of the coarse stage per proposal (the rule: include/sam6d_b200.h,
    sam6d_coarse_pick_distinct).  Rt (B,n1,12), top (B,n2), scores (B,n2) of coarse_select -> R (B,K,3,3), t (B,K,3), score (B,K)
    f32, valid (B,K) u8, count (B) i32; slot 0 is coarse_select's pose, slots from count on are copies of it with valid 0."""
    _check(Rt, torch.float32, "Rt", 3)
    _check(top, torch.int32, "top", 2)
    _check(scores, torch.float32, "scores", 2)
    B, n1, _ = Rt.shape
    n2 = top.shape[1]
    if tuple(scores.shape) != (B, n2) or top.shape[0] != B:
        raise RuntimeError(f"coarse_pick_distinct: Rt (B,n1,12), top and scores (B,n2), got {tuple(Rt.shape)}, {tuple(top.shape)}, "
                           f"{tuple(scores.shape)}")
    cos_thr, d2_min = hypothesis_thresholds(min_angle, min_dist)
    dev = Rt.device
    K = int(K)
    R = torch.empty(B, max(K, 0), 3, 3, dtype=torch.float32, device=dev)
    t = torch.empty(B, max(K, 0), 3, dtype=torch.float32, device=dev)
    score = torch.empty(B, max(K, 0), dtype=torch.float32, device=dev)
    valid = torch.empty(B, max(K, 0), dtype=torch.uint8, device=dev)
    count = torch.empty(B, dtype=torch.int32, device=dev)
    _lib.call("sam6d_coarse_pick_distinct", Rt, top, scores, B, n1, n2, K, cos_thr, d2_min, R, t, score, valid, count)
    return R, t, score, valid, count


PICK_MAX_SYM = 2048             # symmetries per object that sam6d_coarse_pick_distinct_sym stages


def coarse_pick_distinct_sym(Rt: Tensor, top: Tensor, scores: Tensor, K: int, min_angle: float, min_dist: float, symR: Tensor,
                             symt: Tensor, sym_range: Tensor, radius: Tensor, max_count: Optional[int] = None):
    """coarse_pick_distinct with "distinct" read up to each proposal's symmetry set (the rule: include/sam6d_b200.h,
    sam6d_coarse_pick_distinct_sym).  symR (S,3,3) or (S,9), symt (S,3) f32 in metres, sym_range (B,2) i32 (offset, count) of
    each proposal's set, identity first; radius (B) f32 the forward's radius.  max_count: the largest count of any range
    (default min(S, PICK_MAX_SYM), enough for every set symmetry.pack_sets builds).  Same outputs as coarse_pick_distinct;
    with identity-only ranges they are its outputs bit for bit."""
    _check(Rt, torch.float32, "Rt", 3)
    _check(top, torch.int32, "top", 2)
    _check(scores, torch.float32, "scores", 2)
    _check(symR, torch.float32, "symR")
    _check(symt, torch.float32, "symt", 2)
    _check(sym_range, torch.int32, "sym_range", 2)
    _check(radius, torch.float32, "radius", 1)
    B, n1, _ = Rt.shape
    n2 = top.shape[1]
    S = symt.shape[0]
    if tuple(scores.shape) != (B, n2) or top.shape[0] != B:
        raise RuntimeError(f"coarse_pick_distinct_sym: Rt (B,n1,12), top and scores (B,n2), got {tuple(Rt.shape)}, {tuple(top.shape)}, "
                           f"{tuple(scores.shape)}")
    if symR.numel() != S * 9 or symt.shape[1] != 3 or tuple(sym_range.shape) != (B, 2) or tuple(radius.shape) != (B,):
        raise RuntimeError(f"coarse_pick_distinct_sym: symR (S,3,3), symt (S,3), sym_range (B,2), radius (B), got {tuple(symR.shape)}, "
                           f"{tuple(symt.shape)}, {tuple(sym_range.shape)}, {tuple(radius.shape)}")
    cos_thr, d2_min = hypothesis_thresholds(min_angle, min_dist)
    max_count = min(S, PICK_MAX_SYM) if max_count is None else int(max_count)
    dev = Rt.device
    K = int(K)
    R = torch.empty(B, max(K, 0), 3, 3, dtype=torch.float32, device=dev)
    t = torch.empty(B, max(K, 0), 3, dtype=torch.float32, device=dev)
    score = torch.empty(B, max(K, 0), dtype=torch.float32, device=dev)
    valid = torch.empty(B, max(K, 0), dtype=torch.uint8, device=dev)
    count = torch.empty(B, dtype=torch.int32, device=dev)
    _lib.call("sam6d_coarse_pick_distinct_sym", Rt, top, scores, B, n1, n2, K, cos_thr, d2_min, symR, symt, S, sym_range, max_count,
              radius, R, t, score, valid, count)
    return R, t, score, valid, count


# ---------------------------------------------------------------------------------------------- fine stage
def pe_mlp_max(pts: Tensor, idx: Tensor, cnt: Tensor, weights, out: Tensor, out_off: int):
    _check(pts, torch.float32, "pts", 3)
    _check(idx, torch.int32, "idx", 3)
    _check(cnt, torch.int32, "cnt", 2)
    B, N, _ = pts.shape
    ns = idx.shape[2]
    W1, B1, W2, B2, W3, B3 = weights
    _lib.call("sam6d_pe_mlp_max", pts, idx, cnt, B, N, ns, W1, B1, W2, B2, W3, B3, out, out.shape[-1], int(out_off))


def pe_mlp_max_tc(pts: Tensor, idx: Tensor, weights, out: Tensor, out_off: int):
    """tensor-core PE MLP; weights = (W1 f32, B1, W2 bf16, B2, W3 bf16, B3)"""
    _check(pts, torch.float32, "pts", 3)
    _check(idx, torch.int32, "idx", 3)
    B, N, _ = pts.shape
    ns = idx.shape[2]
    W1, B1, W2, B2, W3, B3 = weights
    _check(W2, torch.bfloat16, "W2", 2)
    _check(W3, torch.bfloat16, "W3", 2)
    if out.dtype not in (torch.float32, torch.bfloat16):
        raise RuntimeError("pe_mlp_max_tc: out must be float32 or bfloat16")
    _lib.call("sam6d_pe_mlp_max_tc", pts, idx, B, N, ns, W1, B1, W2, B2, W3, B3, out, int(out.dtype == torch.bfloat16), out.shape[-1],
              int(out_off))


def fine_assign(A: Tensor, pts2: Tensor, shift: float):
    """A: (B,S,S) fp32 as a [:, :, :S] view of a (B,S,ld) allocation with ld % 4 == 0 (the layout compute_feature_similarity
    writes: every row starts on a 16-byte boundary); a contiguous (B,S,S) tensor is re-laid out once."""
    if A.dim() != 3 or A.dtype != torch.float32 or not A.is_cuda:
        raise RuntimeError("atten must be a CUDA fp32 (B,S,S) tensor")
    _check(pts2, torch.float32, "pts2", 3)
    B, S, _ = A.shape
    if A.stride(2) != 1 or A.stride(0) != S * A.stride(1) or A.stride(1) % 4 or A.data_ptr() % 16:
        ld = (S + 3) // 4 * 4
        store = torch.empty(B, S, ld, dtype=torch.float32, device=A.device)
        store[:, :, :S] = A
        A = store[:, :, :S]
    ld = A.stride(1)
    dev = A.device
    tiles = (S + 31) // 32
    if tiles < 4:
        raise RuntimeError("fine_assign: S >= 97 required")
    rsum = torch.empty(B, ld, dtype=torch.float32, device=dev)
    csum = torch.empty(B, ld, dtype=torch.float32, device=dev)
    cpart = torch.empty(B, tiles, ld, dtype=torch.float32, device=dev)
    cpi = torch.empty(B, tiles, ld, dtype=torch.int32, device=dev)
    lab1 = torch.zeros(B, S, dtype=torch.int32, device=dev)
    lab2 = torch.zeros(B, S, dtype=torch.int32, device=dev)
    wts = torch.empty(B, S - 1, dtype=torch.float32, device=dev)
    pred = torch.empty(B, S - 1, 3, dtype=torch.float32, device=dev)
    _lib.call("sam6d_fine_assign", A, B, S, int(ld), shift, pts2, rsum, csum, cpart, cpi, lab1, lab2, wts, pred)
    return lab1, lab2, wts, pred


def fine_assign_tc(f1n: Tensor, f2n: Tensor, pts2: Tensor, alpha: float):
    """the assignment of compute_fine_Rt from the normalised bf16 tokens f1n (B,S,256) [scene, rows] and f2n (B,S,256) [template,
    columns] without forming the (B,S,S) score matrix: 4 wgmma passes (row sums, column sums, column labels, row labels +
    weighted correspondences).  alpha = 1/temp (also the softmax shift: cosine <= 1).  -> lab1 (B,S), lab2 (B,S), wts, pred"""
    _check(f1n, torch.bfloat16, "f1n", 3)
    _check(f2n, torch.bfloat16, "f2n", 3)
    _check(pts2, torch.float32, "pts2", 3)
    B, S, C = f1n.shape
    if C != 256 or f2n.shape != f1n.shape or pts2.shape[1] != S - 1:
        raise RuntimeError("fine_assign_tc: (B,S,256) tokens and (B,S-1,3) points expected")
    dev = f1n.device
    ld = (S + 3) // 4 * 4
    rinv = torch.empty(B, ld, dtype=torch.float32, device=dev)
    cinv = torch.empty(B, ld, dtype=torch.float32, device=dev)
    q4 = torch.empty(B, ld, 4, dtype=torch.float32, device=dev)
    lab1 = torch.zeros(B, S, dtype=torch.int32, device=dev)
    lab2 = torch.zeros(B, S, dtype=torch.int32, device=dev)
    wts = torch.empty(B, S - 1, dtype=torch.float32, device=dev)
    pred = torch.empty(B, S - 1, 3, dtype=torch.float32, device=dev)
    _lib.call("sam6d_fine_pass_tc", f1n, f2n, B, S, alpha, alpha, 0, None, None, ld, None, rinv, None, None, None)
    _lib.call("sam6d_fine_pass_tc", f2n, f1n, B, S, alpha, alpha, 0, None, None, ld, None, cinv, None, None, None)
    _lib.call("sam6d_fine_pass_tc", f2n, f1n, B, S, alpha, alpha, 1, cinv, rinv, ld, None, None, lab2, None, None)
    _lib.call("sam6d_fine_masked_points", lab2, pts2, B, S, ld, q4)
    _lib.call("sam6d_fine_pass_tc", f1n, f2n, B, S, alpha, alpha, 2, rinv, cinv, ld, q4, None, lab1, wts, pred)
    return lab1, lab2, wts, pred


def weighted_procrustes(src: Tensor, ref: Tensor, wts: Tensor, weight_thresh: float = 0.0, eps: float = 1e-5):
    _check(src, torch.float32, "src", 3)
    _check(ref, torch.float32, "ref", 3)
    _check(wts, torch.float32, "weights", 2)
    B, N, _ = src.shape
    R = torch.empty(B, 3, 3, dtype=torch.float32, device=src.device)
    t = torch.empty(B, 3, dtype=torch.float32, device=src.device)
    _lib.call("sam6d_weighted_procrustes", src, ref, wts, B, N, weight_thresh, eps, R, t)
    return R, t


def pose_score(pts1: Tensor, lab1: Tensor, R: Tensor, t: Tensor, model: Tensor, radius: Tensor, dis_thres: float = 0.15):
    _check(pts1, torch.float32, "pts1", 3)
    _check(lab1, torch.int32, "lab1", 2)
    B, N, _ = pts1.shape
    score = torch.empty(B, dtype=torch.float32, device=pts1.device)
    ts = torch.empty(B, 3, dtype=torch.float32, device=pts1.device)
    _lib.call("sam6d_pose_score", pts1, lab1, B, N, R, t, model, model.shape[1], dis_thres, radius, score, ts)
    return score, ts


# ---------------------------------------------------------------------------------------------- depth refinement
def icp_max_samples() -> int:
    """the largest number of samples per object icp_refine accepts on the current device"""
    m = _lib.lib().sam6d_icp_max_samples()
    if m < 0:
        raise _lib.Sam6dError(f"sam6d_icp_max_samples: CUDA error {-m}")
    return m


def icp_refine(R: Tensor, t: Tensor, pts: Tensor, samples: Tensor, normals: Tensor, obj: Tensor, radius: Tensor, iters: int,
               system: bool = False):
    """point-to-plane ICP of B poses against their observed points (the algorithm: include/sam6d_b200.h, sam6d_icp_refine).
    R (B,3,3), t (B,3), pts (B,N,3) f32 camera frame, metres; samples, normals (O,M,3) f32 object frame; obj (B) i32 object of
    each instance; radius (B) f32 -> (R, t refined, inliers (B) i32, rms (B) f32 metres, iters_run (B) i32).  An instance with
    an out-of-range obj or a non-positive radius comes back unrefined with inliers -1.  system=True also returns, of the last
    iteration evaluated, corr (B,N) i32 (j(i) of an inlier, -1 - j(i) of an outlier) and sums (B,29) f64 (the normal
    equations' upper triangle of A, b, the inlier count and sum e^2)."""
    _check(R, torch.float32, "R", 3)
    _check(t, torch.float32, "t", 2)
    _check(pts, torch.float32, "pts", 3)
    _check(samples, torch.float32, "samples", 3)
    _check(normals, torch.float32, "normals", 3)
    _check(obj, torch.int32, "obj", 1)
    _check(radius, torch.float32, "radius", 1)
    B, N, c = pts.shape
    O, M, cs = samples.shape
    if c != 3 or cs != 3 or normals.shape != samples.shape:
        raise RuntimeError(f"icp_refine: pts must be (B,N,3) and samples, normals (O,M,3), got {tuple(pts.shape)}, "
                           f"{tuple(samples.shape)}, {tuple(normals.shape)}")
    if R.shape != (B, 3, 3) or t.shape != (B, 3) or obj.shape != (B,) or radius.shape != (B,):
        raise RuntimeError(f"icp_refine: R (B,3,3), t (B,3), obj (B), radius (B) with B = {B}, got {tuple(R.shape)}, "
                           f"{tuple(t.shape)}, {tuple(obj.shape)}, {tuple(radius.shape)}")
    dev = pts.device
    R_out = torch.empty_like(R)
    t_out = torch.empty_like(t)
    inliers = torch.empty(B, dtype=torch.int32, device=dev)
    rms = torch.empty(B, dtype=torch.float32, device=dev)
    iters_run = torch.empty(B, dtype=torch.int32, device=dev)
    corr = torch.empty(B, N, dtype=torch.int32, device=dev) if system else None
    sums = torch.empty(B, 29, dtype=torch.float64, device=dev) if system else None
    _lib.call("sam6d_icp_refine", R, t, pts, B, N, samples, normals, O, M, obj, radius, int(iters), R_out, t_out, inliers, rms,
              iters_run, corr, sums)
    if system:
        return R_out, t_out, inliers, rms, iters_run, corr, sums
    return R_out, t_out, inliers, rms, iters_run


def track_points(rdepth: Tensor, depth: Tensor, depth_scale: float, K, centre: Tensor, radius: Tensor, margin: int, n: int,
                 return_index: bool = False):
    """observed points of O tracked objects (the rule: include/sam6d_b200.h, sam6d_track_points).  rdepth (O,H,W) f32 rendered
    depth (> 0 = silhouette), depth (H,W) u16 raw, depth_scale and K (3,3) host values (rounded to fp32), centre (O,3) and
    radius (O) f32 gate in metres, margin pixels -> (pts (O,n,3) f32 metres, count (O) i32, cand (O,H,W) u8 candidate mask),
    plus index (O,n) i32 (the pixel y W + x of every point, -1 for an object with no candidate) when return_index."""
    _check(rdepth, torch.float32, "rdepth", 3)
    _check(depth, torch.uint16, "depth", 2)
    _check(centre, torch.float32, "centre", 2)
    _check(radius, torch.float32, "radius", 1)
    O, H, W = rdepth.shape
    if tuple(depth.shape) != (H, W) or tuple(centre.shape) != (O, 3) or tuple(radius.shape) != (O,):
        raise RuntimeError(f"track_points: rdepth (O,H,W), depth (H,W), centre (O,3), radius (O) with (O,H,W) = {(O, H, W)}, got "
                           f"{tuple(depth.shape)}, {tuple(centre.shape)}, {tuple(radius.shape)}")
    if int(margin) < 0 or int(n) < 1:
        raise RuntimeError(f"track_points: margin must be >= 0 and n >= 1, got {margin}, {n}")
    k = np.asarray(K.cpu() if isinstance(K, torch.Tensor) else K, dtype=np.float64).reshape(3, 3).astype(np.float32)
    dev = rdepth.device
    hmask = torch.empty(O, H, W, dtype=torch.uint8, device=dev)
    cand = torch.empty(O, H, W, dtype=torch.uint8, device=dev)
    rows = torch.empty(O, H, dtype=torch.int32, device=dev)
    pts = torch.empty(O, int(n), 3, dtype=torch.float32, device=dev)
    count = torch.empty(O, dtype=torch.int32, device=dev)
    index = torch.empty(O, int(n), dtype=torch.int32, device=dev) if return_index else None
    _lib.call("sam6d_track_points", rdepth, depth, O, H, W, float(np.float32(depth_scale)), float(k[0, 0]), float(k[1, 1]), float(k[0, 2]),
              float(k[1, 2]), centre, radius, int(margin), int(n), hmask, cand, rows, pts, count, index)
    if return_index:
        return pts, count, cand, index
    return pts, count, cand


def track_points_scene(rdepth: Tensor, depth: Tensor, depth_scale: float, K, centre: Tensor, radius: Tensor, margin: int, n: int,
                       return_index: bool = False):
    """track_points over L live tracks of one scene, every pixel given to at most one track: the eligible track rendered in
    front, else the one nearest its gate centre relative to its radius (the rule: include/sam6d_b200.h,
    sam6d_track_points_scene).  Arguments and returns as track_points with O = L; with L = 1 the outputs are track_points'."""
    _check(rdepth, torch.float32, "rdepth", 3)
    _check(depth, torch.uint16, "depth", 2)
    _check(centre, torch.float32, "centre", 2)
    _check(radius, torch.float32, "radius", 1)
    L, H, W = rdepth.shape
    if tuple(depth.shape) != (H, W) or tuple(centre.shape) != (L, 3) or tuple(radius.shape) != (L,):
        raise RuntimeError(f"track_points_scene: rdepth (L,H,W), depth (H,W), centre (L,3), radius (L) with (L,H,W) = {(L, H, W)}, "
                           f"got {tuple(depth.shape)}, {tuple(centre.shape)}, {tuple(radius.shape)}")
    if int(margin) < 0 or int(n) < 1:
        raise RuntimeError(f"track_points_scene: margin must be >= 0 and n >= 1, got {margin}, {n}")
    k = np.asarray(K.cpu() if isinstance(K, torch.Tensor) else K, dtype=np.float64).reshape(3, 3).astype(np.float32)
    dev = rdepth.device
    hmask = torch.empty(L, H, W, dtype=torch.uint8, device=dev)
    dmask = torch.empty(L, H, W, dtype=torch.uint8, device=dev)
    cand = torch.empty(L, H, W, dtype=torch.uint8, device=dev)
    rows = torch.empty(L, H, dtype=torch.int32, device=dev)
    pts = torch.empty(L, int(n), 3, dtype=torch.float32, device=dev)
    count = torch.empty(L, dtype=torch.int32, device=dev)
    index = torch.empty(L, int(n), dtype=torch.int32, device=dev) if return_index else None
    _lib.call("sam6d_track_points_scene", rdepth, depth, L, H, W, float(np.float32(depth_scale)), float(k[0, 0]), float(k[1, 1]),
              float(k[0, 2]), float(k[1, 2]), centre, radius, int(margin), int(n), hmask, dmask, cand, rows, pts, count, index)
    if return_index:
        return pts, count, cand, index
    return pts, count, cand


# ---------------------------------------------------------------------------------------------- pose verification
VERIFY_COUNTS = ("n_sil", "n_occ", "n_fit", "n_viol", "n_mask", "n_mask_fit")
VERIFY_RENDER_BYTES = 1 << 28          # render outputs per chunk of hypotheses in verify_poses, at about 26 B per pixel


def verify_rows(mrow, tau, P: int, M: int):
    """mrow (P) and tau (P, or one number) as sam6d_pose_verify reads them -> host int32 and float32 arrays.  ValueError for an
    mrow outside [0, M) or a tau (after rounding to fp32) that is not finite or is <= 0."""
    mrow = np.asarray(mrow.cpu() if isinstance(mrow, Tensor) else mrow).reshape(-1)
    tau = np.asarray(tau.cpu() if isinstance(tau, Tensor) else tau, dtype=np.float64)
    tau = np.ascontiguousarray(np.broadcast_to(tau.reshape(-1) if tau.ndim else tau, (P,)), dtype=np.float32)
    if mrow.shape != (P,) or (P and not np.issubdtype(mrow.dtype, np.integer)):
        raise ValueError(f"verify: mrow must hold {P} integer mask rows, got {mrow.dtype} {mrow.shape}")
    if P and (mrow.min() < 0 or mrow.max() >= M):
        raise ValueError(f"verify: mrow must lie in [0, {M}), got [{mrow.min()}, {mrow.max()}]")
    if P and not (np.isfinite(tau).all() and (tau > 0).all()):
        raise ValueError("verify: every tau must be finite and > 0 in fp32")
    return np.ascontiguousarray(mrow, dtype=np.int32), tau


def _pose_verify(rdepth: Tensor, depth: Tensor, mask: Tensor, mrow: np.ndarray, tau: np.ndarray, rscale: float, counts: Tensor):
    P, H, W = rdepth.shape
    _lib.call("sam6d_pose_verify", rdepth, depth, mask, mrow.ctypes.data, tau.ctypes.data, P, mask.shape[0], H, W,
              float(np.float32(rscale)), counts)


def verify_counts(rdepth: Tensor, depth: Tensor, mask: Tensor, mrow, tau, rscale: float = 1e-3) -> Tensor:
    """depth agreement of P rendered hypotheses (the rule: include/sam6d_b200.h, sam6d_pose_verify).  rdepth (P,H,W) f32 in
    render units, rscale their factor to metres (rounded to fp32); depth (H,W) f32 metres; mask (M,H,W) u8; mrow (P) each
    hypothesis's mask row; tau (P) metres -> counts (P,6) i32 in the order of VERIFY_COUNTS"""
    _check(rdepth, torch.float32, "rdepth", 3)
    _check(depth, torch.float32, "depth", 2)
    _check(mask, torch.uint8, "mask", 3)
    P, H, W = rdepth.shape
    if tuple(depth.shape) != (H, W) or tuple(mask.shape[1:]) != (H, W):
        raise RuntimeError(f"verify_counts: rdepth (P,H,W), depth (H,W), mask (M,H,W) with (H,W) = {(H, W)}, got "
                           f"{tuple(depth.shape)}, {tuple(mask.shape)}")
    mrow, tau = verify_rows(mrow, tau, P, mask.shape[0])
    counts = torch.empty(P, 6, dtype=torch.int32, device=rdepth.device)
    _pose_verify(rdepth, depth, mask, mrow, tau, rscale, counts)
    return counts


def verify_score(counts: Tensor) -> Tensor:
    """counts (P,6) -> verify (P,) f32 = fit_frac x cover, fit_frac = n_fit / (n_fit + n_viol) and cover = n_mask_fit / n_mask,
    each 0 when its denominator is 0 (fp32; the counts are exact in fp32 up to 2^24 pixels)"""
    c = counts.to(torch.float32)
    seen, n_mask = c[:, 2] + c[:, 3], c[:, 4]
    fit_frac = torch.where(seen > 0, c[:, 2] / seen.clamp_min(1.0), torch.zeros_like(seen))
    cover = torch.where(n_mask > 0, c[:, 5] / n_mask.clamp_min(1.0), torch.zeros_like(n_mask))
    return fit_frac * cover


def verify_poses(R: Tensor, t: Tensor, obj, meshes, depth_m: Tensor, mask: Tensor, mrow, K, tau):
    """render every pose and count its depth agreement with the frame.  R (P,3,3), t (P,3) f32 metres object -> camera; obj (P)
    each hypothesis's index into meshes, CUDA meshes in mm (render.upload); depth_m (H,W) f32 metres (0 = invalid); mask
    (M,H,W) u8 and mrow (P) each hypothesis's mask row; K (3,3) host values; tau (P) tolerances in metres.  Each pose is one
    mesh entry with one view of render.render, translation t x 1000, in chunks that keep the render's outputs under
    VERIFY_RENDER_BYTES.  -> (counts (P,6) i32 as verify_counts, verify (P,) f32 = verify_score(counts))"""
    from . import render
    _check(R, torch.float32, "R", 3)
    _check(t, torch.float32, "t", 2)
    _check(depth_m, torch.float32, "depth_m", 2)
    _check(mask, torch.uint8, "mask", 3)
    P = R.shape[0]
    H, W = depth_m.shape
    if tuple(R.shape) != (P, 3, 3) or tuple(t.shape) != (P, 3) or tuple(mask.shape[1:]) != (H, W):
        raise RuntimeError(f"verify_poses: R (P,3,3), t (P,3), depth_m (H,W), mask (M,H,W), got {tuple(R.shape)}, {tuple(t.shape)}, "
                           f"{tuple(depth_m.shape)}, {tuple(mask.shape)}")
    obj = np.asarray(obj.cpu() if isinstance(obj, Tensor) else obj, dtype=np.int64).reshape(-1)
    if obj.shape != (P,) or (P and (obj.min() < 0 or obj.max() >= len(meshes))):
        raise ValueError(f"verify_poses: obj must hold {P} indices into {len(meshes)} meshes")
    mrow, tau = verify_rows(mrow, tau, P, mask.shape[0])
    dev = R.device
    counts = torch.empty(P, 6, dtype=torch.int32, device=dev)
    step = max(1, VERIFY_RENDER_BYTES // (26 * H * W))
    for p0 in range(0, P, step):
        p1 = min(P, p0 + step)
        poses = torch.zeros(p1 - p0, 1, 4, 4, dtype=torch.float32, device=dev)
        poses[:, 0, :3, :3] = R[p0:p1]
        poses[:, 0, :3, 3] = t[p0:p1] * 1000.0                                          # the meshes are in mm
        poses[:, 0, 3, 3] = 1.0
        rdepth = render.render([meshes[o] for o in obj[p0:p1]], poses, K, H, W)["depth"][:, 0].contiguous()
        _pose_verify(rdepth, depth_m, mask, mrow[p0:p1], tau[p0:p1], 1e-3, counts[p0:p1])
        del rdepth
    return counts, verify_score(counts)


# ---------------------------------------------------------------------------------------------- SAM encoder attention
def attn_relpos(qkv: Tensor, nW: int, Hs: int, Ws: int, nH: int, rel_h: Tensor, rel_w: Tensor, scale: float,
                out_dtype=torch.float32) -> Tensor:
    """qkv (nW*Hs*Ws, 3*nH*D) f32 -> (nW*Hs*Ws, nH*D) f32|bf16, head_dim D = 80 or 64"""
    _check(qkv, torch.float32, "qkv", 2)
    _check(rel_h, torch.float32, "rel_pos_h", 2)
    _check(rel_w, torch.float32, "rel_pos_w", 2)
    T, C3 = qkv.shape
    C = C3 // 3
    if T != nW * Hs * Ws or rel_h.shape[0] != 2 * Hs - 1 or rel_w.shape[0] != 2 * Ws - 1:
        raise RuntimeError("attn_relpos: shape mismatch")
    out = torch.empty(T, C, dtype=out_dtype, device=qkv.device)
    _lib.call("sam6d_attn_relpos", qkv, C3, int(nW), int(Hs), int(Ws), int(nH), C // nH, rel_h, rel_w, scale, out,
              int(out_dtype == torch.bfloat16), C)
    return out


# ---------------------------------------------------------------------------------------------- ISM scoring
def bilinear_gather(up: Tensor, choose: Tensor, G: int, sub: int, C: int, H: int, W: int) -> Tensor:
    """up (B, G*G, sub*sub*C) fp32|bf16, choose (B,K) int64 -> (B,K,C) fp32: bilinear (align_corners=False) samples of the
    (B,C,G*sub,G*sub) map the reference would upsample to (H,W), taken only at the chosen pixels"""
    if up.dtype not in (torch.float32, torch.bfloat16):
        raise RuntimeError("bilinear_gather: up must be float32 or bfloat16")
    _check(up, up.dtype, "up", 3)
    _check(choose, torch.int64, "choose", 2)
    B, K = choose.shape
    if up.shape != (B, G * G, sub * sub * C):
        raise RuntimeError("bilinear_gather: shape mismatch")
    out = torch.empty(B, K, C, dtype=torch.float32, device=up.device)
    _lib.call("sam6d_bilinear_gather", up, int(up.dtype == torch.bfloat16), choose, int(B), int(K), int(G), int(sub), int(C), int(H),
              int(W), out)
    return out


TEMPLATE_AGGREGATIONS = {"mean": 0, "median": 1, "max": 2, "avg_5": 3}     # csrc/ism.cu, matching_config.aggregation_function


def template_score(Qn: Tensor, Rn: Tensor, want_sim: bool = True, aggregation: str = "avg_5"):
    """Qn (P,C), Rn (O,T,C): F.normalize'd descriptors -> sim (P,O,T), obj_score (P,O), best_obj, best_score, best_tmpl.
    aggregation: how obj_score reduces the T similarities, one of TEMPLATE_AGGREGATIONS."""
    _check(Qn, torch.float32, "query", 2)
    _check(Rn, torch.float32, "reference", 3)
    if aggregation not in TEMPLATE_AGGREGATIONS:
        raise NotImplementedError(f"template aggregation {aggregation!r}: one of {sorted(TEMPLATE_AGGREGATIONS)}")
    P, C = Qn.shape
    O, T, _ = Rn.shape
    dev = Qn.device
    sim = torch.empty(P, O, T, dtype=torch.float32, device=dev) if want_sim else None
    obj = torch.empty(P, O, dtype=torch.float32, device=dev)
    obj_t = torch.empty(P, O, dtype=torch.int32, device=dev)
    bo = torch.zeros(P, dtype=torch.int32, device=dev)
    bs = torch.zeros(P, dtype=torch.float32, device=dev)
    bt = torch.zeros(P, dtype=torch.int32, device=dev)
    _lib.call("sam6d_template_score_agg", Qn, Rn, P, O, T, C, TEMPLATE_AGGREGATIONS[aggregation], sim, obj, obj_t, bo, bs, bt)
    return sim, obj, bo, bs, bt


# ---------------------------------------------------------------------------------------------- ISM -> PEM hand-off
def mask_rle(masks: Tensor) -> Tuple[Tensor, Tensor]:
    """masks (n,H,W) f32 (set iff > 0) -> (rle_cum, rle_off) int32 on the device: the cumulative run ends of every mask's
    uncompressed COCO RLE (mask_to_rle of the ISM CLI), concatenated, and the (n+1) offsets: the layout inputs.pack_rle builds.
    One 4-byte device-to-host copy (the total) sizes the output."""
    _check(masks, torch.float32, "masks", 3)
    n, H, W = masks.shape
    dev = masks.device
    col_cnt = torch.empty(n, W, dtype=torch.int32, device=dev)
    band_off = torch.empty(n, (W + 31) // 32, dtype=torch.int32, device=dev)
    rle_off = torch.empty(n + 1, dtype=torch.int32, device=dev)
    _lib.call("sam6d_mask_rle_count", masks, n, H, W, col_cnt, band_off, rle_off)
    rle_cum = torch.empty(int(rle_off[n]), dtype=torch.int32, device=dev)
    _lib.call("sam6d_mask_rle_write", masks, n, H, W, col_cnt, band_off, rle_off, rle_cum)
    return rle_cum, rle_off


# ---------------------------------------------------------------------------------------------- object symmetries (symmetry.py)
SYM_QUERY_CHUNK = 1024          # queries per CTA of sam6d_symmetry_agreement: its scratch holds one int and one float per chunk


def symmetry_agreement(Rt: Tensor, q: Tensor, tg: Tensor, geo_tol: float, color_tol: float = 0.0, qc: Optional[Tensor] = None,
                       tc: Optional[Tensor] = None):
    """C candidate transforms Rt (C,12) (R row-major, t) against query samples q (Nq,3) and target samples tg (M,3), with optional
    colours qc (Nq,3) and tc (M,3) in [0, 1] (the rule: include/sam6d_b200.h, sam6d_symmetry_agreement) -> count (C) i32, the
    queries whose nearest target is within geo_tol (and color_tol in colour), and sumsq (C) f32, their summed squared
    nearest-neighbour distances over all queries"""
    _check(Rt, torch.float32, "Rt", 2)
    _check(q, torch.float32, "q", 2)
    _check(tg, torch.float32, "tg", 2)
    if (qc is None) != (tc is None):
        raise RuntimeError("symmetry_agreement: colours for both sample sets or for neither")
    C, Nq, M = Rt.shape[0], q.shape[0], tg.shape[0]
    if Rt.shape[1] != 12 or q.shape[1] != 3 or tg.shape[1] != 3:
        raise RuntimeError(f"symmetry_agreement: Rt (C,12), q (Nq,3), tg (M,3), got {tuple(Rt.shape)}, {tuple(q.shape)}, {tuple(tg.shape)}")
    if qc is not None:
        _check(qc, torch.float32, "qc", 2)
        _check(tc, torch.float32, "tc", 2)
        if tuple(qc.shape) != (Nq, 3) or tuple(tc.shape) != (M, 3):
            raise RuntimeError(f"symmetry_agreement: qc (Nq,3), tc (M,3), got {tuple(qc.shape)}, {tuple(tc.shape)}")
    dev = Rt.device
    count = torch.empty(C, dtype=torch.int32, device=dev)
    sumsq = torch.empty(C, dtype=torch.float32, device=dev)
    work = torch.empty(max(C, 1) * ((Nq + SYM_QUERY_CHUNK - 1) // SYM_QUERY_CHUNK) * 2, dtype=torch.int32, device=dev)
    _lib.call("sam6d_symmetry_agreement", Rt, C, q, qc, Nq, tg, tc, M, float(geo_tol), float(color_tol), count, sumsq, work)
    return count, sumsq


def point_diameter(pts: Tensor) -> Tensor:
    """pts (V,3) f32 -> (1,) f32 the largest squared distance between two of them (sam6d_point_diameter; its square root is
    models_info's diameter)"""
    _check(pts, torch.float32, "pts", 2)
    if pts.shape[1] != 3:
        raise RuntimeError(f"point_diameter: pts (V,3), got {tuple(pts.shape)}")
    d2 = torch.empty(1, dtype=torch.float32, device=pts.device)
    _lib.call("sam6d_point_diameter", pts, pts.shape[0], d2)
    return d2


# ---------------------------------------------------------------------------------------------- TSDF fusion (fusion.py)
TSDF_MAX_DIM = 512              # voxels per side that sam6d_tsdf_integrate / sam6d_tsdf_mesh_* accept


def _tsdf_volume(tsdf: Tensor, weight: Tensor, csum: Tensor, ccount: Tensor):
    """the volume's four fields -> (nz, ny, nx).  csum holds the u32 colour sums in an int32 tensor (the same bits)."""
    _check(tsdf, torch.float32, "tsdf", 3)
    _check(weight, torch.int32, "weight", 3)
    _check(csum, torch.int32, "csum", 4)
    _check(ccount, torch.int32, "ccount", 3)
    dims = tuple(tsdf.shape)
    if tuple(weight.shape) != dims or tuple(ccount.shape) != dims or tuple(csum.shape) != dims + (3,):
        raise RuntimeError(f"tsdf volume: tsdf, weight, ccount (nz,ny,nx) and csum (nz,ny,nx,3), got {dims}, {tuple(weight.shape)}, "
                           f"{tuple(ccount.shape)}, {tuple(csum.shape)}")
    if min(dims) < 2 or max(dims) > TSDF_MAX_DIM:
        raise RuntimeError(f"tsdf volume: every side in [2, {TSDF_MAX_DIM}] voxels, got {dims}")
    return dims


def _tsdf_box(bbox_min, voxel: float):
    b = [float(x) for x in bbox_min]
    if len(b) != 3 or not all(math.isfinite(x) for x in b):
        raise RuntimeError(f"tsdf volume: bbox_min must be 3 finite numbers, got {bbox_min}")
    if not (math.isfinite(voxel) and voxel > 0):
        raise RuntimeError(f"tsdf volume: voxel must be finite and > 0, got {voxel}")
    return b


def tsdf_integrate(rgb: Tensor, depth: Tensor, mask: Optional[Tensor], K: Tensor, pose: Tensor, tsdf: Tensor, weight: Tensor,
                   csum: Tensor, ccount: Tensor, bbox_min, voxel: float, trunc: float, znear: float):
    """fuse T views into the volume in place (the rule: include/sam6d_b200.h, sam6d_tsdf_integrate).  rgb (T,H,W,3) u8, depth
    (T,H,W) f32 mm (0 = missing), mask (T,H,W) u8 or None, K (T,4) f32 fx, fy, cx, cy, pose (T,12) f32 object -> camera (R
    row-major, t mm); tsdf (nz,ny,nx) f32, weight i32, csum (nz,ny,nx,3) int32 holding u32 sums, ccount i32; bbox_min (3,)
    the lattice's lower corner in mm, voxel, trunc in mm"""
    nz, ny, nx = _tsdf_volume(tsdf, weight, csum, ccount)
    _check(rgb, torch.uint8, "rgb", 4)
    _check(depth, torch.float32, "depth", 3)
    _check(K, torch.float32, "K", 2)
    _check(pose, torch.float32, "pose", 2)
    T, H, W = depth.shape
    if T < 1 or H < 1 or W < 1 or tuple(rgb.shape) != (T, H, W, 3) or tuple(K.shape) != (T, 4) or tuple(pose.shape) != (T, 12):
        raise RuntimeError(f"tsdf_integrate: rgb (T,H,W,3), depth (T,H,W), K (T,4), pose (T,12) with T, H, W >= 1, got "
                           f"{tuple(rgb.shape)}, {tuple(depth.shape)}, {tuple(K.shape)}, {tuple(pose.shape)}")
    if mask is not None:
        _check(mask, torch.uint8, "mask", 3)
        if tuple(mask.shape) != (T, H, W):
            raise RuntimeError(f"tsdf_integrate: mask (T,H,W) = {(T, H, W)}, got {tuple(mask.shape)}")
    if not bool(torch.isfinite(pose).all()) or not bool(torch.isfinite(K).all()):
        raise RuntimeError("tsdf_integrate: K and pose must be finite")
    b = _tsdf_box(bbox_min, float(voxel))
    if not (math.isfinite(float(trunc)) and float(trunc) > 0) or not math.isfinite(float(znear)):
        raise RuntimeError(f"tsdf_integrate: trunc must be finite and > 0 and znear finite, got {trunc}, {znear}")
    _lib.call("sam6d_tsdf_integrate", rgb, depth, mask, K, pose, T, H, W, b[0], b[1], b[2], float(voxel), float(trunc), float(znear),
              nx, ny, nz, tsdf, weight, csum, ccount)


def tsdf_mesh(tsdf: Tensor, weight: Tensor, csum: Tensor, ccount: Tensor, bbox_min, voxel: float, min_weight: int = 1):
    """marching tetrahedra over the volume (the rule: include/sam6d_b200.h, sam6d_tsdf_mesh_count / _emit) -> (verts (V,3) f32 mm,
    colours (V,3) u8, faces (F,3) i32) on the device.  The prefix sums are torch.cumsum; one device-to-host copy reads the two
    totals that size the outputs."""
    nz, ny, nx = _tsdf_volume(tsdf, weight, csum, ccount)
    b = _tsdf_box(bbox_min, float(voxel))
    if int(min_weight) < 1:
        raise RuntimeError(f"tsdf_mesh: min_weight must be >= 1 (a corner no view saw has no distance), got {min_weight}")
    dev = tsdf.device
    N, ncube = nx * ny * nz, (nx - 1) * (ny - 1) * (nz - 1)
    emask = torch.empty(N, dtype=torch.int32, device=dev)
    vcount = torch.empty(N, dtype=torch.int32, device=dev)
    tcount = torch.empty(ncube, dtype=torch.int32, device=dev)
    _lib.call("sam6d_tsdf_mesh_count", tsdf, weight, nx, ny, nz, int(min_weight), emask, vcount, tcount)
    voff = torch.cumsum(vcount, 0, dtype=torch.int32)
    toff = torch.cumsum(tcount, 0, dtype=torch.int32)
    V, F = (int(x) for x in torch.stack([voff[-1], toff[-1]]).cpu())
    verts = torch.empty(V, 3, dtype=torch.float32, device=dev)
    cols = torch.empty(V, 3, dtype=torch.uint8, device=dev)
    faces = torch.empty(F, 3, dtype=torch.int32, device=dev)
    if V > 0 and F > 0:
        _lib.call("sam6d_tsdf_mesh_emit", tsdf, weight, csum, ccount, nx, ny, nz, b[0], b[1], b[2], float(voxel), int(min_weight),
                  emask, voff, toff, verts, cols, faces)
    return verts, cols, faces
