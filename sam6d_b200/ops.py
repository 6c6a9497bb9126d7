"""Tensor-level wrappers over the C ABI (include/sam6d_b200.h).

PyTorch is used here only as the owner of device memory and of the current CUDA stream; every function validates its
arguments the way the reference's native layer does (CUDA, contiguous, dtype -- PEM/model/pointnet2/_ext_src/include/utils.h:10-30
raise through TORCH_CHECK -> RuntimeError) and then hands raw pointers to libsam6d_b200.so.
"""
import ctypes
from typing import Optional, Tuple

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


def _p(t: Optional[Tensor]):
    return ctypes.c_void_p(0 if t is None else t.data_ptr())


def _s():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ll(v):
    return ctypes.c_longlong(int(v))


def _f(v):
    return ctypes.c_float(float(v))


# ---------------------------------------------------------------------------------------------- point-cloud ops
def furthest_point_sampling(xyz: Tensor, m: int) -> Tensor:
    """_ext.furthest_point_sampling: (B,N,3) f32 -> (B,m) i32."""
    _check(xyz, torch.float32, "points", 3)
    b, n, c = xyz.shape
    if c != 3:
        raise RuntimeError("points must be (B,N,3)")
    idx = torch.zeros(b, m, dtype=torch.int32, device=xyz.device)
    temp = torch.empty(b, n, dtype=torch.float32, device=xyz.device) if n > 4096 else None
    _lib.call("sam6d_fps", _p(xyz), b, n, int(m), _p(temp), _p(idx), _s())
    return idx


def furthest_point_sampling_single_cta(xyz: Tensor, m: int) -> Tensor:
    """the one-CTA general-n kernel (comparator of the cluster kernel that furthest_point_sampling uses for large clouds)"""
    _check(xyz, torch.float32, "points", 3)
    b, n, _ = xyz.shape
    idx = torch.zeros(b, m, dtype=torch.int32, device=xyz.device)
    temp = torch.empty(b, n, dtype=torch.float32, device=xyz.device)
    _lib.call("sam6d_fps_single_cta", _p(xyz), b, n, int(m), _p(temp), _p(idx), _s())
    return idx


def gather_points(points: Tensor, idx: Tensor) -> Tensor:
    """_ext.gather_points: (B,C,N) f32, (B,M) i32 -> (B,C,M)."""
    _check(points, torch.float32, "points", 3)
    _check(idx, torch.int32, "idx", 2)
    b, c, n = points.shape
    m = idx.shape[1]
    out = torch.zeros(b, c, m, dtype=torch.float32, device=points.device)
    _lib.call("sam6d_gather_points", _p(points), _p(idx), b, c, n, m, _p(out), _s())
    return out


def gather_rows(src: Tensor, idx: Tensor, n_rows: Optional[int] = None) -> Tensor:
    """channel-last gather: src (B,N,C) f32, idx (B,M) i32 -> (B,M,C)."""
    _check(src, torch.float32, "src", 3)
    _check(idx, torch.int32, "idx", 2)
    b, n, c = src.shape
    m = idx.shape[1]
    out = torch.empty(b, m, c, dtype=torch.float32, device=src.device)
    _lib.call("sam6d_gather_rows", _p(src), _p(idx), b, n, m, c, _ll(n * c), _p(out), _s())
    return out


def ball_query(new_xyz: Tensor, xyz: Tensor, radius: float, nsample: int, return_count: bool = False):
    """_ext.ball_query: new_xyz (B,M,3), xyz (B,N,3) -> (B,M,nsample) i32 [, count (B,M) i32]."""
    _check(new_xyz, torch.float32, "new_xyz", 3)
    _check(xyz, torch.float32, "xyz", 3)
    b, m, _ = new_xyz.shape
    n = xyz.shape[1]
    idx = torch.zeros(b, m, nsample, dtype=torch.int32, device=xyz.device)
    cnt = torch.zeros(b, m, dtype=torch.int32, device=xyz.device) if return_count else None
    _lib.call("sam6d_ball_query", _p(new_xyz), _p(xyz), b, n, m, _f(radius), int(nsample), _p(idx), _p(cnt), _s())
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
    _lib.call("sam6d_ball_query_pair", _p(new_xyz), _p(xyz), b, n, m, _f(ra), int(nsa), _f(rb), int(nsb), _p(ia), _p(ib), _p(ca),
              _p(cb), _s())
    return ia, ca, ib, cb


def group_points(points: Tensor, idx: Tensor) -> Tensor:
    """_ext.group_points: (B,C,N) f32, (B,np,ns) i32 -> (B,C,np,ns)."""
    _check(points, torch.float32, "points", 3)
    _check(idx, torch.int32, "idx", 3)
    b, c, n = points.shape
    _, npnt, ns = idx.shape
    out = torch.zeros(b, c, npnt, ns, dtype=torch.float32, device=points.device)
    _lib.call("sam6d_group_points", _p(points), _p(idx), b, c, n, npnt, ns, _p(out), _s())
    return out


# ---------------------------------------------------------------------------------------------- dense algebra
def gemm(A: Tensor, W: Tensor, bias: Optional[Tensor] = None, residual: Optional[Tensor] = None,
         out: Optional[Tensor] = None, relu=False, alpha: float = 1.0) -> Tensor:
    """out = alpha * A @ W^T (+bias) (act) (+residual); A (M,K), W (N,K) contiguous f32.  relu: False/True or the activation
    code (0 none, 1 ReLU, 2 GELU)."""
    _check(A, torch.float32, "A", 2)
    _check(W, torch.float32, "W", 2)
    M, K = A.shape
    N = W.shape[0]
    if W.shape[1] != K:
        raise RuntimeError("gemm: inner dimensions differ")
    if out is None:
        out = torch.empty(M, N, dtype=torch.float32, device=A.device)
    _lib.call("sam6d_gemm_f32", _p(A), _p(W), _p(bias), _p(residual), _p(out), M, N, K, _ll(K), _ll(K), _ll(N), _ll(N),
              1, _ll(0), _ll(0), _ll(0), _ll(0), _f(alpha), int(relu), _s())
    return out


def gemm_raw(A_ptr, W_ptr, bias, R_ptr, C_ptr, M, N, K, lda, ldw, ldc, ldr, batch=1, sA=0, sW=0, sC=0, sR=0,
             alpha=1.0, relu=False):
    """strided / batched form over raw device addresses (ints)."""
    _lib.call("sam6d_gemm_f32", ctypes.c_void_p(A_ptr), ctypes.c_void_p(W_ptr), _p(bias), ctypes.c_void_p(R_ptr or 0),
              ctypes.c_void_p(C_ptr), int(M), int(N), int(K), _ll(lda), _ll(ldw), _ll(ldc), _ll(ldr), int(batch), _ll(sA),
              _ll(sW), _ll(sC), _ll(sR), _f(alpha), int(relu), _s())


_DT = {torch.float32: 0, torch.bfloat16: 1}


def gemm_tc_raw(A_ptr, a_dt, W_ptr, w_dt, bias, R_ptr, C_ptr, c_dt, M, N, K, lda, ldw, ldc, ldr, batch=1, sA=0, sW=0, sC=0, sR=0,
                alpha=1.0, relu=False):
    """wgmma bf16 GEMM over raw device addresses; *_dt: 0 = fp32, 1 = bf16"""
    _lib.call("sam6d_gemm_bf16", ctypes.c_void_p(A_ptr), int(a_dt), ctypes.c_void_p(W_ptr), int(w_dt), _p(bias),
              ctypes.c_void_p(R_ptr or 0), ctypes.c_void_p(C_ptr), int(c_dt), int(M), int(N), int(K), _ll(lda), _ll(ldw), _ll(ldc),
              _ll(ldr), int(batch), _ll(sA), _ll(sW), _ll(sC), _ll(sR), _f(alpha), int(relu), _s())


def gemm_tc(A: Tensor, W: Tensor, bias: Optional[Tensor] = None, residual: Optional[Tensor] = None, out: Optional[Tensor] = None,
            relu: bool = False, alpha: float = 1.0, out_dtype=torch.float32) -> Tensor:
    """tensor-core form of gemm(): A (M,K) fp32|bf16, W (N,K) fp32|bf16 -> (M,N) fp32|bf16, fp32 accumulate"""
    for t, n in ((A, "A"), (W, "W")):
        if t.dtype not in _DT:
            raise RuntimeError(f"{n} must be float32 or bfloat16")
        _check(t, t.dtype, n, 2)
    M, K = A.shape
    N = W.shape[0]
    if W.shape[1] != K:
        raise RuntimeError("gemm: inner dimensions differ")
    if out is None:
        out = torch.empty(M, N, dtype=out_dtype, device=A.device)
    gemm_tc_raw(A.data_ptr(), _DT[A.dtype], W.data_ptr(), _DT[W.dtype], bias, residual.data_ptr() if residual is not None else 0,
                out.data_ptr(), _DT[out.dtype], M, N, K, K, K, N, N, alpha=alpha, relu=relu)
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
    _lib.call("sam6d_gemm_tma", _p(A), _p(W), _p(bias), _p(residual), _p(out), _DT[out.dtype], M, N, K, _ll(K), _ll(K), _ll(Nout), _ll(N),
              _f(alpha), int(act), _s())
    return out


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
    _lib.call("sam6d_gemm_tma_vt", _p(A), _p(W), _p(bias), _p(out), M, N, K, _ll(K), _ll(K), _ll(vt_col0), _p(vt), int(vt_col0), int(S),
              int(n1), _s())
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
    _lib.call("sam6d_gemm_tma_vt2", _p(A), _p(W), _p(bias), _p(out), M, N, K, _ll(K), _ll(K), _ll(vt_col0), _p(vt), int(vt_col0),
              int(vt_col1), int(S), int(n1), _p(out2), _ll(N - vt_col1), _s())
    return out, vt, out2


def layernorm_raw(x_ptr, x_view, y_ptr, y_view, gamma: Tensor, beta: Tensor, rows: int, C: int, eps: float = 1e-5):
    _lib.call("sam6d_layernorm", ctypes.c_void_p(x_ptr), _ll(x_view[0]), _ll(x_view[1]), _ll(x_view[2]),
              ctypes.c_void_p(y_ptr), _ll(y_view[0]), _ll(y_view[1]), _ll(y_view[2]), _p(gamma), _p(beta), _ll(rows), int(C),
              _f(eps), _s())


def layernorm(x: Tensor, gamma: Tensor, beta: Tensor, eps: float = 1e-5, out: Optional[Tensor] = None) -> Tensor:
    _check(x, torch.float32, "x")
    C = x.shape[-1]
    rows = x.numel() // C
    if out is None:
        out = torch.empty_like(x)
    layernorm_raw(x.data_ptr(), (rows, 0, C), out.data_ptr(), (rows, 0, C), gamma, beta, rows, C, eps)
    return out


def layernorm_bf16(x: Tensor, gamma: Tensor, beta: Tensor, eps: float = 1e-5) -> Tensor:
    """LayerNorm with bf16 output rows (feeds the TMA GEMM directly)"""
    _check(x, torch.float32, "x")
    C = x.shape[-1]
    rows = x.numel() // C
    out = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    _lib.call("sam6d_layernorm_bf16", _p(x), _ll(rows), _ll(0), _ll(C), _p(out), _ll(rows), _ll(0), _ll(C), _p(gamma), _p(beta),
              _ll(rows), int(C), _f(eps), _s())
    return out


def layernorm_bf16io(x: Tensor, gamma: Tensor, beta: Tensor, eps: float = 1e-5, out: Optional[Tensor] = None) -> Tensor:
    """LayerNorm over the last dim of contiguous bf16 rows, bf16 result (statistics in fp32)"""
    _check(x, torch.bfloat16, "x")
    C = x.shape[-1]
    rows = x.numel() // C
    if out is None:
        out = torch.empty_like(x)
    _lib.call("sam6d_layernorm_bf16io", _p(x), _ll(max(rows, 1)), _ll(0), _ll(C), _p(out), _ll(max(rows, 1)), _ll(0), _ll(C),
              _p(gamma), _p(beta), _ll(rows), int(C), _f(eps), _s())
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
    _lib.call("sam6d_transformer_tail_bf16", _p(hid), _ll(256), _p(x), _ll(256), _p(wo), _p(bo), _p(g1), _p(b1), _p(we), _p(be), _p(ws),
              _p(bs), _p(g2), _p(b2), _p(out), _ll(256), int(M), _f(eps), _s())
    return out


def gather_rows_bf16_f32(src: Tensor, idx: Tensor) -> Tensor:
    """out[b,j,:] = float(src[b, idx[b,j], :]) for a bf16 (b,n,c) token matrix; negative index -> zero row"""
    _check(src, torch.bfloat16, "src", 3)
    _check(idx, torch.int32, "idx", 2)
    b, n, c = src.shape
    m = idx.shape[1]
    out = torch.empty(b, m, c, dtype=torch.float32, device=src.device)
    _lib.call("sam6d_gather_rows_bf16_f32", _p(src), _p(idx), b, n, m, c, _ll(n * c), _p(out), _s())
    return out


def gather_rows_bf16(src: Tensor, idx: Tensor) -> Tensor:
    """channel-last gather of bf16 rows (C even): moved as C/2 32-bit words by the fp32 gather kernel"""
    _check(src, torch.bfloat16, "src", 3)
    _check(idx, torch.int32, "idx", 2)
    b, n, c = src.shape
    m = idx.shape[1]
    out = torch.empty(b, m, c, dtype=torch.bfloat16, device=src.device)
    _lib.call("sam6d_gather_rows", _p(src), _p(idx), b, n, m, c // 2, _ll(n * c // 2), _p(out), _s())
    return out


def l2norm_rows(x: Tensor) -> Tensor:
    _check(x, torch.float32, "x")
    C = x.shape[-1]
    rows = x.numel() // C
    out = torch.empty_like(x)
    _lib.call("sam6d_l2norm_rows", _p(x), _ll(rows), _ll(0), _ll(C), _p(out), _ll(rows), _ll(0), _ll(C), _ll(rows), C, _s())
    return out


def l2norm_rows_bf16(x: Tensor) -> Tensor:
    """F.normalize(x, dim=-1) with a bf16 result (operand of the tensor-core score GEMM)"""
    _check(x, torch.float32, "x")
    C = x.shape[-1]
    rows = x.numel() // C
    out = torch.empty(x.shape, dtype=torch.bfloat16, device=x.device)
    _lib.call("sam6d_l2norm_rows_bf16", _p(x), _ll(max(rows, 1)), _ll(0), _ll(C), _p(out), _ll(max(rows, 1)), _ll(0), _ll(C), _ll(rows), C,
              _s())
    return out


def gemm_tma_batched(A: Tensor, W: Tensor, out: Tensor, M: int, N: int, ldc: int, c_bs: int, alpha: float = 1.0,
                     bias: Optional[Tensor] = None, residual: Optional[Tensor] = None, ldr: int = 0, r_bs: int = 0) -> Tensor:
    """A (batch, a_rows, K) bf16; W (batch, w_rows, K) bf16 or one shared (N, K) matrix ->
    out[z, :M, :N] = alpha * A[z,:M] @ W[z,:N]^T (+ bias) (+ residual[z]) for every z, written with row stride ldc and problem
    stride c_bs (elements) into `out` (fp32 or bf16; the residual has out's element type, row stride ldr, problem stride r_bs)"""
    _check(A, torch.bfloat16, "A", 3)
    _check(W, torch.bfloat16, "W")
    batch, a_rows, K = A.shape
    shared = W.dim() == 2
    if W.shape[-1] != K or a_rows < M or (not shared and (W.shape[0] != batch or W.shape[1] < N)) or (shared and W.shape[0] != N):
        raise RuntimeError("gemm_tma_batched: shape mismatch")
    if residual is not None and residual.dtype != out.dtype:
        raise RuntimeError("gemm_tma_batched: the residual must have the output's element type")
    _lib.call("sam6d_gemm_tma_batched", _p(A), _p(W), _p(bias), _p(residual), _p(out), _DT[out.dtype], int(M), int(N), int(K), _ll(K),
              _ll(K), _ll(ldc), _ll(ldr), int(batch), _ll(a_rows), _ll(0 if shared else W.shape[1]), _ll(c_bs), _ll(r_bs), _f(alpha), 0,
              _s())
    return out


def focus_rows_raw(x_ptr, x_view, y_ptr, y_view, sp_scale: Tensor, rows: int, C: int):
    _lib.call("sam6d_focus_rows", ctypes.c_void_p(x_ptr), _ll(x_view[0]), _ll(x_view[1]), _ll(x_view[2]),
              ctypes.c_void_p(y_ptr), _ll(y_view[0]), _ll(y_view[1]), _ll(y_view[2]), _p(sp_scale), _ll(rows), int(C), _s())


def rigid_warp(p: Tensor, R: Tensor, t: Tensor) -> Tensor:
    _check(p, torch.float32, "p", 3)
    _check(R, torch.float32, "R", 3)
    _check(t, torch.float32, "t", 2)
    out = torch.empty_like(p)
    _lib.call("sam6d_rigid_warp", _p(p), _p(R), _p(t), p.shape[0], p.shape[1], _p(out), _s())
    return out


def cloud_radius(po: Tensor) -> Tensor:
    _check(po, torch.float32, "dense_po", 3)
    r = torch.empty(po.shape[0], dtype=torch.float32, device=po.device)
    _lib.call("sam6d_cloud_radius", _p(po), po.shape[0], po.shape[1], _p(r), _s())
    return r


def scale_by_radius(x: Tensor, radius: Tensor) -> Tensor:
    _check(x, torch.float32, "x")
    _check(radius, torch.float32, "radius", 1)
    out = torch.empty_like(x)
    b = x.shape[0]
    _lib.call("sam6d_scale_by_radius", _p(x), _p(radius), b, _ll(x.numel() // max(b, 1)), _p(out), _s())
    return out


# ---------------------------------------------------------------------------------------------- geometric embedding
def geo_indices(pts: Tensor, sigma_d: float, factor_a: float) -> Tensor:
    _check(pts, torch.float32, "points", 3)
    b, s, _ = pts.shape
    T = torch.empty(b, s, s, 4, dtype=torch.float32, device=pts.device)
    _lib.call("sam6d_geo_indices", _p(pts), b, s, _f(sigma_d), _f(factor_a), _p(T), _s())
    return T


def geo_embed_f32(T: Tensor, div_term: Tensor, WaT: Tensor, WdT: Tensor, bias: Tensor) -> Tensor:
    _check(T, torch.float32, "T", 4)
    b, s, _, _ = T.shape
    E = torch.empty(b, s, s, 256, dtype=torch.float32, device=T.device)
    _lib.call("sam6d_geo_embed_f32", _p(T), _ll(b * s * s), _p(div_term), _p(WaT), _p(WdT), _p(bias), _p(E), _s())
    return E


def geo_embed_tc(T: Tensor, div_term: Tensor, Wa_bf16: Tensor, Wd_bf16: Tensor, bias: Tensor, out_dtype=torch.bfloat16) -> Tensor:
    """wgmma version: weights (out,in) bf16, E (B,S,S,256) fp32 or bf16"""
    _check(T, torch.float32, "T", 4)
    _check(Wa_bf16, torch.bfloat16, "Wa", 2)
    _check(Wd_bf16, torch.bfloat16, "Wd", 2)
    b, s, _, _ = T.shape
    E = torch.empty(b, s, s, 256, dtype=out_dtype, device=T.device)
    _lib.call("sam6d_geo_embed_tc", _p(T), _ll(b * s * s), _p(div_term), _p(Wa_bf16), _p(Wd_bf16), _p(bias), _p(E),
              int(out_dtype == torch.bfloat16), _s())
    return E


def geo_embed_dist_tc(T: Tensor, div_term: Tensor, Wd_bf16: Tensor, bias: Tensor) -> Tensor:
    """distance projection only: T (..., 4) f32 -> (..., 256) bf16 = proj_d(emb(T[..., 3])) + bias (wgmma)"""
    if T.dtype != torch.float32 or not T.is_cuda or not T.is_contiguous() or T.shape[-1] != 4:
        raise RuntimeError("T must be a contiguous CUDA float32 tensor (..., 4)")
    _check(Wd_bf16, torch.bfloat16, "Wd", 2)
    n = T.numel() // 4
    E = torch.empty(*T.shape[:-1], 256, dtype=torch.bfloat16, device=T.device)
    _lib.call("sam6d_geo_embed_dist_tc", _p(T), _ll(n), _p(div_term), _p(Wd_bf16), _p(bias), _p(E), _s())
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
    _lib.call("sam6d_geo_embed_lut", _p(T), _ll(b), s, _p(tabA), tabA.shape[0], _f(inv_ha), _p(tabD), tabD.shape[0], _f(inv_hd), _p(far),
              _p(div_term), _p(WdT_bf16), _p(bias), _p(E), _s())
    return E


# ---------------------------------------------------------------------------------------------- attention
def rpe_scores(E: Tensor, U: Tensor, u_ptr: Optional[int] = None, u_ld: int = 1024) -> Tensor:
    """E (B,S,S,256) f32|bf16, U (B,S,4,256) f32 (or a raw address + row stride) -> (B,4,S,S) f32."""
    if E.dtype not in (torch.float32, torch.bfloat16):
        raise RuntimeError("E must be float32 or bfloat16")
    _check(E, E.dtype, "E", 4)
    if u_ptr is None:
        _check(U, torch.float32, "U", 4)
        u_ptr = U.data_ptr()
    B, S = E.shape[0], E.shape[1]
    SP = torch.empty(B, 4, S, S, dtype=torch.float32, device=E.device)
    _lib.call("sam6d_rpe_scores", _p(E), int(E.dtype == torch.bfloat16), ctypes.c_void_p(u_ptr), _ll(u_ld), B, S, _p(SP), _s())
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
    _lib.call("sam6d_rpe_scores_tc_ld", _p(E), _p(U), B, S, _p(SP), int(ld), _s())
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
    _lib.call("sam6d_attn_tc_bias_ld", _p(Q), _ll(Q.shape[1]), int(q_col0), _p(K), _ll(K.shape[1]), int(k_col0), _p(Vt), _ll(Vt.shape[1]),
              int(B), int(H), int(Sq), int(Sk), int(D), _p(bias), _ll(bias.shape[3]), _f(scale), _p(out),
              int(out_dtype == torch.bfloat16), _ll(H * D), _s())
    return out


def mha_raw(q_ptr, q_ld, q_bs, k_ptr, k_ld, k_bs, v_ptr, v_ld, v_bs, bias: Optional[Tensor], B, H, Sq, Sk, scale,
            o_ptr, o_ld, o_bs):
    _lib.call("sam6d_mha", ctypes.c_void_p(q_ptr), _ll(q_ld), _ll(q_bs), ctypes.c_void_p(k_ptr), _ll(k_ld), _ll(k_bs),
              ctypes.c_void_p(v_ptr), _ll(v_ld), _ll(v_bs), _p(bias), int(B), int(H), int(Sq), int(Sk), _f(scale),
              ctypes.c_void_p(o_ptr), _ll(o_ld), _ll(o_bs), _s())


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
    _lib.call("sam6d_attn_global_tc_ex", _p(qkv), _ll(qkv.shape[1]), _p(vt), _ll(vt.shape[1]), _p(rel_blob), int(B), int(H), int(grid),
              int(D), _f(scale), _p(out), int(out_dtype == torch.bfloat16), _ll(H * D), _s())
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
    _lib.call("sam6d_attn_tc", _p(Q), _ll(Q.shape[1]), int(q_col0), _p(K), _ll(K.shape[1]), int(k_col0), _p(Vt), _ll(Vt.shape[1]),
              int(B), int(H), int(Sq), int(Sk), int(D), mode, _p(bias), _p(rh), _p(rw), int(Hs), int(Ws), _p(bv), _f(scale), _p(out),
              int(out_dtype == torch.bfloat16), _ll(H * D), _s())
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
    _lib.call("sam6d_attn_tc_ex", _p(Q), _ll(Q.shape[1]), int(q_col0), _p(K), _ll(K.shape[1]), int(k_col0), _p(Vt), _ll(Vt.shape[1]),
              int(B), int(H), int(Sq), int(Sk), int(D), _f(scale), int(k_brows), int(k_row0), int(v_col0), _p(lse), _p(out),
              int(out_dtype == torch.bfloat16), _ll(H * D), _s())
    return out, lse


def attn_merge_key(Q: Tensor, q_col0: int, K: Tensor, k_col0: int, k_brows: int, key_row: int, Vt: Tensor, key_col: int, lse: Tensor,
                   B: int, H: int, Sq: int, scale: float, out: Tensor) -> Tensor:
    """folds one more key (row key_row of every batch's K rows, column key_col of its V^T rows) into the bf16 result `out` of
    attn_tc_ex (head dim 64), in place"""
    _check(out, torch.bfloat16, "out", 2)
    _check(lse, torch.float32, "lse", 3)
    _lib.call("sam6d_attn_merge_key", _p(Q), _ll(Q.shape[1]), int(q_col0), _p(K), _ll(K.shape[1]), int(k_col0), int(k_brows), int(key_row),
              _p(Vt), _ll(Vt.shape[1]), int(key_col), _p(lse), int(B), int(H), int(Sq), _f(scale), _p(out), _ll(out.shape[1]), _s())
    return out


def transpose_tokens(src: Tensor, col0: int, C: int, nB: int, L: int) -> Tensor:
    """V^T for attn_tc: src bf16 (nB*L, ld) -> (nB*C, ceil16(L)) bf16, zero padded keys"""
    _check(src, torch.bfloat16, "src", 2)
    N1 = (L + 15) // 16 * 16
    out = torch.empty(nB * C, N1, dtype=torch.bfloat16, device=src.device)
    _lib.call("sam6d_transpose_tokens_bf16", _p(src), _ll(src.shape[1]), int(col0), int(C), int(nB), int(L), int(N1), _p(out), _s())
    return out


def linattn_kv_raw(k_ptr, k_ld, k_bs, v_ptr, v_ld, v_bs, B, H, J, KV: Tensor, KS: Tensor):
    _lib.call("sam6d_linattn_kv", ctypes.c_void_p(k_ptr), _ll(k_ld), _ll(k_bs), ctypes.c_void_p(v_ptr), _ll(v_ld), _ll(v_bs),
              int(B), int(H), int(J), _p(KV), _p(KS), _s())


def linattn_apply_raw(q_ptr, q_rpb, q_bs, q_ld, KV: Tensor, KS: Tensor, B, H, x_ptr, x_bs, x_ld):
    _lib.call("sam6d_linattn_apply", ctypes.c_void_p(q_ptr), _ll(q_rpb), _ll(q_bs), _ll(q_ld), _p(KV), _p(KS), int(B), int(H),
              ctypes.c_void_p(x_ptr), _ll(x_bs), _ll(x_ld), _s())


# ---------------------------------------------------------------------------------------------- coarse pose
def linattn_kv_pack_raw(k_ptr, k_ld, k_bs, v_ptr, v_ld, v_bs, B, J, device):
    """focused keys / values ((B,J,256) fp32 views) -> (blob: B x 32 KB bf16 wgmma image of KV_h^T, KS (B,4,64) fp32)"""
    blob = torch.empty(B, 4 * 64 * 64, dtype=torch.bfloat16, device=device)
    KS = torch.empty(B, 4, 64, dtype=torch.float32, device=device)
    _lib.call("sam6d_linattn_kv_pack", ctypes.c_void_p(k_ptr), _ll(k_ld), _ll(k_bs), ctypes.c_void_p(v_ptr), _ll(v_ld), _ll(v_bs),
              int(B), int(J), _p(blob), _p(KS), _s())
    return blob, KS


def linattn_tc_raw(q_ptr, q_ld, q_bs, blob: Tensor, KS: Tensor, sp_scale: Tensor, B, rpb, x_ptr, x_ld, x_bs):
    """dense tokens (bf16): focusing feature map + per-head (q' KV) / (q' . ksum) on wgmma"""
    _lib.call("sam6d_linattn_tc", ctypes.c_void_p(q_ptr), _ll(q_ld), _ll(q_bs), _p(blob), _p(KS), _p(sp_scale), int(B), int(rpb),
              ctypes.c_void_p(x_ptr), _ll(x_ld), _ll(x_bs), _s())


def coarse_assign(A: Tensor) -> Tuple[Tensor, Tensor]:
    _check(A, torch.float32, "atten", 3)
    B, S, _ = A.shape
    n = S - 1
    W = torch.empty(B, n * n, dtype=torch.float32, device=A.device)
    w1 = torch.empty(B, n, dtype=torch.float32, device=A.device)
    _lib.call("sam6d_coarse_assign", _p(A), B, S, _p(W), _p(w1), _s())
    return W, w1


def coarse_sample(W: Tensor, rand: Tensor) -> Tensor:
    _check(W, torch.float32, "W", 2)
    _check(rand, torch.float32, "rand", 2)
    B, L = W.shape
    nr = rand.shape[1]
    idx = torch.empty(B, nr, dtype=torch.int32, device=W.device)
    _lib.call("sam6d_coarse_sample", _p(W), B, L, _p(rand), nr, _p(idx), _s())
    return idx


def coarse_hypotheses(idx: Tensor, pts1: Tensor, pts2: Tensor) -> Tuple[Tensor, Tensor]:
    _check(idx, torch.int32, "idx", 2)
    _check(pts1, torch.float32, "pts1", 3)
    _check(pts2, torch.float32, "pts2", 3)
    B, n, _ = pts1.shape
    n1 = idx.shape[1] // 3
    Rt = torch.empty(B, n1, 12, dtype=torch.float32, device=idx.device)
    resid = torch.empty(B, n1, dtype=torch.float32, device=idx.device)
    _lib.call("sam6d_coarse_hypotheses", _p(idx), _p(pts1), _p(pts2), B, n, n1, _p(Rt), _p(resid), _s())
    return Rt, resid


def topk_smallest(v: Tensor, k: int) -> Tensor:
    _check(v, torch.float32, "v", 2)
    B, n = v.shape
    out = torch.empty(B, k, dtype=torch.int32, device=v.device)
    _lib.call("sam6d_topk_smallest", _p(v), B, n, int(k), _p(out), _s())
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
    _lib.call("sam6d_coarse_select", _p(Rt), _p(top), B, n1, n2, _p(pts1), _p(w1), n, _p(model), model.shape[1], _p(scores),
              _p(R), _p(t), _s())
    return R, t, scores


# ---------------------------------------------------------------------------------------------- fine stage
def pe_mlp_max(pts: Tensor, idx: Tensor, cnt: Tensor, weights, out: Tensor, out_off: int):
    _check(pts, torch.float32, "pts", 3)
    _check(idx, torch.int32, "idx", 3)
    _check(cnt, torch.int32, "cnt", 2)
    B, N, _ = pts.shape
    ns = idx.shape[2]
    W1, B1, W2, B2, W3, B3 = weights
    _lib.call("sam6d_pe_mlp_max", _p(pts), _p(idx), _p(cnt), B, N, ns, _p(W1), _p(B1), _p(W2), _p(B2), _p(W3), _p(B3),
              _p(out), out.shape[-1], int(out_off), _s())


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
    _lib.call("sam6d_pe_mlp_max_tc", _p(pts), _p(idx), B, N, ns, _p(W1), _p(B1), _p(W2), _p(B2), _p(W3), _p(B3), _p(out),
              int(out.dtype == torch.bfloat16), out.shape[-1], int(out_off), _s())


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
    _lib.call("sam6d_fine_assign", _p(A), B, S, int(ld), _f(shift), _p(pts2), _p(rsum), _p(csum), _p(cpart), _p(cpi), _p(lab1),
              _p(lab2), _p(wts), _p(pred), _s())
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
    a, sh = _f(alpha), _f(alpha)
    _lib.call("sam6d_fine_pass_tc", _p(f1n), _p(f2n), B, S, a, sh, 0, None, None, ld, None, _p(rinv), None, None, None, _s())
    _lib.call("sam6d_fine_pass_tc", _p(f2n), _p(f1n), B, S, a, sh, 0, None, None, ld, None, _p(cinv), None, None, None, _s())
    _lib.call("sam6d_fine_pass_tc", _p(f2n), _p(f1n), B, S, a, sh, 1, _p(cinv), _p(rinv), ld, None, None, _p(lab2), None, None, _s())
    _lib.call("sam6d_fine_masked_points", _p(lab2), _p(pts2), B, S, ld, _p(q4), _s())
    _lib.call("sam6d_fine_pass_tc", _p(f1n), _p(f2n), B, S, a, sh, 2, _p(rinv), _p(cinv), ld, _p(q4), None, _p(lab1), _p(wts), _p(pred),
              _s())
    return lab1, lab2, wts, pred


def weighted_procrustes(src: Tensor, ref: Tensor, wts: Tensor, weight_thresh: float = 0.0, eps: float = 1e-5):
    _check(src, torch.float32, "src", 3)
    _check(ref, torch.float32, "ref", 3)
    _check(wts, torch.float32, "weights", 2)
    B, N, _ = src.shape
    R = torch.empty(B, 3, 3, dtype=torch.float32, device=src.device)
    t = torch.empty(B, 3, dtype=torch.float32, device=src.device)
    _lib.call("sam6d_weighted_procrustes", _p(src), _p(ref), _p(wts), B, N, _f(weight_thresh), _f(eps), _p(R), _p(t), _s())
    return R, t


def pose_score(pts1: Tensor, lab1: Tensor, R: Tensor, t: Tensor, model: Tensor, radius: Tensor, dis_thres: float = 0.15):
    _check(pts1, torch.float32, "pts1", 3)
    _check(lab1, torch.int32, "lab1", 2)
    B, N, _ = pts1.shape
    score = torch.empty(B, dtype=torch.float32, device=pts1.device)
    ts = torch.empty(B, 3, dtype=torch.float32, device=pts1.device)
    _lib.call("sam6d_pose_score", _p(pts1), _p(lab1), B, N, _p(R), _p(t), _p(model), model.shape[1], _f(dis_thres),
              _p(radius), _p(score), _p(ts), _s())
    return score, ts


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
    _lib.call("sam6d_attn_relpos", _p(qkv), _ll(C3), int(nW), int(Hs), int(Ws), int(nH), C // nH, _p(rel_h), _p(rel_w), _f(scale),
              _p(out), int(out_dtype == torch.bfloat16), _ll(C), _s())
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
    _lib.call("sam6d_bilinear_gather", _p(up), int(up.dtype == torch.bfloat16), _p(choose), int(B), int(K), int(G), int(sub), int(C),
              int(H), int(W), _p(out), _s())
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
    _lib.call("sam6d_template_score_agg", _p(Qn), _p(Rn), P, O, T, C, TEMPLATE_AGGREGATIONS[aggregation], _p(sim), _p(obj), _p(obj_t),
              _p(bo), _p(bs), _p(bt), _s())
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
    _lib.call("sam6d_mask_rle_count", _p(masks), n, H, W, _p(col_cnt), _p(band_off), _p(rle_off), _s())
    rle_cum = torch.empty(int(rle_off[n]), dtype=torch.int32, device=dev)
    _lib.call("sam6d_mask_rle_write", _p(masks), n, H, W, _p(col_cnt), _p(band_off), _p(rle_off), _p(rle_cum), _s())
    return rle_cum, rle_off
