"""Module parameters in kernel form, and the pre-norm ViT trunk shared by the PEM RGB branch (vit.py), the DINOv2 descriptor
(dinov2.py) and the SAM image encoder (sam.py).

Every model module keeps its weights packed for the kernels in a `_Packed` cache, rebuilt when a parameter or buffer of the
module it keys on changes.  The three ViT encoders run the same block on the fp32 residual stream
    x = x + proj(attend(LN1(x)));  x = x + fc2(act(fc1(LN2(x))))
and differ only in `attend`, which each encoder passes in."""
from typing import Optional

import torch
import torch.nn as nn

from . import ops

# Arithmetic of the dense projections.  "fp32": CUDA-core kernels, fp32 storage (exact path, parity reference).
# "bf16": wgmma tensor-core kernels -- operands rounded to bf16, fp32 accumulation in registers.
PRECISIONS = ("fp32", "bf16")


class _W:
    """a weight matrix in both operand formats"""
    __slots__ = ("f32", "bf16")

    def __init__(self, w: torch.Tensor):
        self.f32 = w.detach().to(torch.float32).contiguous()
        self.bf16 = self.f32.to(torch.bfloat16).contiguous()


def _f32(t: torch.Tensor) -> torch.Tensor:
    return t.detach().to(torch.float32).contiguous()


def _gemm(prec, A, W: "_W", bias=None, residual=None, relu=False, out=None):
    """A, residual and out are row views (ops.gemm)"""
    if prec == "bf16":
        if A.dtype == torch.bfloat16 and residual is None and out is None and A.is_contiguous() and A.shape[1] % 64 == 0:
            # bf16 token matrix: the persistent TMA kernel (fp32 output); the register-staged kernel below is for fp32 operands
            return ops.gemm_tma(A, W.bf16, bias, act=1 if relu else 0)
        return ops.gemm_tc(A, W.bf16, bias, residual=residual, out=out, relu=relu)
    return ops.gemm(A, W.f32, bias, residual=residual, out=out, relu=relu)


def _param_key(*modules: nn.Module):
    """identifies the current values of the modules' parameters and buffers: in-place updates (load_state_dict's copies
    among them) bump `_version`, and .to() replaces the storage"""
    return tuple((t.data_ptr(), t._version) for m in modules for t in (*m.parameters(), *m.buffers()))


class _Packed:
    """device-resident, kernel-ready weights derived from modules' parameters: get(build, *modules) returns build()'s result,
    calling it again only when a parameter or buffer of the modules has changed since.  `key` identifies the parameters the
    weights were built from, for caches derived from them."""

    def __init__(self):
        self.key = None
        self.w = None

    def get(self, build, *modules: nn.Module):
        key = _param_key(*modules)
        if self.key != key:
            self.w, self.key = build(), key
        return self.w


# ---------------------------------------------------------------------------------------------------------------------
# pre-norm ViT trunk
# ---------------------------------------------------------------------------------------------------------------------
class _PatchEmbed(nn.Module):
    def __init__(self, patch_size, in_chans, embed_dim):
        super().__init__()
        self.proj = nn.Conv2d(in_chans, embed_dim, kernel_size=patch_size, stride=patch_size)


class _Attention(nn.Module):
    def __init__(self, dim, qkv_bias=True):
        super().__init__()
        self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        self.proj = nn.Linear(dim, dim)


class _Mlp(nn.Module):
    def __init__(self, dim, hidden):
        super().__init__()
        self.fc1 = nn.Linear(dim, hidden)
        self.fc2 = nn.Linear(hidden, dim)


def patch_rows(x: torch.Tensor, P: int, Kp: Optional[int] = None) -> torch.Tensor:
    """(B, Cin, Gh*P, Gw*P) -> fp32 rows (B*Gh*Gw, Cin*P*P) in the (c, kh, kw) order of a Conv2d weight: a non-overlapping
    conv is a GEMM over them.  With Kp, the rows are zero-padded to Kp columns."""
    B, Cin, H, W = x.shape
    Gh, Gw = H // P, W // P
    K = Cin * P * P
    rows = x.float().reshape(B, Cin, Gh, P, Gw, P).permute(0, 2, 4, 1, 3, 5).reshape(B * Gh * Gw, K)
    if Kp is None:
        return rows.contiguous()
    padded = torch.zeros(B * Gh * Gw, Kp, dtype=torch.float32, device=x.device)
    padded[:, :K] = rows
    return padded


def patch_embed(precision, rows: torch.Tensor, pe_w: _W, pe_b: torch.Tensor, pos: torch.Tensor, out: torch.Tensor):
    """out (B, L, C) view <- rows pe_w^T + pe_b + pos (L, C): gemm_tc on the bf16 weights, or gemm on the fp32 ones"""
    B, L, C = out.shape
    gemm, w = (ops.gemm_tc, pe_w.bf16) if precision == "bf16" else (ops.gemm, pe_w.f32)
    gemm(rows.view(B, L, -1), w, pe_b, residual=pos.expand(B, L, C), out=out)


def pack_block(norm1: nn.LayerNorm, qkv_w, qkv_b, proj_w, proj_b, norm2: nn.LayerNorm, fc1_w, fc1_b, fc2_w, fc2_b):
    """one block's weights for `block` (l1 / l2: the first and second MLP Linear); a missing qkv bias becomes zeros"""
    if qkv_b is None:
        qkv_b = torch.zeros(qkv_w.shape[0], dtype=torch.float32, device=qkv_w.device)
    return dict(n1w=_f32(norm1.weight), n1b=_f32(norm1.bias), eps1=norm1.eps, qkv=_W(qkv_w), qkv_b=_f32(qkv_b),
                proj=_W(proj_w), proj_b=_f32(proj_b), n2w=_f32(norm2.weight), n2b=_f32(norm2.bias), eps2=norm2.eps,
                l1=_W(fc1_w), l1b=_f32(fc1_b), l2=_W(fc2_w), l2b=_f32(fc2_b))


def block(precision, bw, tok: torch.Tensor, attend, act=ops.ACT_GELU) -> torch.Tensor:
    """x = x + proj(attend(norm1(x)));  x = x + fc2(act(fc1(norm2(x))))  on the fp32 residual stream tok (rows, C).
    attend(LayerNorm rows) -> attention rows ahead of proj.  bf16: the LayerNorms write bf16 GEMM operands and the hidden
    activations are bf16; fp32: CUDA-core kernels throughout."""
    if precision == "bf16":
        att = attend(ops.layernorm_bf16(tok, bw["n1w"], bw["n1b"], eps=bw["eps1"]))
        tok = ops.gemm_tma(att, bw["proj"].bf16, bw["proj_b"], residual=tok)
        xn = ops.layernorm_bf16(tok, bw["n2w"], bw["n2b"], eps=bw["eps2"])
        h = ops.gemm_tma(xn, bw["l1"].bf16, bw["l1b"], act=act, out_dtype=torch.bfloat16)
        return ops.gemm_tma(h, bw["l2"].bf16, bw["l2b"], residual=tok)
    att = attend(ops.layernorm(tok, bw["n1w"], bw["n1b"], eps=bw["eps1"]))
    tok = ops.gemm(att, bw["proj"].f32, bw["proj_b"], residual=tok)
    xn = ops.layernorm(tok, bw["n2w"], bw["n2b"], eps=bw["eps2"])
    h = ops.gemm(xn, bw["l1"].f32, bw["l1b"], relu=act)
    return ops.gemm(h, bw["l2"].f32, bw["l2b"], residual=tok)
