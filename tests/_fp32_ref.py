"""Float64 restatements of the CUDA-core fp32 kernels (gemm_simt.cu, attn.cu, geo.cu: geo_embed_f32, pe.cu, rowops.cu) and
the error bounds tests/test_gpu_fp32_kernels.py holds them to.

Each restatement is plain torch in float64 on the fp32 operands the kernel reads; the constants are the fp32 values the kernel
uses (1e-6f, 1e-12f, 0.70710678f, the eps passed in).  tests/test_fp32_reference_cpu.py pins every restatement to
oracle/pem_oracle.py or to the torch functional form of the same operation.

Bounds use the notation of tests/test_gpu_pem_kernels.py: u = 2^-24 (fp32 unit roundoff), gamma_n = n u / (1 - n u) for a
chain of n fp32 roundings.  One rounding is charged per fp32 operation, in the order the kernel performs it (named next to each
bound).  Where nvcc may or may not contract a multiply and an add into an fma, both roundings are charged: contraction only
removes one.  Math functions (the build has no --use_fast_math): __expf 2 + floor(1.173 |x|) ulp, rsqrtf 2 ulp, sincosf and
erff 2 ulp, sqrtf and division IEEE (correctly rounded).  An ulp of a result y is at most 2 u |y|.  Each bound helper returns
a per-element bound on |kernel - reference| alongside the float64 reference."""
import math

import numpy as np
import torch

F64 = torch.float64
U = 2.0 ** -24                      # fp32 unit roundoff
UB = 2.0 ** -8                      # bf16 unit roundoff


def f32(v):
    """the fp32 value of a Python float constant, as the kernel uses it"""
    return float(np.float32(v))


EPS6 = f32(1e-6)                    # 1e-6f of focus_kernel, linattn_apply_kernel, scale_by_radius_kernel
EPS12 = f32(1e-12)                  # 1e-12f of l2norm_kernel
RSQRT2 = f32(0.70710678118654752)   # the GELU constant of s6_act


def gamma(n):
    """gamma_n = n u / (1 - n u): the relative bound of a chain of n fp32 roundings"""
    return n * U / (1.0 - n * U)


def exp_rel(x):
    """relative error of __expf(s - m) for an argument x = s - m <= 0: 2 + floor(1.173 |x|) ulp of the result, plus the
    rounding of the subtraction (u |x| in the argument)"""
    x = x.abs()
    return (2.0 + 1.173 * x) * 2 * U + U * x


def bf(v):
    """the bf16 value a kernel stores for an fp32 value equal to v (fp64 -> fp32 -> bf16, round to nearest even)"""
    return v.float().bfloat16().to(F64)


def spread(v, e):
    """bound on |bf16(kernel fp32 value) - bf(v)| when the kernel's fp32 value is within e of v: rounding is monotone, so the
    kernel's bf16 value lies in [bf(v - e), bf(v + e)]"""
    return bf(v + e) - bf(v - e)


# ================================================================================================== gemm_simt.cu
def gelu(x):
    """s6_act(x, 2) = 0.5 x (1 + erf(x * 0.70710678f)), with the kernel's fp32 constant"""
    return 0.5 * x * (1.0 + torch.erf(x * RSQRT2))


def gemm(A, W, bias=None, residual=None, alpha=1.0, act=0):
    """alpha * A W^T (+bias) (act) (+residual) in float64; A (..., M, K), W (N, K) or (batch, N, K) -> (out, bound).

    Kernel order: acc = a sequential fma chain over k = 0..K-1 (K roundings), then acc * alpha, + bias (two roundings, or one if
    contracted): gamma_{K+2} (|alpha| sum_k |a w| + |bias|) before the activation.  ReLU is 1-Lipschitz; GELU's slope
    Phi(x) + x phi(x) is at most 1.13, and its own arithmetic is x * c (u |x c|, through erf' <= 2 / sqrt(pi)), erff (2 ulp),
    1 + erf (u), 0.5 x (exact) and the product (u).  The residual add is one more rounding of the result."""
    A, W = A.to(F64), W.to(F64)
    Wt = W.transpose(-1, -2)
    z = alpha * (A @ Wt)
    mag = abs(alpha) * (A.abs() @ Wt.abs())
    if bias is not None:
        b = bias.to(F64)
        z = z + b
        mag = mag + b.abs()
    e = gamma(A.shape[-1] + 2) * mag
    if act == 1:
        y = torch.relu(z)
    elif act == 2:
        y = gelu(z)
        t = z * RSQRT2
        er = torch.erf(t)
        own = 0.5 * z.abs() * (1.1284 * t.abs() * U + 4 * U * er.abs() + U * (1 + er).abs()) + U * y.abs()
        e = 1.13 * e + own
    else:
        y = z
    if residual is not None:
        y = y + residual.to(F64)
        e = e + U * y.abs()
    return y, e * (1 + 1e-6)


# ================================================================================================== attn.cu
def rpe_scores(E, U4):
    """SP[b,h,n,m] = sum_c U[b*S+n, 256 h + c] E[b,n,m,c]; E (B,S,S,256), U (B*S, 1024) -> ((B,4,S,S), bound).

    Kernel order: lane l sums channels [8l, 8l+8) as an fma chain from 0 (8 roundings), then five shuffle additions (the four
    transpose-halving steps and the final xor-1): gamma_13 sum_c |u e|."""
    B, S = E.shape[0], E.shape[1]
    Uh = U4.to(F64).reshape(B, S, 4, 256)
    sp = torch.empty(B, 4, S, S, dtype=F64, device=E.device)
    mag = torch.empty_like(sp)
    for b in range(B):
        for n0 in range(0, S, 64):
            e = E[b, n0:n0 + 64].to(F64)                                   # (n, m, c)
            u = Uh[b, n0:n0 + 64]                                          # (n, h, c)
            sp[b, :, n0:n0 + 64] = torch.einsum("nhc,nmc->hnm", u, e)
            mag[b, :, n0:n0 + 64] = torch.einsum("nhc,nmc->hnm", u.abs(), e.abs())
    return sp, gamma(13) * mag


def mha(q, k, v, bias, scale, drop_last_key=False):
    """softmax((q k^T + bias) * scale) v per head of 64 channels; q (B,Sq,H*64), k, v (B,Sk,H*64), bias (B,H,Sq,Sk) or None
    -> ((B,Sq,H*64), bound).  drop_last_key leaves key Sk-1 out of the softmax (a deliberately wrong answer).

    Kernel order, per query:
      score  a = fma chain over the 64 channels from 0 (64 roundings), + bias, * scale (two roundings): the fp32 score is within
             d = gamma_66 |scale| (sum_c |q k| + |bias|) of s;
      exp    e = __expf(a - max) (exp_rel, at an argument within 2 max d of x); score errors |delta_j| <= d_j move p_m by a
             factor between exp(-(d_m + D)) and exp(d_m + D), D = log sum_j p_j exp(d_j) (Jensen bounds the other side);
      sum    each lane adds its <= 8 keys in turn, then a 5-level butterfly: gamma_13 (all terms positive);
      p      1 / sum (IEEE division) and e * (1/sum): two roundings;
      out    fma chain over the keys m = 0..Sk-1 from 0: gamma_Sk sum_m p |v|."""
    B, Sq, HD = q.shape
    Sk, H = k.shape[1], HD // 64
    qh = q.to(F64).reshape(B, Sq, H, 64).transpose(1, 2)
    kh = k.to(F64).reshape(B, Sk, H, 64).transpose(1, 2)
    vh = v.to(F64).reshape(B, Sk, H, 64).transpose(1, 2)
    raw = qh @ kh.transpose(-1, -2)
    mag = qh.abs() @ kh.abs().transpose(-1, -2)
    if bias is not None:
        raw = raw + bias.to(F64)
        mag = mag + bias.to(F64).abs()
    s = raw * scale
    d = gamma(66) * abs(scale) * mag
    if drop_last_key:
        s = s.clone()
        s[..., -1] = -math.inf
    p = torch.softmax(s, dim=-1)
    x = s - s.amax(-1, keepdim=True)
    xa = torch.nan_to_num(x, neginf=0.0).abs() + 2 * d.amax(-1, keepdim=True)
    eta = torch.where(p > 0, exp_rel(xa), torch.zeros_like(p))
    eta_sum = (p * eta).sum(-1, keepdim=True) + gamma(13)
    D = torch.log((p * torch.exp(d)).sum(-1, keepdim=True))
    rel = eta + eta_sum + gamma(2) + torch.expm1(d + D)
    out = p @ vh
    e = (p * rel) @ vh.abs() + gamma(Sk) * (p * (1 + rel)) @ vh.abs()
    return out.transpose(1, 2).reshape(B, Sq, HD), (e * (1 + 1e-6)).transpose(1, 2).reshape(B, Sq, HD)


def linattn_kv(k, v):
    """KV[b,h] = sum_j k_j v_j^T, KS[b,h] = sum_j k_j per head of 64; k, v (B,J,H*64) -> (KV (B,H,64,64), KS (B,H,64), bounds).

    Kernel order: one thread per (c, 16 d) runs fma chains over j = 0..J-1 from 0 (J roundings), and the plain sum of k[j, c]
    alongside (J roundings): gamma_J sum_j |k v|, gamma_J sum_j |k|."""
    B, J, HD = k.shape
    H = HD // 64
    kh = k.to(F64).reshape(B, J, H, 64).permute(0, 2, 3, 1)             # (B,H,c,J)
    vh = v.to(F64).reshape(B, J, H, 64).transpose(1, 2)                 # (B,H,J,d)
    KV = kh @ vh
    KS = kh.sum(-1)
    return KV, KS, gamma(J) * (kh.abs() @ vh.abs()), gamma(J) * kh.abs().sum(-1)


def linattn_apply(q, KV, KS):
    """x_h = (q_h KV_h) / (q_h . KS_h + 1e-6f); q (B,N,H*64), KV (B,H,64,64), KS (B,H,64) -> ((B,N,H*64), bound).

    Kernel order, per token and head:
      zden  q0 ks0 + q1 ks1 per lane (two or three roundings), then a 5-level warp sum: gamma_8 (q, KS >= 0, as the focused
            features the model passes); + 1e-6f and 1 / (.) one rounding each: z within gamma_10 |z|;
      o     fma chain over the 64 channels c from 0: gamma_64 sum_c |q KV|;
      x     o * z: one rounding.
    For operands of either sign the zden term is charged as gamma_8 sum |q KS| |z|^2 |o| instead."""
    B, N, HD = q.shape
    H = HD // 64
    qh = q.to(F64).reshape(B, N, H, 64).transpose(1, 2)                 # (B,H,N,c)
    KV, KS = KV.to(F64), KS.to(F64)
    den = (qh * KS.unsqueeze(2)).sum(-1, keepdim=True)
    dmag = (qh.abs() * KS.abs().unsqueeze(2)).sum(-1, keepdim=True)
    z = 1.0 / (den + EPS6)
    o = qh @ KV
    x = o * z
    e_o = gamma(64) * (qh.abs() @ KV.abs())
    e_z = gamma(8) * dmag * z.abs() ** 2 + gamma(2) * z.abs()
    e = e_o * z.abs() + o.abs() * e_z + U * x.abs() + e_o * e_z
    return x.transpose(1, 2).reshape(B, N, HD), (e * (1 + 1e-6)).transpose(1, 2).reshape(B, N, HD)


# ================================================================================================== rowops.cu
def layernorm(x, g, b, eps, eps_scale=1.0):
    """LayerNorm over the last dim (biased variance, eps inside the square root); x (R, C) -> (out, bound).  eps_scale != 1 is a
    deliberately wrong answer.

    Kernel order (one warp per row, nv = C / 32 values per lane):
      mean  each lane adds its nv values in turn, then a 5-level butterfly, / C: gamma_{nv+5} mean |x| + u |mean|;
      d     x - mean: one rounding, on top of the mean's error;
      var   d * d per lane (fma or mul + add), 5-level butterfly: gamma_{nv+5} sum d~^2; / C and + eps one rounding each;
      rstd  rsqrtf: 2 ulp, plus half the relative error of var + eps;
      out   d * rstd * gamma + beta: three roundings (two if the last two contract)."""
    x, g, b = x.to(F64), g.to(F64), b.to(F64)
    C = x.shape[-1]
    nv = C // 32
    mu = x.mean(-1, keepdim=True)
    d = x - mu
    var = d.pow(2).mean(-1, keepdim=True)
    r = 1.0 / torch.sqrt(var + eps * eps_scale)
    out = d * r * g + b
    e_mu = gamma(nv + 5) * x.abs().mean(-1, keepdim=True) + U * mu.abs()
    e_d = e_mu + U * (d.abs() + e_mu)
    e_q = (2 * d.abs() * e_d + e_d ** 2).mean(-1, keepdim=True) + gamma(nv + 6) * (d.abs() + e_d).pow(2).mean(-1, keepdim=True)
    e_ve = e_q + 2 * U * (var + eps + e_q)
    xr = e_ve / (var + eps)
    e_r = 0.5 * xr * (1 + xr) + 4 * U                    # (1 + x)^-1/2 - 1 within x/2 (1 + x) for 0 <= x <= 1/2
    e = g.abs() * r * (e_d + (d.abs() + e_d) * (e_r + 3 * U)) + U * out.abs()
    return out, e * (1 + 1e-6) + 1e-30


def l2norm(x):
    """F.normalize(x, dim=-1) with the kernel's clamp: x / max(||x||, 1e-12f); x (R, C) -> (out, bound).

    Kernel order: x * x summed per lane (nv terms), 5-level butterfly: gamma_{nv+5} (positive terms); sqrtf: half that plus u;
    fmaxf with the clamp exact (1-Lipschitz); x / n: one rounding."""
    x = x.to(F64)
    nv = x.shape[-1] // 32
    n = x.norm(dim=-1, keepdim=True)
    nc = n.clamp_min(EPS12)
    out = x / nc
    e_n = (0.5 * gamma(nv + 5) + U) * n
    return out, (x.abs() * e_n / (nc * (nc - e_n).clamp_min(EPS12 * 0.5)) + U * out.abs()) * (1 + 1e-6)


def focus(x, sp):
    """the focused-linear-attention feature map, PEM transformer.py:541-550 with FOCUS = 3:
    q = (relu(x) + 1e-6f) / sp;  out = q^3 / ||q^3|| * ||q||;  x (R, C), sp (C) -> (out, bound).

    Kernel order (all quantities positive, so every error is relative):
      q     + 1e-6f and / sp: two roundings;  q^3 = q * q * q: two more (q^3 within 8u);
      s1    q * q summed per lane (nv terms) and over a 5-level butterfly: 2 x 2u from q, gamma_{nv+6};
      s3    (q^3)^2 likewise: 2 x 8u from q^3, gamma_{nv+6};
      n     sqrtf: half the relative error of s, plus u;
      out   (q^3 / n3) * n1: two roundings.
    Valid while every (q^3)^2 is a normal fp32 number: for an all-negative row every q = 1e-6f / sp, and (q^3)^2 < 2^-126 once
    sp exceeds about 2.1 (the sum of squares then loses relative accuracy, and vanishes for sp above about 33)."""
    x, sp = x.to(F64), sp.to(F64)
    nv = x.shape[-1] // 32
    q = (torch.relu(x) + EPS6) / sp
    q3 = q ** 3
    out = q3 / q3.norm(dim=-1, keepdim=True) * q.norm(dim=-1, keepdim=True)
    r_q, r_q3 = gamma(2), gamma(8)
    r_s1 = 2 * r_q + gamma(nv + 6)
    r_s3 = 2 * r_q3 + gamma(nv + 6)
    rel = r_q3 + (0.5 * r_s1 + U) + (0.5 * r_s3 + U) + gamma(2)
    return out, rel * 1.001 * out.abs()


# ================================================================================================== geo.cu
def sin_emb(x, div, arg_fp32=True):
    """[sin(x w_0), cos(x w_0), sin(x w_1), ...] (transformer.py:262-283), x (...), div (128) -> (..., 256).  With arg_fp32 the
    argument is the fp32 product x * div_term[f], as geo_embed_f32_kernel forms it before sincosf."""
    if arg_fp32:
        om = (x.float().unsqueeze(-1) * div.float()).to(F64)
    else:
        om = x.to(F64).unsqueeze(-1) * div.to(F64)
    return torch.stack([torch.sin(om), torch.cos(om)], dim=-1).flatten(-2)


def geo_embed(T, div, WaT, WdT, bias, drop_last_pair=False, arg_fp32=True, chunk=16384):
    """E = proj_d(emb(T[..., 3])) + max_t proj_a(emb(T[..., t])) (transformer.py:334-349); T (P, 4) angle / distance indices,
    WaT, WdT (256 k, 256 c), bias = b_a + b_d -> ((P, 256), bound).  drop_last_pair leaves out k = 254, 255 (a deliberately wrong
    answer).

    Kernel order: sincosf on the fp32 argument (2 ulp each: 4u |sin|), the projections as fma chains over k = 0..255 from 0
    (gamma_256 sum_k |w emb|, plus sum_k |w| 4u |emb|), max over the three angle rows (exact, 1-Lipschitz), then
    acc_d + max + bias: two roundings."""
    P = T.shape[0]
    Wa, Wd, b = WaT.to(F64), WdT.to(F64), bias.to(F64)
    if drop_last_pair:
        Wa, Wd = Wa.clone(), Wd.clone()
        Wa[254:], Wd[254:] = 0, 0
    out = torch.empty(P, 256, dtype=F64, device=T.device)
    err = torch.empty_like(out)
    for p0 in range(0, P, chunk):
        e = sin_emb(T[p0:p0 + chunk], div, arg_fp32)                   # (p, 4, 256)
        ea = e.abs()
        acc_a = e[:, :3] @ Wa
        acc_d = e[:, 3] @ Wd
        ma = (gamma(256) + 4 * U) * (ea[:, :3] @ WaT.to(F64).abs())
        md = (gamma(256) + 4 * U) * (ea[:, 3] @ WdT.to(F64).abs())
        mx = acc_a.amax(1)
        o = acc_d + mx + b
        out[p0:p0 + chunk] = o
        err[p0:p0 + chunk] = ma.amax(1) + md + 2 * U * (acc_d.abs() + mx.abs() + b.abs()) + U * o.abs()
    return out, err * (1 + 1e-6)


# ================================================================================================== pe.cu
def pe_mlp_max(pts, idx, cnt, weights):
    """max over the samples s < max(cnt, 1) of relu(W3 relu(W2 relu(W1 [p_j - p_i, p_j] + b1) + b2) + b3), j = idx[i, s]: the
    PositionalEncoding SharedMLP of fine_point_matching.py:90-125 with BatchNorm folded into (W, b); pts (B,N,3), idx (B,N,ns),
    cnt (B,N) -> ((B,N,128), bound).

    Kernel order: p_j - p_i one rounding; each layer an fma chain from the bias over its inputs (6, 32, 64 roundings):
    gamma_n (|b| + |W| |h|) plus |W| times the input's error (ReLU and the max over samples are 1-Lipschitz)."""
    W1, B1, W2, B2, W3, B3 = (w.to(F64) for w in weights)
    B, N, ns = idx.shape
    P = pts.to(F64)
    out = torch.empty(B, N, 128, dtype=F64, device=pts.device)
    err = torch.empty_like(out)
    valid = torch.arange(ns, device=idx.device) < cnt.clamp_min(1).unsqueeze(-1)          # (B,N,ns)
    for b in range(B):
        pj = P[b][idx[b].long()]                                                          # (N,ns,3)
        pi = P[b].unsqueeze(1)
        rel = pj - pi
        x = torch.cat([rel, pj], -1)
        ex = torch.cat([U * rel.abs(), torch.zeros_like(pj)], -1)
        h, e = x, ex
        for W, bb, n in ((W1, B1, 6), (W2, B2, 32), (W3, B3, 64)):
            pre = h @ W.t() + bb
            e = e @ W.abs().t() + gamma(n) * (bb.abs() + h.abs() @ W.abs().t())
            h = torch.relu(pre)
        m = valid[b].unsqueeze(-1)
        out[b] = torch.where(m, h, torch.full_like(h, -math.inf)).amax(1)
        err[b] = torch.where(m, e, torch.zeros_like(e)).amax(1)
    return out, err * (1 + 1e-6)


def fold_bn(conv_w, bn_w, bn_b, mean, var, eps=1e-5):
    """Conv (no bias) + BatchNorm (eval) -> (W, b), folded in float64 as sam6d_b200.pem folds them"""
    s = bn_w.double() / torch.sqrt(var.double() + eps)
    return conv_w.double().reshape(conv_w.shape[0], -1) * s[:, None], bn_b.double() - mean.double() * s


# ================================================================================================== point-cloud row ops
def rigid_warp(p, R, t):
    """(p - t) @ R per cloud; p (B,n,3), R (B,3,3), t (B,3) -> (out, bound).  Kernel order: the difference one rounding, then
    three products and two additions (gamma_3, or fewer roundings if contracted)."""
    d = p.to(F64) - t.to(F64).unsqueeze(1)
    Rd = R.to(F64)
    out = d @ Rd
    return out, (U * d.abs() @ Rd.abs() + gamma(3) * (d.abs() @ Rd.abs())) * (1 + U)


def cloud_radius(po):
    """max_i ||po[b, i]||; po (B,n,3) -> (radius, bound).  Kernel order: three squares summed (gamma_3, positive), sqrtf (half
    plus u); the max is exact."""
    r = po.to(F64).norm(dim=-1).amax(-1)
    return r, (0.5 * gamma(3) + U) * r * (1 + U)


def scale_by_radius(x, radius):
    """x / (radius + 1e-6f) per cloud; x (B, ...) -> (out, bound).  Kernel order: the add and the division, one rounding each."""
    shape = (-1,) + (1,) * (x.dim() - 1)
    out = x.to(F64) / (radius.to(F64).view(shape) + EPS6)
    return out, gamma(2) * out.abs()
