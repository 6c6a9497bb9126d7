"""Float64 restatements of the PEM pose kernels (geo.cu: geo_indices; coarse.cu; fine.cu: fine_assign, weighted_procrustes,
pose_score; svd3.cuh) and the error-bound helpers tests/test_gpu_pose_kernels.py holds them to.

Each restatement is plain torch in float64 on the fp32 operands the kernel reads (constants included: 1e-8f, 1e-6f, the
hypothesis weight 1/(3+1e-5) and dis_thres are the fp32 values the kernel uses), in the order of operations of the reference
(PEM/utils/model_utils.py, PEM/model/transformer.py) where that order decides a discrete output.  Ties are broken the way the
kernels break them: the first index wins (torch.max, torch.searchsorted(right=False)).  tests/test_pose_reference_cpu.py pins
every function here to oracle/pem_oracle.py.  Bound helpers return a per-element bound and, for every discrete output, the
mask of elements whose choice the bound decides."""
import math

import numpy as np
import torch

F64 = torch.float64
U = 2.0 ** -24                   # fp32 unit roundoff
U64 = 2.0 ** -53
EPS8 = float(np.float32(1e-8))   # the fp32 constants the kernels add
EPS6 = float(np.float32(1e-6))
W3 = float(np.float32(1.0) / (np.float32(3.0) + np.float32(1e-5)))   # coarse_hyp_kernel's weight 1.f / (3.f + 1e-5f)


def f32(v):
    """the fp32 value of a Python float constant, as the kernel receives it"""
    return float(np.float32(v))


def gamma(n):
    """gamma_n = n u / (1 - n u): the relative bound of a chain of n fp32 roundings"""
    return n * U / (1.0 - n * U)


def first_argmax(x, dim):
    """index of the first maximum along dim (torch.max's documented choice, stated without relying on it)"""
    m = x.amax(dim, keepdim=True)
    ar = torch.arange(x.shape[dim], device=x.device).view([-1 if d == (dim % x.dim()) else 1 for d in range(x.dim())])
    return torch.where(x == m, ar, x.shape[dim]).amin(dim)


# ================================================================================================ geometric indices
def pair_dist(p, q):
    """|q_j - p_i| (B,I,3), (B,J,3) -> (B,I,J) from the differences (not the expanded form the kernel uses)"""
    return (q.to(F64).unsqueeze(1) - p.to(F64).unsqueeze(2)).pow(2).sum(-1).sqrt()


def knn_sorted(d, k):
    """the k+1 nearest points by (distance, index): a stable sort, self (distance 0) first unless an earlier duplicate ties it"""
    v, i = torch.sort(d, dim=-1, stable=True)
    return v[..., :k + 1], i[..., :k + 1]


def triplet_angles(pts, anchors, knn, factor_a):
    """atan2(|r x a|, r . a) * factor_a for r = p[knn_k] - p_i (k = 1..3), a = p_j - p_i; exactly 0 where r or a is 0
    (transformer.py:318-331; the + 0.0 makes an all-(-0) dot product +0, as torch.sum does)  -> (B,A,S,3), and |r|, |a|"""
    P = pts.to(F64)
    B = P.shape[0]
    pi = P[:, anchors]                                                      # (B,A,3)
    bidx = torch.arange(B, device=P.device).view(B, 1, 1)
    r = P[bidx, knn[..., 1:]] - pi.unsqueeze(2)                             # (B,A,3,3)
    a = P.unsqueeze(1) - pi.unsqueeze(2)                                    # (B,A,S,3)
    rr, aa = r.unsqueeze(2), a.unsqueeze(3)                                 # (B,A,1,3,3), (B,A,S,1,3)
    s = torch.linalg.cross(rr.expand(-1, -1, aa.shape[2], -1, -1), aa.expand(-1, -1, -1, 3, -1), dim=-1).norm(dim=-1)
    c = (rr * aa).sum(-1) + 0.0
    return torch.atan2(s, c) * factor_a, r.norm(dim=-1), a.norm(dim=-1)


def geo_indices(pts, sigma_d, factor_a, anchors=None):
    """restatement of sam6d_geo_indices for the given anchor rows: d_idx (B,A,S), a_idx (B,A,S,3), the distances (B,A,S),
    knn (B,A,4) (entry 0 is dropped by the kernel), |r| (B,A,3), |a| (B,A,S)"""
    S = pts.shape[1]
    anchors = torch.arange(S, device=pts.device) if anchors is None else anchors
    d = pair_dist(pts[:, anchors], pts)
    _, knn = knn_sorted(d, 3)
    ang, rn, an = triplet_angles(pts, anchors, knn, f32(factor_a))
    return d / f32(sigma_d), ang, d, knn, rn, an


def sqdist_err(xn, mn, n):
    """bound on the fp32 error of |x|^2 - 2 x.y + |y|^2 (expanded form, n roundings on the longest path), |x| = xn, |y| = mn"""
    return gamma(n) * (xn + mn) ** 2


def dist_err(d, e):
    """bound on |sqrtf(clamp(s, 0)) - d| when |s - d^2| <= e: min(sqrt(e), e / d) plus the sqrtf rounding"""
    return torch.minimum(e.sqrt(), e / d.clamp_min(1e-300)) + U * (d + e.sqrt())


# ================================================================================================ coarse soft assignment
def soft_assignment(A):
    """P = softmax_row(A) * softmax_col(A) (model_utils.py:206-214) and the first-max labels of every row / column
    -> P (B,S,S), lab1 (B,S) (row i -> column), lab2 (B,S) (column j -> row)"""
    A = A.to(F64)
    P = torch.softmax(A, 2) * torch.softmax(A, 1)
    return P, first_argmax(P, 2), first_argmax(P, 1)


def coarse_weights(P, lab1, lab2):
    """the kernel's outputs from P and labels: W (B,n*n) = (P_inner * [lab1 > 0] * [lab2 > 0]) ** 1.5, w1 (B,n)"""
    B, S, _ = P.shape
    m1, m2 = (lab1[:, 1:] > 0).to(F64), (lab2[:, 1:] > 0).to(F64)
    inner = P[:, 1:, 1:] * m1.unsqueeze(2) * m2.unsqueeze(1)
    return inner.pow(1.5).reshape(B, (S - 1) ** 2), m1


def argmax_decided(x, e, dim):
    """first-max index of x along dim, whether the bound e (same shape) decides it (the winner's lower end above every other
    element's upper end), and the mask of elements the bound allows as the kernel's choice (upper end >= the winner's lower end)"""
    i = first_argmax(x, dim)
    lo = (x - e).gather(dim, i.unsqueeze(dim))
    hi = x + e
    allowed = hi >= lo
    decided = allowed.sum(dim) == 1
    return i, decided, allowed


# ================================================================================================ cdf + searchsorted
def cdf(W):
    """cumsum(W) / (sum + 1e-8f)  (model_utils.py:217-218)"""
    c = torch.cumsum(W.to(F64), 1)
    return c / (c[:, -1:] + EPS8)


def searchsorted(c, v):
    """first i with c[i] >= v; L if there is none (torch.searchsorted, right=False)"""
    return torch.searchsorted(c.contiguous(), v.to(F64).contiguous(), right=False)


def cdf_err(c):
    """bound on the kernel's cdf: the double running sum rounded to fp32 (u), the total rounded (u), + 1e-8f (u), the
    division (u); the double sums themselves (L terms, 2^-53 each) are charged 1e-12"""
    return (4 * U + 1e-12) * c.abs() * 1.001


# ================================================================================================ Procrustes
def triplet_ranks(i1, i2):
    """(rank1, rank0) of hypotheses (...,3) whose triplet repeats a point (pem_oracle._triplet_ranks)"""
    eq = lambda a: (a[..., 0] == a[..., 1]).int() + (a[..., 0] == a[..., 2]).int() + (a[..., 1] == a[..., 2]).int()  # noqa: E731
    e1, e2 = eq(i1), eq(i2)
    rank0 = (e1 == 3) | (e2 == 3)
    return ~rank0 & ((e1 + e2) > 0), rank0


def any_orth(a):
    """unit vector orthogonal to the unit vectors a (n,3): a x e_k, k = the first smallest |component| (svd3.cuh: any_orth)"""
    ab = a.abs()
    k = torch.where((ab[:, 0] <= ab[:, 1]) & (ab[:, 0] <= ab[:, 2]), 0, torch.where(ab[:, 1] <= ab[:, 2], 1, 2))
    o = torch.linalg.cross(a, torch.nn.functional.one_hot(k, 3).to(a.dtype))
    return o / o.norm(dim=1, keepdim=True)


def rank1_rotation(u1, v1):
    """the least rotation taking u1 to v1: c I + [w]x + w w^T / (1 + c), w = u1 x v1, c = u1 . v1; the half turn about
    any_orth(u1) when 1 + c < 1e-9 (pem_oracle.rank1_rotation)  -> R (n,3,3), c (n,)"""
    c = (u1 * v1).sum(1)
    w = torch.linalg.cross(u1, v1)
    eye = torch.eye(3, dtype=F64, device=u1.device).expand(u1.shape[0], 3, 3)
    K = torch.zeros_like(eye)
    K[:, 0, 1], K[:, 0, 2], K[:, 1, 0], K[:, 1, 2], K[:, 2, 0], K[:, 2, 1] = -w[:, 2], w[:, 1], w[:, 2], -w[:, 0], -w[:, 1], w[:, 0]
    R = c[:, None, None] * eye + K + w[:, :, None] * w[:, None, :] / (1.0 + c).clamp_min(1e-300)[:, None, None]
    flip = (1.0 + c) < 1e-9
    if flip.any():
        a = any_orth(u1[flip])
        R[flip] = 2.0 * a[:, :, None] * a[:, None, :] - torch.eye(3, dtype=F64, device=u1.device)
    return R, c


def procrustes_rotation(H, rank1=None, rank0=None):
    """R = V diag(1, 1, sign det(V U^T)) U^T for H = U S V^T (model_utils.py:352-358); R = I where H = 0 or rank0; the
    rank-1 completion where rank1.  H (n,3,3) float64 -> R (n,3,3), singular values (n,3), sign(det H) (n,), c (n,) of the
    rank-1 rule (nan elsewhere)"""
    n = H.shape[0]
    U_, S, Vh = torch.linalg.svd(H)
    V = Vh.transpose(1, 2)
    D = torch.eye(3, dtype=F64, device=H.device).repeat(n, 1, 1)
    D[:, 2, 2] = torch.sign(torch.det(V @ U_.transpose(1, 2)))
    R = V @ D @ U_.transpose(1, 2)
    c = torch.full((n,), float("nan"), dtype=F64, device=H.device)
    if rank1 is not None and rank1.any():
        R[rank1], c[rank1] = rank1_rotation(U_[rank1, :, 0], Vh[rank1, 0, :])
    zero = ~(S[:, 0] > 0)
    if rank0 is not None:
        zero = zero | rank0
    R[zero] = torch.eye(3, dtype=F64, device=H.device)
    return R, S, torch.sign(torch.det(H)), c


def triplets(idx, pts1, pts2):
    """the clamped pair indices of the kernel's flat samples idx (B,3*n1) -> i1, i2 (B,n1,3) and the points p1, p2 (B,n1,3,3)"""
    B, n, _ = pts1.shape
    idx = idx.long()
    i1 = torch.clamp(idx // n, max=n - 1).view(B, -1, 3)
    i2 = torch.clamp(idx % n, max=n - 1).view(B, -1, 3)
    bidx = torch.arange(B, device=idx.device).view(B, 1, 1)
    return i1, i2, pts1.to(F64)[bidx, i1], pts2.to(F64)[bidx, i2]


def triplet_procrustes(idx, pts1, pts2):
    """sam6d_coarse_hypotheses: weighted_procrustes(src = p2, ref = p1, weights 1 / (3 + 1e-5)), the rank rule of
    _triplet_ranks, t = c_r - R c_s, resid = mean_k |(p1_k - t) R - p2_k|.  -> dict of (B,n1,...) tensors"""
    i1, i2, p1, p2 = triplets(idx, pts1, pts2)
    B, n1 = i1.shape[:2]
    r1, r0 = triplet_ranks(i1, i2)
    cs, cr = (p2 * W3).sum(2), (p1 * W3).sum(2)                               # (B,n1,3)
    a, b = p2 - cs.unsqueeze(2), W3 * (p1 - cr.unsqueeze(2))
    H = a.transpose(2, 3) @ b                                                 # (B,n1,3,3)
    R, S, sdet, c = procrustes_rotation(H.reshape(-1, 3, 3), r1.reshape(-1), r0.reshape(-1))
    R = R.view(B, n1, 3, 3)
    t = cr - (R @ cs.unsqueeze(3)).squeeze(3)
    resid = ((p1 - t.unsqueeze(2)) @ R - p2).norm(dim=3).mean(2)
    return dict(R=R, t=t, resid=resid, H=H, S=S.view(B, n1, 3), sdet=sdet.view(B, n1), c=c.view(B, n1), rank1=r1, rank0=r0,
                p1=p1, p2=p2, cs=cs, cr=cr, a=a, b=b)


def weighted_procrustes(src, ref, wts, weight_thresh=0.0, eps=1e-5):
    """sam6d_weighted_procrustes (model_utils.py:287-363): weights below weight_thresh (strictly) dropped, normalised by
    sum + eps, ref ~= R src + t  -> dict with R (B,3,3), t (B,3) and the intermediates the bound needs"""
    s, r, w = src.to(F64), ref.to(F64), wts.to(F64)
    w = torch.where(w < f32(weight_thresh), torch.zeros_like(w), w)
    wn = w / (w.sum(1, keepdim=True) + f32(eps))
    cs, cr = (s * wn.unsqueeze(2)).sum(1), (r * wn.unsqueeze(2)).sum(1)
    a, b = s - cs.unsqueeze(1), wn.unsqueeze(2) * (r - cr.unsqueeze(1))
    H = a.transpose(1, 2) @ b
    R, S, sdet, _ = procrustes_rotation(H)
    t = cr - (R @ cs.unsqueeze(2)).squeeze(2)
    return dict(R=R, t=t, H=H, S=S, sdet=sdet, wn=wn, cs=cs, cr=cr, a=a, b=b)


def cross_cov_err(a, b, da, db):
    """Frobenius bound on the error of H = sum_k a_k b_k^T when |a_k - a^_k| <= da, |b_k - b^_k| <= db (elementwise, (...,N,3)):
    |dH_ij| <= sum_k da_ki |b_kj| + |a_ki| db_kj + da_ki db_kj, plus 1e-15 sum |a||b| for the double accumulation"""
    A, Bm = a.abs(), b.abs()
    dH = da.transpose(-1, -2) @ Bm + A.transpose(-1, -2) @ db + da.transpose(-1, -2) @ db + 1e-15 * (A.transpose(-1, -2) @ Bm)
    return dH.flatten(-2).norm(dim=-1)


def rotation_err(dHF, S, sdet, rank1=None, rank0=None, c=None):
    """bound on |R^ - R|_F from a perturbation |dH|_F <= dHF of the cross-covariance.

    Full rank path.  R maximises tr(R H) over SO(3); with H = U S V^T and s = sign(det H) it is V D U^T, D = diag(1, 1, s),
    and tr(R H) = tr(Q S) for Q = V^T R U = D.  Perturb H by dH and the maximiser by R -> V D exp([w]x) U^T.  With
    E = U^T dH V (dH in the singular bases, |E|_F = |dH|_F), stationarity of tr(D exp([w]x) (S + E)) in w at first order reads
    w_k (s~_i + s~_j) = E_ij - E_ji for each pair (i, j, k) cyclic, where s~ = (s1, s2, s s3) are the signed singular values
    (the Hessian of tr(D exp([w]x) S) is diagonal in this basis with the pair sums on its diagonal).  So
    |w|^2 <= sum (E_ij - E_ji)^2 / gap^2 <= 2 |E|_F^2 / gap^2, gap = min pair sum = s2 + s s3, and
    |dR|_F = |[w]x|_F = sqrt(2) |w| <= 2 |dH|_F / (s2 + s s3): the first-order bound of the special orthogonal Procrustes
    problem.  Charged 1.1x for the second-order terms, used while dHF / gap <= 0.05 (beyond that the trivial bound 2 sqrt 2
    between two rotations), plus the double-precision Jacobi of H^T H (eigenvectors to 2^-53 (s1 / gap)^2, charged 8x) and
    the fp32 rounding of R (sqrt(3) u).

    Rank-1 path (the triplet repeats a point).  The leading singular pair moves by at most sqrt(2) dHF / (s1 - s2) each
    (Wedin); the least rotation c I + [w]x + w w^T / (1 + c) moves by |du| + |dv| times (5 + 3 (1 + q)^2),
    q = |w| / (1 + c) = sqrt((1 - c) / (1 + c)) (the Frobenius norms of the three terms' derivatives); the half-turn branch
    2 a a^T - I moves by 4 |da| <= 4 sqrt(3/2) 2 |du| (|u1 x e_k| >= sqrt(2/3) for the smallest component k).
    Rank 0: R = I exactly."""
    s1, s2, s3 = S.unbind(-1)
    gap = s2 + sdet * s3
    ratio = dHF / gap.clamp_min(1e-300)
    b = 1.1 * 2 * ratio + 8 * U64 * (s1 / gap.clamp_min(1e-300)) ** 2 + 2 * U
    b = torch.where(ratio <= 0.05, b, torch.full_like(b, 2 * math.sqrt(2)))
    if rank1 is not None and rank1.any():
        du = 1.1 * math.sqrt(2) * dHF / (s1 - s2).clamp_min(1e-300)
        q = ((1 - c) / (1 + c).clamp_min(1e-300)).clamp_min(0).sqrt()
        b1 = torch.where(1 + c < 1e-9, 4 * math.sqrt(1.5) * 2 * du, 2 * du * (5 + 3 * (1 + q) ** 2)) + 2 * U
        b1 = torch.where(du <= 0.05, b1, torch.full_like(b1, 2 * math.sqrt(2)))
        b = torch.where(rank1, b1, b)
    if rank0 is not None:
        b = torch.where(rank0, torch.zeros_like(b), b)
    return b


# ================================================================================================ selection, fine stage
def transform(p, R, t):
    """(p - t) R, row vectors: p (B,N,3), R (B,H,3,3), t (B,H,3) -> (B,H,N,3)"""
    return (p.to(F64).unsqueeze(1) - t.to(F64).unsqueeze(2)) @ R.to(F64)


def transform_err(p, R, t):
    """bound on |fp32 (p - t) R - exact| (per point, Euclidean): p - t one rounding, each output an fma chain of 3: gamma_4
    on sum_j |x_j R_jk|"""
    x = (p.to(F64).unsqueeze(1) - t.to(F64).unsqueeze(2)).abs()
    return (gamma(4) * (x @ R.to(F64).abs())).norm(dim=-1)


def min_dist(x, model, chunk=8):
    """min_m |x_n - model_m| for x (B,H,N,3), model (B,M,3), from the differences, chunked over H"""
    m = model.to(F64)
    out = []
    for h in range(0, x.shape[1], chunk):
        xs = x[:, h:h + chunk]
        d = torch.cdist(xs.reshape(x.shape[0], -1, 3), m, compute_mode="donot_use_mm_for_euclid_dist").amin(-1)
        out.append(d.view(xs.shape[:3]))
    return torch.cat(out, 1)


def select_scores(R, t, pts1, w1, model):
    """sum(w1) / (sum_i w1_i min_m |(p_i - t) R - m| + 1e-8f) per hypothesis (model_utils.py:239-246); R (B,H,3,3), t (B,H,3)
    -> scores (B,H), distances (B,H,N)"""
    d = min_dist(transform(pts1, R, t), model)
    w = w1.to(F64).unsqueeze(1)
    return w.sum(2) / ((d * w).sum(2) + EPS8), d


def fine_assign(A, shift):
    """the assignment of sam6d_fine_assign: e = exp(A - shift); P = (e / row sums) (e / column sums) (the dual softmax with
    the fixed shift)  -> P (B,S,S), lab1 (B,S) row labels (entry 0 is never written by the kernel), lab2 (B,S) column labels
    (wts and pred: fine_weights)"""
    e = torch.exp(A.to(F64) - f32(shift))
    P = e / e.sum(2, keepdim=True) * (e / e.sum(1, keepdim=True))
    return P, first_argmax(P, 2), first_argmax(P, 1)


def fine_weights(P, lab1, lab2, pts2):
    """wts and pred of sam6d_fine_assign from P and the given labels (fine_Rt, model_utils.py:262-270):
    w_i = [lab1_i > 0] sum_{j>=1, lab2_j>0} P_ij, pred_i = sum_{j>=1} [lab1_i > 0][lab2_j > 0] P_ij pts2_j / (w_i + 1e-6f)
    -> w (B,N), pred (B,N,3), the masked inner block (B,N,N)"""
    m1, m2 = (lab1[:, 1:] > 0).to(F64), (lab2[:, 1:] > 0).to(F64)
    inner = P[:, 1:, 1:] * m1.unsqueeze(2) * m2.unsqueeze(1)
    w = inner.sum(2)
    pred = (inner @ pts2.to(F64)) / (w.unsqueeze(2) + EPS6)
    return w, pred, inner


def pose_score(pts1, lab1, R, t, model, radius, dis_thres=0.15):
    """sam6d_pose_score (model_utils.py:271-281, fine_point_matching.py:80): d_i = min_m |(p_i - t) R - m|,
    hits = #{lab1_i > 0, d_i < dis_thres}, valid = #{lab1_i > 0}, score = hits / (valid + 1e-8f) * valid / N,
    t_scaled = t (radius + 1e-6f)  -> d (B,N), hits, valid, score, t_scaled"""
    d = min_dist(transform(pts1, R.unsqueeze(1), t.unsqueeze(1)), model).squeeze(1)
    mk = lab1[:, 1:] > 0
    hits = ((d < f32(dis_thres)) & mk).sum(1)
    valid = mk.sum(1)
    N = d.shape[1]
    score = hits.to(F64) / (valid.to(F64) + EPS8) * (valid.to(F64) / N)
    return d, hits, valid, score, t.to(F64) * (radius.to(F64) + EPS6).unsqueeze(1)
