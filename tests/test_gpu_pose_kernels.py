"""GPU: the CUDA-core kernels that turn the PEM's score matrices into poses (geo.cu: geo_indices; coarse.cu: coarse_assign,
coarse_sample, coarse_hypotheses, topk_smallest, coarse_select; fine.cu: fine_assign, weighted_procrustes, pose_score; the
3x3 solver of svd3.cuh), called directly through the C ABI at the shapes bench.py runs (B = 32 proposals, S = 197 sparse
points with the background point, n1 = 6000 hypotheses, n2 = 300 kept, nm = 1024 CAD samples, N = 2048 dense points,
dis_thres = 0.15 on clouds in the unit ball) and at the edges of their loops, each against the float64 restatement of
tests/_pose_ref.py on the fp32 operands the kernel reads.

Every bound is derived from the kernel's arithmetic and written next to its check.  Notation: u = 2^-24 (fp32 unit
roundoff), gamma_n ~ n u for a chain of n fp32 roundings.  Documented accuracy of the math functions used: expf 2 ulp,
__expf 2 + floor(1.173 |x|) ulp (|x| <= 2 / temp = 20 in fine.cu), atan2f 3 ulp; sqrtf and division are IEEE (nvcc's
defaults).  An ulp of a result in [2^k, 2^(k+1)) is 2u 2^k, so k ulp are at most 2k u relative.  Sums in double precision
are charged 1e-12 relative.

Discrete outputs (labels, k-NN sets, sample indices, hits, the picked hypothesis): where the float64 decision margin exceeds
the derived error the kernel must match exactly; elsewhere its choice must be one the bound allows, and the count of such
undecided elements is printed (~0 on random data).  Planted exact ties must go to the first index.  Each check prints its
largest error / bound ratio; where a bound could hide a mistake, a plausible wrong answer computed in torch must fail it."""
import math

import numpy as np
import pytest
import torch

import _pose_ref as pr   # noqa: E402

pytestmark = pytest.mark.gpu

U = pr.U
F64 = torch.float64
DEV = "cuda"
SIGMA_D, FACTOR_A = 0.2, 180.0 / (15.0 * math.pi)      # transformer.py: sigma_d, 180 / (sigma_a pi)
THR = 0.15


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from sam6d_b200 import ops as _ops
    return _ops


@pytest.fixture(scope="module")
def refused():
    from sam6d_b200._lib import Sam6dError
    return Sam6dError


def _gc(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _ratio(err, bound):
    """max over elements of err / bound (0 / 0 counts as 0: outputs that must be exact)"""
    err, bound = err.to(F64), bound.to(F64)
    assert torch.isfinite(err).all(), "non-finite output"
    return (err / bound.clamp_min(1e-300)).max().item() if err.numel() else 0.0


def _check(name, err, bound):
    r = _ratio(err, bound)
    print(f"{name}: max error / bound = {r:.3g}  (max error {err.max().item() if err.numel() else 0:.3g})")
    assert r <= 1.0, f"{name}: error exceeds its bound by {r:.3g}x"
    return r


def _negative(name, err, bound):
    """a plausible wrong answer must fail the bound the kernel passes"""
    r = _ratio(err, bound)
    print(f"{name} (negative control): max error / bound = {r:.3g}")
    assert r > 1.0, f"{name}: the bound does not tell a wrong answer apart"


def _undecided(name, undecided, total):
    n = int(undecided)
    print(f"{name}: {n} undecided of {int(total)}")


def _ball(B, n, g, r=1.0):
    x = torch.randn(B, n, 3, generator=g, device=DEV)
    return x / x.norm(dim=2, keepdim=True) * torch.rand(B, n, 1, generator=g, device=DEV) ** (1 / 3) * r


def _rotations(B, g):
    q = torch.randn(B, 4, generator=g, device=DEV, dtype=F64)
    q = q / q.norm(dim=1, keepdim=True)
    w, x, y, z = q.unbind(1)
    return torch.stack([1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w),
                        2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w),
                        2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)], 1).view(B, 3, 3)


def _frob(x):
    return x.flatten(-2).norm(dim=-1)


# ================================================================================================== 1. geo_indices (geo.cu)
def _angle_bound(theta, fa):
    """angle of the kernel in the fp32 difference vectors r, a (each component one rounding: |dr| <= u |r|, 2u of angle for
    both); the cross product (fma + product per component: |ds| <= gamma_2 sqrt(2) |r||a| + the norm's gamma_3 + sqrtf) and
    the dot product (fma chain of 3: |dc| <= gamma_3 |r||a|) move atan2 by at most (|ds| + |dc|) / (|r||a|) <= 9u; atan2f
    3 ulp <= 6u theta; times factor_a one rounding.  Rounded up: 14u + 6u theta radians."""
    return fa * (14 * U + 6 * U * theta) * (1 + 2 * U) + U * fa * theta


def _geo_check(ops, pts, name, chunk=256):
    B, S, _ = pts.shape
    T = ops.geo_indices(pts, SIGMA_D, FACTOR_A)
    sig, fa = pr.f32(SIGMA_D), pr.f32(FACTOR_A)
    nrm = pts.to(F64).norm(dim=2)
    r_d = r_a = 0.0
    und = tot = 0
    neg = []
    for a0 in range(0, S, chunk):
        anc = torch.arange(a0, min(S, a0 + chunk), device=DEV)
        d_idx, ang, dist, knn, rn, an = pr.geo_indices(pts, SIGMA_D, FACTOR_A, anc)
        Tk = T[:, anc].to(F64)
        # distance: expanded form |x|^2 - 2 x.y + |y|^2, three fma chains + two combining roundings: gamma_5 on
        # (|x| + |y|)^2 >= |x|^2 + 2 sum |x_i y_i| + |y|^2; then sqrtf and the division by sigma_d (one rounding each)
        ed = pr.dist_err(dist, pr.sqdist_err(nrm[:, anc].unsqueeze(2), nrm.unsqueeze(1), 5))
        r_d = max(r_d, _check(f"geo_indices {name} d/sigma_d", (Tk[..., 3] - d_idx).abs(), ed / sig * (1 + U) + U * d_idx))
        # k-NN: decided when each consecutive gap of the five smallest (distance, index) exceeds both bounds, or the two
        # points are bitwise duplicates (identical fp32 distances, ordered by index in the kernel as in the stable sort)
        v5, i5 = pr.knn_sorted(dist, 4)
        e5 = ed.gather(2, i5)
        bidx = torch.arange(B, device=DEV).view(B, 1, 1)
        p5 = pts[bidx, i5]
        same = (p5[..., 1:, :] == p5[..., :-1, :]).all(-1)
        dec = ((v5[..., 1:] - v5[..., :-1] > e5[..., 1:] + e5[..., :-1]) | same).all(-1)      # (B,A)
        und += int((~dec).sum())
        tot += dec.numel()
        # angles: exactly 0 where r or a vanishes (j = i, coincident duplicates: the + 0.0f rule), else the bound
        zero = (rn.unsqueeze(2) == 0) | (an.unsqueeze(3) == 0)
        bnd = torch.where(zero, torch.zeros_like(ang), _angle_bound(ang / fa, fa))
        err = (Tk[..., :3] - ang).abs()
        r_a = max(r_a, _check(f"geo_indices {name} angles (decided anchors)", err[dec], bnd[dec]))
        # a neighbour-order mistake (slots 1 and 2 swapped) must fail the same bound
        sw = torch.where(bnd > 0, (Tk[..., [1, 0, 2]] - ang).abs() / bnd.clamp_min(1e-300), torch.zeros_like(bnd))
        neg.append(sw[dec].amax().item() if dec.any() else 0.0)
        # undecided anchors: each slot's angle must be the one of a neighbour the distance bound allows in that slot
        for b, ai in (~dec).nonzero().tolist():
            i = int(anc[ai])
            lo, hi = dist[b, ai] - ed[b, ai], dist[b, ai] + ed[b, ai]
            for k in range(1, 4):
                cand = ((lo <= v5[b, ai, k] + e5[b, ai, k]) & (hi >= v5[b, ai, k] - e5[b, ai, k])).nonzero().flatten()
                best = math.inf
                for j in cand.tolist():
                    kn = torch.tensor([[[i, j, j, j]]], device=DEV)
                    a_j, rn_j, _ = pr.triplet_angles(pts[b:b + 1], torch.tensor([i], device=DEV), kn, fa)
                    z = (rn_j[0, 0, 0] == 0) | (an[b, ai] == 0)
                    bj = torch.where(z, torch.zeros_like(a_j[0, 0, :, 0]), _angle_bound(a_j[0, 0, :, 0] / fa, fa))
                    best = min(best, _ratio((Tk[b, ai, :, k - 1] - a_j[0, 0, :, 0]).abs(), bj))
                assert best <= 1.0, f"geo_indices {name}: anchor {i} slot {k} matches no allowed neighbour"
    _undecided(f"geo_indices {name} k-NN", und, tot)
    if S > 4:
        _negative(f"geo_indices {name} angles, neighbours 1 and 2 swapped", torch.tensor([max(neg)]), torch.ones(1))
    return T, r_d, r_a


def test_geo_indices_bench_layout(ops):
    """64 clouds of 197 points, the background point (100, 100, 100) as row 0 (2B clouds per step)"""
    g = _gc(11)
    pts = _ball(64, 197, g)
    pts[:, 0] = 100.0
    _geo_check(ops, pts, "B=64 S=197")


@pytest.mark.parametrize("B,S", [(3, 4), (1, 4096)])
def test_geo_indices_size_limits(ops, refused, B, S):
    """S = 4 (the minimum: three neighbours besides the anchor) and S = 4096 (the shared-memory maximum); 4097 is refused"""
    g = _gc(S)
    _geo_check(ops, _ball(B, S, g), f"B={B} S={S}")
    if S == 4096:
        with pytest.raises(refused, match="invalid argument"):
            ops.geo_indices(_ball(1, 4097, g), SIGMA_D, FACTOR_A)


def test_geo_indices_duplicate_points(ops):
    """bitwise-duplicate points (FPS on a mask with few distinct pixels): their zero distances are exact, ties go to the
    smaller index in the kernel as in the stable sort, and every angle against a coincident point is exactly 0"""
    g = _gc(12)
    base = _ball(4, 40, g)
    pick = torch.randint(0, 40, (4, 197), generator=g, device=DEV)
    pick[:, :40] = torch.arange(40, device=DEV)
    pts = base.gather(1, pick.unsqueeze(2).expand(-1, -1, 3)).contiguous()
    pts[:, 0] = 100.0
    T, _, _ = _geo_check(ops, pts, "duplicates")
    # the + 0.0f rule, directly: the anchor against itself and against its coincident copies
    eq = (pts.unsqueeze(2) == pts.unsqueeze(1)).all(-1)
    assert (T[..., :3][eq] == 0).all() and not torch.signbit(T[..., :3][eq]).any()


# ================================================================================================== 2. coarse_assign
def _score_matrix(B, S, g, bg_rows=0.15, dim=32, noise=0.6):
    """|A| <= 10 (cosine / temp): planted correspondences, background row / column 0, a share of rows matching it"""
    f1 = torch.nn.functional.normalize(torch.randn(B, S, dim, generator=g, device=DEV), dim=2)
    perm = torch.argsort(torch.rand(B, S, generator=g, device=DEV), 1)
    perm[:, 0] = 0
    f2 = f1.gather(1, perm.unsqueeze(2).expand(-1, -1, dim)) + noise * torch.randn(B, S, dim, generator=g, device=DEV)
    f2 = torch.nn.functional.normalize(f2, dim=2)
    bg = torch.rand(B, S, generator=g, device=DEV) < bg_rows
    f1 = torch.where(bg.unsqueeze(2), torch.nn.functional.normalize(f2[:, :1] + noise * torch.randn(B, S, dim, generator=g,
                                                                                                   device=DEV), dim=2), f1)
    return ((f1 @ f2.transpose(1, 2)) * 10.0).clamp(-10, 10).contiguous()


def _assign_bound(A):
    """relative bound on the kernel's P = (expf(a - rmax) / rsum) (expf(a - cmax) / csum): expf 2 ulp (4u) and the argument
    rounding (u |a - max|) per factor; the row sum (per lane ceil(S/32) terms, 5 shuffle levels) and the column sum (S
    serial terms) carry their terms' worst relative error plus gamma of their depth; two divisions and the product 3u"""
    A = A.to(F64)
    B, S, _ = A.shape
    xr, xc = (A - A.amax(2, keepdim=True)).abs(), (A - A.amax(1, keepdim=True)).abs()
    rs = 4 * U + U * xr.amax(2, keepdim=True) + pr.gamma(-(-S // 32) + 5)
    cs = 4 * U + U * xc.amax(1, keepdim=True) + pr.gamma(S)
    return 1.01 * (8 * U + U * (xr + xc) + rs + cs + 3 * U)


def _coarse_assign_check(ops, A, name):
    B, S, _ = A.shape
    n = S - 1
    W, w1 = ops.coarse_assign(A)
    P, l1, l2 = pr.soft_assignment(A)
    eP = _assign_bound(A) * P
    _, dec1, al1 = pr.argmax_decided(P, eP, 2)
    _, dec2, al2 = pr.argmax_decided(P, eP, 1)
    dec1, dec2, al1, al2 = dec1[:, 1:], dec2[:, 1:], al1[:, 1:], al2.transpose(1, 2)[:, 1:]
    _undecided(f"coarse_assign {name} row labels", (~dec1).sum(), dec1.numel())
    _undecided(f"coarse_assign {name} column labels", (~dec2).sum(), dec2.numel())
    fg_ref = (l1[:, 1:] > 0).to(F64)
    assert torch.equal(w1.to(F64)[dec1], fg_ref[dec1]), f"coarse_assign {name}: w1 differs on a decided row"
    ok = torch.where(w1 > 0, al1[..., 1:].any(-1), al1[..., 0])
    assert ok.all(), f"coarse_assign {name}: w1 on an undecided row is a label the bound does not allow"
    # W: v * sqrtf(v) -> 1.5 x P's relative bound, sqrtf and the product 2u; rows with w1 = 0 exactly 0; an undecided
    # column may be masked either way
    Wr = P[:, 1:, 1:].pow(1.5)
    eW = (1.5 * _assign_bound(A)[:, 1:, 1:] + 2.01 * U) * Wr
    Wk = W.view(B, n, n).to(F64)
    m2 = (l2[:, 1:] > 0).to(F64).unsqueeze(1)
    err = (Wk - Wr * w1.to(F64).unsqueeze(2) * m2).abs()
    err_alt = torch.minimum(Wk.abs(), (Wk - Wr).abs())
    err = torch.where(dec2.unsqueeze(1) | (w1.unsqueeze(2) == 0), err, torch.minimum(err, err_alt))
    assert (Wk[w1 == 0] == 0).all()
    r = _check(f"coarse_assign {name} W", err, eW)
    return W, w1, r


def test_coarse_assign_bench(ops):
    """B = 32, S = 197, |A| <= 10, rows and columns whose argmax is the background"""
    _coarse_assign_check(ops, _score_matrix(32, 197, _gc(21)), "B=32 S=197")


def test_coarse_assign_edges(ops):
    """a proposal with every row background (W = 0, w1 = 0); planted exact ties in P between the background and a
    foreground column / row, which go to the first index (background): w1 = 0 for the tied rows, W = 0 for the tied columns"""
    g = _gc(22)
    A = _score_matrix(3, 197, g)
    A[0, :, 0] = 10.0                                      # every row's maximum is the background column
    A[0, :, 1:] = A[0, :, 1:].clamp(-1, 1)
    A[1, :, 0] = A[1, :, 1]                                 # columns 0 and 1 identical: P ties exactly in every row
    A[1, 5:25, 2:] = A[1, 5:25, 2:].clamp(max=0.0)
    A[1, 5:25, :2] = 10.0
    A[2, 0, :] = A[2, 1, :]                                 # rows 0 and 1 identical: P ties exactly in every column
    A[2, 2:, 30:45] = A[2, 2:, 30:45].clamp(max=0.0)
    A[2, :2, 30:45] = 10.0
    W, w1, _ = _coarse_assign_check(ops, A.contiguous(), "edges")
    assert (W[0] == 0).all() and (w1[0] == 0).all()
    assert (w1[1, 4:24] == 0).all(), "a row tied between background and column 1 must take the background"
    assert (W[2].view(196, 196)[:, 29:44] == 0).all(), "a column tied between background and row 1 must take the background"
    assert (W[2].view(196, 196)[:, 50:] != 0).any()


def test_coarse_assign_size_limit(ops, refused):
    """S = 234 fills 220 KB of shared memory; S = 235 is refused"""
    _coarse_assign_check(ops, _score_matrix(2, 234, _gc(23)), "S=234")
    with pytest.raises(refused, match="invalid argument"):
        ops.coarse_assign(_score_matrix(1, 235, _gc(24)))


# ================================================================================================== 3. coarse_sample
def _sample_check(ops, W, rand, name):
    B, L = W.shape
    idx = ops.coarse_sample(W, rand).long()
    c = pr.cdf(W)
    e = pr.cdf_err(c)
    ref = pr.searchsorted(c, rand)
    v = rand.to(F64)
    # whatever the kernel's cdf^ looks like, its binary search ends at an index k with cdf^[k-1] < v (or k = 0) and
    # cdf^[k] >= v (or k = L): both were probed.  With |cdf^ - cdf| <= e elementwise that makes the draw decided when
    # cdf[ref] - e >= v (or ref = L) and cdf[ref-1] + e < v (or ref = 0), and bounds k by the same test otherwise
    cp = torch.cat([torch.full((B, 1), -1.0, dtype=F64, device=DEV), c], 1)     # cp[i] = cdf[i-1]
    ep = torch.cat([torch.zeros(B, 1, dtype=F64, device=DEV), e], 1)
    cx = torch.cat([c, torch.full((B, 1), 2.0, dtype=F64, device=DEV)], 1)      # cx[L] = beyond every draw
    ex = torch.cat([e, torch.zeros(B, 1, dtype=F64, device=DEV)], 1)
    dec = (cx.gather(1, ref) - ex.gather(1, ref) >= v) & (cp.gather(1, ref) + ep.gather(1, ref) < v)
    _undecided(f"coarse_sample {name}", (~dec).sum(), dec.numel())
    assert torch.equal(idx[dec], ref[dec]), f"coarse_sample {name}: a decided draw differs"
    allowed = (cx.gather(1, idx) + ex.gather(1, idx) >= v) & (cp.gather(1, idx) - ep.gather(1, idx) < v)
    assert allowed.all(), f"coarse_sample {name}: an undecided draw outside the bound"
    # a zero run is a plateau of the cdf: the search never lands inside it.  Within one thread's chunk of ceil(L / 1024)
    # entries cdf^ is a running double sum rounded to fp32, so W = 0 repeats the previous value exactly; a chunk's first
    # entry comes from the double scan of the partials instead and may round differently from its predecessor
    per = -(-L // 1024)
    inside = (idx > 0) & (idx < L) & (idx % per != 0)
    assert (W.gather(1, idx.clamp(max=L - 1))[inside] > 0).all(), f"coarse_sample {name}: index inside a plateau"
    return idx, ref


def test_coarse_sample_bench(ops):
    """L = 196^2, nr = 18 000 draws per proposal at B = 32, on the kernel's own W"""
    W, _, _ = _coarse_assign_check(ops, _score_matrix(32, 197, _gc(31)), "for sampling")
    _sample_check(ops, W, torch.rand(32, 18000, generator=_gc(32), device=DEV), "L=196^2")


@pytest.mark.parametrize("L", [700, 5000])
def test_coarse_sample_edges(ops, L):
    """L < 1024 and L not a multiple of 1024; zero runs (the first index of a plateau, also at the start: rand = 0 -> 0);
    W = 0 (every draw with rand > 0 gives L); a tiny total so that rand > cdf[L-1] gives L"""
    g = _gc(L)
    W = torch.rand(4, L, generator=g, device=DEV) ** 3
    W[:, :10] = 0.0
    W[:, L // 3:L // 3 + 50] = 0.0
    W[:, L // 2:L // 2 + 1] = 0.0
    W[1] = 0.0
    W[2] *= 1e-8 / W[2].sum()                               # cdf[L-1] = 1e-8 / (1e-8 + 1e-8f) ~ 0.5
    rand = torch.rand(4, 3000, generator=g, device=DEV)
    rand[:, :5] = 0.0
    rand[:, 5:10] = 0.9999999
    c = pr.cdf(W)
    rand[:, 10] = c[:, L // 3].float()                      # a draw equal to a plateau's value
    idx, ref = _sample_check(ops, W, rand, f"L={L}")
    assert (idx[:, :5] == 0).all(), "rand = 0 is the first index: cdf[0] = 0 >= 0"
    assert (idx[1][rand[1] > 0] == L).all() and (idx[2, 5:10] == L).all()


# ================================================================================================== 4. coarse_hypotheses
def _hyp_check(ops, idx, pts1, pts2, name, neg=False):
    Rt, resid = ops.coarse_hypotheses(idx, pts1, pts2)
    B, n1 = Rt.shape[:2]
    h = pr.triplet_procrustes(idx, pts1, pts2)
    W3 = pr.W3
    p1, p2, a, b = h["p1"], h["p2"], h["a"], h["b"]
    # centroids: p_0 w + p_1 w + p_2 w, a product and two fma: gamma_3 on w sum |p| (w is the fp32 constant)
    dcs = pr.gamma(3) * W3 * p2.abs().sum(2) * 1.01
    dcr = pr.gamma(3) * W3 * p1.abs().sum(2) * 1.01
    # centred points: one rounding of p - c^; the reference side times w, one more rounding
    da = dcs.unsqueeze(2) + U * (a.abs() + dcs.unsqueeze(2))
    db = 1.01 * (W3 * (dcr.unsqueeze(2) + U * (p1 - h["cr"].unsqueeze(2)).abs()) + U * b.abs())
    dHF = pr.cross_cov_err(a, b, da, db)
    bR = pr.rotation_err(dHF.reshape(-1), h["S"].reshape(-1, 3), h["sdet"].reshape(-1), h["rank1"].reshape(-1),
                         h["rank0"].reshape(-1), h["c"].reshape(-1)).view(B, n1)
    Rk, tk = Rt[..., :9].view(B, n1, 3, 3).to(F64), Rt[..., 9:].to(F64)
    rR = _check(f"coarse_hypotheses {name} R (Frobenius)", _frob(Rk - h["R"]), bR)
    assert torch.equal(Rk[h["rank0"]], torch.eye(3, dtype=F64, device=DEV).expand(int(h["rank0"].sum()), 3, 3))
    # t = c_r - R c_s (fp32 R; fma chain of 3 and the subtraction: gamma_4)
    R, cs, cr = h["R"], h["cs"], h["cr"]
    bt = 1.01 * (dcr + bR.unsqueeze(2) * cs.norm(dim=2, keepdim=True) + (R.abs() @ dcs.unsqueeze(3)).squeeze(3)
                 + pr.gamma(4) * (cr.abs() + (R.abs() @ cs.abs().unsqueeze(3)).squeeze(3)))
    rt = _check(f"coarse_hypotheses {name} t", (tk - h["t"]).abs(), bt)
    # residual: x = p1 - t (one rounding, and the t error), y = x R - p2 (fma chain of 3 and the subtraction: gamma_4 on
    # |x||R| + |p2|; the R error |dR|_2 |x|), its norm (gamma_3 under sqrtf, sqrtf: 3u |y|), sum of three and / 3 (3u)
    x = p1 - h["t"].unsqueeze(2)
    y = x @ R - p2
    dy = (bR.view(B, n1, 1) * x.norm(dim=3) + bt.norm(dim=2, keepdim=True)
          + (pr.gamma(4) * (x.abs() @ R.abs() + p2.abs()) + U * x.abs() @ R.abs()).norm(dim=3) + 3 * U * y.norm(dim=3))
    bres = 1.02 * (dy.mean(2) + 3 * U * h["resid"])
    rr = _check(f"coarse_hypotheses {name} resid", (resid.to(F64) - h["resid"]).abs(), bres)
    if neg:
        # the plain mean (weights 1/3) instead of 1 / (3 + 1e-5): t moves by 3.3e-6 |c|
        cs3, cr3 = p2.mean(2), p1.mean(2)
        _negative(f"coarse_hypotheses {name} t with the plain mean", (cr3 - (R @ cs3.unsqueeze(3)).squeeze(3) - h["t"]).abs(),
                  bt)
        # no determinant correction (R = V U^T): a reflection for about half the rank-2 triplets
        full = ~(h["rank1"] | h["rank0"])
        Uq, _, Vh = torch.linalg.svd(h["H"][full])
        _negative(f"coarse_hypotheses {name} R without det correction", _frob(Vh.transpose(1, 2) @ Uq.transpose(1, 2) - R[full]),
                  bR[full])
    return Rt, resid, h, (rR, rt, rr)


def _bench_draw(B, n, n1, g, wrong=0.3):
    pts2 = _ball(B, n, g)
    Rg = _rotations(B, g).float()
    pts1 = (pts2 @ Rg.transpose(1, 2) + 0.1 * torch.randn(B, 1, 3, generator=g, device=DEV)
            + 0.01 * torch.randn(B, n, 3, generator=g, device=DEV)).contiguous()
    i = torch.randint(0, n, (B, 3 * n1), generator=g, device=DEV)
    idx = i * n + i
    bad = torch.rand(B, 3 * n1, generator=g, device=DEV) < wrong
    idx = torch.where(bad, torch.randint(0, n * n, (B, 3 * n1), generator=g, device=DEV), idx)
    idx[:, :30] = n * n                                     # idx = L (no cdf entry >= rand): the clamp to n - 1
    return idx.int().contiguous(), pts1, pts2


def test_coarse_hypotheses_bench(ops):
    """B = 32, n1 = 6000 on 196 points: a planted pose, noise, 30 % wrong correspondences, idx = L; every hypothesis (the
    rank-1 and rank-0 triplets that repeat a point included) inside its bound"""
    idx, pts1, pts2 = _bench_draw(32, 196, 6000, _gc(41))
    _, _, h, _ = _hyp_check(ops, idx, pts1, pts2, "bench", neg=True)
    print(f"coarse_hypotheses bench: {int(h['rank1'].sum())} rank-1, {int(h['rank0'].sum())} rank-0 hypotheses")


def test_coarse_hypotheses_hand_built(ops):
    """nearly collinear triplets (sigma2/sigma1 ~ 1e-3, 1e-5), a mirror image, an exact half turn, rank-1 triplets (one
    with antiparallel directions: c = -1, the half-turn branch), rank-0 triplets, coincident points with distinct indices"""
    n = 24
    g = _gc(42)
    p2 = _ball(1, n, g)[0].clone()
    Rg = _rotations(1, g)[0].float()
    p1 = p2 @ Rg.T + 0.05
    tri = []
    for k, eps in ((0, 0.028), (3, 0.0028)):               # nearly collinear: sigma2/sigma1 ~ eps^2
        p2[k] = torch.tensor([-0.5, 0.1, 0.2], device=DEV)
        p2[k + 1] = torch.tensor([0.5, 0.1, 0.2], device=DEV)
        p2[k + 2] = torch.tensor([0.0, 0.1 + eps, 0.2], device=DEV)
        p1[k:k + 3] = p2[k:k + 3] @ Rg.T + 0.05
        tri.append([(k, k), (k + 1, k + 1), (k + 2, k + 2)])
    p1[6:9] = p2[6:9] * torch.tensor([-1.0, 1.0, 1.0], device=DEV)      # mirror image
    tri.append([(6, 6), (7, 7), (8, 8)])
    p1[9:12] = p2[9:12] * torch.tensor([-1.0, -1.0, 1.0], device=DEV)   # exact half turn about z
    tri.append([(9, 9), (10, 10), (11, 11)])
    e = torch.tensor([3.0, 2.0, 1.0], device=DEV) / math.sqrt(14.0)
    p2[12], p2[13] = 0.0, e                                 # rank 1, antiparallel: p1 runs along -e where p2 runs along e
    p1[12], p1[13] = 0.0, -e
    tri.append([(12, 12), (12, 12), (13, 13)])
    tri.append([(14, 15), (14, 16), (17, 18)])              # rank 1, generic
    tri.append([(19, 1), (19, 2), (19, 5)])                 # rank 0 (one point of pts1)
    tri.append([(1, 20), (2, 20), (5, 20)])                 # rank 0 (one point of pts2)
    p1[21], p2[21] = p1[20], p2[20]                         # coincident points, distinct indices: the full path
    tri.append([(20, 20), (21, 21), (22, 22)])
    idx = torch.tensor([[i1 * n + i2 for t in tri for (i1, i2) in t]], dtype=torch.int32, device=DEV)
    Rt, _, h, _ = _hyp_check(ops, idx, p1.unsqueeze(0).contiguous(), p2.unsqueeze(0).contiguous(), "hand-built")
    assert h["rank1"][0].tolist() == [False] * 4 + [True, True, False, False, False]
    assert h["rank0"][0].tolist() == [False] * 6 + [True, True, False]
    assert (1 + h["c"][0, 4]).abs() < 1e-9, "the antiparallel triplet takes the half-turn branch"
    print("coarse_hypotheses hand-built sigma2/sigma1:", [f"{v:.2g}" for v in (h["S"][0, :, 1] / h["S"][0, :, 0]).tolist()])


# ================================================================================================== 5. topk_smallest
def _topk_expected(v, k):
    return torch.sort(v, dim=1, stable=True)[1][:, :k]


@pytest.mark.parametrize("B,n,k,kind", [(32, 6000, 300, "resid"), (3, 100, 100, "ties"), (2, 1, 1, "rand"), (2, 2, 2, "ties"),
                                        (2, 2, 1, "rand"), (2, 1000, 7, "equal"), (2, 16384, 500, "ties")])
def test_topk_smallest_order(ops, B, n, k, kind):
    """exact (value, index) order against a stable sort of the kernel's own input: n = 6000, k = 300 on the hypothesis
    kernel's residuals; k = n; n = 1 and 2; all-equal rows; n = 16 384 (the largest power of two under the 200 KB key
    buffer); many exact ties (quantised values)"""
    g = _gc(n + k)
    if kind == "resid":
        idx, pts1, pts2 = _bench_draw(B, 196, n, g)
        _, v = ops.coarse_hypotheses(idx, pts1, pts2)
    elif kind == "ties":
        v = torch.randint(0, 37, (B, n), generator=g, device=DEV).float() / 7
    elif kind == "equal":
        v = torch.full((B, n), 0.25, device=DEV)
    else:
        v = torch.rand(B, n, generator=g, device=DEV)
    out = ops.topk_smallest(v.contiguous(), k).long()
    assert torch.equal(out, _topk_expected(v, k))


def test_topk_smallest_size_limit(ops, refused):
    with pytest.raises(refused, match="invalid argument"):
        ops.topk_smallest(torch.rand(1, 16385, device=DEV), 10)


def test_topk_smallest_signed_zero_and_nan_contract(ops):
    """the documented key order: ascending by the order-preserving map of the fp32 bit pattern, then index.  It equals
    (value, index) for ordinary values; -0.0 sorts before +0.0 whatever their indices; a NaN with the sign bit set sorts
    before everything and one without it after +inf.  (Residuals are norms: never -0, never NaN from finite inputs.)"""
    vals = [0.5, 0.0, -0.0, float("inf"), 0.0, -1.0, -0.0, -float("inf"), 0.25]
    v = torch.tensor([vals], device=DEV)
    nan_neg = torch.from_numpy(np.array([0xFFC00000], dtype=np.uint32).view(np.float32))
    v = torch.cat([v, torch.tensor([[float("nan")]], device=DEV), nan_neg.to(DEV).view(1, 1), torch.tensor([[0.1]], device=DEV)], 1)
    out = ops.topk_smallest(v.contiguous(), v.shape[1]).tolist()[0]
    u = v.cpu().view(torch.int32).numpy().view(np.uint32).astype(np.uint64)[0]
    key = np.where(u & 0x80000000, ~u & 0xFFFFFFFF, u | 0x80000000)
    assert out == sorted(range(len(key)), key=lambda i: (int(key[i]), i))
    assert out[:3] == [10, 7, 5] and out[3:5] == [2, 6] and out[5:7] == [1, 4] and out[-1] == 9


# ================================================================================================== 6. coarse_select + pick
def _select_check(ops, Rt, top, pts1, w1, model, name, neg=False):
    B, n1, _ = Rt.shape
    n2, n, nm = top.shape[1], pts1.shape[1], model.shape[1]
    R, t, sc = ops.coarse_select(Rt, top, pts1, w1, model)
    bidx = torch.arange(B, device=DEV).view(B, 1)
    sel = Rt[bidx, top.long()]                              # (B,n2,12)
    Rs, ts = sel[..., :9].view(B, n2, 3, 3), sel[..., 9:]
    ref, d = pr.select_scores(Rs, ts, pts1, w1, model)
    # per (hypothesis, point): the transformed point (p - t one rounding, fma chains of 3) within transform_err; the
    # squared distance |x|^2 + min_m (|m|^2 - 2 x.m) in fp32 (|m|^2 a chain of 3, x.m an fma chain of 3 onto it, |x|^2 a
    # chain of 3, the sum one rounding): gamma_8 on (|x| + max |m|)^2; sqrtf.  The minimum is exact.
    xt = pr.transform(pts1, Rs, ts)
    M = model.to(F64).norm(dim=2).amax(1).view(B, 1, 1)
    dd = pr.transform_err(pts1, Rs, ts) + pr.dist_err(d, pr.sqdist_err(xt.norm(dim=3), M, 8))
    w = w1.to(F64).unsqueeze(1)
    den = (d * w).sum(2)
    # the sums: per thread ceil(n / 224) points, 5 shuffle levels, 7 warps, and the final + 1e-8f and division
    depth = -(-n // 224) + 5 + 7 + 1
    den_err = (dd * w).sum(2) + pr.gamma(depth) * den
    bound = 1.01 * ref * ((den_err + U * (den + pr.EPS8)) / (den + pr.EPS8) + 2 * U)
    r = _check(f"coarse_select {name} scores", (sc.to(F64) - ref).abs(), bound)
    # the pick: the first maximum of the kernel's own scores, its R, t copied bitwise; its fp64 score within twice the
    # bound of the fp64 maximum
    pick = pr.first_argmax(sc, 1)
    win = Rt[torch.arange(B, device=DEV), top[torch.arange(B, device=DEV), pick].long()]
    assert torch.equal(R.view(B, 9), win[:, :9]) and torch.equal(t, win[:, 9:]), f"coarse_select {name}: pick not copied"
    best = ref.amax(1)
    got = ref.gather(1, pick.unsqueeze(1)).squeeze(1)
    assert (got >= best - 2 * bound.amax(1)).all(), f"coarse_select {name}: the pick is not a maximum within the bound"
    if neg:
        # the odd tail dropped (the last CAD sample never scored)
        wrong, _ = pr.select_scores(Rs, ts, pts1, w1, model[:, :nm - 1])
        _negative(f"coarse_select {name} scores without the last CAD sample", (wrong - ref).abs(), bound)
    return sc, pick, ref


def _select_case(B, n, n1, n2, nm, g):
    Rt = torch.cat([_rotations(B * n1, g).view(B, n1, 9), 0.1 * torch.randn(B, n1, 3, generator=g, device=DEV, dtype=F64)],
                   2).float().contiguous()
    top = torch.argsort(torch.rand(B, n1, generator=g, device=DEV), 1)[:, :n2].int().contiguous()
    pts1 = _ball(B, n, g)
    w1 = (torch.rand(B, n, generator=g, device=DEV) < 0.8).float()
    model = _ball(B, nm, g)                                  # a different CAD model per proposal
    return Rt, top, pts1, w1, model


@pytest.mark.parametrize("n2,nm", [(300, 1024), (301, 1023), (1, 1024), (300, 1), (5, 1023)])
def test_coarse_select_shapes(ops, n2, nm):
    """n2 = 300, 301 and 1 (a partial last SEL_PP group); nm = 1024, 1023 and 1 (the odd tail); B = 32, n = 196, n1 = 6000,
    a different CAD model per proposal"""
    Rt, top, pts1, w1, model = _select_case(32 if n2 >= 300 else 4, 196, 6000, n2, nm, _gc(n2 * 7 + nm))
    _select_check(ops, Rt, top, pts1, w1, model, f"n2={n2} nm={nm}", neg=(nm == 1023))


def test_coarse_select_edges(ops, refused):
    """nm = 12 800 (the 200 KB limit) and 12 801 refused; w1 = 0 (every score 0, pick 0); duplicate hypotheses (equal
    scores: the first wins)"""
    g = _gc(61)
    Rt, top, pts1, w1, model = _select_case(3, 196, 500, 40, 12800, g)
    w1[1] = 0.0
    top[2] = top[2, 0]                                      # one hypothesis 40 times
    top[0, 10:20] = top[0, :10]
    sc, pick, _ = _select_check(ops, Rt, top.contiguous(), pts1, w1, model, "nm=12800")
    assert (sc[1] == 0).all() and pick[1] == 0
    assert (sc[2] == sc[2, 0]).all() and pick[2] == 0
    assert torch.equal(sc[0, 10:20], sc[0, :10]) and not (10 <= int(pick[0]) < 20), "a duplicate's first copy wins"
    with pytest.raises(refused, match="invalid argument"):
        ops.coarse_select(Rt, top.contiguous(), pts1, w1, _ball(3, 12801, g))


# ================================================================================================== 7. fine_assign (fp32 arm)
def _fine_bound(A, shift):
    """relative bound on the kernel's P = (e rinv)(e cinv), e = __expf(a - shift): per factor 2 + floor(1.173 |x|) ulp and
    the argument's rounding (u |x|); row sums: pairs of 4 columns, ceil(S/1024) groups, 5 shuffle levels, 8 warps and the
    tail (gamma of that depth); column sums: 32 rows per tile then `tiles` partials (gamma_{32 + tiles}); the two
    reciprocals and three products"""
    x = (A.to(F64) - pr.f32(shift)).abs()
    S = A.shape[1]
    ee = (2 + 1.173 * x) * 2 * U + U * x
    rs = ee.amax(2, keepdim=True) + pr.gamma(2 + -(-S // 1024) + 5 + 8 + 1)
    cs = ee.amax(1, keepdim=True) + pr.gamma(32 + -(-S // 32))
    return 1.01 * (2 * ee + rs + cs + 5 * U)


def _fine_check(ops, A, pts2, name, neg=False):
    """A: (B,S,S) view with row stride ld"""
    B, S, _ = A.shape
    N = S - 1
    lab1, lab2, wts, pred = ops.fine_assign(A, pts2, 10.0)
    lab1, lab2 = lab1.long(), lab2.long()
    r = {}
    und = [0, 0]
    wk, pk = [], []
    for b in range(B):
        Ab = A[b:b + 1].contiguous()
        P, l1, l2 = pr.fine_assign(Ab, 10.0)
        rel = _fine_bound(Ab, 10.0)
        eP = rel * P
        _, dec1, al1 = pr.argmax_decided(P, eP, 2)
        _, dec2, al2 = pr.argmax_decided(P, eP, 1)
        dec1, al1 = dec1[:, 1:], al1[:, 1:]
        und[0] += int((~dec1).sum())
        und[1] += int((~dec2).sum())
        assert torch.equal(lab1[b:b + 1, 1:][dec1], l1[:, 1:][dec1]), f"fine_assign {name}: decided row label differs"
        assert torch.equal(lab2[b:b + 1][dec2], l2[dec2]), f"fine_assign {name}: decided column label differs"
        assert al1.gather(2, lab1[b:b + 1, 1:].unsqueeze(2)).all() and al2.gather(1, lab2[b:b + 1].unsqueeze(1)).all()
        # wts, pred from the kernel's own labels: per lane 4 ceil(S/128) sequential adds (or fma), 5 shuffle levels
        w, pd, inner = pr.fine_weights(P, lab1[b:b + 1], lab2[b:b + 1], pts2[b:b + 1])
        inner_e = inner * rel[:, 1:, 1:]
        depth = 4 * -(-S // 128) + 5
        we = 1.01 * (inner_e.sum(2) + pr.gamma(depth) * w)
        q = pts2[b:b + 1].to(F64)
        num = inner @ q
        ne = inner_e @ q.abs() + pr.gamma(depth) * (inner @ q.abs())
        dw = we + U * (w + pr.EPS6)
        pe = 1.01 * (ne + pd.abs() * dw.unsqueeze(2)) / (w + pr.EPS6).unsqueeze(2) + U * pd.abs()
        wk.append(((wts[b:b + 1].to(F64) - w).abs(), we))
        pk.append(((pred[b:b + 1].to(F64) - pd).abs(), pe))
        if neg and b == 0:
            _negative(f"fine_assign {name} pred without + 1e-6", (num / w.clamp_min(1e-300).unsqueeze(2) - pd).abs(), pe)
    bg = lab1[:, 1:] == 0
    assert (wts[bg] == 0).all() and (pred[bg] == 0).all(), "rows labelled background carry no weight"
    _undecided(f"fine_assign {name} row labels", und[0], B * N)
    _undecided(f"fine_assign {name} column labels", und[1], B * S)
    r["wts"] = _check(f"fine_assign {name} wts", torch.cat([e for e, _ in wk]), torch.cat([b for _, b in wk]))
    r["pred"] = _check(f"fine_assign {name} pred", torch.cat([e for e, _ in pk]), torch.cat([b for _, b in pk]))
    return lab1, lab2, wts, pred


def _padded(A, ld, fill=0.0):
    B, S, _ = A.shape
    store = torch.full((B, S, ld), fill, device=DEV)
    store[:, :, :S] = A
    return store[:, :, :S]


@pytest.mark.parametrize("B,S", [(32, 2049), (2, 97), (2, 1025), (2, 1028), (2, 1029), (2, 2052)])
def test_fine_assign_shapes(ops, B, S):
    """S = 2049 at B = 32 (N = 2048), the S = 97 minimum, either side of the row-parallel tail switch (S & 1023 in 1..4):
    1025, 1028 (tail), 1029 and 2052 (no tail)"""
    g = _gc(S)
    A = _score_matrix(B, S, g, dim=48)
    pts2 = _ball(B, S - 1, g)
    _fine_check(ops, _padded(A, (S + 3) // 4 * 4), pts2, f"B={B} S={S}", neg=(S == 2049))


@pytest.mark.parametrize("S", [1027, 2049])
def test_fine_assign_nan_padding(ops, S):
    """padding columns hold arbitrary bits: with S % 4 != 0 the last 16-byte load of every row and of the row-parallel tail
    reads padding columns (1027 at S = 1027, 2049..2051 at S = 2049), and ld is well above round4(S).  NaN there must give
    results bit-identical to clean padding (exp4 selects, never multiplies: NaN * 0 is NaN)"""
    g = _gc(S + 7)
    A = _score_matrix(2, S, g, dim=48)
    pts2 = _ball(2, S - 1, g)
    ld = (S + 3) // 4 * 4 + 100
    clean = ops.fine_assign(_padded(A, ld), pts2, 10.0)
    out = _fine_check(ops, _padded(A, ld, float("nan")), pts2, f"S={S} ld={ld} NaN padding")
    for a, b in zip(clean, out):
        assert torch.equal(a.view(torch.int32) if a.is_floating_point() else a,
                           b.view(torch.int32) if b.is_floating_point() else b), "padding bits leaked into the result"


def test_fine_assign_edges(ops, refused):
    """S = 1027 (three tail columns 1024..1026, handled row-parallel): exact ties across the 32-row tile boundary (column
    labels take row 31); two identical rows of one tile whose maxima sit in a tail column (the tail's lane-level argmax
    takes row 40); identical tail columns (row labels take column 1025); all-background rows; S = 96 refused"""
    g = _gc(71)
    S = 1027
    A = _score_matrix(2, S, g, dim=48)
    A[:, :, 100:110] = A[:, :, 100:110].clamp(max=0.0)
    A[:, :, 1024] = A[:, :, 1024].clamp(max=0.0)
    A[:, 200:220] = A[:, 200:220].clamp(max=0.0)
    A[:, 400:430, 1:] = A[:, 400:430, 1:].clamp(max=0.0)    # background rows
    A[:, 31, 100:110] = 10.0
    A[:, 40, 1024] = 10.0
    A[:, 200:220, 1025] = 10.0
    A[:, 400:430, 0] = 10.0
    A[:, 32] = A[:, 31]                                     # rows 31 and 32 identical: tiles 0 and 1
    A[:, 45] = A[:, 40]                                     # rows 40 and 45 identical: both in tile 1
    A[:, :, 1026] = A[:, :, 1025]                           # tail columns 1025 and 1026 identical
    pts2 = _ball(2, S - 1, g)
    lab1, lab2, _, _ = _fine_check(ops, _padded(A, (S + 3) // 4 * 4), pts2, "S=1027 ties")
    assert (lab2[:, 100:110] == 31).all(), "a column tie across the tile boundary goes to the first row"
    assert (lab2[:, 1024] == 40).all(), "a column tie inside one tile, in a tail column, goes to the first row"
    assert (lab1[:, 200:220] == 1025).all(), "a row tie between tail columns goes to the first column"
    assert (lab1[:, 400:430] == 0).all()
    # S = 96 (three 32-row tiles) through the C ABI itself, with every buffer sized for it
    from sam6d_b200 import _lib
    S, ld = 96, 96
    A96, pts96 = _score_matrix(1, S, g), _ball(1, S - 1, g)
    f = lambda *s: torch.zeros(*s, device=DEV)              # noqa: E731
    i = lambda *s: torch.zeros(*s, dtype=torch.int32, device=DEV)   # noqa: E731
    bufs = [f(1, ld), f(1, ld), f(1, 3, ld), i(1, 3, ld), i(1, S), i(1, S), f(1, S - 1), f(1, S - 1, 3)]
    with pytest.raises(refused, match="invalid argument"):
        _lib.call("sam6d_fine_assign", A96, 1, S, ld, 10.0, pts96, *bufs)


# ================================================================================================== 8. weighted_procrustes
def _wp_check(ops, src, ref, wts, thresh, name, neg=None):
    eps = 1e-5
    R, t = ops.weighted_procrustes(src, ref, wts, thresh, eps)
    h = pr.weighted_procrustes(src, ref, wts, thresh, eps)
    s, r = src.to(F64), ref.to(F64)
    wn, cs, cr, a, b = h["wn"], h["cs"], h["cr"], h["a"], h["b"]
    # normalised weights: the double sum rounded to fp32, + eps, the division: 3u; centroids: each term s w^ one rounding
    # (plus the weight's error), a double sum rounded to fp32 (u)
    dwn = 1.01 * (3 * U + 1e-12) * wn
    dcs = 1.01 * ((s.abs() * (dwn + U * wn).unsqueeze(2)).sum(1) + U * cs.abs()) + 1e-15 * (s.abs() * wn.unsqueeze(2)).sum(1)
    dcr = 1.01 * ((r.abs() * (dwn + U * wn).unsqueeze(2)).sum(1) + U * cr.abs()) + 1e-15 * (r.abs() * wn.unsqueeze(2)).sum(1)
    # centred products: sc = s - c^ (one rounding), rc = w^ (r - c^) (two roundings and the weight's error)
    da = dcs.unsqueeze(1) + U * (a.abs() + dcs.unsqueeze(1))
    rcn = (r - cr.unsqueeze(1)).abs()
    db = 1.01 * (wn.unsqueeze(2) * (dcr.unsqueeze(1) + U * (rcn + dcr.unsqueeze(1))) + dwn.unsqueeze(2) * (rcn + dcr.unsqueeze(1))
                 + U * b.abs())
    dHF = pr.cross_cov_err(a, b, da, db)
    bR = pr.rotation_err(dHF, h["S"], h["sdet"])
    rR = _check(f"weighted_procrustes {name} R (Frobenius)", _frob(R.to(F64) - h["R"]), bR)
    Rr = h["R"]
    bt = 1.01 * (dcr + bR.unsqueeze(1) * cs.norm(dim=1, keepdim=True) + (Rr.abs() @ dcs.unsqueeze(2)).squeeze(2)
                 + pr.gamma(4) * (cr.abs() + (Rr.abs() @ cs.abs().unsqueeze(2)).squeeze(2)))
    rt = _check(f"weighted_procrustes {name} t", (t.to(F64) - h["t"]).abs(), bt)
    if neg is not None:
        if neg == "le":
            w2 = torch.where(wts <= pr.f32(thresh), torch.zeros_like(wts), wts)
            hw = pr.weighted_procrustes(src, ref, w2, thresh, eps)
            _negative(f"weighted_procrustes {name} t with weights == thresh dropped", (hw["t"] - h["t"]).abs(), bt)
        if neg == "det":
            Uq, _, Vh = torch.linalg.svd(h["H"])
            _negative(f"weighted_procrustes {name} R without det correction", _frob(Vh.transpose(1, 2) @ Uq.transpose(1, 2) - Rr), bR)
    return R, t, h, (rR, rt)


def test_weighted_procrustes_bench(ops):
    """N = 2048 at B = 32: pred-like sources, a planted pose with noise, weights like the fine stage's"""
    g = _gc(81)
    src = _ball(32, 2048, g)
    Rg = _rotations(32, g).float()
    ref = (src @ Rg.transpose(1, 2) + 0.1 * torch.randn(32, 1, 3, generator=g, device=DEV)
           + 0.02 * torch.randn(32, 2048, 3, generator=g, device=DEV)).contiguous()
    wts = torch.rand(32, 2048, generator=g, device=DEV) ** 2
    _wp_check(ops, src, ref, wts, 0.0, "B=32 N=2048")


def test_weighted_procrustes_geometry(ops):
    """near-isotropic (sigma1 ~ sigma2 ~ sigma3: clustered eigenvalues for the fixed 8 Jacobi sweeps), planar (sigma3 ~ 0),
    and a mirror image (det H < 0: the determinant correction, bound over sigma2 - sigma3)"""
    g = _gc(82)
    oct6 = torch.tensor([[1.0, 0, 0], [-1, 0, 0], [0, 1, 0], [0, -1, 0], [0, 0, 1], [0, 0, -1]], device=DEV)
    iso = (oct6.repeat(1, 50, 1) + 1e-3 * torch.randn(1, 300, 3, generator=g, device=DEV))
    planar = _ball(1, 300, g) * torch.tensor([1.0, 0.6, 0.0], device=DEV)
    aniso = _ball(1, 300, g) * torch.tensor([3.0, 2.0, 1.0], device=DEV)
    Rg = _rotations(3, g).float()
    src = torch.cat([iso, planar, aniso]).contiguous()
    ref = src @ Rg.transpose(1, 2) + 0.3
    ref[2] = src[2] * torch.tensor([-1.0, 1.0, 1.0], device=DEV)
    ref = (ref + 1e-3 * torch.randn(3, 300, 3, generator=g, device=DEV)).contiguous()
    wts = torch.rand(3, 300, generator=g, device=DEV) + 0.5
    _, _, h, _ = _wp_check(ops, src, ref, wts, 0.0, "geometry", neg="det")
    assert h["sdet"][2] < 0
    print("weighted_procrustes geometry singular values:", [[f"{x:.3g}" for x in s] for s in h["S"].tolist()])


def test_weighted_procrustes_weights(ops):
    """weights exactly 0, below weight_thresh, exactly at it (kept: the test is <), all 0 (R = I, t = 0); the points below
    and at the threshold are outliers, so dropping or keeping them moves the pose"""
    g = _gc(83)
    B, N, th = 3, 600, 0.25
    src = _ball(B, N, g)
    Rg = _rotations(B, g).float()
    ref = src @ Rg.transpose(1, 2) + 0.05 * torch.randn(B, N, 3, generator=g, device=DEV)
    wts = 0.3 + 0.7 * torch.rand(B, N, generator=g, device=DEV)
    wts[:, :100] = 0.0
    wts[:, 100:200] = 0.1
    wts[:, 200:260] = pr.f32(th)
    ref[:, 100:200] -= 0.7                                  # outliers below the threshold (dropped)
    ref[:, 200:260] += 0.5                                  # outliers at the threshold (kept)
    wts[2] = 0.0
    R, t, _, _ = _wp_check(ops, src, ref.contiguous(), wts.contiguous(), th, "thresholds", neg="le")
    assert torch.equal(R[2], torch.eye(3, device=DEV)) and (t[2] == 0).all()


# ================================================================================================== 9. pose_score
def _score_case(B, N, nm, g, bg=0.2):
    model = _ball(B, nm, g)
    Rg = _rotations(B, g).float()
    tg = 0.2 * torch.randn(B, 3, generator=g, device=DEV)
    m = model[:, torch.randint(0, nm, (N,), generator=g, device=DEV)]
    pts1 = ((m + 0.1 * torch.randn(B, N, 3, generator=g, device=DEV)) @ Rg.transpose(1, 2) + tg.unsqueeze(1)).contiguous()
    lab1 = torch.randint(1, N + 1, (B, N + 1), generator=g, device=DEV)
    lab1 = torch.where(torch.rand(B, N + 1, generator=g, device=DEV) < bg, 0, lab1)
    lab1[:, 0] = 0
    radius = 0.05 + torch.rand(B, generator=g, device=DEV)
    return pts1, lab1.int().contiguous(), Rg.contiguous(), tg.contiguous(), model, radius


def _pose_score_check(ops, pts1, lab1, R, t, model, radius, name, neg=False):
    B, N, _ = pts1.shape
    score, ts = ops.pose_score(pts1, lab1, R, t, model, radius, THR)
    d, hits, valid, ref, tsr = pr.pose_score(pts1, lab1, R, t, model, radius, THR)
    # d: the transformed point within transform_err; |x|^2 - 2 x.m + |m|^2 with |x|^2, x.m and |m|^2 chains of 3 and two
    # combining roundings: gamma_9 on (|x| + max |m|)^2; sqrtf.  A hit is decided when |d - dis_thres| exceeds that.
    xt = pr.transform(pts1, R.unsqueeze(1), t.unsqueeze(1)).squeeze(1)
    M = model.to(F64).norm(dim=2).amax(1, keepdim=True)
    dd = pr.transform_err(pts1, R.unsqueeze(1), t.unsqueeze(1)).squeeze(1) + pr.dist_err(d, pr.sqdist_err(xt.norm(dim=2), M, 9))
    mk = lab1[:, 1:] > 0
    dec = (d - pr.f32(THR)).abs() > dd
    h_lo = ((d < pr.f32(THR)) & mk & dec).sum(1)
    h_hi = h_lo + (mk & ~dec).sum(1)
    _undecided(f"pose_score {name} hits", (mk & ~dec).sum(), mk.sum())
    # the kernel's hit count from its score (score = h / (valid + 1e-8f) * valid / N, four roundings: h is recovered exactly)
    v = valid.to(F64)
    hk = torch.where(valid > 0, torch.round(score.to(F64) * N * (v + pr.EPS8) / v.clamp_min(1)), torch.zeros_like(v)).long()
    assert ((hk >= h_lo) & (hk <= h_hi)).all(), f"pose_score {name}: hit count {hk.tolist()} outside [{h_lo.tolist()}, {h_hi.tolist()}]"
    assert torch.equal(hk[h_lo == h_hi], hits[h_lo == h_hi])
    fk = hk.to(F64) / (v + pr.EPS8) * (v / N)
    r = _check(f"pose_score {name} score", (score.to(F64) - fk).abs(), 4.01 * U * fk)
    assert (score[valid == 0] == 0).all()
    # t_scaled = t (radius + 1e-6f): two roundings
    _check(f"pose_score {name} t_scaled", (ts.to(F64) - tsr).abs(), 2.01 * U * tsr.abs())
    if neg:
        all_rows = ((d < pr.f32(THR)) & dec).sum(1)        # hits += 1: background rows counted
        drop = torch.arange(N, device=DEV)
        drop = ((drop // 256) % 8 == 7)                      # CTA 0 sums 7 slots: the last CTA's slice lost
        lost = h_hi - ((d < pr.f32(THR)) & mk & dec & drop).sum(1)
        bad1 = ~((all_rows >= h_lo) & (all_rows <= h_hi))
        bad2 = lost < h_lo
        print(f"pose_score {name} (negative controls): background counted leaves the allowed range in {int(bad1.sum())} of "
              f"{B} proposals, a lost cluster slice in {int(bad2.sum())}")
        assert bad1.any() and bad2.any()
    return score, ts, r


@pytest.mark.parametrize("B,N,nm", [(32, 2048, 1024), (3, 1, 1024), (3, 255, 1023), (3, 2049, 1023), (3, 2048, 1)])
def test_pose_score_shapes(ops, B, N, nm):
    """N = 2048 at B = 32; N = 1, 255 and 2049 (uneven slices over the 8 CTAs of a cluster); odd nm; per-proposal radius and
    CAD model"""
    case = _score_case(B, N, nm, _gc(N + nm))
    _pose_score_check(ops, *case, f"B={B} N={N} nm={nm}", neg=(N == 2048 and nm == 1024))


def test_pose_score_all_background(ops):
    """lab1 all background for one proposal: score 0; and rows labelled background never count as hits"""
    pts1, lab1, R, t, model, radius = _score_case(2, 2048, 1024, _gc(91))
    lab1[0] = 0
    score, _, _ = _pose_score_check(ops, pts1, lab1.contiguous(), R, t, model, radius, "all background")
    assert score[0] == 0 and score[1] > 0
