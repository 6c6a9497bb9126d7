"""CPU: the float64 restatements that tests/test_gpu_pose_kernels.py holds the pose kernels to (tests/_pose_ref.py), pinned
to oracle/pem_oracle.py (soft_assignment, coarse_Rt(completion="deterministic"), fine_Rt, geo_embedding_indices), which is
pinned to the reference modules.  Discrete outputs (labels, indices, k-NN sets) must match exactly on inputs without near
ties; floats within fp32 noise (the oracle runs in fp32).  A wrong restatement would make every bound of the GPU file
meaningless."""
import math

import pytest
import torch

import _pose_ref as pr   # noqa: E402
from oracle import pem_oracle as po

F64 = torch.float64
FACTOR_A = 180.0 / (po.SIGMA_A * math.pi)


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _ball(B, n, g):
    x = torch.randn(B, n, 3, generator=g)
    return x / x.norm(dim=2, keepdim=True) * torch.rand(B, n, 1, generator=g) ** (1 / 3)


def test_geo_indices_match_oracle():
    """d_idx and the triplet angles == geo_embedding_indices (fp32 topk) within fp32 noise; the k-NN sets equal the oracle's
    topk sets, the background point at (100, 100, 100) included"""
    g = _g(1)
    pts = _ball(3, 60, g)
    pts[:, 0] = 100.0
    d_ref, a_ref = po.geo_embedding_indices(pts)
    d, a, dist, knn, _, _ = pr.geo_indices(pts, po.SIGMA_D, FACTOR_A)
    # the oracle's fp32 expanded form loses up to sqrt(gamma |x|^2) near d = 0 (|x| ~ 170 at the background point)
    nrm = pts.to(F64).norm(dim=2)
    e = pr.sqdist_err(nrm.unsqueeze(2), nrm.unsqueeze(1), 16)
    assert ((d - d_ref.to(F64)).abs() * po.SIGMA_D <= pr.dist_err(dist, e)).all()
    fg = torch.ones(60, dtype=torch.bool)
    fg[0] = False
    torch.testing.assert_close(a[:, fg][:, :, fg], a_ref.to(F64)[:, fg][:, :, fg], rtol=0, atol=2e-4)
    ref_knn = torch.sqrt(po.pairwise_sqdist(pts, pts)).topk(4, dim=2, largest=False)[1]
    assert torch.equal(knn.sort(-1)[0], ref_knn.sort(-1)[0])
    assert (knn[..., 0] == torch.arange(60)).all(), "self is the first entry without duplicates"


def test_knn_ties_go_to_the_first_index():
    """bitwise-duplicate points: zero distances tie exactly and the stable order keeps the smaller index first, so an anchor
    whose duplicate has a smaller index lists that duplicate before itself, and the angle against a coincident point is 0"""
    g = _g(2)
    pts = _ball(1, 20, g)
    pts[0, 7] = pts[0, 3]
    pts[0, 12] = pts[0, 3]
    _, a, _, knn, rn, _ = pr.geo_indices(pts, po.SIGMA_D, FACTOR_A)
    assert knn[0, 3, :3].tolist() == [3, 7, 12]
    assert knn[0, 7, :3].tolist() == [3, 7, 12]
    assert knn[0, 12, :3].tolist() == [3, 7, 12]
    assert (rn[0, 7, :2] == 0).all() and (a[0, 7, :, :2] == 0).all()     # both references of anchor 7 coincide with it
    assert (a[0, 3, 12] == 0).all() and (a[0, 3, 3] == 0).all() and (a[0, 5, 5] == 0).all()


def test_soft_assignment_matches_oracle():
    g = _g(3)
    A = torch.randn(2, 41, 41, generator=g) * 3
    A[1, :, 0] += 4.0                                    # mostly background rows in proposal 1
    inner, w1, w2, lab1, lab2 = po.soft_assignment(A)
    P, l1, l2 = pr.soft_assignment(A)
    assert torch.equal(l1[:, 1:], lab1) and torch.equal(l2[:, 1:], lab2)
    W, m1 = pr.coarse_weights(P, l1, l2)
    assert torch.equal(m1, w1.to(F64))
    torch.testing.assert_close(W, (inner.reshape(2, -1) ** 1.5).to(F64), rtol=1e-5, atol=1e-12)


def test_first_argmax_and_decided():
    x = torch.tensor([[1.0, 3.0, 3.0, 2.0], [5.0, 1.0, 4.999, 0.0]], dtype=F64)
    assert pr.first_argmax(x, 1).tolist() == [1, 0]
    i, dec, allowed = pr.argmax_decided(x, torch.full_like(x, 1e-4), 1)
    assert i.tolist() == [1, 0] and dec.tolist() == [False, True]
    assert allowed[0].tolist() == [False, True, True, False]
    i, dec, allowed = pr.argmax_decided(x, torch.full_like(x, 1e-3), 1)
    assert dec.tolist() == [False, False] and allowed[1].tolist() == [True, False, True, False]


def _coarse_case(seed, B=2, n=30, n1=400):
    g = _g(seed)
    pts1 = _ball(B, n, g)
    R = torch.linalg.qr(torch.randn(3, 3, generator=g))[0]
    if torch.det(R) < 0:
        R = -R
    pts2 = (pts1 - 0.1) @ R + 0.01 * torch.randn(B, n, 3, generator=g)
    A = torch.randn(B, n + 1, n + 1, generator=g)
    A[:, 1:, 1:] += 6 * torch.eye(n)
    model = _ball(B, 200, g)
    rand = torch.rand(B, 3 * n1, generator=g)
    return A, pts1, pts2, model, rand


def test_coarse_chain_matches_oracle():
    """cdf, searchsorted, triplet Procrustes (rank-1 completion and identity for rank 0 included) and the selection score
    == coarse_Rt(completion="deterministic")'s intermediates"""
    A, pts1, pts2, model, rand = _coarse_case(4)
    B, n = pts1.shape[:2]
    _, _, dbg = po.coarse_Rt(A, pts1, pts2, model, rand=rand, n1=400, n2=50, return_debug=True, completion="deterministic")
    P, l1, l2 = pr.soft_assignment(A)
    W, w1 = pr.coarse_weights(P, l1, l2)
    c = pr.cdf(W)
    torch.testing.assert_close(c, dbg["cdf"].to(F64), rtol=1e-5, atol=1e-6)
    idx = pr.searchsorted(c, rand)
    # the fp32 cdf of the oracle may differ within its rounding: every sample index agrees unless rand is that close
    e = pr.cdf_err(c) * 64
    near = ((c.unsqueeze(1) - rand.to(F64).unsqueeze(2)).abs() <= e.unsqueeze(1)).any(2)
    assert (near | (idx == dbg["idx"])).all() and (~near).float().mean() > 0.99
    idx = dbg["idx"]
    h = pr.triplet_procrustes(idx.int(), pts1, pts2)
    assert torch.equal(h["rank1"].reshape(-1), po._triplet_ranks(idx.div(n, rounding_mode="floor").clamp(max=n - 1),
                                                                 (idx % n).clamp(max=n - 1), B, 400)[0])
    assert h["rank1"].any() and not h["rank0"].any()
    torch.testing.assert_close(h["R"], dbg["Rs"].to(F64), rtol=0, atol=2e-4)
    torch.testing.assert_close(h["t"], dbg["ts"].to(F64), rtol=0, atol=2e-4)
    torch.testing.assert_close(h["resid"], dbg["resid"].to(F64), rtol=0, atol=2e-4)
    top = dbg["top"]
    bi = torch.arange(B).view(B, 1)
    sc, _ = pr.select_scores(dbg["Rs"][bi, top], dbg["ts"][bi, top], pts1, w1, model)
    torch.testing.assert_close(sc, dbg["sel_scores"].to(F64), rtol=1e-4, atol=1e-5)
    assert torch.equal(pr.first_argmax(sc, 1), dbg["best"])


def test_procrustes_special_cases():
    """rank 0 -> identity; H = 0 -> identity; a rank-1 triplet with antiparallel directions -> the half turn of rank1_rotation;
    a mirrored full-rank cloud -> a proper rotation"""
    H = torch.zeros(1, 3, 3, dtype=F64)
    R, _, _, _ = pr.procrustes_rotation(H)
    assert torch.equal(R[0], torch.eye(3, dtype=F64))
    u = torch.tensor([[3.0, 2.0, 1.0]], dtype=F64)
    u = u / u.norm()
    H = 2.0 * u.view(1, 3, 1) * (-u).view(1, 1, 3)
    R, _, _, c = pr.procrustes_rotation(H, rank1=torch.tensor([True]))
    assert abs(c.item() + 1) < 1e-12
    torch.testing.assert_close(R, po.rank1_rotation(H), rtol=0, atol=1e-12)
    torch.testing.assert_close(R[0] @ u[0], -u[0], rtol=0, atol=1e-12)
    g = _g(5)
    src = torch.randn(1, 50, 3, generator=g) * torch.tensor([3.0, 2.0, 1.0])
    ref = src * torch.tensor([-1.0, 1.0, 1.0])
    h = pr.weighted_procrustes(src, ref, torch.ones(1, 50))
    assert h["sdet"].item() < 0
    assert abs(torch.det(h["R"][0]).item() - 1) < 1e-12
    R_ref, _ = po.weighted_procrustes(src, ref, torch.ones(1, 50))
    torch.testing.assert_close(h["R"], R_ref.to(F64), rtol=0, atol=1e-5)


@pytest.mark.parametrize("thresh", [0.0, 0.3])
def test_fine_chain_matches_oracle(thresh):
    """fine_assign's labels, weights and pred, weighted Procrustes and the pose score == fine_Rt (weight_thresh 0) and
    pem_oracle.weighted_procrustes (a positive threshold)"""
    g = _g(6)
    B, N = 2, 120
    pts1 = _ball(B, N, g)
    pts2 = pts1 @ torch.linalg.qr(torch.randn(3, 3, generator=g))[0] + 0.05
    f1 = torch.nn.functional.normalize(torch.randn(B, N + 1, 16, generator=g), dim=2)
    f2 = torch.nn.functional.normalize(f1 + 0.3 * torch.randn(B, N + 1, 16, generator=g), dim=2)
    A = (f1 @ f2.transpose(1, 2)) / po.TEMP
    A[1, 1:20, 0] = 10.0                                 # background rows
    model = _ball(B, 300, g)
    R_ref, t_ref, s_ref, dbg = po.fine_Rt(A, pts1, pts2, model, return_debug=True)
    P, l1, l2 = pr.fine_assign(A, 1.0 / po.TEMP)
    assert torch.equal(l1[:, 1:], dbg["lab1"]) and torch.equal(l2[:, 1:], dbg["lab2"])
    w, pred, _ = pr.fine_weights(P, l1, l2, pts2)
    torch.testing.assert_close(w, dbg["wts"].to(F64), rtol=1e-5, atol=1e-9)
    torch.testing.assert_close(pred, dbg["pred"].to(F64), rtol=1e-4, atol=1e-5)
    wts = w.float()
    if thresh > 0:
        wts = torch.rand(B, N, generator=g)
        R_ref, t_ref = po.weighted_procrustes(pred.float(), pts1, wts, weight_thresh=thresh)
    h = pr.weighted_procrustes(pred.float(), pts1, wts, weight_thresh=thresh)
    torch.testing.assert_close(h["R"], R_ref.to(F64), rtol=0, atol=1e-4)
    torch.testing.assert_close(h["t"], t_ref.to(F64), rtol=0, atol=1e-4)
    if thresh == 0:
        radius = torch.tensor([0.5, 2.0])
        d, hits, valid, score, ts = pr.pose_score(pts1, l1, R_ref, t_ref, model, radius)
        torch.testing.assert_close(score, s_ref.to(F64), rtol=1e-6, atol=1e-7)
        assert torch.equal(valid, (dbg["lab1"] > 0).sum(1))
