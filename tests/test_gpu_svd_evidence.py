"""Evidence for the one documented deviation of the CUDA path (DESIGN.md section 3): the reference's rotation for a
rank-deficient pose hypothesis is not a function of its inputs.

compute_coarse_Rt (PEM/utils/model_utils.py:218-234) draws its 3-point hypotheses WITH replacement; a triplet that repeats a
point has collinear centred points, so its 3x3 cross-covariance has one singular value above fp32 rounding noise.
weighted_procrustes (model_utils.py:352-358) then builds R = V diag(1,1,det) U^T from torch.svd's noise-level second and
third singular vectors.  This test runs that exact torch code on the host (LAPACK) and on the GPU (cuSOLVER / batched
Jacobi) for the same triplets and prints the disagreement: ~1e-6 for triplets of distinct points, O(1) for repeated ones."""
import json

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import pem_oracle as po      # noqa: E402


def _reference_procrustes(src, ref):
    """weighted_procrustes(src, ref, None, weight_thresh=0.5) as the reference writes it, on whatever device src lives"""
    bsz = src.shape[0]
    w = torch.ones_like(src[:, :, 0])
    w = (w / (w.sum(dim=1, keepdim=True) + 1e-5)).unsqueeze(2)
    c_s = (src * w).sum(dim=1, keepdim=True)
    c_r = (ref * w).sum(dim=1, keepdim=True)
    H = (src - c_s).permute(0, 2, 1) @ (w * (ref - c_r))
    U, _, V = torch.svd(H)
    Ut = U.transpose(1, 2)
    eye = torch.eye(3, device=src.device).unsqueeze(0).repeat(bsz, 1, 1)
    eye[:, -1, -1] = torch.sign(torch.det(V @ Ut))
    return V @ eye @ Ut


def test_reference_svd_disagrees_with_itself_on_rank_deficient_triplets():
    g = torch.Generator().manual_seed(5)
    n, n1 = 196, 6000
    pts2 = torch.randn(1, n, 3, generator=g) * 0.4
    R = po.random_rotation(1, g)
    pts1 = pts2 @ R.transpose(1, 2) + 0.1 + 0.002 * torch.randn(1, n, 3, generator=g)
    i1 = torch.randint(0, n, (1, n1 * 3), generator=g)
    i2 = i1.clone()                                              # correct correspondences
    rep = torch.arange(n1) % 2 == 1                              # every second triplet repeats its first correspondence
    i1v, i2v = i1.view(n1, 3), i2.view(n1, 3)
    i1v[rep, 1], i2v[rep, 1] = i1v[rep, 0], i2v[rep, 0]
    r1, r0 = po._triplet_ranks(i1, i2, 1, n1)
    deg = r1 | r0
    p1 = pts1[0][i1.view(-1)].reshape(n1, 3, 3)
    p2 = pts2[0][i2.view(-1)].reshape(n1, 3, 3)
    R_cpu = _reference_procrustes(p2, p1)
    R_gpu = _reference_procrustes(p2.cuda(), p1.cuda()).cpu()
    d = (R_cpu - R_gpu).abs().amax(dim=(1, 2))
    # the deterministic completion: CPU restatement (float64 LAPACK) vs the CUDA kernel (fp64 Jacobi)
    from sam6d_b200 import ops
    Rs, _ = po.weighted_procrustes(p2, p1, None, weight_thresh=0.5, rank1=r1, rank0=r0)
    Rt, _ = ops.coarse_hypotheses((i1 * n + i2).int().cuda(), pts1.cuda(), pts2.cuda())
    d_ours = (Rt.cpu()[0, :, :9].reshape(n1, 3, 3) - Rs).abs().amax(dim=(1, 2))
    rec = dict(
        what="max |R_cpu - R_cuda| of the reference's own weighted_procrustes (torch.svd) on identical 3-point hypotheses",
        torch=torch.__version__, device=torch.cuda.get_device_name(0), hypotheses=n1,
        distinct_triplets=dict(count=int((~deg).sum()), median=d[~deg].median().item(), q99=d[~deg].quantile(0.99).item(),
                               max=d[~deg].max().item()),
        repeated_point_triplets=dict(count=int(deg.sum()), median=d[deg].median().item(), q10=d[deg].quantile(0.1).item(),
                                     max=d[deg].max().item(), frac_above_0p1=(d[deg] > 0.1).float().mean().item()),
        deterministic_completion_cpu_vs_cuda=dict(max_rank_deficient=d_ours[deg].max().item(),
                                                  q999_distinct=d_ours[~deg].quantile(0.999).item()),
    )
    print(json.dumps(rec, indent=1))
    assert d[~deg].quantile(0.99).item() < 1e-3            # well-posed hypotheses: the two devices agree
    assert (d[deg] > 0.1).float().mean().item() > 0.5      # rank-deficient ones: they do not
    assert d_ours[deg].max().item() < 1e-4                 # the completion is reproducible across implementations
