"""GPU parity: every C-ABI kernel against the CPU oracle / plain torch fp32 on the same seeded inputs.

Index-valued outputs (FPS, ball query, gathers, top-k, labels, template indices) must be bit-exact; floating-point outputs
carry the tolerance written next to each check."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import pem_oracle as po      # noqa: E402
from oracle import pn2                   # noqa: E402
from oracle import ism_oracle as io      # noqa: E402
from _helpers import exact_indices as _exact_indices, exact_geo_embedding   # noqa: E402


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from sam6d_b200 import ops as _ops
    return _ops


def G(seed):
    return torch.Generator().manual_seed(seed)


# ------------------------------------------------------------------------------------------------- point cloud ops
@pytest.mark.parametrize("b,n,m", [(3, 2048, 196), (2, 1000, 64), (2, 300, 40), (1, 4096, 128), (1, 5000, 50), (1, 37, 9)])
def test_fps_exact(ops, b, n, m):
    x = torch.randn(b, n, 3, generator=G(n))
    ref = pn2.furthest_point_sampling(x, m)
    got = ops.furthest_point_sampling(x.cuda(), m).cpu()
    assert got.dtype == torch.int32
    assert torch.equal(got, ref)


def test_fps_duplicates_and_ties(ops):
    # masks with < 2048 px are sampled with replacement upstream -> many exact duplicates (SURVEY Q2)
    base = torch.randn(2, 300, 3, generator=G(5))
    pick = torch.randint(0, 300, (2, 2048), generator=G(6))
    x = torch.gather(base, 1, pick.unsqueeze(2).expand(2, 2048, 3)).contiguous()
    assert torch.equal(ops.furthest_point_sampling(x.cuda(), 196).cpu(), pn2.furthest_point_sampling(x, 196))
    # symmetric lattice: plenty of exact distance ties
    g = torch.stack(torch.meshgrid(torch.arange(8.), torch.arange(8.), torch.arange(8.), indexing="ij"), -1).reshape(1, 512, 3)
    assert torch.equal(ops.furthest_point_sampling(g.cuda(), 100).cpu(), pn2.furthest_point_sampling(g, 100))
    ones = torch.ones(1, 100, 3)
    assert ops.furthest_point_sampling(ones.cuda(), 5).cpu().tolist() == [[0, 0, 0, 0, 0]]


def test_gather_and_group_exact(ops):
    pts = torch.randn(2, 7, 300, generator=G(1))
    idx = torch.randint(0, 300, (2, 50), generator=G(2), dtype=torch.int32)
    assert torch.equal(ops.gather_points(pts.cuda(), idx.cuda()).cpu(), pn2.gather_points(pts, idx))
    gi = torch.randint(0, 300, (2, 50, 16), generator=G(3), dtype=torch.int32)
    assert torch.equal(ops.group_points(pts.cuda(), gi.cuda()).cpu(), pn2.group_points(pts, gi))
    rows = torch.randn(2, 300, 256, generator=G(4))
    got = ops.gather_rows(rows.cuda(), idx.cuda()).cpu()
    assert torch.equal(got, torch.gather(rows, 1, idx.long().unsqueeze(2).expand(2, 50, 256)))
    rows3 = torch.randn(2, 300, 3, generator=G(4))
    got = ops.gather_rows(rows3.cuda(), idx.cuda()).cpu()
    assert torch.equal(got, torch.gather(rows3, 1, idx.long().unsqueeze(2).expand(2, 50, 3)))


@pytest.mark.parametrize("n,r,ns", [(2048, 0.1, 32), (2048, 0.2, 64), (1500, 0.15, 32), (100, 0.5, 64)])
def test_ball_query_exact(ops, n, r, ns):
    d = torch.randn(2, n, 3, generator=G(n + ns))
    x = (d / d.norm(dim=2, keepdim=True) * (0.6 + 0.4 * torch.rand(2, n, 1, generator=G(1)))).contiguous()
    ref = pn2.ball_query(x, x, r, ns)
    got, cnt = ops.ball_query(x.cuda(), x.cuda(), r, ns, return_count=True)
    assert torch.equal(got.cpu(), ref)
    # cnt = number of distinct leading hits
    d2 = ((x.unsqueeze(2) - x.unsqueeze(1)) ** 2).sum(-1)
    approx = (d2 < r * r).sum(-1).clamp(max=ns)
    assert (cnt.cpu() - approx).abs().max() <= 1
    # empty balls -> zeros
    far = torch.full((2, 5, 3), 50.0)
    assert ops.ball_query(far.cuda(), x.cuda(), r, ns).abs().sum().item() == 0


def test_ball_query_pair_matches_two_queries(ops):
    xyz = (torch.rand(3, 2048, 3, generator=G(5)) - 0.5).cuda()
    ia, ca, ib, cb = ops.ball_query_pair(xyz, xyz, 0.1, 32, 0.2, 64)
    ra, rca = ops.ball_query(xyz, xyz, 0.1, 32, return_count=True)
    rb, rcb = ops.ball_query(xyz, xyz, 0.2, 64, return_count=True)
    assert torch.equal(ia, ra) and torch.equal(ca, rca) and torch.equal(ib, rb) and torch.equal(cb, rcb)


def test_native_layer_argument_errors(ops):
    x = torch.randn(1, 64, 3)
    with pytest.raises(RuntimeError):
        ops.furthest_point_sampling(x, 8)                         # CPU tensor: "CPU not supported" in the reference
    with pytest.raises(RuntimeError):
        ops.furthest_point_sampling(x.cuda().double(), 8)         # dtype
    with pytest.raises(RuntimeError):
        ops.gather_points(torch.randn(1, 3, 64).cuda().transpose(1, 2), torch.zeros(1, 4, dtype=torch.int32).cuda())


# ------------------------------------------------------------------------------------------------- dense algebra / rows
@pytest.mark.parametrize("M,N,K", [(197 * 3, 1792, 256), (1000, 512, 256), (77, 33, 19), (4096, 256, 512), (130, 64, 6)])
def test_gemm(ops, M, N, K):
    A = torch.randn(M, K, generator=G(1))
    W = torch.randn(N, K, generator=G(2)) / math.sqrt(K)
    bias = torch.randn(N, generator=G(3))
    R = torch.randn(M, N, generator=G(4))
    ref = torch.relu(A.double() @ W.double().t() * 0.5 + bias.double()) + R.double()
    got = ops.gemm(A.cuda(), W.cuda(), bias.cuda(), residual=R.cuda(), relu=True, alpha=0.5).cpu()
    torch.testing.assert_close(got.double(), ref, atol=2e-5, rtol=1e-5)     # fp32 accumulate over K <= 512


def test_gemm_batched_strided_views(ops):
    B, N, M, C = 3, 65, 70, 256
    f1 = torch.randn(B, N, C, generator=G(1))
    f2 = torch.randn(B, M, C, generator=G(2))
    out = torch.empty(B, N, M).cuda()
    a, w = f1.cuda(), f2.cuda()
    ops.gemm(a, w, out=out, alpha=10.0)
    torch.testing.assert_close(out.cpu(), 10.0 * f1 @ f2.transpose(1, 2), atol=2e-4, rtol=1e-5)


def test_row_ops_views(ops):
    x = torch.randn(500, 256, generator=G(1)) * 3 + 0.5
    g, b = torch.randn(256, generator=G(2)), torch.randn(256, generator=G(3))
    torch.testing.assert_close(ops.layernorm(x.cuda(), g.cuda(), b.cuda()).cpu(),
                               torch.nn.functional.layer_norm(x, (256,), g, b, 1e-5), atol=2e-5, rtol=1e-5)
    torch.testing.assert_close(ops.l2norm_rows(x.cuda()).cpu(), torch.nn.functional.normalize(x, dim=-1), atol=1e-6, rtol=1e-5)
    x1024 = torch.randn(9, 1024, generator=G(4))
    torch.testing.assert_close(ops.l2norm_rows(x1024.cuda()).cpu(), torch.nn.functional.normalize(x1024, dim=-1), atol=1e-6, rtol=1e-5)
    # focus map (transformer.py:541-550)
    scale = torch.nn.functional.softplus(0.2 * torch.randn(256, generator=G(5)))
    q = torch.relu(x) + 1e-6
    q = q / scale
    qn = q.norm(dim=-1, keepdim=True)
    q = q ** 3
    ref = q / q.norm(dim=-1, keepdim=True) * qn
    xc = x.cuda()
    out = torch.empty_like(xc)
    ops.focus_rows(xc, scale.cuda(), out=out)
    torch.testing.assert_close(out.cpu(), ref, atol=1e-5, rtol=2e-5)
    # rigid warp, radius
    p = torch.randn(2, 100, 3, generator=G(6))
    R = po.random_rotation(2, G(7))
    t = torch.randn(2, 3, generator=G(8))
    torch.testing.assert_close(ops.rigid_warp(p.cuda(), R.cuda(), t.cuda()).cpu(), (p - t.unsqueeze(1)) @ R, atol=1e-5, rtol=1e-5)
    rad = torch.norm(p, dim=2).max(1)[0]
    torch.testing.assert_close(ops.cloud_radius(p.cuda()).cpu(), rad, atol=0, rtol=1e-6)
    torch.testing.assert_close(ops.scale_by_radius(p.cuda(), rad.cuda()).cpu(), p / (rad.reshape(-1, 1, 1) + 1e-6), atol=0, rtol=1e-6)


# ------------------------------------------------------------------------------------------------- geometric embedding
def _sparse_cloud(B, S, seed, scale=1.0, offset=0.0):
    d = torch.randn(B, S - 1, 3, generator=G(seed))
    pts = d / d.norm(dim=2, keepdim=True) * (0.5 + 0.5 * torch.rand(B, S - 1, 1, generator=G(seed + 1))) * scale + offset
    return torch.cat([torch.ones(B, 1, 3) * 100, pts], dim=1).contiguous()


def test_geo_indices(ops):
    pts = _sparse_cloud(2, 197, 3)
    d_ref, a_ref = _exact_indices(pts)
    T = ops.geo_indices(pts.cuda(), po.SIGMA_D, 180.0 / (po.SIGMA_A * math.pi)).cpu()
    torch.testing.assert_close(T[..., 3], d_ref, atol=2e-3, rtol=1e-5)         # the reference's own fp32 noise level
    d_cpu, _ = po.geo_embedding_indices(pts)
    assert (T[..., 3] - d_ref).abs().max() <= (d_cpu - d_ref).abs().max() + 1e-4   # no worse than the fp32 reference
    # the neighbour *set* matters (max over k): compare sorted angle triplets, allow a vanishing fraction of knn ties
    got, ref = T[..., :3].sort(dim=-1)[0], a_ref.sort(dim=-1)[0]
    bad = ((got - ref).abs() > 2e-3).any(dim=-1).float().mean().item()
    assert bad < 2e-3, f"{bad:.2e} of pairs differ in their angle triplet"


def test_geo_embed(ops):
    sd = po.make_state_dict(seed=2)
    pts = _sparse_cloud(2, 64, 9)
    ref = exact_geo_embedding(sd, pts)
    T = ops.geo_indices(pts.cuda(), po.SIGMA_D, 180.0 / (po.SIGMA_A * math.pi))
    E = ops.geo_embed_f32(T, sd["geo_embedding.embedding.div_term"].cuda(), sd["geo_embedding.proj_a.weight"].t().contiguous().cuda(),
                          sd["geo_embedding.proj_d.weight"].t().contiguous().cuda(),
                          (sd["geo_embedding.proj_a.bias"] + sd["geo_embedding.proj_d.bias"]).cuda()).cpu()
    err = (E - ref).abs()
    assert (err > 5e-3).float().mean().item() < 2e-3
    assert err.median().item() < 1e-4


# ------------------------------------------------------------------------------------------------- attention
def test_rpe_scores_and_mha_views(ops):
    B, S, C, H = 2, 197, 256, 4
    E = torch.randn(B, S, S, C, generator=G(1))
    U = torch.randn(B, S, H, C, generator=G(2))
    ref = torch.einsum("bnhc,bnmc->bhnm", U, E)
    got = ops.rpe_scores(E.cuda(), U.cuda()).cpu()
    torch.testing.assert_close(got, ref, atol=2e-4, rtol=1e-5)
    got16 = ops.rpe_scores(E.cuda().bfloat16(), U.cuda()).cpu()
    ref16 = torch.einsum("bnhc,bnmc->bhnm", U, E.bfloat16().float())
    torch.testing.assert_close(got16, ref16, atol=2e-4, rtol=1e-5)
    q = torch.randn(B, S, C, generator=G(3))
    k = torch.randn(B, 150, C, generator=G(4))
    v = torch.randn(B, 150, C, generator=G(5))
    bias = torch.randn(B, H, S, 150, generator=G(6))
    qh, kh, vh = (t.view(B, -1, H, 64).permute(0, 2, 1, 3) for t in (q, k, v))
    att = torch.softmax((qh @ kh.transpose(-1, -2) + bias) / 8.0, dim=-1)
    ref = (att @ vh).permute(0, 2, 1, 3).reshape(B, S, C)
    qc, kc, vc = q.cuda(), k.cuda(), v.cuda()
    out = torch.empty(B, S, C).cuda()
    ops.mha(qc, kc, vc, bias.cuda(), 0.125, out)
    torch.testing.assert_close(out.cpu(), ref, atol=2e-5, rtol=1e-4)


@pytest.mark.parametrize("B,S", [(2, 197), (3, 65), (5, 129), (1, 200), (64, 197)])
def test_rpe_scores_tensor_core(ops, B, S):
    """TMA + wgmma stream over E (csrc/rpe_tc.cu) against the einsum on the same bf16 operands; B = 64, S = 197 is the
    launch shape of the bench step (more query rows than SMs: every CTA walks a range and the ring stages wrap)"""
    E = (torch.randn(B, S, S, 256, generator=G(1)) * 0.7).bfloat16()
    U = torch.randn(B * S, 1024, generator=G(2)).bfloat16()
    got = ops.rpe_scores_tc(E.cuda(), U.cuda())
    if B <= 8:
        ref = torch.einsum("bnhc,bnmc->bhnm", U.float().view(B, S, 4, 256), E.float())
        torch.testing.assert_close(got.cpu(), ref, atol=2e-3, rtol=1e-4)
    else:   # compare on the device in fp32 (the reference einsum of the full shape is slow on the host)
        ref = torch.einsum("bnhc,bnmc->bhnm", U.cuda().float().view(B, S, 4, 256), E.cuda().float())
        torch.testing.assert_close(got, ref, atol=2e-3, rtol=1e-4)
    # and the CUDA-core kernel agrees on the same operands
    old = ops.rpe_scores(E.cuda(), U.cuda().float().view(B, S, 4, 256).contiguous())
    torch.testing.assert_close(got, old, atol=2e-3, rtol=1e-4)


@pytest.mark.parametrize("B,S", [(2, 197), (3, 65), (2, 130), (1, 200)])
def test_padded_bias_attention_equals_dense_bias(ops, B, S):
    """score planes with 16-key padded rows (sam6d_rpe_scores_tc_ld) + the cp.async-streamed bias of sam6d_attn_tc_bias_ld:
    same scores bit for bit, same attention output bit for bit as the dense-bias kernel (identical arithmetic, other data path)"""
    H, D = 4, 64
    E = (torch.randn(B, S, S, 256, generator=G(1)) * 0.7).bfloat16().cuda()
    U = torch.randn(B * S, 1024, generator=G(2)).bfloat16().cuda()
    sp = ops.rpe_scores_tc(E, U)
    spp = ops.rpe_scores_tc_padded(E, U)
    assert spp.shape[3] % 16 == 0 and spp.shape[3] >= S
    assert torch.equal(spp[..., :S], sp)
    qk = torch.randn(B * S, 2 * H * D, generator=G(3)).bfloat16().cuda()
    v = torch.randn(B * S, H * D, generator=G(4)).bfloat16().cuda()
    # V^T per (batch, head): (B*H*D, ceil16(S))
    N1 = (S + 15) // 16 * 16
    vt = torch.zeros(B * H * D, N1, dtype=torch.bfloat16, device="cuda")
    vt[:, :S] = v.view(B, S, H * D).permute(0, 2, 1).reshape(B * H * D, S)
    want = ops.attn_tc(qk, 0, qk, H * D, vt, B, H, S, S, D, 0.125, bias=sp, out_dtype=torch.bfloat16)
    spp[..., S:] = float("nan")                               # the padding must never be read into a result
    got = ops.attn_tc_padded_bias(qk, 0, qk, H * D, vt, B, H, S, S, D, 0.125, spp)
    assert torch.equal(got, want)


@pytest.mark.parametrize("M", [100, 128, 1000, 12608, 40000])
def test_transformer_tail_fused(ops, M):
    """csrc/tail_tc.cu against the same math in fp64 on the bf16-rounded operands (y and h rounded to bf16 where the kernel
    rounds them): 12608 rows = the sparse stream of the bench step (one tile per SM), 40000 = several tiles per CTA"""
    g = G(M)
    bf = torch.bfloat16
    hid = torch.randn(M, 256, generator=g).to(bf)
    x = torch.randn(M, 256, generator=g).to(bf)
    wo = (torch.randn(256, 256, generator=g) / 16).to(bf)
    we = (torch.randn(512, 256, generator=g) / 16).to(bf)
    ws = (torch.randn(256, 512, generator=g) / 22).to(bf)
    bo, be, bs = (torch.randn(n, generator=g) * 0.1 for n in (256, 512, 256))
    g1, g2 = (1 + 0.1 * torch.randn(256, generator=g) for _ in range(2))
    b1, b2 = (0.1 * torch.randn(256, generator=g) for _ in range(2))
    dev = lambda t: t.cuda()      # noqa: E731
    got = ops.transformer_tail_bf16(dev(hid), dev(x), dev(wo), dev(bo), dev(g1), dev(b1), dev(we), dev(be), dev(ws), dev(bs), dev(g2),
                                    dev(b2))
    d = lambda t: t.cuda().double()   # noqa: E731
    ln = torch.nn.functional.layer_norm
    y = ln(d(hid) @ d(wo).t() + d(bo) + d(x), (256,), d(g1), d(b1), 1e-5).to(bf).double()
    h = torch.relu(y @ d(we).t() + d(be)).to(bf).double()
    ref = ln(y + h @ d(ws).t() + d(bs), (256,), d(g2), d(b2), 1e-5)
    err = (got.double() - ref).abs()
    # one bf16 rounding of an O(1) output (2^-8 relative), plus the occasional flipped rounding of y / h
    assert err.max().item() < 6e-2 and err.mean().item() < 4e-3, (err.max().item(), err.mean().item())


def test_linear_attention_views(ops):
    sd = po.make_state_dict(seed=4)
    p = "fine_point_matching.transformers.0.dense_layer.attention.attention"
    B, N, J, C = 2, 300, 50, 256
    xq = torch.randn(B, N, C, generator=G(1))
    xkv = torch.randn(B, J, C, generator=G(2))
    ref = po.linear_attention(sd, p, xq, xkv)
    q = torch.nn.functional.linear(xq, sd[p + ".proj_q.weight"], sd[p + ".proj_q.bias"]).cuda().contiguous()
    k = torch.nn.functional.linear(xkv, sd[p + ".proj_k.weight"], sd[p + ".proj_k.bias"]).cuda().contiguous()
    v = torch.nn.functional.linear(xkv, sd[p + ".proj_v.weight"], sd[p + ".proj_v.bias"]).cuda().contiguous()
    sp = torch.nn.functional.softplus(sd[p + ".scale"]).reshape(-1).cuda()
    ops.focus_rows(q.view(B * N, C), sp, out=q.view(B * N, C))
    ops.focus_rows(k.view(B * J, C), sp, out=k.view(B * J, C))
    KV = torch.empty(B, 4, 64, 64).cuda()
    KS = torch.empty(B, 4, 64).cuda()
    ops.linattn_kv(k, v, KV, KS)
    x = torch.empty(B, N, C).cuda()
    ops.linattn_apply(q, KV, KS, x)
    torch.testing.assert_close(x.cpu(), ref, atol=1e-4, rtol=1e-3)


@pytest.mark.parametrize("B,N,J", [(2, 300, 50), (3, 2048, 196), (1, 129, 7)])
def test_linear_attention_tensor_core_views(ops, B, N, J):
    """bf16 dense tokens: feature map + per-head (q' KV)/(q' . ksum) in one wgmma kernel, against fp64 math on the same
    bf16-rounded query projection.  The token rows sit behind a bg row (the (B,N+1,C) layout of the fine stage)."""
    C = 256
    sp = (torch.rand(C, generator=G(5)) + 0.5)
    q = torch.randn(B, N + 1, C, generator=G(1)).bfloat16()
    k = torch.randn(B, J, C, generator=G(2))
    v = torch.randn(B, J, C, generator=G(3))

    def focus(x):
        x = (torch.relu(x) + 1e-6) / sp.double()
        n = x.norm(dim=-1, keepdim=True)
        x = x ** 3
        return x / x.norm(dim=-1, keepdim=True) * n

    qf, kf = focus(q[:, 1:].double()), focus(k.double())
    qh = qf.view(B, N, 4, 64).permute(0, 2, 1, 3)
    kh = kf.view(B, J, 4, 64).permute(0, 2, 1, 3)
    vh = v.double().view(B, J, 4, 64).permute(0, 2, 1, 3)
    z = 1.0 / (qh @ kh.sum(dim=2).unsqueeze(-1) + 1e-6)
    ref = ((qh @ (kh.transpose(-1, -2) @ vh)) * z).permute(0, 2, 1, 3).reshape(B, N, C)

    kd, vd, spd = k.cuda().contiguous(), v.cuda().contiguous(), sp.cuda()
    ops.focus_rows(kd.view(B * J, C), spd, out=kd.view(B * J, C))
    blob, KS = ops.linattn_kv_pack(kd, vd)
    torch.testing.assert_close(KS.cpu().double(), kh.sum(dim=2), atol=1e-4, rtol=1e-4)
    qd = q.cuda()
    x = torch.full((B, N + 1, C), 7.0, dtype=torch.bfloat16, device="cuda")
    ops.linattn_tc(qd[:, 1:, :], blob, KS, spd, x[:, 1:, :])
    x = x.cpu()
    assert (x[:, 0] == 7.0).all()                                     # rows outside the view are untouched
    torch.testing.assert_close(x[:, 1:].double(), ref, atol=2e-2 * ref.abs().max().item(), rtol=3e-2)


def test_bf16_row_ops(ops):
    x = torch.randn(5, 77, 256, generator=G(1)).bfloat16()
    g, b = torch.randn(256, generator=G(2)), torch.randn(256, generator=G(3))
    ref = torch.nn.functional.layer_norm(x.float(), (256,), g, b)
    got = ops.layernorm_bf16io(x.cuda(), g.cuda(), b.cuda()).cpu()
    assert got.dtype == torch.bfloat16
    torch.testing.assert_close(got.float(), ref, atol=3e-2, rtol=1e-2)
    idx = torch.randint(0, 77, (5, 40), generator=G(4), dtype=torch.int32)
    idx[0, 3] = -1
    out = ops.gather_rows_bf16_f32(x.cuda(), idx.cuda()).cpu()
    ref = torch.gather(x.float(), 1, idx.clamp(min=0).long().unsqueeze(-1).expand(-1, -1, 256))
    ref[0, 3] = 0
    assert torch.equal(out, ref)


# ------------------------------------------------------------------------------------------------- coarse pose pieces
def _score_matrix(B, S, seed, peak=6.0):
    """cosine/temp-like matrix in [-10,10] with a planted permutation so that labels are decisive"""
    g = G(seed)
    A = torch.rand(B, S, S, generator=g) * 4 - 2
    for b in range(B):
        perm = torch.randperm(S - 1, generator=g) + 1
        keep = torch.rand(S - 1, generator=g) < 0.8
        rows = torch.arange(1, S)[keep]
        A[b, rows, perm[keep]] += peak
        A[b, torch.arange(1, S)[~keep], 0] += peak
    return A.clamp(-10, 10).contiguous()


def test_coarse_assign_sample(ops):
    A = _score_matrix(3, 197, 1)
    inner, w1, _, _, _ = po.soft_assignment(A)
    ref = inner.reshape(3, -1) ** 1.5
    W, w1g = ops.coarse_assign(A.cuda())
    assert torch.equal(w1g.cpu(), w1)
    torch.testing.assert_close(W.cpu(), ref, atol=1e-7, rtol=2e-5)
    # cdf + searchsorted on identical weights must give identical indices (double accumulation like the CPU cumsum)
    rand = torch.rand(3, 18000, generator=G(2))
    cdf = torch.cumsum(ref, dim=1)
    cdf = cdf / (cdf[:, -1].unsqueeze(1) + 1e-8)
    idx_ref = torch.searchsorted(cdf, rand)
    idx = ops.coarse_sample(ref.cuda().contiguous(), rand.cuda()).cpu()
    mism = (idx.long() != idx_ref).float().mean().item()
    assert mism < 1e-3, f"searchsorted mismatch fraction {mism}"


def test_hypotheses_topk_select(ops):
    B, n, n1, n2, nm = 2, 196, 6000, 300, 1024
    g = G(3)
    pts2 = torch.randn(B, n, 3, generator=g) * 0.4
    R = po.random_rotation(B, g)
    t = torch.randn(B, 3, generator=g) * 0.2
    pts1 = pts2 @ R.transpose(1, 2) + t.unsqueeze(1) + 0.002 * torch.randn(B, n, 3, generator=g)
    model = torch.cat([pts2, torch.randn(B, nm - n, 3, generator=g) * 0.4], dim=1).contiguous()
    i1 = torch.randint(0, n, (B, n1 * 3), generator=g)
    # 70% correct correspondences, 30% random
    i2 = torch.where(torch.rand(B, n1 * 3, generator=g) < 0.7, i1, torch.randint(0, n, (B, n1 * 3), generator=g))
    idx = (i1 * n + i2).int()
    p1 = torch.gather(pts1, 1, i1.unsqueeze(2).repeat(1, 1, 3)).reshape(B * n1, 3, 3)
    p2 = torch.gather(pts2, 1, i2.unsqueeze(2).repeat(1, 1, 3)).reshape(B * n1, 3, 3)
    # rank-deficient triplets (a repeated point on either side) follow the deterministic completion -- the one documented
    # deviation (oracle: rank1_rotation); with it EVERY hypothesis is comparable
    r1, r0 = po._triplet_ranks(i1, i2, B, n1)
    assert 0.02 < r1.float().mean() < 0.2
    Rs, ts = po.weighted_procrustes(p2, p1, None, weight_thresh=0.5, rank1=r1, rank0=r0)
    resid_ref = torch.norm((p1 - ts.unsqueeze(1)) @ Rs - p2, dim=2).mean(1).reshape(B, n1)
    Rt, resid = ops.coarse_hypotheses(idx.cuda(), pts1.cuda(), pts2.cuda())
    Rt, resid = Rt.cpu(), resid.cpu()
    dR = (Rt[..., :9].reshape(B, n1, 3, 3) - Rs.reshape(B, n1, 3, 3)).abs().amax(dim=(2, 3))
    dt = (Rt[..., 9:] - ts.reshape(B, n1, 3)).abs().amax(dim=2)
    deg = (r1 | r0).reshape(B, n1)
    print(f"hypotheses: {int(deg.sum())} rank-deficient of {deg.numel()}; max dR on them {dR[deg].max().item():.2e}, "
          f"on the others median {dR[~deg].median().item():.2e} / q99.9 {dR[~deg].quantile(0.999).item():.2e}")
    assert dR[deg].max().item() < 1e-4 and dt[deg].max().item() < 1e-4
    # full-rank triplets: the reference's fp32 svd against the fp64 Jacobi (nearly collinear triplets are ill-conditioned)
    assert dR[~deg].quantile(0.999).item() < 2e-3 and dR[~deg].median().item() < 1e-5
    assert dt[~deg].quantile(0.999).item() < 2e-3
    torch.testing.assert_close(resid, resid_ref, atol=2e-5, rtol=1e-3)
    # top-k: same set as torch.topk on the same values, ascending (value, index) order
    top = ops.topk_smallest(resid.cuda(), n2).cpu().long()
    vals = torch.gather(resid, 1, top)
    assert (vals[:, 1:] >= vals[:, :-1]).all()
    ref_vals = torch.topk(resid, n2, dim=1, largest=False)[0]
    assert torch.equal(vals, ref_vals)
    # selection: score every retained hypothesis like the reference and take the first maximum
    w1 = (torch.rand(B, n, generator=g) < 0.8).float()
    Rsel = torch.gather(Rt[..., :9], 1, top.unsqueeze(2).expand(B, n2, 9)).reshape(B, n2, 3, 3)
    tsel = torch.gather(Rt[..., 9:], 1, top.unsqueeze(2).expand(B, n2, 3)).reshape(B, n2, 1, 3)
    tp = ((pts1.unsqueeze(1) - tsel) @ Rsel).reshape(B * n2, -1, 3)
    mp = model.unsqueeze(1).repeat(1, n2, 1, 1).reshape(B * n2, -1, 3)
    dis = torch.sqrt(po.pairwise_sqdist(tp, mp)).min(2)[0].reshape(B, n2, -1)
    sc_ref = w1.unsqueeze(1).sum(2) / ((dis * w1.unsqueeze(1)).sum(2) + 1e-8)
    Rb, tb, sc = ops.coarse_select(Rt.cuda(), top.int().cuda(), pts1.cuda(), w1.cuda(), model.cuda())
    # sqrt of the reference's expanded-form squared distance amplifies fp32 cancellation noise near d = 0
    torch.testing.assert_close(sc.cpu(), sc_ref, atol=0, rtol=5e-3)
    best = sc.cpu().max(1)[1]
    torch.testing.assert_close(Rb.cpu(), Rsel[torch.arange(B), best], atol=0, rtol=0)
    torch.testing.assert_close(tb.cpu(), tsel[torch.arange(B), best, 0], atol=0, rtol=0)
    # and the chosen pose is the planted one
    torch.testing.assert_close(Rb.cpu(), R, atol=2e-2, rtol=0)


def test_procrustes_rank_deficient_completion(ops):
    """all three correspondences identical -> identity; two identical (either side, or both at different slots) -> the least
    rotation taking the source direction onto the reference direction; compared with the oracle's restatement of the rule"""
    g = G(1)
    n = 10
    pts1 = torch.randn(1, n, 3, generator=g)
    pts2 = torch.randn(1, n, 3, generator=g)
    f = lambda a, b: a * n + b      # noqa: E731  flat index of the correspondence (point a of cloud 1, point b of cloud 2)
    trip = [[f(3, 4)] * 3, [f(3, 4), f(3, 4), f(5, 6)], [f(3, 4), f(3, 7), f(5, 6)], [f(1, 4), f(2, 4), f(5, 6)],
            [f(1, 4), f(1, 5), f(2, 5)], [f(1, 2), f(1, 3), f(1, 4)], [f(1, 1), f(2, 3), f(3, 5)]]
    idx = torch.tensor([sum(trip, [])], dtype=torch.int32)
    n1 = len(trip)
    Rt, resid = ops.coarse_hypotheses(idx.cuda(), pts1.cuda(), pts2.cuda())
    R = Rt.cpu()[0, :, :9].reshape(n1, 3, 3)
    assert torch.isfinite(R).all() and torch.isfinite(resid).all()
    torch.testing.assert_close(R @ R.transpose(1, 2), torch.eye(3).expand(n1, 3, 3), atol=1e-5, rtol=0)
    torch.testing.assert_close(torch.det(R), torch.ones(n1), atol=1e-5, rtol=0)
    i1, i2 = (idx.long() // n), (idx.long() % n)
    r1, r0 = po._triplet_ranks(i1, i2, 1, n1)
    assert r0.tolist() == [True, False, False, False, False, True, False]
    assert r1.tolist() == [False, True, True, True, True, False, False]
    p1 = pts1[0][i1.reshape(-1)].reshape(n1, 3, 3)
    p2 = pts2[0][i2.reshape(-1)].reshape(n1, 3, 3)
    Rs, ts = po.weighted_procrustes(p2, p1, None, weight_thresh=0.5, rank1=r1, rank0=r0)
    torch.testing.assert_close(R, Rs, atol=1e-5, rtol=0)
    torch.testing.assert_close(Rt.cpu()[0, :, 9:], ts, atol=1e-5, rtol=0)
    torch.testing.assert_close(R[0], torch.eye(3), atol=0, rtol=0)
    # the rank-1 rotation maps the source segment direction onto the reference segment direction
    d2 = torch.nn.functional.normalize(pts2[0, 6] - pts2[0, 4], dim=0)
    d1 = torch.nn.functional.normalize(pts1[0, 5] - pts1[0, 3], dim=0)
    torch.testing.assert_close(R[1] @ d2, d1, atol=1e-5, rtol=0)


# ------------------------------------------------------------------------------------------------- fine stage pieces
def test_positional_encoding_kernel(ops):
    from sam6d_b200.pem import PositionalEncoding
    sd = po.make_state_dict(seed=5)
    pe = PositionalEncoding(256).cuda().eval()
    pe.load_state_dict({k[len("fine_point_matching.PE."):]: v for k, v in sd.items() if k.startswith("fine_point_matching.PE.")})
    inp = po.make_inputs(B=2, n=2048, seed=5)
    pts = inp["dense_po"] / (torch.norm(inp["dense_po"], dim=2).max(1)[0].reshape(-1, 1, 1) + 1e-6)
    ref = po.positional_encoding(sd, pts)
    got = pe(pts.cuda()).cpu()
    torch.testing.assert_close(got, ref, atol=5e-4, rtol=1e-4)


def test_fine_assign_procrustes_score(ops):
    B, S, nm = 2, 513, 256
    A = _score_matrix(B, S, 7, peak=8.0)
    g = G(8)
    pts2 = torch.randn(B, S - 1, 3, generator=g) * 0.4
    R = po.random_rotation(B, g)
    t = torch.randn(B, 3, generator=g) * 0.1
    pts1 = pts2 @ R.transpose(1, 2) + t.unsqueeze(1)
    model = pts2[:, :nm].contiguous()
    Rr, tr, sr, dbg = po.fine_Rt(A, pts1, pts2, model, return_debug=True)
    lab1, lab2, wts, pred = ops.fine_assign(A.cuda(), pts2.cuda(), shift=10.0)
    assert torch.equal(lab1.cpu()[:, 1:].long(), dbg["lab1"])
    assert torch.equal(lab2.cpu()[:, 1:].long(), dbg["lab2"])
    torch.testing.assert_close(wts.cpu(), dbg["wts"], atol=1e-6, rtol=2e-4)
    torch.testing.assert_close(pred.cpu(), dbg["pred"], atol=1e-5, rtol=1e-4)
    Rg, tg = ops.weighted_procrustes(pred, pts1.cuda(), wts)
    torch.testing.assert_close(Rg.cpu(), Rr, atol=1e-4, rtol=0)
    torch.testing.assert_close(tg.cpu(), tr, atol=1e-4, rtol=0)
    radius = torch.tensor([0.7, 1.3])
    score, ts = ops.pose_score(pts1.cuda(), lab1, Rg, tg, model.cuda(), radius.cuda(), 0.15)
    torch.testing.assert_close(score.cpu(), sr, atol=2e-3, rtol=0)
    torch.testing.assert_close(ts.cpu(), tr * (radius.reshape(-1, 1) + 1e-6), atol=2e-4, rtol=0)


# ------------------------------------------------------------------------------------------------- ISM template scoring
@pytest.mark.parametrize("P,O,T", [(64, 8, 42), (200, 21, 42), (5, 1, 3)])
def test_template_score(ops, P, O, T):
    from sam6d_b200 import ism
    q, r = io.make_descriptors(P=P, O=O, T=T, C=1024, seed=P)
    idx_sel, pred_obj, sem, best_t, scores, per_obj = io.compute_semantic_score(q, r)
    sim = ism.PairwiseSimilarity()(q.cuda(), r.cuda()).cpu()
    torch.testing.assert_close(sim, scores, atol=2e-6, rtol=1e-5)
    g_sel, g_obj, g_sem, g_t = ism.compute_semantic_score(q.cuda(), r.cuda())
    assert torch.equal(g_sel.cpu(), idx_sel)
    assert torch.equal(g_obj.cpu(), pred_obj)                     # bit-exact argmax object
    assert torch.equal(g_t.cpu(), best_t)                         # bit-exact argmax template indices
    assert g_t.dtype == torch.int64 and g_obj.dtype == torch.int64
    torch.testing.assert_close(g_sem.cpu(), sem, atol=2e-6, rtol=1e-5)


@pytest.mark.parametrize("case", ["config5_ycbv", "config3_ism"])
def test_template_score_matches_reference_golden(ops, golden_dir, case):
    """the fused scoring kernel against the outputs of the reference's OWN PairwiseSimilarity / compute_semantic_score /
    best_template_pose (tests/golden/ism_scoring.pt, tools/make_golden_ism.py): bit-exact object and template indices"""
    import os
    from sam6d_b200 import ism
    c = torch.load(os.path.join(golden_dir, "ism_scoring.pt"), weights_only=False)["cases"][case]
    q, r = io.make_descriptors(P=c["P"], O=c["O"], T=c["T"], C=c["C"], seed=c["seed"])
    assert q.double().sum().item() == c["input_checksum"]["q"] and r.double().sum().item() == c["input_checksum"]["ref"]
    scorer = ism.SemanticScorer(r.cuda())
    g_sel, g_obj, g_sem, g_t = scorer.compute_semantic_score(q.cuda())
    assert torch.equal(g_sel.cpu(), c["idx_selected"])
    assert torch.equal(g_obj.cpu(), c["pred_idx_objects"])
    assert torch.equal(g_t.cpu(), c["best_template"])
    torch.testing.assert_close(g_sem.cpu(), c["semantic_score"], atol=2e-6, rtol=1e-5)
    sim = scorer.matching_config.metric(q.cuda(), r.cuda()).cpu()
    torch.testing.assert_close(sim, c["sim"], atol=2e-6, rtol=1e-5)


# ------------------------------------------------------------------------------------------------- wgmma GEMM
@pytest.mark.parametrize("M,N,K", [(197 * 3, 1792, 256), (1000, 512, 256), (4096, 256, 512), (130, 40, 64), (2049, 2049, 256)])
@pytest.mark.parametrize("adt,wdt,odt", [(torch.float32, torch.bfloat16, torch.float32), (torch.float32, torch.float32, torch.float32),
                                         (torch.bfloat16, torch.bfloat16, torch.bfloat16)])
def test_gemm_tc(ops, M, N, K, adt, wdt, odt):
    A = torch.randn(M, K, generator=G(1))
    W = torch.randn(N, K, generator=G(2)) / math.sqrt(K)
    bias = torch.randn(N, generator=G(3))
    R = torch.randn(M, N, generator=G(4))
    # the kernel rounds both operands to bf16 and accumulates in fp32: compare with exactly that arithmetic
    ref = torch.relu(A.bfloat16().double() @ W.bfloat16().double().t() * 0.5 + bias.double()) + R.double()
    got = ops.gemm_tc(A.cuda().to(adt), W.cuda().to(wdt), bias.cuda(), residual=R.cuda(), relu=True, alpha=0.5, out_dtype=odt).cpu()
    assert got.dtype == odt
    tol = 2e-5 if odt == torch.float32 else 2e-2
    torch.testing.assert_close(got.double(), ref, atol=tol, rtol=1e-5 if odt == torch.float32 else 1e-2)


def test_gemm_tc_batched_strided_views(ops):
    B, N, M, C = 3, 300, 257, 256
    f1 = torch.randn(B, N, C, generator=G(1))
    f2 = torch.randn(B, M, C, generator=G(2))
    out = torch.empty(B, N, M).cuda()
    a, w = f1.cuda(), f2.cuda()
    ops.gemm_tc(a, w, out=out, alpha=10.0)
    ref = 10.0 * f1.bfloat16().double() @ f2.bfloat16().double().transpose(1, 2)
    torch.testing.assert_close(out.cpu().double(), ref, atol=2e-4, rtol=1e-5)


@pytest.mark.parametrize("S,edt", [(64, torch.float32), (197, torch.bfloat16), (197, torch.float32), (33, torch.bfloat16)])
def test_geo_embed_tc(ops, S, edt):
    """wgmma geometric embedding: bf16 operands (sin/cos and weights), fp32 accumulation, E in fp32 or bf16"""
    sd = po.make_state_dict(seed=2)
    pts = _sparse_cloud(3, S, 9)
    ref = exact_geo_embedding(sd, pts)
    T = ops.geo_indices(pts.cuda(), po.SIGMA_D, 180.0 / (po.SIGMA_A * math.pi))
    E = ops.geo_embed_tc(T, sd["geo_embedding.embedding.div_term"].cuda(), sd["geo_embedding.proj_a.weight"].cuda().bfloat16().contiguous(),
                         sd["geo_embedding.proj_d.weight"].cuda().bfloat16().contiguous(),
                         (sd["geo_embedding.proj_a.bias"] + sd["geo_embedding.proj_d.bias"]).cuda(), out_dtype=edt).float().cpu()
    assert E.shape == ref.shape and torch.isfinite(E).all()
    err = (E - ref).abs()
    # bf16 rounding of 256-term dot products of O(1) values: ~3e-3 typical, a few 1e-2 worst case
    assert err.median().item() < 4e-3, err.median().item()
    assert (err > 6e-2).float().mean().item() < 2e-3
    # and it must agree with the fp32 CUDA-core kernel within the same budget (same indices, so no knn-tie outliers)
    E32 = ops.geo_embed_f32(T, sd["geo_embedding.embedding.div_term"].cuda(), sd["geo_embedding.proj_a.weight"].t().contiguous().cuda(),
                            sd["geo_embedding.proj_d.weight"].t().contiguous().cuda(),
                            (sd["geo_embedding.proj_a.bias"] + sd["geo_embedding.proj_d.bias"]).cuda()).cpu()
    torch.testing.assert_close(E, E32, atol=6e-2, rtol=0)


@pytest.mark.parametrize("S,far_point", [(197, False), (64, False), (197, True), (33, True)])
def test_geo_embed_lut(ops, S, far_point):
    """table-interpolated geometric embedding (csrc/geo_lut.cu) through the module, against the float64-index embedding: at least as
    close as the tensor-core product, incl. the background point's row / column (exact distance projection, `far`) and -- far_point
    -- an ordinary point 40 units away, whose pairs take the exact per-pair fallback"""
    from sam6d_b200 import pem
    sd = po.make_state_dict(seed=2)
    pts = _sparse_cloud(3, S, 9)
    if far_point:
        pts[:, 5, :] = torch.tensor([30.0, -20.0, 10.0])
    ref = exact_geo_embedding(sd, pts)
    geo = pem.GeometricStructureEmbedding(pem.DEFAULT_MODEL_CFG["geo_embedding"]).cuda()
    geo.load_state_dict({k[len("geo_embedding."):]: v for k, v in sd.items() if k.startswith("geo_embedding.")})
    geo.precision = "bf16"
    E = geo(pts.cuda())
    assert E.dtype == torch.bfloat16 and E.shape == ref.shape
    E = E.float().cpu()
    assert torch.isfinite(E).all()
    err = (E - ref).abs()
    assert err.median().item() < 4e-3, err.median().item()
    assert (err > 6e-2).float().mean().item() < 2e-3
    T = ops.geo_indices(pts.cuda(), po.SIGMA_D, 180.0 / (po.SIGMA_A * math.pi))
    w = geo._weights()
    wa_bf = geo.proj_a.weight.detach().to(torch.bfloat16).contiguous()
    Etc = ops.geo_embed_tc(T, w["div"], wa_bf, w["wd_bf"], w["bias"], out_dtype=torch.bfloat16).float().cpu()
    # same indices: the two kernels differ only by their bf16 roundings (no knn-tie outliers)
    torch.testing.assert_close(E, Etc, atol=4e-2, rtol=0)
    rms_lut, rms_tc = (E - ref).pow(2).mean().sqrt().item(), (Etc - ref).pow(2).mean().sqrt().item()
    print(f"geo S={S} far_point={far_point}: rms error vs float64-index embedding: table {rms_lut:.3e}, tensor-core {rms_tc:.3e}")
    assert rms_lut < 1.1 * rms_tc + 1e-4
    # rows / columns whose distance index is outside the table
    far_rows = [0, 5] if far_point else [0]
    for r in far_rows:
        others = [m for m in range(S) if m != r]
        assert (T[:, r, others, 3] > 32).all()
        assert (E[:, r] - ref[:, r]).abs().median().item() < 4e-3 and (E[:, :, r] - ref[:, :, r]).abs().median().item() < 4e-3
    # the distance-only tensor-core projection that feeds `far`
    far = ops.geo_embed_dist_tc(T[:, 0].contiguous(), w["div"], w["wd_bf"], w["bias"]).float().cpu()
    want = po._lin(sd, "geo_embedding.proj_d", po.sinusoidal_embedding(T[:, 0, :, 3].cpu(), 256)) + sd["geo_embedding.proj_a.bias"]
    torch.testing.assert_close(far, want, atol=3e-2, rtol=0)


def test_positional_encoding_tensor_core(ops):
    """layers 2/3 of the PE shared MLP on wgmma (bf16 operands) against the fp32 oracle"""
    from sam6d_b200.pem import PositionalEncoding
    sd = po.make_state_dict(seed=5)
    pe = PositionalEncoding(256).cuda().eval()
    pe.load_state_dict({k[len("fine_point_matching.PE."):]: v for k, v in sd.items() if k.startswith("fine_point_matching.PE.")})
    inp = po.make_inputs(B=3, n=2048, seed=5)
    pts = inp["dense_po"] / (torch.norm(inp["dense_po"], dim=2).max(1)[0].reshape(-1, 1, 1) + 1e-6)
    ref_local = torch.cat([po._shared_mlp(sd, "fine_point_matching.PE.mlp1", po._query_and_group(pts, po.PE_R1, po.PE_NS1)).max(dim=3)[0],
                           po._shared_mlp(sd, "fine_point_matching.PE.mlp2", po._query_and_group(pts, po.PE_R2, po.PE_NS2)).max(dim=3)[0]],
                          dim=1).transpose(1, 2)
    pe.precision = "fp32"
    l32 = pe.local_features(pts.cuda()).cpu()
    torch.testing.assert_close(l32, ref_local, atol=2e-4, rtol=1e-4)
    pe.precision = "bf16"
    l16 = pe.local_features(pts.cuda()).cpu().float()          # bf16 features in this mode
    err = (l16 - ref_local).abs()
    scale = ref_local.abs().mean().item()
    print("PE tc: mean |ref|", scale, "median err", err.median().item(), "max err", err.max().item())
    assert err.median().item() < 1e-2 * max(scale, 1.0)
    torch.testing.assert_close(l16, ref_local, atol=8e-2 * max(scale, 1.0), rtol=5e-2)
    # odd sizes: N not a multiple of the points-per-tile
    pts2 = pts[:, :1023].contiguous()
    pe.precision = "fp32"
    a = pe.local_features(pts2.cuda()).cpu()
    pe.precision = "bf16"
    b = pe.local_features(pts2.cuda()).cpu().float()
    torch.testing.assert_close(b, a, atol=8e-2 * max(scale, 1.0), rtol=5e-2)


@pytest.mark.parametrize("M,N,K", [(4096, 3840, 1280), (1000, 512, 256), (130, 40, 64), (2049, 2049, 256), (300, 1280, 5120)])
@pytest.mark.parametrize("odt", [torch.float32, torch.bfloat16])
def test_gemm_tma(ops, M, N, K, odt):
    A = torch.randn(M, K, generator=G(1))
    W = torch.randn(N, K, generator=G(2)) / math.sqrt(K)
    bias = torch.randn(N, generator=G(3))
    R = torch.randn(M, N, generator=G(4))
    R = R.to(odt)                           # the residual stream has the element type of the output
    ref = torch.nn.functional.gelu(A.bfloat16().double() @ W.bfloat16().double().t() * 0.5 + bias.double()) + R.double()
    got = ops.gemm_tma(A.cuda().bfloat16(), W.cuda().bfloat16(), bias.cuda(), residual=R.cuda(), act=2, alpha=0.5, out_dtype=odt).cpu()
    assert got.dtype == odt
    if odt == torch.float32:
        torch.testing.assert_close(got.double(), ref, atol=1e-4, rtol=1e-5)     # fp32 accumulation order over K <= 5120
    else:
        torch.testing.assert_close(got.double(), ref, atol=3e-2, rtol=1e-2)


def _dense_attention(q, k, v, H, scale, bias=None):
    B, Sq, C = q.shape
    Sk = k.shape[1]
    d = C // H
    qh, kh, vh = (t.view(B, -1, H, d).permute(0, 2, 1, 3) for t in (q, k, v))
    s = qh @ kh.transpose(-1, -2)
    if bias is not None:
        s = s + bias
    att = torch.softmax(s * scale, dim=-1)
    return (att @ vh).permute(0, 2, 1, 3).reshape(B * Sq, C)


@pytest.mark.parametrize("B,Sq,Sk,H,D,with_bias", [(3, 197, 197, 4, 64, True), (2, 197, 150, 4, 64, False), (5, 196, 196, 2, 80, False),
                                                    (1, 33, 256, 1, 64, True)])
def test_attn_tc_dense(ops, B, Sq, Sk, H, D, with_bias):
    """wgmma attention against fp64 softmax attention on the bf16-rounded operands"""
    g = G(Sq + Sk)
    q = torch.randn(B, Sq, H * D, generator=g)
    k = torch.randn(B, Sk, H * D, generator=g)
    v = torch.randn(B, Sk, H * D, generator=g)
    bias = torch.randn(B, H, Sq, Sk, generator=g) if with_bias else None
    bv = torch.randn(H * D, generator=g)
    qb, kb, vb = q.bfloat16(), k.bfloat16(), v.bfloat16()
    ref = _dense_attention(qb.double(), kb.double(), vb.double(), H, D ** -0.5, bias.double() if with_bias else None) + bv.double()
    N1 = (Sk + 15) // 16 * 16
    vt = torch.zeros(B * H * D, N1, dtype=torch.bfloat16)
    vt[:, :Sk] = vb.view(B, Sk, H, D).permute(0, 2, 3, 1).reshape(B * H * D, Sk)
    qk = torch.cat([qb.view(B * Sq, -1), torch.zeros(B * Sq, 8, dtype=torch.bfloat16)], dim=1).contiguous()   # odd leading dim
    got = ops.attn_tc(qk.cuda(), 0, kb.view(B * Sk, -1).contiguous().cuda(), 0, vt.cuda(), B, H, Sq, Sk, D, D ** -0.5,
                      bias=bias.cuda() if with_bias else None, bv=bv.cuda()).cpu()
    # P is rounded to bf16 before the PV product: ~2^-9 relative on O(1) outputs
    torch.testing.assert_close(got.double(), ref, atol=2e-2, rtol=2e-2)
    assert (got.double() - ref).abs().mean().item() < 3e-3


def test_attn_tc_sam_window(ops):
    """decomposed rel-pos bias mode against the reference formula (image_encoder.py:325-361)"""
    from oracle import sam_oracle as so
    nW, S, H, D = 4, 14, 2, 80
    g = G(77)
    qkv = torch.randn(nW * S * S, 3 * H * D, generator=g)
    rel_h = torch.randn(2 * S - 1, D, generator=g) * 0.1
    rel_w = torch.randn(2 * S - 1, D, generator=g) * 0.1
    qkv_b = qkv.bfloat16()
    x = qkv_b.float().view(nW, S * S, 3, H, D).permute(2, 0, 3, 1, 4).reshape(3, nW * H, S * S, D)
    q, k, v = x.unbind(0)
    attn = (q * D ** -0.5) @ k.transpose(-2, -1)
    Rh, Rw = so.rel_pos_table(S, rel_h), so.rel_pos_table(S, rel_w)
    rq = q.reshape(nW * H, S, S, D)
    attn = (attn.view(-1, S, S, S, S) + torch.einsum("bhwc,hkc->bhwk", rq, Rh)[:, :, :, :, None] +
            torch.einsum("bhwc,wkc->bhwk", rq, Rw)[:, :, :, None, :]).view(-1, S * S, S * S).softmax(dim=-1)
    ref = (attn @ v).view(nW, H, S * S, D).permute(0, 2, 1, 3).reshape(nW * S * S, H * D)
    L = S * S
    N1 = (L + 15) // 16 * 16
    vt = torch.zeros(nW * H * D, N1, dtype=torch.bfloat16)
    vt[:, :L] = qkv_b[:, 2 * H * D:].view(nW, L, H, D).permute(0, 2, 3, 1).reshape(nW * H * D, L)
    qk = qkv_b[:, :2 * H * D].contiguous()
    got = ops.attn_tc(qk.cuda(), 0, qk.cuda(), H * D, vt.cuda(), nW, H, L, L, D, D ** -0.5,
                      rel=(ops.pack_rel_pos(rel_h.cuda(), rel_w.cuda()), S, S)).cpu()
    torch.testing.assert_close(got, ref, atol=2e-2, rtol=2e-2)
    assert (got - ref).abs().mean().item() < 3e-3


def test_attn_global_tensor_core(ops):
    """SAM global attention (64 x 64 tokens, online softmax on wgmma) against the reference formula
    (image_encoder.py:224-240, 325-361) evaluated in fp32 on the same bf16-rounded q, k, v."""
    from oracle import sam_oracle as so
    B, S, H, D = 2, 64, 2, 80
    L = S * S
    g = G(78)
    qkv = (torch.randn(B * L, 3 * H * D, generator=g) * 1.5).bfloat16()
    rel_h = torch.randn(2 * S - 1, D, generator=g) * 0.2
    rel_w = torch.randn(2 * S - 1, D, generator=g) * 0.2
    x = qkv.float().cuda().view(B, L, 3, H, D).permute(2, 0, 3, 1, 4).reshape(3, B * H, L, D)
    q, k, v = x.unbind(0)
    attn = (q * D ** -0.5) @ k.transpose(-2, -1)
    Rh, Rw = so.rel_pos_table(S, rel_h).cuda(), so.rel_pos_table(S, rel_w).cuda()
    rq = q.reshape(B * H, S, S, D)
    attn = (attn.view(-1, S, S, S, S) + torch.einsum("bhwc,hkc->bhwk", rq, Rh)[:, :, :, :, None] +
            torch.einsum("bhwc,wkc->bhwk", rq, Rw)[:, :, :, None, :]).view(-1, L, L).softmax(dim=-1)
    ref = (attn @ v).view(B, H, L, D).permute(0, 2, 1, 3).reshape(B * L, H * D).cpu()
    qd = qkv.cuda()
    vt = ops.transpose_tokens(qd, 2 * H * D, H * D, B, L)
    blob = ops.pack_rel_pos(rel_h.cuda(), rel_w.cuda(), slab_rows=128)
    # bf16 P and bf16 rel-pos tables (|q . rel| ~ 3 here): worst-case logit error ~1e-2 -> output error of a few 1e-2 on a
    # handful of peaked rows, mean error an order of magnitude lower
    for odt in (torch.float32, torch.bfloat16):
        got = ops.attn_global_tc(qd, vt, blob, B, H, S, D ** -0.5, out_dtype=odt).cpu().float()
        torch.testing.assert_close(got, ref, atol=6e-2, rtol=2e-2)
        assert (got - ref).abs().mean().item() < 3e-3


@pytest.mark.parametrize("B,S,T", [(3, 197, 197), (2, 2049, 2049), (4, 130, 77)])
def test_gemm_tma_batched_scores_view(ops, B, S, T):
    """stacked per-proposal score matrices: tiles that run into the next proposal's rows must not leak into the output"""
    C = 256
    a = torch.randn(B, S, C, generator=G(1))
    w = torch.randn(B, T, C, generator=G(2))
    ld = (T + 3) // 4 * 4
    out = torch.full((B, S, ld), 7.0, device="cuda")
    an, wn = ops.l2norm_rows_bf16(a.cuda()), ops.l2norm_rows_bf16(w.cuda())
    ops.gemm_tma_batched(an, wn, out[:, :, :T], alpha=10.0)
    ref = 10.0 * an.float().cpu().double() @ wn.float().cpu().double().transpose(1, 2)
    torch.testing.assert_close(out.cpu()[:, :, :T].double(), ref, atol=2e-4, rtol=1e-5)
    assert (out.cpu()[:, :, T:] == 7.0).all()
    torch.testing.assert_close(an.float().cpu(), torch.nn.functional.normalize(a, dim=-1), atol=4e-3, rtol=4e-3)


@pytest.mark.parametrize("nB,S,C,K", [(5, 197, 256, 256), (3, 196, 1280, 1280), (1, 4096, 160, 256)])
def test_gemm_tma_vt_matches_gemm_plus_transpose(ops, nB, S, C, K):
    """QKV projection with the value columns written as V^T by the epilogue == plain GEMM followed by transpose_tokens"""
    M, N = nB * S, 3 * C
    A = torch.randn(M, K, generator=G(1)).bfloat16().cuda()
    W = (torch.randn(N, K, generator=G(2)) / math.sqrt(K)).bfloat16().cuda()
    b = torch.randn(N, generator=G(3)).cuda()
    full = ops.gemm_tma(A, W, b, out_dtype=torch.bfloat16)
    vt_ref = ops.transpose_tokens(full, 2 * C, C, nB, S)
    qk, vt = ops.gemm_tma_vt(A, W, b, 2 * C, S, slot=7)
    assert torch.equal(qk, full[:, :2 * C])
    assert torch.equal(vt, vt_ref)


@pytest.mark.parametrize("nB,S", [(5, 197), (64, 197), (2, 64)])
def test_gemm_tma_vt2_three_column_ranges(ops, nB, S):
    """q | k rows, V^T and the folded rel-pos queries u from ONE launch == the plain GEMM's columns, bit for bit"""
    C, K = 256, 256
    M, N = nB * S, 3 * C + 4 * C
    A = torch.randn(M, K, generator=G(1)).bfloat16().cuda()
    W = (torch.randn(N, K, generator=G(2)) / math.sqrt(K)).bfloat16().cuda()
    b = torch.randn(N, generator=G(3)).cuda()
    full = ops.gemm_tma(A, W, b, out_dtype=torch.bfloat16)
    vt_ref = ops.transpose_tokens(full, 2 * C, C, nB, S)
    qk, vt, u = ops.gemm_tma_vt2(A, W, b, 2 * C, 3 * C, S, slot=9)
    assert torch.equal(qk, full[:, :2 * C])
    assert torch.equal(vt, vt_ref)
    assert torch.equal(u, full[:, 3 * C:])


@pytest.mark.parametrize("B,S", [(2, 513), (3, 2049), (1, 130)])
def test_fine_assign_tensor_core_fused(ops, B, S):
    """compute_fine_Rt's assignment recomputed tile by tile on wgmma (no (B,S,S) matrix) against fp64 math on the same
    bf16-rounded normalised tokens: labels exact (planted matches make them decisive), weights / correspondences to 1e-3"""
    g = G(31)
    C, temp = 256, 0.1
    f2 = torch.randn(B, S, C, generator=g)
    perm = torch.stack([torch.randperm(S, generator=g) for _ in range(B)])
    f1 = torch.gather(f2, 1, perm[:, :, None].expand(-1, -1, C)) + 0.35 * torch.randn(B, S, C, generator=g)
    pts2 = torch.randn(B, S - 1, 3, generator=g) * 0.4
    f1n, f2n = ops.l2norm_rows_bf16(f1.cuda()), ops.l2norm_rows_bf16(f2.cuda())
    a, b = f1n.cpu().double(), f2n.cpu().double()
    A = a @ b.transpose(1, 2) / temp
    P = torch.softmax(A, dim=2) * torch.softmax(A, dim=1)
    lab1_ref = P.argmax(dim=2)                                   # (B,S) incl. the bg row 0 (unused)
    lab2_ref = P.argmax(dim=1)
    mask = (lab2_ref[:, 1:] > 0).double()                        # columns j >= 1 matched to a non-background row
    Pm = P[:, 1:, 1:] * mask[:, None, :]
    w_ref = Pm.sum(dim=2) * (lab1_ref[:, 1:] > 0)
    pred_ref = (Pm @ pts2.double()) * (lab1_ref[:, 1:] > 0)[:, :, None] / (w_ref[:, :, None] + 1e-6)
    lab1, lab2, wts, pred = ops.fine_assign_tc(f1n, f2n, pts2.cuda(), 1.0 / temp)
    assert torch.equal(lab1.cpu()[:, 1:].long(), lab1_ref[:, 1:])
    assert torch.equal(lab2.cpu().long(), lab2_ref)
    torch.testing.assert_close(wts.cpu().double(), w_ref, atol=1e-6, rtol=2e-3)
    torch.testing.assert_close(pred.cpu().double(), pred_ref, atol=2e-5, rtol=2e-3)


@pytest.mark.parametrize("C", [96, 256, 384, 1280, 2048])
def test_layernorm_f32_to_bf16(ops, C):
    """LayerNorm writing bf16 rows (A operand of the next GEMM): vector kernel for C % 128 == 0, generic otherwise"""
    x = torch.randn(3, 41, C, generator=G(C)) * 2 + 0.5
    g, b = torch.randn(C, generator=G(2)), torch.randn(C, generator=G(3))
    ref = torch.nn.functional.layer_norm(x, (C,), g, b, eps=1e-6)
    got = ops.layernorm_bf16(x.cuda(), g.cuda(), b.cuda(), eps=1e-6).cpu()
    assert got.dtype == torch.bfloat16 and got.shape == x.shape
    torch.testing.assert_close(got.float(), ref, atol=3e-2, rtol=1e-2)
