"""Routing of the PEM modules: each module runs one route per precision, whatever allocation its two clouds arrive in.

The modules stack the scene cloud and the template cloud into one (2B, ...) batch themselves (a view of the caller's
allocation when the clouds are its two halves, as Net passes them, a copy otherwise), so the same values must give the same
bits and the same dtype either way."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from sam6d_b200 import synth     # noqa: E402

B, S, N = 2, 197, 2048           # S = 196 FPS samples + the background point (the coarse_npoint of the bench)


@pytest.fixture(scope="module")
def net():
    from sam6d_b200.pem import Net
    net = Net().cuda().eval()
    net.load_state_dict(synth.make_pem_state_dict(seed=1), strict=True)
    return net


def _randn(*shape, seed, scale=1.0, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).cuda()


def _split(t):
    """a (2B, ...) tensor -> its two halves (one allocation) and two separately allocated copies of them"""
    return (t[:B], t[B:]), (t[:B].clone(), t[B:].clone())


def _clouds(net, seed):
    """(2B, S-1, 3) sparse points of unit-radius clouds and their (2B, S, S, 256) geometric embedding with the background
    point, both clouds of every proposal in one allocation; the embedding has the dtype Net hands on in this precision"""
    g = torch.Generator().manual_seed(seed)
    d = torch.randn(2 * B, S - 1, 3, generator=g)
    pts = (d / d.norm(dim=2, keepdim=True) * torch.rand(2 * B, S - 1, 1, generator=g)).cuda()
    bg = torch.full((2 * B, 1, 3), 100.0, device="cuda")
    return pts, net.geo_embedding(torch.cat([bg, pts], dim=1))


def _assert_same(got, want):
    assert len(got) == len(want)
    for i, (a, b) in enumerate(zip(got, want)):
        assert a.dtype == b.dtype, (i, a.dtype, b.dtype)
        assert torch.equal(a, b), (i, (a.float() - b.float()).abs().max().item())


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_geometric_transformer_allocation_independent(net, precision):
    net.set_precision(precision)
    _, emb = _clouds(net, seed=1)
    (f0, f1), (g0, g1) = _split(_randn(2 * B, S, 256, seed=2))
    (e0, e1), (d0, d1) = _split(emb)
    blk = net.coarse_point_matching.transformers[0]
    _assert_same(blk(g0, d0, g1, d1), blk(f0, e0, f1, e1))


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_coarse_point_matching_allocation_independent(net, precision):
    net.set_precision(precision)
    pts, emb = _clouds(net, seed=3)
    (p0, p1), (q0, q1) = _split(pts)
    (f0, f1), (g0, g1) = _split(_randn(2 * B, S - 1, 256, seed=4))
    (e0, e1), (d0, d1) = _split(emb)
    radius = torch.full((B,), 0.1, device="cuda")
    model = _randn(B, 1024, 3, seed=5, scale=0.5)
    rand = torch.rand(B, synth.N_PROPOSAL1 * 3, generator=torch.Generator().manual_seed(6)).cuda()
    cpm = net.coarse_point_matching
    cpm.return_feat = True
    try:
        outs = []
        for args in ((p0, f0, e0, p1, f1, e1), (q0, g0, d0, q1, g1, d1)):
            ep, o1, o2 = cpm(*args, radius, {"model": model}, rand=rand)
            outs.append((ep["init_R"], ep["init_t"], cpm.last_select_scores, o1, o2))
    finally:
        cpm.return_feat = False
    _assert_same(outs[1], outs[0])


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_sparse_to_dense_allocation_independent(net, precision):
    net.set_precision(precision)
    _, emb = _clouds(net, seed=7)
    dense_dtype = torch.bfloat16 if precision == "bf16" else torch.float32     # the fine stage's token stream
    (x0, x1), (y0, y1) = _split(_randn(2 * B, N + 1, 256, seed=8, dtype=dense_dtype))
    (e0, e1), (d0, d1) = _split(emb)
    g = torch.Generator().manual_seed(9)
    idx = torch.stack([torch.randperm(N, generator=g)[:S - 1] for _ in range(2 * B)]).to(torch.int32).cuda()
    (i0, i1), (j0, j1) = _split(idx)
    blk = net.fine_point_matching.transformers[0]
    _assert_same(blk(y0, d0, j0, y1, d1, j1), blk(x0, e0, i0, x1, e1, i1))


def test_net_unequal_point_counts_run_one_sparse_stage(monkeypatch):
    """a template bank with more points than the scene: FPS brings both clouds down to coarse_npoint, and the geometric
    embedding and the coarse stage run on the 2B sparse clouds as one batch.  The fine stage is replaced by a pass-through:
    its assignment kernels take equal point counts only, and this test is about the sparse stage."""
    from sam6d_b200 import _lib
    from sam6d_b200.pem import Net
    net = Net(precision="bf16").cuda().eval()
    net.load_state_dict(synth.make_pem_state_dict(seed=1), strict=True)
    monkeypatch.setattr(net.fine_point_matching, "forward", lambda *args: args[-1])
    scene = synth.make_pem_inputs(B=B, n=2048, seed=10)
    bank = synth.make_pem_inputs(B=B, n=2560, seed=11)
    ep = {"pts": scene["pts"], "dense_fm": scene["dense_fm"], "dense_po": bank["dense_po"], "dense_fo": bank["dense_fo"],
          "model": bank["model"]}
    ep = {k: v.cuda() for k, v in ep.items()}
    rand = torch.rand(B, synth.N_PROPOSAL1 * 3, generator=torch.Generator().manual_seed(12)).cuda()
    _lib.time_kernel("sam6d_geo_embed_lut", True)
    try:
        out = net(dict(ep), rand=rand)
        torch.cuda.synchronize()
        launches = len(_lib.timed_events("sam6d_geo_embed_lut"))
    finally:
        _lib.time_kernel("sam6d_geo_embed_lut", False)
    assert launches == 1
    R, t = out["init_R"].cpu(), out["init_t"].cpu()
    assert R.shape == (B, 3, 3) and torch.isfinite(R).all() and torch.isfinite(t).all()
    torch.testing.assert_close(R @ R.transpose(1, 2), torch.eye(3).expand_as(R), atol=1e-5, rtol=0)
    torch.testing.assert_close(torch.det(R), torch.ones(B), atol=1e-5, rtol=0)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_positional_encoding_larger_first_radius(precision):
    """r1 > r2: the features equal those built from two ball_query calls, scale by scale"""
    from sam6d_b200 import ops
    from sam6d_b200.pem import PositionalEncoding
    sd = synth.make_pem_state_dict(seed=5)
    pe = PositionalEncoding(256, r1=0.2, r2=0.1).cuda().eval()
    pe.load_state_dict({k[len("fine_point_matching.PE."):]: v for k, v in sd.items() if k.startswith("fine_point_matching.PE.")})
    pe.precision = precision
    po = synth.make_pem_inputs(B=B, n=N, seed=13)["dense_po"]
    pts = (po / po.norm(dim=2).max(1)[0].reshape(-1, 1, 1)).cuda()
    got = pe.local_features(pts)
    w = pe._weights()
    want = torch.empty_like(got)
    for r, ns, name, off in ((pe.r1, pe.ns1, "m1", 0), (pe.r2, pe.ns2, "m2", 128)):
        idx, cnt = ops.ball_query(pts, pts, r, ns, return_count=True)
        if precision == "bf16":
            ops.pe_mlp_max_tc(pts, idx, w[name + "_tc"], want, off)
        else:
            ops.pe_mlp_max(pts, idx, cnt, w[name], want, off)
    assert torch.equal(got, want)
