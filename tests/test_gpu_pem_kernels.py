"""GPU: the PEM's bf16 hot-path kernels (the ones bench.py times) called directly through the C ABI, each against a float64
evaluation of the same operation in plain torch on the operands rounded exactly as the kernel reads them.

Every bound is derived from the kernel's arithmetic and written next to its check.  Notation: u = 2^-24 (fp32 unit roundoff),
ub = 2^-8 (bf16 unit roundoff: one round-to-nearest bf16 store moves a value by at most ub |x|), gamma_n ~ n u for a chain of n
fp32 roundings.  A tensor-core (wgmma) fp32 accumulation is charged 2u per added product: the accumulator may truncate rather
than round.  Documented accuracy of the math functions used: ex2.approx.f32 and __expf 2 ulp of the result (plus, for __expf,
the rounding of its argument: 2 + floor(|1.173 x|) ulp), rsqrtf 2 ulp, sincosf 2 ulp; sqrtf and divisions are IEEE (nvcc's
defaults).  An ulp of a result in [1, 2) is 2u.

Where a kernel rounds an intermediate to bf16 (y and h of the layer tail, h1 and h2 of the PE MLP, q' of the linear attention)
the float64 chain rounds the float64 value at the same place (fp64 -> fp32 -> bf16, as the kernel's fp32 value is rounded).
The kernel's fp32 value lies within a derived distance e of the float64 one, and rounding is monotone, so the two bf16 values
differ by at most bf16(v + e) - bf16(v - e): zero unless v sits within e of a rounding boundary, one bf16 ulp (plus e) if it
does (`_spread`).  That difference is carried through the rest of the chain with magnitude products.

Each check prints its largest error / bound ratio; where a bound is loose enough to leave doubt, a deliberately wrong answer
computed in torch must fail the same bound."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24          # fp32 unit roundoff
UB = 2.0 ** -8          # bf16 unit roundoff
F64 = torch.float64
EPS6 = float(np.float32(1e-6))     # the fp32 constant 1e-6f the kernels add


@pytest.fixture(scope="module")
def lib():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from sam6d_b200 import _lib
    return _lib


@pytest.fixture(scope="module")
def ops(lib):
    from sam6d_b200 import ops as _ops
    return _ops


def _g(seed):
    return torch.Generator().manual_seed(seed)


def _gc(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _ratio(err, bound):
    """max over elements of err / bound (0 / 0 counts as 0: outputs that must be exact)"""
    err, bound = err.to(F64), bound.to(F64)
    assert torch.isfinite(err).all(), "non-finite output"
    return (err / bound.clamp_min(1e-300)).max().item()


def _check(name, err, bound):
    r = _ratio(err, bound)
    print(f"{name}: max error / bound = {r:.3g}  (max error {err.max().item():.3g})")
    assert r <= 1.0, f"{name}: error exceeds its bound by {r:.3g}x"
    return r


def _bf(v):
    """the bf16 value a kernel stores for an fp32 value equal to v (fp64 -> fp32 -> bf16, round to nearest even)"""
    return v.float().bfloat16().to(F64)


def _spread(v, e):
    """bound on |bf16(kernel fp32 value) - _bf(v)| when the kernel's fp32 value is within e of v (module docstring)"""
    return _bf(v + e) - _bf(v - e)


def _exp_err(xr):
    """relative error of __expf over arguments down to -xr, plus the rounding of the subtraction s - m"""
    return (2.0 + 1.173 * xr) * 2 * U + U * xr


# ================================================================================================== 1. layer tail (tail_tc.cu)
def _ln_stats(z, eps):
    mu = z.mean(-1, keepdim=True)
    d = z - mu
    var = d.pow(2).mean(-1, keepdim=True)
    return mu, d, var, 1.0 / torch.sqrt(var + eps)


def _ln_bound(z, dz, g, b, eps):
    """LayerNorm of the kernel (fp32, one-pass statistics, 256 channels in the four threads of a quad) on an input known to
    within dz of z -> (float64 LayerNorm of z, bound on the kernel's fp32 result)"""
    mu, d, var, r = _ln_stats(z, eps)
    zh = d * r
    out = zh * g + b
    # input error, first order through the Jacobian (g r)(I - 11^T/n - zh zh^T/n):
    #   |d out_i| <= |g_i| r (dz_i + mean dz + |zh_i| mean(|zh| dz)); 2 % covers the second-order terms (dz << sigma here)
    prop = 1.02 * g.abs() * r * (dz + dz.mean(-1, keepdim=True) + zh.abs() * (zh.abs() * dz).mean(-1, keepdim=True))
    # own arithmetic.  mean: per thread 32 pair sums (33 roundings per element) + 2 quad levels, times 1/256 (exact)
    e_mu = 35 * U * z.abs().mean(-1, keepdim=True)
    # E[z^2]: a 64-term fma chain + 2 quad levels; var = E[z^2] - mu^2 (square and difference one rounding each, the
    # cancellation of a large common offset is what makes this term matter), + eps one rounding
    e_var = 66 * U * z.pow(2).mean(-1, keepdim=True) + 2 * mu.abs() * e_mu + e_mu ** 2 + U * mu ** 2 + U * var + U * (var + eps)
    e_r = 0.5 * e_var / (var + eps) + 4 * U                    # rsqrtf 2 ulp; half the relative error of var + eps
    # (z - mu) one rounding, times rstd one rounding, fma with gamma / beta one rounding
    own = g.abs() * r * (e_mu + U * d.abs() + d.abs() * (e_r + U)) + U * out.abs()
    return out, prop + own


def _tail_inputs(M, kind, seed):
    g = _gc(seed)
    dev = "cuda"
    # hid on a 2^-2 grid (|hid| <= 3), W_o on a 2^-6 grid (|w| <= 1/4): every product is a multiple of 2^-8 and every partial
    # sum of a row stays below 192 = 2^15.6 of them, so G1 accumulates exactly in fp32 in any order (see _tail_ref)
    hid = (torch.randn(M, 256, generator=g, device=dev) * 4).round().clamp(-12, 12) / 4
    x = torch.randn(M, 256, generator=g, device=dev)
    if kind == "offset":
        x = x + 50.0                                            # LayerNorm 1 cancels a common offset of 50 sigma
    if kind == "flat":
        hid = torch.zeros(M, 256, device=dev)                   # z1 = x in {-2^-9, 0, 2^-9}: variance ~2.5e-6 < eps
        x = 2.0 ** -9 * torch.randint(-1, 2, (M, 256), generator=g, device=dev).float()
    wo = (torch.randn(256, 256, generator=g, device=dev) * 4).round().clamp(-16, 16) / 64
    we = torch.randn(512, 256, generator=g, device=dev) / 16
    ws = torch.randn(256, 512, generator=g, device=dev) / 22
    bo, be, bs = (torch.randn(n, generator=g, device=dev) * 0.1 for n in (256, 512, 256))
    if kind == "flat":
        bo = torch.zeros(256, device=dev)
    g1, g2 = (1 + 0.1 * torch.randn(256, generator=g, device=dev) for _ in range(2))
    b1, b2 = (0.1 * torch.randn(256, generator=g, device=dev) for _ in range(2))
    bf = torch.bfloat16
    return dict(hid=hid.to(bf), x=x.to(bf), wo=wo.to(bf), bo=bo, g1=g1, b1=b1, we=we.to(bf), be=be, ws=ws.to(bf), bs=bs, g2=g2, b2=b2)


def _tail_ref(t, eps, drop_bs=False):
    """float64 layer tail on the kernel's operands, y and h rounded where the kernel rounds them -> (out, bound)"""
    d = {k: v.to(F64) for k, v in t.items()}
    # G1: exact (products on a 2^-8 grid, partial sums below 2^24 grid steps: _tail_inputs); E1: acc + (b_o + x), two roundings
    assert (d["hid"] * 4).frac().eq(0).all() and (d["wo"] * 64).frac().eq(0).all()
    assert (d["hid"].abs() @ d["wo"].abs().t()).max().item() * 2 ** 8 < 2 ** 24
    z1 = d["hid"] @ d["wo"].t() + d["bo"] + d["x"]
    e_z1 = U * (d["bo"] + d["x"]).abs() + U * z1.abs()
    y64, e_y = _ln_bound(z1, e_z1, d["g1"], d["b1"], eps)
    y = _bf(y64)                                                 # the bf16 y: A operand of G2 and residual of E3
    dy = _spread(y64, e_y)
    # G2: relu(y W_e^T + b_e), 256 products, bias one rounding; then the bf16 rounding of h
    pre = y @ d["we"].t() + d["be"]
    e_pre = dy @ d["we"].abs().t() + 512 * U * (y.abs() @ d["we"].abs().t()) + U * pre.abs()
    h64 = torch.relu(pre)
    h = _bf(h64)
    dh = _spread(h64, e_pre)                                     # relu is monotone: the spread of relu(pre +- e_pre)
    # G3 + E3: 512 products, acc + (b_s + y): two roundings; then LayerNorm 2 and one bf16 rounding of the output
    z2 = y + h @ d["ws"].t() + (0 if drop_bs else d["bs"])
    e_z2 = dy + dh @ d["ws"].abs().t() + 1024 * U * (h @ d["ws"].abs().t()) + U * (d["bs"] + y).abs() + U * z2.abs()
    out, e_out = _ln_bound(z2, e_z2, d["g2"], d["b2"], eps)
    return out, e_out + UB * (out.abs() + e_out)


_TAIL_CASES = [(1, "rand", 1e-5), (63, "rand", 1e-5), (64, "rand", 1e-5), (65, "rand", 1e-5), (127, "rand", 1e-5), (129, "rand", 1e-5),
               (12608, "rand", 1e-5), (131136, "rand", 1e-5), (1000, "offset", 1e-5), (1000, "flat", 1e-5), (1000, "flat", 1e-4),
               (300, "rand", 1e-3)]


@pytest.mark.parametrize("M,kind,eps", _TAIL_CASES)
def test_transformer_tail(ops, M, kind, eps):
    """sam6d_transformer_tail_bf16.  M = 1..129: partial 128-row tiles, one warpgroup without rows (M <= 64); 12608 = 32 x 2 x 197
    (the sparse stream of a bench step), 131136 = 32 x 2 x 2049 (the dense stream: several tiles per CTA).  `offset` rows carry a
    common offset of 50 (LayerNorm 1 cancellation), `flat` rows have a variance below eps (eps dominates rstd).  out is the head
    of a larger allocation: the sentinel rows past M must stay unwritten."""
    t = _tail_inputs(M, kind, seed=M + len(kind) + int(1e6 * eps))
    buf = torch.full((M + 5, 256), 7.0, dtype=torch.bfloat16, device="cuda")
    ops.transformer_tail_bf16(t["hid"], t["x"], t["wo"], t["bo"], t["g1"], t["b1"], t["we"], t["be"], t["ws"], t["bs"], t["g2"], t["b2"],
                              out=buf[:M], eps=eps)
    got = buf[:M].to(F64)
    assert (buf[M:] == 7.0).all(), "rows past M were written"
    ref, bound = _tail_ref(t, eps)
    _check(f"transformer_tail M={M} {kind} eps={eps:g}", (got - ref).abs(), bound)
    if kind == "flat":
        # negative control: the same LayerNorms with eps / 10 (a wrong eps only shows where the variance is below it)
        wrong, _ = _tail_ref(t, eps / 10)
        r = _ratio((got - wrong).abs(), bound)
        print(f"  eps / 10: ratio {r:.3g}")
        assert r > 1.0
    if M in (129, 12608):
        # negative control: b_s dropped
        wrong, _ = _tail_ref(t, eps, drop_bs=True)
        assert _ratio((got - wrong).abs(), bound) > 1.0


# ================================================================================================== 2. fine assignment (fine_tc.cu)
LOG2E32 = float(np.float32(1.4426950408889634))


def _fine_tokens(B, S, seed, twins, bg_rows, all_bg_cloud):
    """normalised bf16 tokens: F2 = a noisy permutation of F1 (every row has a clear best column), planted exact column twins
    (identical tokens at j < j'), rows whose best match is the background column 0, and optionally a last cloud whose every
    column matches scene row 0 best (so every column label is background)"""
    g = _gc(seed)
    F1 = torch.nn.functional.normalize(torch.randn(B, S, 256, generator=g, device="cuda", dtype=F64), dim=-1)
    perm = torch.randperm(S, generator=torch.Generator().manual_seed(seed)).cuda()
    F2 = torch.nn.functional.normalize(F1[:, perm] + 0.3 * torch.randn(B, S, 256, generator=g, device="cuda", dtype=F64) / 16, dim=-1)
    if all_bg_cloud:
        F2[-1] = torch.nn.functional.normalize(F1[-1, 0] + 0.2 * torch.randn(S, 256, generator=g, device="cuda", dtype=F64) / 16, dim=-1)
    for j, j2 in twins:
        F2[:, j2] = F2[:, j]
    nb = B - 1 if all_bg_cloud else B
    for i in bg_rows:
        F1[:nb, i] = F2[:nb, 0]
    return F1.to(torch.bfloat16).contiguous(), F2.to(torch.bfloat16).contiguous()


def _fine_e(Fa, Fb, alpha):
    """float64 e = exp(alpha s - alpha) of the bf16 tokens + its relative error bound eta in the kernel (wgmma score, ex2)"""
    a, b = Fa.to(F64), Fb.to(F64)
    s = a @ b.transpose(1, 2)
    e_acc = 512 * U * (a.abs() @ b.abs().transpose(1, 2))            # 256 products on the tensor cores
    a2 = alpha * LOG2E32
    # ex2 argument fma(acc, a2, -s2) in log2 units: acc error times a2; a2 = fl(alpha * fl(log2 e)) and s2 likewise carry
    # 1.5u each; the fma rounds once
    e_arg = a2 * e_acc + 1.5 * U * a2 * (s.abs() + 1) + U * a2 * (s - 1).abs()
    eta = math.log(2.0) * e_arg * 1.001 + 4 * U                      # ex2.approx: 2 ulp
    return torch.exp(alpha * (s - 1)), eta


def _first_argmax_with_gap(P, eps_rel, cls):
    """first arg-max of every row of P (float64) and whether the kernel's label is determined: the best value beats every
    column that is not a twin of it by more than the relative error bound of both"""
    a1 = P.argmax(-1)
    P1 = P.gather(-1, a1[..., None])
    same = cls[None, None, :] == cls[a1][..., None]
    P2 = torch.where(same, torch.full_like(P, -1.0), P).amax(-1, keepdim=True)
    er = eps_rel.amax(-1, keepdim=True)
    ok = (P1 * (1 - er) > P2 * (1 + er)).squeeze(-1)
    return a1, ok


@pytest.mark.parametrize("B,S", [(2, 65), (2, 128), (3, 129), (2, 197), (2, 257), (2, 2049), (32, 2049)])
def test_fine_assignment_passes(lib, B, S):
    """the passes of ops.fine_assign_tc one by one: ROWSUM (F1, F2), ROWSUM (F2, F1), ARGMAX (F2, F1) -> column labels, the
    masked points, ASSIGN (F1, F2) -> row labels, weights and weighted correspondences.  B = 32, S = 2049 is the bench shape."""
    alpha = 10.0                                                      # 1 / temp of SAM-6D's fine stage
    twins = [(5, 6), (9, 11), (20, 33)] + ([(40, 40 + 256)] if S > 300 else [])
    bg_rows = [3, S - 2]
    F1, F2 = _fine_tokens(B, S, 100 + S + B, twins, bg_rows, all_bg_cloud=True)
    g = _g(200 + S)
    pts2 = torch.randn(B, S - 1, 3, generator=g).cuda()
    ld = (S + 3) // 4 * 4
    dev = "cuda"
    a, sh = alpha, alpha
    rinv = torch.full((B, ld), float("nan"), device=dev)
    cinv = torch.full((B, ld), float("nan"), device=dev)
    lib.call("sam6d_fine_pass_tc", F1, F2, B, S, a, sh, 0, None, None, ld, None, rinv, None, None, None)
    lib.call("sam6d_fine_pass_tc", F2, F1, B, S, a, sh, 0, None, None, ld, None, cinv, None, None, None)

    # ---- ROWSUM: inv_i = 1 / sum_j e_ij.  Per row 64 columns of every 256-column tile in one thread's chain, then 2 quad levels
    e, eta = _fine_e(F1, F2, alpha)
    n_chain = 64 * ((S + 255) // 256) + 2
    for name, ee, et, inv in (("rows", e, eta, rinv), ("cols", e.transpose(1, 2), eta.transpose(1, 2), cinv)):
        tot = ee.sum(-1)
        rho = (ee * et).sum(-1) / tot + n_chain * U
        ref = 1.0 / tot
        bound = ref * (1.01 * rho + U)                                # + the IEEE reciprocal
        got = inv[:, :S].to(F64)
        _check(f"fine ROWSUM {name} B={B} S={S}", (got - ref).abs(), bound)
        # negative control: the last column left out of the sum
        assert _ratio((got - 1.0 / ee[..., :S - 1].sum(-1)).abs(), bound) > 1.0
    del eta

    # ties: identical tokens, and identical factors, so the kernel computes bit-identical products for the twins
    rf, cf = rinv.clone(), cinv.clone()
    for j, j2 in twins:
        cf[:, j2] = cf[:, j]
    cls = torch.arange(S, device=dev)
    for j, j2 in twins:
        cls[j2] = j

    # ---- ARGMAX (F2, F1): column labels.  P = (e rf) (e cf): two ex2 errors, three roundings
    lab2 = torch.full((B, S), -7, dtype=torch.int32, device=dev)
    lib.call("sam6d_fine_pass_tc", F2, F1, B, S, a, sh, 1, cf, rf, ld, None, None, lab2, None, None)
    eT, etaT = _fine_e(F2, F1, alpha)
    P2 = eT * eT * cf[:, :S, None].to(F64) * rf[:, None, :S].to(F64)
    a2, ok2 = _first_argmax_with_gap(P2, 2 * etaT + 3 * U, torch.arange(S, device=dev))
    del eT, etaT, P2
    frac = ok2[:-1].double().mean().item()
    print(f"fine ARGMAX cols B={B} S={S}: {frac:.4f} of the labels (all clouds but the all-background one) are determined")
    assert frac > 0.9 and ok2[-1].all()
    assert torch.equal(lab2[ok2].long(), a2[ok2]), "column label differs from the float64 first arg-max where it is determined"
    assert (lab2[-1] == 0).all(), "the all-background cloud must label every column 0"

    # ---- masked points: q4[b,j] = (pts2[b,j-1], 1) where column j >= 1 carries a non-background label, else 0 (also j >= S)
    q4 = torch.full((B, ld, 4), float("nan"), device=dev)
    lib.call("sam6d_fine_masked_points", lab2, pts2, B, S, ld, q4)
    want = torch.zeros(B, ld, 4, device=dev)
    keep = (lab2[:, 1:] > 0)[..., None]
    want[:, 1:S, :3] = torch.where(keep, pts2, torch.zeros_like(pts2))
    want[:, 1:S, 3:] = keep.float()
    assert torch.equal(q4, want)

    # ---- ASSIGN (F1, F2): row labels, w_i = sum_j P_ij q4_j.w, pred_i = sum_j P_ij q4_j.xyz / (w_i + 1e-6), rows i >= 1
    lab1 = torch.full((B, S), -7, dtype=torch.int32, device=dev)
    wts = torch.full((B, S - 1), float("nan"), device=dev)
    pred = torch.full((B, S - 1, 3), float("nan"), device=dev)
    lib.call("sam6d_fine_pass_tc", F1, F2, B, S, a, sh, 2, rf, cf, ld, q4, None, lab1, wts, pred)
    e, eta = _fine_e(F1, F2, alpha)
    P = e * e * rf[:, :S, None].to(F64) * cf[:, None, :S].to(F64)
    del e
    eps_p = 2 * eta + 3 * U
    del eta
    a1, ok1 = _first_argmax_with_gap(P, eps_p, cls)
    frac = ok1[:-1].double().mean().item()
    print(f"fine ASSIGN rows B={B} S={S}: {frac:.4f} of the labels (all clouds but the all-background one) are determined")
    assert frac > 0.9
    assert torch.equal(lab1[ok1].long(), a1[ok1]), "row label differs from the float64 first arg-max where it is determined"
    for i in bg_rows:
        assert ok1[:-1, i].all() and (lab1[:-1, i] == 0).all(), "a row matching the background column best must get label 0"
    # planted ties: the first maximum wins, and the rows that decide it exist
    tie_rows = 0
    for j, j2 in twins:
        rows = ok1 & (a1 == j)
        tie_rows += rows.sum().item()
        assert (lab1[rows] == j).all()
    assert tie_rows >= len(twins)
    # weights and points, rows 1.. (q4.w in {0, 1}: the products p q.w are exact).  One chain per thread as in ROWSUM, the
    # point sums one more rounding (fma); d = w + 1e-6f one rounding, the division IEEE
    q = q4[:, :S].to(F64)
    Pr = P[:, 1:]
    w_ref = Pr @ q[..., 3:]
    n_ref = Pr @ q[..., :3]
    rel = eps_p[:, 1:] + n_chain * U
    e_w = (Pr * rel) @ q[..., 3:]
    e_n = (Pr * (rel + U)) @ q[..., :3].abs()
    den = w_ref + EPS6
    pred_ref = n_ref / den
    e_pred = (e_n + pred_ref.abs() * (e_w + U * den)) / den * 1.001 + U * pred_ref.abs()
    lab = lab1[:, 1:]
    bgl = lab == 0
    assert (wts[bgl] == 0).all() and (pred[bgl] == 0).all(), "a background-labelled row must carry no weight and no point"
    fg = ~bgl
    _check(f"fine ASSIGN w B={B} S={S}", (wts.to(F64) - w_ref.squeeze(-1))[fg].abs(), e_w.squeeze(-1)[fg])
    _check(f"fine ASSIGN pred B={B} S={S}", (pred.to(F64) - pred_ref)[fg].abs(), e_pred[fg])
    # the all-background cloud: no column keeps a point, so every row has w = 0 and pred = 0 / (0 + 1e-6) = 0
    assert (wts[-1] == 0).all() and (pred[-1] == 0).all()
    # negative control: the background rows would fail if they kept their weight
    bgw = w_ref.squeeze(-1)[:-1, [i - 1 for i in bg_rows]]
    assert (bgw > e_w.squeeze(-1)[:-1, [i - 1 for i in bg_rows]]).any()


# ================================================================================================== 3. PE MLP (pe_tc.cu)
def _pe_weights(seed):
    g = _gc(seed)
    dev = "cuda"
    W1 = torch.randn(32, 6, generator=g, device=dev) * 0.8
    B1 = torch.randn(32, generator=g, device=dev) * 0.1
    W2 = (torch.randn(64, 32, generator=g, device=dev) * 0.3).bfloat16()
    B2 = torch.randn(64, generator=g, device=dev) * 0.1
    W3 = (torch.randn(128, 64, generator=g, device=dev) * 0.2).bfloat16()
    B3 = torch.randn(128, generator=g, device=dev) * 0.2
    return W1, B1, W2, B2, W3, B3


def _pe_ref(pts, idx, w, drop_b3=False):
    """float64 shared MLP + max-pool over every (point, sample) pair -> (out (B,N,128), fp32 bound before the output rounding)"""
    W1, B1, W2, B2, W3, B3 = (t.to(F64) for t in w)
    p = pts.to(F64)
    B, N, ns = idx.shape
    pj = torch.gather(p, 1, idx.long().reshape(B, N * ns, 1).expand(B, N * ns, 3)).view(B, N, ns, 3)
    dlt = pj - p[:, :, None]
    x = torch.cat([dlt, pj], dim=-1)
    # layer 1 on the CUDA cores: p_j - p_i one rounding; b1 + six fmas (gamma_6 of the magnitudes)
    pre1 = x @ W1.t() + B1
    e1 = (U * dlt.abs()) @ W1[:, :3].abs().t() + 6 * U * (x.abs() @ W1.abs().t() + B1.abs())
    h1_64 = torch.relu(pre1)
    h1 = _bf(h1_64)
    d1 = _spread(h1_64, e1)
    # layer 2: 32 bf16 products on the tensor cores, + b2 one rounding, relu, bf16
    pre2 = h1 @ W2.t() + B2
    e2 = d1 @ W2.abs().t() + 64 * U * (h1 @ W2.abs().t()) + U * pre2.abs()
    h2_64 = torch.relu(pre2)
    h2 = _bf(h2_64)
    d2 = _spread(h2_64, e2)
    # layer 3: 64 products; the max over the group moves by at most the largest per-sample error; + b3 one rounding; relu
    pre3 = h2 @ W3.t()
    e3 = d2 @ W3.abs().t() + 128 * U * (h2 @ W3.abs().t())
    m = pre3.amax(2) + (0 if drop_b3 else B3)
    out = torch.relu(m)
    return out, e3.amax(2) + U * m.abs()


def _run_pe(lib, pts, idx, w, out, off):
    B, N, _ = pts.shape
    W1, B1, W2, B2, W3, B3 = w
    lib.call("sam6d_pe_mlp_max_tc", pts, idx, B, N, idx.shape[2], W1, B1, W2, B2, W3, B3, out, int(out.dtype == torch.bfloat16),
             out.shape[-1], off)


def _pe_check(lib, name, pts, idx, w, odt, off):
    B, N, _ = pts.shape
    out = torch.full((B, N, 256), 7.0, dtype=odt, device="cuda")
    _run_pe(lib, pts, idx, w, out, off)
    ref, e = _pe_ref(pts, idx, w)
    bound = e + (UB * (ref.abs() + e) if odt == torch.bfloat16 else 0)
    got = out[..., off:off + 128].to(F64)
    _check(f"pe_mlp_max_tc {name} {str(odt)[6:]} off={off}", (got - ref).abs(), bound)
    other = torch.ones(256, dtype=torch.bool, device="cuda")
    other[off:off + 128] = False
    assert (out[..., other] == 7.0).all(), "columns outside [out_off, out_off + 128) were written"
    return got, bound


@pytest.mark.parametrize("odt", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("N", [2048, 1023])
@pytest.mark.parametrize("ns", [32, 64])
def test_pe_mlp_max_ball_query(ops, lib, ns, N, odt):
    """both instantiations (ns 32: 4 points per 128-row tile; ns 64: 2) on the real ball_query_pair indices; B N = 3 x 1023 is
    not a multiple of either.  ns 64 writes columns [128, 256) of the 256-wide feature row (as the model does), ns 32 columns
    [0, 128); the other half holds a sentinel."""
    B = 3
    g = _gc(300 + N)
    pts = (torch.randn(B, N, 3, generator=g, device="cuda") * 0.3).contiguous()
    ia, _, ib, _ = ops.ball_query_pair(pts, pts, 0.1, 32, 0.2, 64)
    idx = ia if ns == 32 else ib
    w = _pe_weights(310 + ns)
    off = 0 if ns == 32 else 128
    got, bound = _pe_check(lib, f"ball query ns={ns} N={N}", pts, idx, w, odt, off)
    # negative control: b3 left out
    wrong, _ = _pe_ref(pts, idx, w, drop_b3=True)
    assert _ratio((got - wrong).abs(), bound) > 1.0


@pytest.mark.parametrize("ns", [32, 64])
def test_pe_mlp_max_padding_and_duplicates(lib, ns):
    """hand-built groups: empty balls (every index 0), heavy first-hit padding (one neighbour repeated over the group), and
    duplicate points (a small mask sampled with replacement)"""
    B, N = 2, 517
    g = _gc(400 + ns)
    base = torch.randn(B, 40, 3, generator=g, device="cuda") * 0.3
    pick = torch.randint(0, 40, (B, N), generator=g, device="cuda")
    pts = torch.gather(base, 1, pick[..., None].expand(B, N, 3)).contiguous()      # duplicates
    idx = torch.randint(0, N, (B, N, ns), generator=g, device="cuda", dtype=torch.int32)
    idx[:, ::7] = 0                                                                  # empty balls
    first = idx[:, 1::5, :1].clone()
    idx[:, 1::5, 3:] = first                                                         # first hit repeated over the group
    idx = idx.contiguous()
    w = _pe_weights(410 + ns)
    _pe_check(lib, f"padding/duplicates ns={ns}", pts, idx, w, torch.bfloat16, 128)
    _pe_check(lib, f"padding/duplicates ns={ns}", pts, idx, w, torch.float32, 0)


# ================================================================================================== 4. linear attention (linattn_tc.cu)
def _blob_index():
    """element index of KV_h^T[e][d] inside one 64 x 64 SWIZZLE_128B slab (row e = 128 bytes, 16-byte chunks XOR (e & 7))"""
    e = torch.arange(64)[:, None]
    d = torch.arange(64)[None, :]
    off = e * 128 + ((((d >> 3) ^ (e & 7)) << 4) | ((d & 7) << 1))
    return (off // 2).reshape(-1)


def _focus64(x, sp):
    t = (torch.relu(x) + EPS6) / sp
    n = t.norm(dim=-1, keepdim=True)
    t3 = t ** 3
    return t3 / t3.norm(dim=-1, keepdim=True) * n


@pytest.mark.parametrize("N", [1, 129, 2048])
@pytest.mark.parametrize("J", [1, 7, 197])
def test_linear_attention(lib, J, N):
    """sam6d_linattn_kv_pack (KV image and ksum of the focused keys) and sam6d_linattn_tc (feature map of the bf16 queries,
    per-head (q' KV) / (q' . ksum + 1e-6)) for B = 64 clouds.  Every 5th query row is all negative: its feature map is
    q = 1e-6 / softplus, and the normaliser's + 1e-6 is no longer negligible.  Row 0 of every cloud is outside the view."""
    B, C = 64, 256
    g = _gc(500 + J * 10 + N)
    dev = "cuda"
    sp = torch.rand(C, generator=g, device=dev) + 0.5
    k = torch.randn(B, J, C, generator=g, device=dev)
    Kf = _focus64(k.to(F64), sp.to(F64)).float().contiguous()
    V = torch.randn(B, J, C, generator=g, device=dev)
    blob = torch.empty(B, 4 * 64 * 64, dtype=torch.bfloat16, device=dev)
    KS = torch.empty(B, 4, 64, device=dev)
    lib.call("sam6d_linattn_kv_pack", Kf, C, J * C, V, C, J * C, B, J, blob, KS)
    kh = Kf.to(F64).view(B, J, 4, 64)
    vh = V.to(F64).view(B, J, 4, 64)
    # ksum: one fp32 chain of J terms
    ks_ref = kh.sum(1)
    _check(f"linattn ksum J={J}", (KS.to(F64) - ks_ref).abs(), J * U * kh.abs().sum(1))
    # KV_h[d][e]: one fp32 fma chain of J terms, then one bf16 rounding
    kv_ref = torch.einsum("bjhd,bjhe->bhde", kh, vh)
    e_kv = J * U * torch.einsum("bjhd,bjhe->bhde", kh.abs(), vh.abs())
    KVimg = blob.view(B, 4, 4096)[..., _blob_index().to(dev)].view(B, 4, 64, 64).transpose(-1, -2).to(F64)   # -> [d][e]
    _check(f"linattn KV image J={J}", (KVimg - kv_ref).abs(), e_kv + UB * (kv_ref.abs() + e_kv))
    # ---- dense side: (B, N + 1, C) rows, row 0 outside the view
    q = torch.randn(B, N + 1, C, generator=g, device=dev)
    q[:, 1::5] = -q[:, 1::5].abs() - 0.01
    q = q.bfloat16()
    x = torch.full((B, N + 1, C), 7.0, dtype=torch.bfloat16, device=dev)
    lib.call("sam6d_linattn_tc", q[:, 1:], C, (N + 1) * C, blob, KS, sp, B, N, x[:, 1:], C, (N + 1) * C)
    assert (x[:, 0] == 7.0).all(), "a row outside the view was written"
    qf = _focus64(q[:, 1:].to(F64), sp.to(F64))
    # feature map in fp32: t = (q+ + 1e-6) / s (3u), sums of t^2 and t^6 (8-term chains + a 5-level warp tree: gamma_13),
    # t^3 (two roundings), n = sqrtf * rsqrtf (1u + 2 ulp + 1u), q' = t^3 n (1u): <= 50u relative
    e_q = 50 * U * qf
    qr = _bf(qf)
    dq = _spread(qf, e_q)
    qh, qrh, dqh = (t.view(B, N, 4, 64) for t in (qf, qr, dq))
    KVb = KVimg                                                  # the kernel's bf16 KV, as it reads it
    KSk = KS.to(F64)
    num = torch.einsum("bnhd,bhde->bnhe", qrh, KVb)
    e_num = torch.einsum("bnhd,bhde->bnhe", dqh, KVb.abs()) + 128 * U * torch.einsum("bnhd,bhde->bnhe", qrh, KVb.abs())

    def den_of(plus):
        return torch.einsum("bnhd,bhd->bnh", qh, KSk) + plus

    den = den_of(EPS6)
    # q' . ksum: 8-term fma chains + 3 shuffle sums (gamma_11), + 1e-6 one rounding; 1 / den one rounding, x = acc z one rounding
    e_den = torch.einsum("bnhd,bhd->bnh", e_q.view(B, N, 4, 64) + 11 * U * qh, KSk.abs()) + U * den
    ref = num / den[..., None]
    e_x = (e_num + ref.abs() * e_den[..., None]) / den[..., None] * 1.001 + 2 * U * ref.abs()
    bound = e_x + UB * (ref.abs() + e_x)
    got = x[:, 1:].to(F64).view(B, N, 4, 64)
    _check(f"linattn_tc J={J} N={N}", (got - ref).abs(), bound)
    if J == 1 and N > 1:
        # negative control: the normaliser without its + 1e-6 (visible on the all-negative rows)
        wrong = num / den_of(0.0)[..., None]
        r = _ratio((got - wrong).abs(), bound)
        print(f"  without + 1e-6: ratio {r:.3g}")
        assert r > 1.0


# ================================================================================================== 5. geometric embedding (geo_lut.cu)
def _geo_module(seed):
    from sam6d_b200 import pem
    torch.manual_seed(seed)
    geo = pem.GeometricStructureEmbedding(pem.DEFAULT_MODEL_CFG["geo_embedding"]).cuda()
    with torch.no_grad():
        geo.proj_a.bias.normal_(0, 0.1)
        geo.proj_d.bias.normal_(0, 0.1)
    geo.precision = "bf16"
    return geo, geo._weights(), pem.GEO_LUT_INV_H


def _emb(x, div):
    om = x[..., None] * div
    return torch.stack([torch.sin(om), torch.cos(om)], dim=-1).flatten(-2)       # interleaved (sin, cos) per frequency


def _lut_bound(x, tab, inv_h, g2):
    """bound on |fp32 interpolation of the bf16 table - g(x)| for table positions x (..., ) -> (..., 256)"""
    n = tab.shape[0]
    u = x * inv_h                                                               # inv_h = 8: exact
    i = u.floor().clamp(0, n - 2).long()
    lo, hi = tab.to(F64)[i], tab.to(F64)[i + 1]
    h = 1.0 / inv_h
    # interpolation error h^2 / 8 max|g''|; the table's bf16 rounding (from fp32: ub + u of the entry, interpolation takes the
    # larger); the fma t (hi - lo) + lo: two roundings
    return (h * h / 8) * g2 + (UB + U) * torch.maximum(lo.abs(), hi.abs()) + U * ((hi - lo).abs() + torch.maximum(lo.abs(), hi.abs()))


def _geo_ref(T, w, inv_h, far):
    """float64 E = g_d(d) + max_k g_a(a_k) at the given indices, g = W emb(x) (+ b_a + b_d) from the fp32 weights, with the kernel's
    three routes: table pairs, row 0 / column 0 through `far`, other out-of-table distances through the exact fp32 path
    -> (ref, bound, lerp-free wrong answer of the table pairs)"""
    div = w["div"].to(F64)
    Wa, Wd = w["waT"].to(F64).t(), w["wdT"].to(F64).t()
    bias = w["bias"].to(F64)
    # max |g''| per output channel: sum_k div_k^2 |(W[c, 2k], W[c, 2k + 1])|
    d2 = div ** 2
    g2a = (d2 * torch.hypot(Wa[:, 0::2], Wa[:, 1::2])).sum(1)
    g2d = (d2 * torch.hypot(Wd[:, 0::2], Wd[:, 1::2])).sum(1)
    Td = T.to(F64)
    ga = _emb(Td[..., :3], div) @ Wa.t()                                      # (C,S,S,3,256)
    ea = _lut_bound(Td[..., :3], w["tab_a"], inv_h, g2a)
    amax = ga.amax(-2)
    e_amax = ea.amax(-2)
    gd = _emb(Td[..., 3], div) @ Wd.t() + bias
    ed = _lut_bound(Td[..., 3], w["tab_d"], inv_h, g2d)
    nd = w["tab_d"].shape[0]
    in_tab = Td[..., 3] < (nd - 1) / inv_h
    C, S = T.shape[0], T.shape[1]
    row0 = torch.zeros(C, S, S, dtype=torch.bool, device=T.device)
    row0[:, 0, :] = True
    col0 = torch.zeros_like(row0)
    col0[:, 1:, 0] = True
    slow = ~in_tab & ~row0 & ~col0
    # far pairs: the kernel's bf16 far value is the g_d term (far itself is checked against float64 in its own test)
    fd = torch.zeros_like(gd)
    farv = far.to(F64)
    fd[row0] = farv[:, 0][:, None].expand(C, S, S, 256)[row0]
    fd[col0] = farv[:, 1][:, :, None].expand(C, S, S, 256)[col0]
    use_far = (~in_tab) & (row0 | col0)
    gd = torch.where(use_far[..., None], fd, gd)
    ed = torch.where(use_far[..., None], torch.zeros_like(ed), ed)
    # slow pairs: sincosf 2 ulp (<= 2^-22) of the fp32 product x div (one rounding: u |x div|); b + 256 fmas with the bf16
    # W_d^T (gamma_256 of the magnitudes).  The reference uses the bf16 W_d the kernel reads.
    Wdb = w["wdT_bf"].to(F64).t()
    xs = Td[..., 3][slow]
    es = _emb(xs, div)
    gd_s = es @ Wdb.t() + bias
    e_emb = 2.0 ** -22 + U * (xs[:, None] * div).abs()
    e_emb = torch.stack([e_emb, e_emb], dim=-1).flatten(-2)
    e_s = e_emb @ Wdb.abs().t() + 256 * U * (es.abs() @ Wdb.abs().t() + bias.abs())
    e_s = e_s + UB * (gd_s.abs() + e_s)                          # the exact path returns g_d rounded to bf16, then adds the max
    gd[slow] = gd_s
    ed[slow] = e_s
    ref = gd + amax
    # fd + max: one rounding; then one bf16 rounding of E
    e = ed + e_amax + U * ref.abs()
    bound = e + UB * (ref.abs() + e)
    # lerp-free wrong answer: every table lookup reads the lower row only
    lo_a = w["tab_a"].to(F64)[(Td[..., :3] * inv_h).floor().clamp(0, w["tab_a"].shape[0] - 2).long()].amax(-2)
    lo_d = w["tab_d"].to(F64)[(Td[..., 3] * inv_h).floor().clamp(0, nd - 2).long()]
    wrong = torch.where(in_tab[..., None], lo_d, gd) + lo_a
    return ref, bound, wrong, in_tab, use_far, slow


def _geo_T(C, S, seed, d_lim):
    g = _gc(seed)
    dev = "cuda"
    T = torch.empty(C, S, S, 4, device=dev)
    T[..., :3] = torch.rand(C, S, S, 3, generator=g, device=dev) * 12.0
    T[..., 3] = torch.rand(C, S, S, generator=g, device=dev) * d_lim
    flat = torch.arange(S * S, device=dev).view(S, S)
    inner = torch.zeros(S, S, dtype=torch.bool, device=dev)
    inner[1:, 1:] = True
    # edges: angle index exactly 0 and exactly 180 / sigma_a = 12 (the last table row)
    T[:, inner & (flat % 11 == 0), 0] = 0.0
    T[:, inner & (flat % 13 == 1), 1] = 12.0
    T[:, 2, 3, :3] = 12.0
    T[:, 3, 2, :3] = 0.0
    # distance index just below and exactly at the table limit (nd - 1) / inv_hd
    below = float(np.nextafter(np.float32(d_lim), np.float32(0)))
    T[:, inner & (flat % 17 == 5), 3] = below
    T[:, 4, 5, 3] = below
    T[:, 5, 4, 3] = d_lim                                                    # -> the exact path
    # other out-of-table pairs (exact path)
    T[:, 6, 7, 3] = 33.5
    T[:, 6, 8, 3] = 40.0
    # row 0 and column 0 out of the table (the background point), deliberately not symmetric
    T[:, 0, 1:, 3] = 33.0 + 7.0 * torch.rand(C, S - 1, generator=g, device=dev)
    T[:, 1:, 0, 3] = 36.0 + 5.0 * torch.rand(C, S - 1, generator=g, device=dev)
    T[:, 0, 0, 3] = 0.0
    return T.contiguous()


@pytest.mark.parametrize("C,S", [(3, 33), (2, 197)])
def test_geo_embed_lut(ops, C, S):
    """sam6d_geo_embed_lut on index tensors built by hand (so knn ties do not enter) with `far` from sam6d_geo_embed_dist_tc:
    angle indices exactly 0 and 12, distances just below and exactly at the table limit, row 0 / column 0 through `far`, other
    out-of-table pairs through the exact path.  C S^2 = 3267 and 77618 are not multiples of the 32 pairs of a warp."""
    geo, w, inv_h = _geo_module(600 + S)
    nd = w["tab_d"].shape[0]
    d_lim = (nd - 1) / inv_h
    T = _geo_T(C, S, 610 + S, d_lim)
    far = ops.geo_embed_dist_tc(torch.stack([T[:, 0], T[:, :, 0]], dim=1).contiguous(), w["div"], w["wd_bf"], w["bias"])
    _check_far(T, far, w, f"geo_embed_dist_tc (far) C={C} S={S}")
    E = ops.geo_embed_lut(T, w["tab_a"], inv_h, w["tab_d"], inv_h, far, w["div"], w["wdT_bf"], w["bias"]).to(F64)
    ref, bound, wrong, in_tab, use_far, slow = _geo_ref(T, w, inv_h, far)
    assert use_far.any() and slow.any() and in_tab.any()
    print(f"geo lut C={C} S={S}: {in_tab.sum().item()} table pairs, {use_far.sum().item()} far pairs, {slow.sum().item()} exact-path pairs")
    for name, m in (("table", in_tab), ("far", use_far), ("exact path", slow)):
        _check(f"geo_embed_lut {name} C={C} S={S}", (E - ref)[m].abs(), bound[m])
    # negative controls: no interpolation (the lower table row only); the far row / column slots exchanged
    assert _ratio((E - wrong)[in_tab].abs(), bound[in_tab]) > 1.0
    swapped = ref.clone()
    row0 = use_far.clone()
    row0[:, 1:] = False
    swapped[row0] = ref[row0] - far.to(F64)[:, 0][:, None].expand(C, S, S, 256)[row0] + far.to(F64)[:, 1][:, None].expand(C, S, S, 256)[row0]
    assert _ratio((E - swapped)[row0].abs(), bound[row0]) > 1.0


def _check_far(T, far, w, name):
    """far = bf16(W_d(bf16) bf16(emb(x)) + b): __sincosf of the fp32 product x div (documented 2^-21.41 absolute in [-pi, pi];
    beyond, the argument reduction in fp32 adds about u |x div|, charged twice) rounded to bf16 (spread), 256 products on the
    tensor cores, + bias one rounding, one bf16 rounding"""
    div = w["div"].to(F64)
    Wdb = w["wd_bf"].to(F64)
    bias = w["bias"].to(F64)
    x = torch.stack([T[:, 0, :, 3], T[:, :, 0, 3]], dim=1).to(F64)
    em = _emb(x, div)
    om = (x[..., None] * div).abs()
    e_em = 2.0 ** -21.41 + 3 * U * om
    e_em = torch.stack([e_em, e_em], dim=-1).flatten(-2)
    emr = _bf(em)
    dem = _spread(em, e_em)
    ref = emr @ Wdb.t() + bias
    e = dem @ Wdb.abs().t() + 512 * U * (emr.abs() @ Wdb.abs().t()) + U * ref.abs()
    _check(name, (far.to(F64) - ref).abs(), e + UB * (ref.abs() + e))


def test_geo_embed_lut_coincident_points(ops):
    """sparse points with repeats (FPS on a tiny cloud returns them) through geo_indices -> dist_tc -> lut: finite and within
    the bound at the indices geo_indices produced"""
    from oracle import pem_oracle as po
    geo, w, inv_h = _geo_module(700)
    C, S = 2, 24
    g = _gc(701)
    base = torch.randn(C, 6, 3, generator=g, device="cuda") * 0.2
    pick = torch.randint(0, 6, (C, S), generator=g, device="cuda")
    pts = torch.gather(base, 1, pick[..., None].expand(C, S, 3)).contiguous()
    T = ops.geo_indices(pts, po.SIGMA_D, 180.0 / (po.SIGMA_A * math.pi))
    assert torch.isfinite(T).all()
    far = ops.geo_embed_dist_tc(torch.stack([T[:, 0], T[:, :, 0]], dim=1).contiguous(), w["div"], w["wd_bf"], w["bias"])
    E = ops.geo_embed_lut(T, w["tab_a"], inv_h, w["tab_d"], inv_h, far, w["div"], w["wdT_bf"], w["bias"]).to(F64)
    assert torch.isfinite(E).all()
    ref, bound, _, _, _, _ = _geo_ref(T, w, inv_h, far)
    _check("geo_embed_lut coincident points", (E - ref).abs(), bound)


# ================================================================================================== 6. RPE self-attention
@pytest.mark.parametrize("B,S", [(64, 197), (3, 65), (3, 130)])
def test_rpe_self_attention(ops, B, S):
    """the bf16 self-attention of the PEM as Transformer._self_bf16 runs it: gemm_tma_vt2 (q | k rows, V^T, the folded
    rel-pos queries u) -> rpe_scores_tc_padded (u . E score planes) -> attn_tc_padded_bias.  B = 64, S = 197 is the bench
    launch.  Each stage against float64 on the previous stage's bf16 / fp32 outputs."""
    H, D, C = 4, 64, 256
    g = _gc(800 + S)
    dev = "cuda"
    x = torch.randn(B * S, C, generator=g, device=dev).bfloat16()
    W = (torch.randn(7 * C, C, generator=g, device=dev) / 16).bfloat16()
    bw = torch.randn(7 * C, generator=g, device=dev) * 0.1
    E = (torch.randn(B, S, S, C, generator=g, device=dev) * 0.7).bfloat16()
    qk, vt, u = ops.gemm_tma_vt2(x, W, bw, 2 * C, 3 * C, S)
    # ---- projection: 256 products on the tensor cores, + bias one rounding, one bf16 rounding
    R = x.to(F64) @ W.to(F64).t() + bw.to(F64)
    eR = 512 * U * (x.to(F64).abs() @ W.to(F64).abs().t()) + U * R.abs()
    bR = eR + UB * (R.abs() + eR)
    n1 = vt.shape[1]
    vt_got = vt[:B * C].view(B, C, n1)[:, :, :S].transpose(1, 2).reshape(B * S, C)
    _check(f"gemm_tma_vt2 q|k B={B} S={S}", (qk.to(F64) - R[:, :2 * C]).abs(), bR[:, :2 * C])
    _check(f"gemm_tma_vt2 V^T B={B} S={S}", (vt_got.to(F64) - R[:, 2 * C:3 * C]).abs(), bR[:, 2 * C:3 * C])
    _check(f"gemm_tma_vt2 u B={B} S={S}", (u.to(F64) - R[:, 3 * C:]).abs(), bR[:, 3 * C:])
    del R, eR, bR
    # ---- score planes: 256 bf16 products on the tensor cores
    sp = ops.rpe_scores_tc_padded(E, u)
    uh = u.to(F64).view(B, S, H, C)
    sp_ref = torch.empty(B, H, S, S, dtype=F64, device=dev)
    e_sp = torch.empty_like(sp_ref)
    for b0 in range(0, B, 4):
        Ed = E[b0:b0 + 4].to(F64)
        sp_ref[b0:b0 + 4] = torch.einsum("bnmc,bnhc->bhnm", Ed, uh[b0:b0 + 4])
        e_sp[b0:b0 + 4] = 512 * U * torch.einsum("bnmc,bnhc->bhnm", Ed.abs(), uh[b0:b0 + 4].abs())
        del Ed
    _check(f"rpe_scores_tc_padded B={B} S={S}", (sp[..., :S].to(F64) - sp_ref).abs(), e_sp)
    # ---- attention on the kernel's q, k, V^T and score planes: x = (q.k + s_p) / 8
    scale = 1.0 / math.sqrt(D)
    qh = qk[:, :C].to(F64).view(B, S, H, D).permute(0, 2, 1, 3)
    kh = qk[:, C:].to(F64).view(B, S, H, D).permute(0, 2, 1, 3)
    vh = vt_got.to(F64).view(B, S, H, D).permute(0, 2, 1, 3)
    spk = sp[..., :S].to(F64)

    def attn(bias):
        s = (qh @ kh.transpose(-1, -2) + bias) * scale
        p = torch.softmax(s, dim=-1)
        return s, p @ vh, p @ vh.abs()

    s, o, pv = attn(spk)
    # logits: 64 products on the tensor cores (2u each) + the plane value (one rounding), times 1/8 (exact); the row max carries
    # the same error
    dlog = ((128 * U * (qh.abs() @ kh.abs().transpose(-1, -2)) + U * (s.abs() / scale)) * scale).amax(-1)
    xr = s.amax(-1) - s.amin(-1)
    eta = 2 * dlog + _exp_err(xr)
    # P rounded to bf16 for the P V product (ub per weight), exp / logit error, the fp32 row sum (a chain of S/4 pair sums + 2
    # quad levels), the P V accumulation on the tensor cores (2u per key), 1 / sum and one product; then one bf16 rounding
    n_sum = (S + 3) // 4 + 3
    e32 = pv * (UB + 2 * eta + (2 * n_sum + 2 * S + 2) * U)[..., None]
    bound = e32 + UB * (o.abs() + e32)
    hid = ops.attn_tc_padded_bias(qk, 0, qk, C, vt, B, H, S, S, D, scale, sp)
    got = hid.to(F64).view(B, S, H, D).permute(0, 2, 1, 3)
    _check(f"attn_tc_padded_bias B={B} S={S}", (got - o).abs(), bound)
    # negative control: the plane value of the last key dropped
    spw = spk.clone()
    spw[..., S - 1] = 0.0
    _, ow, _ = attn(spw)
    assert _ratio((got - ow).abs(), bound) > 1.0
    # and the float64 score planes in place of the kernel's: within the planes' own bound (checked above) of the same answer
    _, o64, _ = attn(sp_ref)
    e_plane = pv * (2 * scale * e_sp.amax(-1))[..., None]
    _check(f"attn on float64 planes B={B} S={S}", (got - o64).abs(), bound + e_plane)
