"""GPU: the CUDA-core fp32 kernels (gemm_simt.cu, attn.cu, geo.cu: geo_embed_f32, pe.cu, rowops.cu) through their public entry
points, each against its float64 restatement in tests/_fp32_ref.py (pinned to the oracle by tests/test_fp32_reference_cpu.py)
and held to the bound derived there from the kernel's arithmetic.  These kernels are the fp32 route, Net(precision="fp32"), the
fp32 ViT and SAM encoder, and the row ops the bf16 routes still call.

The references run on the device in float64 on exactly the fp32 operands the kernel reads.  Each check prints its largest
error / bound ratio and asserts it is at most 1; where a bound is loose enough to leave doubt (the long fma chains of the GEMM,
the softmax, the geometric embedding, the linear attention, the PE max), a deliberately wrong answer must exceed it.  Output
views are pre-filled with a sentinel, and everything outside the rows and columns a kernel owns must keep it."""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _fp32_ref as R   # noqa: E402

pytestmark = pytest.mark.gpu

F64 = torch.float64
SENT = -12345.5          # sentinel of every output buffer


@pytest.fixture(scope="module")
def lib():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from sam6d_b200 import _lib
    return _lib


@pytest.fixture(scope="module")
def ops(lib):
    from sam6d_b200 import ops as _ops
    return _ops


def _gc(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _randn(g, *shape, scale=1.0):
    return torch.randn(*shape, generator=g, device="cuda") * scale


def _ratio(got, ref, bound):
    err = (got.to(F64) - ref).abs()
    assert torch.isfinite(got).all(), "non-finite output"
    return (err / bound.clamp_min(1e-300)).max().item(), err.max().item()


def _check(name, got, ref, bound):
    r, e = _ratio(got, ref, bound)
    print(f"{name}: max error / bound = {r:.3g}  (max error {e:.3g})")
    assert r <= 1.0, f"{name}: error exceeds its bound by {r:.3g}x"
    return r


def _wrong(name, got, ref, bound):
    """a deliberately wrong float64 answer must be refused by the same bound"""
    r, _ = _ratio(got, ref, bound)
    print(f"{name} (wrong answer): max error / bound = {r:.3g}")
    assert r > 1.0, f"{name}: the bound does not tell a wrong answer apart (ratio {r:.3g})"


def _untouched(name, t):
    assert bool((t == SENT).all()), f"{name}: a kernel wrote outside its output rows / columns"


def _sent(*shape):
    return torch.full(shape, SENT, device="cuda")


# ================================================================================================== gemm_simt.cu
def _gemm_case(ops, name, A, W, bias=None, act=0, res=None, alpha=1.0, out=None, wrong=False):
    """runs ops.gemm and checks it; res is copied into out first when out is the residual (residual aliasing out)"""
    if res is not None and out is not None:
        out.copy_(res)
        got = ops.gemm(A, W, bias, residual=out, out=out, relu=act, alpha=alpha)
    else:
        got = ops.gemm(A, W, bias, residual=res, out=out, relu=act, alpha=alpha)
    ref, bound = R.gemm(A, W, bias, res, alpha, act)
    _check(name, got, ref, bound)
    if wrong:
        K = A.shape[-1]
        kk = (K - 1) // 16 * 16                                # the last 16-wide K slab dropped
        wref, wb = R.gemm(A[..., :kk], W[..., :kk], bias, res, alpha, act)
        _wrong(name + " without the last K slab", got, wref, wb)
    return got


def test_gemm_model_shapes(ops):
    g = _gc(0)
    B, C = 2, 256
    # the fused RPE projection of the fp32 self layer: q | k | v | u0..u3
    x = _randn(g, B * 197, C)
    _gemm_case(ops, "gemm qkvu 394x256->1792", x, _randn(g, 1792, C, scale=C ** -0.5), _randn(g, 1792, scale=0.1), wrong=True)
    # dense fine-stage rows: the (B, N+1, C)[:, 1:] token views, the residual written in place into out[:, 1:, :]
    N = 2048
    xb = _randn(g, B, N + 1, C)
    ob = _sent(B, N + 1, C)
    res = _randn(g, B, N, C)
    _gemm_case(ops, "gemm dense 2x2048x256->256 +res in place", xb[:, 1:], _randn(g, C, C, scale=C ** -0.5),
               _randn(g, C, scale=0.1), res=res, out=ob[:, 1:])
    _untouched("gemm dense: background rows", ob[:, 0])
    _gemm_case(ops, "gemm dense 2x2048x256->512 relu", xb[:, 1:], _randn(g, 512, C, scale=C ** -0.5), _randn(g, 512, scale=0.1),
               act=1)
    # the feature similarity: per-batch W, alpha = 1 / temp, into the (B, 197, ld) store
    f1, f2 = _randn(g, B, 197, C, scale=0.06), _randn(g, B, 197, C, scale=0.06)
    store = _sent(B, 197, 208)
    _gemm_case(ops, "gemm similarity (2,197,197) alpha 10", f1, f2, alpha=1.0 / 0.1, out=store[:, :, :197], wrong=True)
    _untouched("gemm similarity: padding columns", store[:, :, 197:])
    # the PEM ViT in fp32: ViT-B (768) and ViT-L (1024) widths, qkv, the GELU MLP and the residual projection
    for D in (768, 1024):
        t = _randn(g, B * 197, D)
        _gemm_case(ops, f"gemm vit qkv {D}->{3 * D}", t, _randn(g, 3 * D, D, scale=D ** -0.5), _randn(g, 3 * D, scale=0.1))
        h = _gemm_case(ops, f"gemm vit fc1 {D}->{4 * D} gelu", t, _randn(g, 4 * D, D, scale=D ** -0.5),
                       _randn(g, 4 * D, scale=0.1), act=2)
        _gemm_case(ops, f"gemm vit fc2 {4 * D}->{D} +res", h, _randn(g, D, 4 * D, scale=(4 * D) ** -0.5),
                   _randn(g, D, scale=0.1), res=t, wrong=(D == 1024))


def test_gemm_edges(ops):
    g = _gc(1)
    # M % 128, N % 64 and K % 16 tails, every activation, bias None
    for M, N, K in ((130, 70, 40), (257, 65, 17), (1, 1, 1), (128, 64, 16)):
        A, W = _randn(g, M, K), _randn(g, N, K, scale=K ** -0.5)
        for act in (0, 1, 2):
            _gemm_case(ops, f"gemm {M}x{K}->{N} act {act}", A, W, _randn(g, N) if act else None, act=act)
    # K % 4 != 0 and lda % 4 != 0 take the scalar loader
    A, W = _randn(g, 150, 37), _randn(g, 90, 37, scale=0.2)
    _gemm_case(ops, "gemm K 37 (scalar loader)", A, W, _randn(g, 90), wrong=True)
    Ab = _randn(g, 150, 41)
    _gemm_case(ops, "gemm lda 41 (scalar loader)", Ab[:, :40], _randn(g, 90, 40, scale=0.2), _randn(g, 90), wrong=True)
    # batched: one W shared by every problem, and one W per problem, residual batched
    A3 = _randn(g, 3, 50, 48)
    res = _randn(g, 3, 50, 70)
    _gemm_case(ops, "gemm batched shared W", A3, _randn(g, 70, 48, scale=0.2), _randn(g, 70), act=1, res=res)
    _gemm_case(ops, "gemm batched per-batch W", A3, _randn(g, 3, 70, 48, scale=0.2), None, act=2, res=res, alpha=0.5)


# ================================================================================================== rpe_scores
def _rpe_case(ops, name, E, U4, wrong=False):
    got = ops.rpe_scores(E, U4)
    ref, bound = R.rpe_scores(E, U4)
    _check(name, got, ref, bound)
    if wrong:                                                   # the channels of the last lane left out
        Ew = E.clone()
        Ew[..., 248:] = 0
        wref, wb = R.rpe_scores(Ew, U4)
        _wrong(name + " without channels 248..255", got, wref, wb)


def test_rpe_scores(ops, lib):
    g = _gc(2)
    # fp32 E at (2B, 197) with U the qkvu[:, 768:] columns of the fused projection (row stride 1792)
    B2, S = 4, 197
    qkvu = _randn(g, B2 * S, 1792)
    E = _randn(g, B2, S, S, 256)
    _rpe_case(ops, "rpe_scores f32 (4,197) u_ld 1792", E, qkvu[:, 768:], wrong=True)
    # the score planes fill SP exactly: nothing past its end is written
    SP = _sent(B2 * 4 * S * S + 97)
    lib.call("sam6d_rpe_scores", E, 0, qkvu[:, 768:], 1792, B2, S, SP)
    ref, bound = R.rpe_scores(E, qkvu[:, 768:])
    _check("rpe_scores f32 into a larger buffer", SP[:-97].view(B2, 4, S, S), ref, bound)
    _untouched("rpe_scores: past the score planes", SP[-97:])
    del E
    # bf16 E: the route of the bf16 forward above 200 points
    for Bs, S in ((2, 201), (2, 257), (1, 1025)):
        E = _randn(g, Bs, S, S, 256).bfloat16()
        _rpe_case(ops, f"rpe_scores bf16 ({Bs},{S})", E, _randn(g, Bs * S, 1024), wrong=(S == 201))
        del E
    # S - 1 clamps the last chunk of four keys
    for S in (4, 5, 33):
        _rpe_case(ops, f"rpe_scores f32 (3,{S})", _randn(g, 3, S, S, 256), _randn(g, 3 * S, 1024))


def test_rpe_scores_argument_checks(ops, lib):
    g = _gc(3)
    S = 8
    E = _randn(g, 1, S, S, 256)
    ub = _randn(g, S, 1028)
    SP = _sent(4 * S * S)
    # U one float past a 16-byte boundary (row stride still a multiple of 4): refused by the C ABI, and so by the wrapper
    with pytest.raises(RuntimeError, match="invalid argument"):
        ops.rpe_scores(E, ub[:, 1:1025])
    with pytest.raises(RuntimeError, match="invalid argument"):
        lib.call("sam6d_rpe_scores", E, 0, ub[:, 1:1025], 1028, 1, S, SP)
    Eb = torch.zeros(S * S * 256 + 1, device="cuda")[1:].view(1, S, S, 256)
    with pytest.raises(RuntimeError, match="invalid argument"):
        lib.call("sam6d_rpe_scores", Eb, 0, ub[:, :1024], 1028, 1, S, SP)
    with pytest.raises(RuntimeError, match="invalid argument"):
        lib.call("sam6d_rpe_scores", E, 0, ub[:, :1024], 1026, 1, S, SP)
    torch.cuda.synchronize()
    _untouched("rpe_scores: refused calls", SP)


# ================================================================================================== mha
def _mha_case(ops, name, q, k, v, bias, scale, out, wrong=False):
    ops.mha(q, k, v, bias, scale, out)
    ref, bound = R.mha(q, k, v, bias, scale)
    r = _check(name, out, ref, bound)
    if wrong:
        wref, wb = R.mha(q, k, v, bias, scale, drop_last_key=True)
        _wrong(name + " with the last key left out", out, wref, wb)
    return r


def test_mha_model_shapes(ops):
    g = _gc(4)
    B, S, C = 2, 197, 256
    # self RPE: q / k / v column slices of the (B, 197, 1792) qkvu view, bias from rpe_scores; out a view with o_ld 320
    x = _randn(g, B * S, C)
    qkvu = ops.gemm(x, _randn(g, 1792, C, scale=C ** -0.5), _randn(g, 1792, scale=0.1))
    E = _randn(g, B, S, S, 256, scale=0.5)
    sp = ops.rpe_scores(E, qkvu[:, 3 * C:])
    qkv = qkvu.view(B, S, -1)
    ob = _sent(B, S, 320)
    _mha_case(ops, "mha self rpe (2,197,197) H 4", qkv[..., :C], qkv[..., C:2 * C], qkv[..., 2 * C:3 * C], sp, 0.125,
              ob[..., :C], wrong=True)
    _untouched("mha self: columns past H*64", ob[..., C:])
    # cross: Sq = Sk = 197, k / v the halves of one (B, 197, 512) projection, no bias
    q = _randn(g, B, S, C)
    kv = _randn(g, B, S, 2 * C)
    _mha_case(ops, "mha cross (2,197,197) H 4", q, kv[..., :C], kv[..., C:], None, 0.125, torch.empty(B, S, C, device="cuda"),
              wrong=True)
    # the fp32 ViT: H = 12 (ViT-B) and 16 (ViT-L), S = 197
    for H in (12, 16):
        HD = 64 * H
        qkv = _randn(g, B, S, 3 * HD)
        _mha_case(ops, f"mha vit H {H}", qkv[..., :HD], qkv[..., HD:2 * HD], qkv[..., 2 * HD:], None, 0.125,
                  torch.empty(B, S, HD, device="cuda"))


def test_mha_edges(ops):
    """every key count the register tile treats differently (1, the lane count and one past it, 255, 256) against the query
    tails of a 4-query warp and a 32-query CTA; one dominant score per row drives __expf down to arguments near -50"""
    g = _gc(5)
    B, H = 2, 4
    HD = 64 * H
    worst = 0.0
    for Sk in (1, 31, 32, 33, 255, 256):
        k, v = _randn(g, B, Sk, HD), _randn(g, B, Sk, HD)
        for Sq in (1, 3, 4, 5, 33):
            q = _randn(g, B, Sq, HD)
            bias = _randn(g, B, H, Sq, Sk)
            ob = _sent(B, Sq, HD + 64)
            worst = max(worst, _mha_case(ops, f"mha Sq {Sq} Sk {Sk}", q, k, v, bias, 0.125, ob[..., :HD],
                                         wrong=(Sk > 1 and Sq == 5)))
            _untouched(f"mha Sq {Sq} Sk {Sk}: columns past H*64", ob[..., HD:])
        dom = torch.zeros(B, H, 33, Sk, device="cuda")
        pick = torch.randint(0, Sk, (B, H, 33, 1), generator=_gc(100 + Sk), device="cuda")
        dom.scatter_(-1, pick, 400.0)                                                       # + 50 after the scale
        q = _randn(g, B, 33, HD)
        _mha_case(ops, f"mha Sk {Sk} one dominant score per row", q, k, v, dom, 0.125, torch.empty(B, 33, HD, device="cuda"))
    print(f"mha edges: worst ratio {worst:.3g}")


def test_mha_argument_checks(ops, lib):
    g = _gc(6)
    B, S, HD = 2, 9, 256
    q, k, v = _randn(g, B, S, HD), _randn(g, B, S, HD), _randn(g, B, S, HD)
    out = _sent(B, S, HD)
    bias = _randn(g, B, 4, S, S)
    bad = {
        "bf16 q": dict(q=q.bfloat16()), "bf16 k": dict(k=k.bfloat16()), "bf16 v": dict(v=v.bfloat16()),
        "bf16 out": dict(out=out.bfloat16()), "bf16 bias": dict(bias=bias.bfloat16()),
        "HD % 64": dict(q=q[..., :96], k=k[..., :96], v=v[..., :96], out=out[..., :96], bias=None),
        "k width": dict(k=k[..., :192]), "v width": dict(v=v[..., :192]), "out width": dict(out=out[..., :192]),
        "v keys": dict(v=v[:, :8]), "bias keys": dict(bias=bias[..., :8]),
        "padded bias rows": dict(bias=torch.zeros(B, 4, S, 12, device="cuda")[..., :S]),
        "transposed bias": dict(bias=bias.transpose(-1, -2)),
        "bias heads": dict(bias=bias[:, :2]),
        "257 keys": dict(k=_randn(g, B, 257, HD), v=_randn(g, B, 257, HD), bias=None),
    }
    for name, over in bad.items():
        a = dict(q=q, k=k, v=v, bias=bias, out=out)
        a.update(over)
        with pytest.raises(RuntimeError):
            ops.mha(a["q"], a["k"], a["v"], a["bias"], 0.125, a["out"])
            pytest.fail(f"mha accepted {name}")
    # K or V one float past a 16-byte boundary (strides still multiples of 4): the wrapper and the C ABI refuse them
    kb = _randn(g, B, S, HD + 4)
    with pytest.raises(RuntimeError, match="invalid argument"):
        ops.mha(q, kb[..., 1:HD + 1], v, None, 0.125, out)
    with pytest.raises(RuntimeError, match="invalid argument"):
        ops.mha(q, k, kb[..., 1:HD + 1], None, 0.125, out)
    ld = HD + 4
    with pytest.raises(RuntimeError, match="invalid argument"):
        lib.call("sam6d_mha", q, HD, S * HD, kb[..., 1:], ld, S * ld, v, HD, S * HD, None, B, 4, S, S, 0.125, out, HD, S * HD)
    # B * H is the grid's y extent
    with pytest.raises(RuntimeError, match="invalid argument"):
        lib.call("sam6d_mha", q, HD, S * HD, k, HD, S * HD, v, HD, S * HD, None, 16384, 4, S, S, 0.125, out, HD, S * HD)
    torch.cuda.synchronize()
    _untouched("mha: refused calls", out)


# ================================================================================================== linear attention
def _focused(g, *shape):
    """non-negative features of the magnitude the feature map leaves (|q| ~ ||relu(x) + 1e-6|| / sqrt(C))"""
    return _randn(g, *shape).abs() * 0.5 + 1e-7


def test_linattn(ops, lib):
    g = _gc(7)
    C = 256
    for B, J, N in ((2, 196, 2048), (32, 196, 2048), (2, 1, 8), (2, 7, 9), (3, 400, 513), (2, 196, 1)):
        kv = _randn(g, B, J, 2 * C)
        kv[..., :C] = _focused(g, B, J, C)
        KV, KS = _sent(B, 4, 64, 64), _sent(B, 4, 64)
        ops.linattn_kv(kv[..., :C], kv[..., C:], KV, KS)
        rKV, rKS, eKV, eKS = R.linattn_kv(kv[..., :C], kv[..., C:])
        _check(f"linattn_kv B {B} J {J} KV", KV, rKV, eKV)
        _check(f"linattn_kv B {B} J {J} KS", KS, rKS, eKS)
        if J == 196 and B == 2:
            wKV, _, weKV, _ = R.linattn_kv(kv[:, :-1, :C], kv[:, :-1, C:])
            _wrong(f"linattn_kv B {B} J {J} without the last key", KV, wKV, weKV)
        # queries and output are rows 1..N of (B, N+1, C) sequences
        qb = _randn(g, B, N + 1, C)
        qb[:, 1:] = _focused(g, B, N, C)
        ob = _sent(B, N + 1, C)
        ops.linattn_apply(qb[:, 1:], KV, KS, ob[:, 1:])
        ref, bound = R.linattn_apply(qb[:, 1:], KV, KS)
        _check(f"linattn_apply B {B} J {J} N {N}", ob[:, 1:], ref, bound)
        _untouched(f"linattn_apply B {B} N {N}: background rows", ob[:, 0])
        if N == 2048 and B == 2:
            qw = qb[:, 1:].clone()
            qw[..., 63::64] = 0                                      # the last channel of every head left out
            wref, wb = R.linattn_apply(qw, KV, KS)
            _wrong(f"linattn_apply N {N} without channel 63 of each head", ob[:, 1:], wref, wb)
    # 401 keys need more shared memory than the kernel takes
    kv = _randn(g, 1, 401, 2 * C)
    KV, KS = _sent(1, 4, 64, 64), _sent(1, 4, 64)
    with pytest.raises(RuntimeError, match="invalid argument"):
        ops.linattn_kv(kv[..., :C], kv[..., C:], KV, KS)
    torch.cuda.synchronize()
    _untouched("linattn_kv: refused call", KV)


# ================================================================================================== rowops.cu
def test_focus_rows(ops):
    g = _gc(8)
    C = 256
    sp = torch.nn.functional.softplus(_randn(g, C, scale=0.3))
    # in place on the queries of the dense layer, B * 2048 rows
    q = _randn(g, 2 * 2048, C)
    x0 = q.clone()
    ops.focus_rows(q, sp, out=q)
    ref, bound = R.focus(x0, sp)
    _check("focus_rows in place (4096, 256)", q, ref, bound)
    # in place on the k half of the (B*J, 2C) key / value projection: the v half keeps its values; B*J % 8 = 4
    kv = _randn(g, 3 * 196, 2 * C)
    kv[:, C:] = SENT
    x0 = kv[:, :C].clone()
    ops.focus_rows(kv[:, :C], sp, out=kv[:, :C])
    ref, bound = R.focus(x0, sp)
    _check("focus_rows kv[:, :C] (588 rows, ld 512)", kv[:, :C], ref, bound)
    _untouched("focus_rows: the v half", kv[:, C:])
    # all-negative rows (every q = 1e-6f / sp) across sp in [0.5, 2]: every (q^3)^2 stays a normal fp32 number (the
    # docstring of _fp32_ref.focus states the subnormal limit near sp = 2.1); one dominant channel; 13 rows (13 % 8 = 5)
    spn = torch.linspace(0.5, 2.0, C, device="cuda")
    x = _randn(g, 13, C)
    x[:6] = -x[:6].abs() - 0.1
    x[6:9] = x[6:9].abs() * 1e-3
    x[6:9, 17] = 50.0
    out = _sent(13, C)
    ops.focus_rows(x, spn, out=out)
    ref, bound = R.focus(x, spn)
    _check("focus_rows all-negative and dominant-channel rows", out, ref, bound)
    for spc in (0.5, 2.0):
        xs = -torch.ones(8, C, device="cuda")
        ys = ops.focus_rows(xs, torch.full((C,), spc, device="cuda"))
        ref, bound = R.focus(xs, torch.full((C,), spc, device="cuda"))
        _check(f"focus_rows all-negative rows at sp {spc}", ys, ref, bound)


LN_CASES = [(32, 1e-5), (256, 1e-5), (288, 1e-5), (384, 1e-6), (768, 1e-6), (1024, 1e-6), (1056, 1e-5), (1280, 1e-6),
            (1536, 1e-6), (2048, 1e-5), (768, 1e-5), (1024, 1e-5)]


def _ln_rows(g, rows, C):
    """random rows, rows with |mean| = 100 sigma, constant rows"""
    x = _randn(g, rows, C) * 2 + 0.5
    x[rows // 3: rows // 2] = _randn(g, rows // 2 - rows // 3, C) + 100.0
    x[-3:] = torch.tensor([0.1, -7.25, 100.0], device="cuda").view(3, 1)
    return x


@pytest.mark.parametrize("C,eps", LN_CASES)
def test_layernorm(ops, C, eps):
    """C = 256 (PEM), 384 / 768 / 1024 / 1536 at eps 1e-6 (the DINOv2 final norm), 768 / 1024 / 1280 (the fp32 SAM encoder and
    the PEM ViT), and all three register tiles with their edges (288, 1056, 2048)"""
    g = _gc(9 + C)
    x = _ln_rows(g, 37, C)
    gm, bt = 1 + 0.2 * _randn(g, C), 0.2 * _randn(g, C)
    y = ops.layernorm(x, gm, bt, eps)
    ref, bound = R.layernorm(x, gm, bt, eps)
    _check(f"layernorm C {C} eps {eps:g}", y, ref, bound)
    if C == 256 and eps == 1e-5:
        wref, wb = R.layernorm(x, gm, bt, eps, eps_scale=10)
        _wrong(f"layernorm C {C} with eps x 10", y, wref, wb)
    # row views: rows 1..N of (B, N+1, C) sequences in and out
    xb = _randn(g, 3, 12, C)
    ob = _sent(3, 12, C)
    ops.layernorm(xb[:, 1:], gm, bt, eps, out=ob[:, 1:])
    ref, bound = R.layernorm(xb[:, 1:].reshape(-1, C), gm, bt, eps)
    _check(f"layernorm C {C} row views", ob[:, 1:].reshape(-1, C), ref, bound)
    _untouched(f"layernorm C {C}: background rows", ob[:, 0])


def test_layernorm_refuses_wide_rows(ops):
    x = torch.zeros(4, 2080, device="cuda")
    g = torch.ones(2080, device="cuda")
    with pytest.raises(RuntimeError, match="invalid argument"):
        ops.layernorm(x, g, g, 1e-5)


@pytest.mark.parametrize("C", [256, 384, 768, 1024, 1536])
def test_l2norm_rows(ops, C):
    """ISM descriptor widths and the PEM's 256; zero rows (the 1e-12 clamp) and norms around it; fp32 and bf16 results"""
    g = _gc(20 + C)
    x = _randn(g, 45, C)
    x[3] = 0
    for i, n in enumerate((0.25e-12, 0.9e-12, 1e-12, 1.1e-12, 4e-12, 1e-9)):
        x[5 + i] = x[5 + i] / x[5 + i].norm() * n
    y = ops.l2norm_rows(x)
    ref, bound = R.l2norm(x)
    _check(f"l2norm_rows C {C}", y, ref, bound)
    assert bool((y[3] == 0).all())
    yb = ops.l2norm_rows_bf16(x)
    _check(f"l2norm_rows_bf16 C {C}", yb, R.bf(ref), R.spread(ref, bound))


# ================================================================================================== geo_embed_f32
def _geo_weights(g):
    div = torch.exp(torch.arange(0, 256, 2, device="cuda").float() * (-math.log(10000.0) / 256))
    WaT, WdT = _randn(g, 256, 256, scale=1 / 16), _randn(g, 256, 256, scale=1 / 16)
    return div, WaT, WdT, _randn(g, 256, scale=0.1)


def _geo_pts(g, B, S):
    """clouds of radius ~0.1 whose point 0 is the far background point: distance indices near 866 in its row and column"""
    p = _randn(g, B, S, 3, scale=0.05)
    p[:, 0] = 100.0
    return p


def test_geo_embed_f32(ops, lib):
    g = _gc(30)
    div, WaT, WdT, bias = _geo_weights(g)
    fa = 180.0 / (15.0 * math.pi)
    T = ops.geo_indices(_geo_pts(g, 4, 197), 0.2, fa)
    assert T[:, 0, 1:, 3].min().item() > 800                     # the background row reaches the large-argument sincosf
    E = ops.geo_embed_f32(T, div, WaT, WdT, bias)
    ref, bound = R.geo_embed(T.view(-1, 4), div, WaT, WdT, bias)
    _check("geo_embed_f32 (4,197,197)", E.view(-1, 256), ref, bound)
    wref, wb = R.geo_embed(T.view(-1, 4), div, WaT, WdT, bias, drop_last_pair=True)
    _wrong("geo_embed_f32 without k = 254, 255", E.view(-1, 256), wref, wb)
    del E, ref, bound, wref, wb
    # 33 x 33 pairs: npairs % 16 = 1; nothing past the last pair is written
    T = ops.geo_indices(_geo_pts(g, 1, 33), 0.2, fa)
    P = 33 * 33
    out = _sent(P + 16, 256)
    lib.call("sam6d_geo_embed_f32", T, P, div, WaT, WdT, bias, out)
    ref, bound = R.geo_embed(T.view(-1, 4), div, WaT, WdT, bias)
    _check("geo_embed_f32 (1,33,33)", out[:P], ref, bound)
    _untouched("geo_embed_f32: past the last pair", out[P:])


# ================================================================================================== pe_mlp_max
def _pe_weights(g):
    w = []
    for cin, cout in ((6, 32), (32, 64), (64, 128)):
        w += [_randn(g, cout, cin, scale=(2.0 / cin) ** 0.5), _randn(g, cout, scale=0.1)]
    return w


def test_pe_mlp_max(ops):
    g = _gc(40)
    for B, N in ((2, 2048), (2, 13), (1, 6)):
        pts = _randn(g, B, N, 3, scale=0.08)
        pts[:, :N // 8] *= 5                                        # a sparse fringe: balls with fewer than ns points
        far = N - 1
        pts[:, far] = 3.0                                           # a valid point far from the rest
        out = _sent(B, N, 256)
        ia, ca, ib, cb = ops.ball_query_pair(pts, pts, 0.1, 32, 0.2, 64)
        for ns, idx, cnt, off in ((32, ia, ca, 0), (64, ib, cb, 128)):
            idx, cnt = idx.clone(), cnt.clone()
            s = torch.arange(ns, device="cuda")
            idx = torch.where(s < cnt.unsqueeze(-1), idx, torch.full_like(idx, far))     # never read: would win the max
            cnt[:, :3] = 0                                        # empty balls: one sample, idx[..., 0]
            idx[:, :3, 0] = 0
            idx[:, :3, 1:] = far
            assert bool((cnt[:, 3:-1] < ns).any())
            w = _pe_weights(g)
            ops.pe_mlp_max(pts, idx, cnt, w, out, off)
            ref, bound = R.pe_mlp_max(pts, idx, cnt, w)
            _check(f"pe_mlp_max B {B} N {N} ns {ns}", out[..., off:off + 128], ref, bound)
            wref, wb = R.pe_mlp_max(pts, idx, torch.full_like(cnt, ns), w)
            _wrong(f"pe_mlp_max B {B} N {N} ns {ns} reading every sample", out[..., off:off + 128], wref, wb)
            if off == 0:
                _untouched(f"pe_mlp_max N {N}: channels 128..255 before their call", out[..., 128:])


# ================================================================================================== point-cloud row ops
def test_point_ops(ops, lib):
    from oracle import pem_oracle as po
    inp = po.make_inputs(B=4, n=2048, seed=2)
    g = _gc(50)
    for p in (inp["dense_po"].cuda(), inp["pts"].cuda(), _randn(g, 3, 1, 3)):
        B = p.shape[0]
        Rm = torch.linalg.qr(_randn(g, B, 3, 3))[0].contiguous()
        t = _randn(g, B, 3, scale=0.1)
        out = ops.rigid_warp(p, Rm, t)
        ref, bound = R.rigid_warp(p, Rm, t)
        _check(f"rigid_warp {tuple(p.shape)}", out, ref, bound)
        r = ops.cloud_radius(p)
        ref, bound = R.cloud_radius(p)
        _check(f"cloud_radius {tuple(p.shape)}", r, ref, bound)
        s = ops.scale_by_radius(p, r)
        ref, bound = R.scale_by_radius(p, r)
        _check(f"scale_by_radius {tuple(p.shape)}", s, ref, bound)
    # b = 0: nothing to do, nothing launched, empty results
    e = torch.empty(0, 5, 3, device="cuda")
    assert ops.rigid_warp(e, torch.empty(0, 3, 3, device="cuda"), torch.empty(0, 3, device="cuda")).shape == (0, 5, 3)
    assert ops.cloud_radius(e).shape == (0,)
    assert ops.scale_by_radius(e, torch.empty(0, device="cuda")).shape == (0, 5, 3)
    assert lib.call("sam6d_rigid_warp", None, None, None, 0, 5, None) == 0
    assert lib.call("sam6d_cloud_radius", None, 0, 5, None) == 0
    assert lib.call("sam6d_scale_by_radius", None, None, 0, 15, None) == 0
    torch.cuda.synchronize()
