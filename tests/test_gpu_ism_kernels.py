"""GPU: the ISM's decoder, descriptor and GEMM-epilogue kernels called directly through the C ABI, each against a float64
evaluation of the same operation in plain torch on the operands rounded exactly as the kernel reads them.

Every bound is derived from the kernel's arithmetic and written next to its check.  Notation: u = 2^-24 (fp32 unit roundoff),
ub = 2^-8 (bf16 unit roundoff: one round-to-nearest bf16 store moves a value by at most ub |x|), gamma_n ~ n u for a chain of n
fp32 roundings.  A tensor-core (wgmma) fp32 accumulation is charged 2u per added product: the accumulator may truncate rather
than round.  CUDA's documented accuracy of the math functions used: __expf(x) 2 + floor(|1.173 x|) ulp, sinf / cosf / erff /
rsqrtf 2 ulp, __logf 3 ulp (an ulp of a result in [1, 2) is 2u).  Each check prints its largest error / bound ratio; where a
bound is loose enough to leave doubt, a deliberately wrong answer computed in torch must fail the same bound."""
import itertools
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import ism_oracle as io          # noqa: E402
from oracle import sam_dec_oracle as so      # noqa: E402
from sam6d_b200 import synth                 # noqa: E402

U = 2.0 ** -24          # fp32 unit roundoff
UB = 2.0 ** -8          # bf16 unit roundoff
F64 = torch.float64


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


def _softmax_terms(s, v):
    """fp64 softmax attention pieces: s (..., Lk) logits, v (..., Lk, d) -> (out, sum_j p_j |v_j| / sum_j p_j, max_j (m - s_j))"""
    p = torch.softmax(s, dim=-1)
    return p @ v, p @ v.abs(), (s.amax(-1) - s.amin(-1))


def _exp_err(xr):
    """relative error of __expf over arguments down to -xr, plus the rounding of the subtraction s - m"""
    return (2.0 + 1.173 * xr) * 2 * U + U * xr


# ================================================================================================== A. SAM mask decoder
@pytest.mark.parametrize("G", [1, 3, 64])
@pytest.mark.parametrize("B", [1, 3])
def test_sam_mask_dot_every_subpixel(lib, B, G):
    """the pixel shuffle of both transposed convolutions folded into sam_mask_dot's output index, at all 16 sub-positions"""
    g = _g(100 + 10 * B + G)
    up = torch.randn(B * G * G * 4, 128, generator=g).bfloat16()
    hyper = torch.randn(B, 4, 32, generator=g)
    hyper[:, 0] = float("nan")                   # mask token 0 (the single-mask output) must never reach the multimask slice
    up_d, hyper_d = up.cuda(), hyper.cuda()
    masks = torch.full((B, 3, 4 * G, 4 * G), float("nan"), device="cuda")
    lib.call("sam6d_sam_mask_dot", up_d, hyper_d, B, G, masks)
    got = masks.double()
    assert torch.isfinite(got).all(), "a pixel was not written or mask token 0 leaked in"
    # up rows (b, y, x, i, j), columns (i', j', o) -> pixel (4y + 2i + i', 4x + 2j + j')
    Ud = up_d.double().view(B, G, G, 2, 2, 2, 2, 32)
    Uimg = Ud.permute(0, 7, 1, 3, 5, 2, 4, 6).reshape(B, 32, 4 * G, 4 * G)
    h = hyper_d[:, 1:4].double()
    ref = torch.einsum("bmo,boyx->bmyx", h, Uimg)
    # one fp32 fma chain over 32 products: |err| <= gamma_32 sum_o |h_o u_o|
    bound = 33 * U * torch.einsum("bmo,boyx->bmyx", h.abs(), Uimg.abs())
    _check(f"sam_mask_dot B={B} G={G}", (got - ref).abs(), bound)
    # negative control: i' and j' swapped inside every 2 x 2 sub-block
    wrong = torch.einsum("bmo,boyx->bmyx", h, Ud.permute(0, 7, 1, 3, 6, 2, 4, 5).reshape(B, 32, 4 * G, 4 * G))
    assert _ratio((got - wrong).abs(), bound) > 1.0


def _build_sam_decoder(seed):
    from sam6d_b200.sam_amg import MaskDecoder, PromptEncoder, Sam
    sd = so.make_state_dict(seed=seed)
    enc = torch.nn.Module()
    enc.img_size = 1024
    sam = Sam(enc, PromptEncoder(), MaskDecoder()).cuda().eval()
    sam.prompt_encoder.load_state_dict({k[len("prompt_encoder."):]: v for k, v in sd.items() if k.startswith("prompt_encoder.")}, strict=True)
    sam.mask_decoder.load_state_dict({k[len("mask_decoder."):]: v for k, v in sd.items() if k.startswith("mask_decoder.")}, strict=True)
    return sd, sam


def _subpixel_classes(low, ref):
    """per (Y % 4, X % 4) class: (relative rms error, sign agreement)"""
    B = low.shape[0]
    lo, rf = low.reshape(B, 3, 64, 4, 64, 4), ref.reshape(B, 3, 64, 4, 64, 4)
    out = {}
    for a, c in itertools.product(range(4), range(4)):
        x, y = lo[:, :, :, a, :, c], rf[:, :, :, a, :, c]
        rel = ((x - y).pow(2).mean().sqrt() / y.pow(2).mean().sqrt()).item()
        out[(a, c)] = (rel, ((x > 0) == (y > 0)).float().mean().item())
    return out


def test_mask_decoder_full_resolution_every_subpixel(golden_dir):
    """all 3 x 256 x 256 logits of 4 point prompts against the pinned CPU oracle, per sub-pixel class (Y % 4, X % 4): this covers
    the (kh, kw, out, in) packing of both ConvTranspose2d weights (MaskDecoder._weights), which a comparison on the ::8 lattice
    samples at one class only.  Bounds as test_gpu_sam_dec.py (bf16 image-side operands): rel rms < 3e-2, signs > 0.99."""
    seed = torch.load(os.path.join(golden_dir, "sam_dec.pt"), weights_only=False)["meta"]["seed"]
    sd, sam = _build_sam_decoder(seed)
    feat = synth.make_image_embedding(seed=seed)
    pts = so.build_point_grid(8)[[0, 19, 36, 63]] * np.array([640, 480])[None, :]
    c = so.apply_coords(pts, (480, 640))
    sparse_ref = so.embed_points(sd, torch.as_tensor(c)[:, None, :].float(), torch.ones(4, 1))
    ref, _ = so.mask_decoder(sd, feat, so.dense_pe(sd), sparse_ref)
    with torch.no_grad():
        sparse, dense = sam.prompt_encoder(points=(torch.as_tensor(c, device="cuda")[:, None, :],
                                                   torch.ones(4, 1, dtype=torch.int, device="cuda")))
        low, _ = sam.mask_decoder(feat.cuda(), sam.prompt_encoder.dense_pe_rows(), sparse, dense, True)
    low = low.cpu()
    assert low.shape == ref.shape == (4, 3, 256, 256)
    cls = _subpixel_classes(low, ref)
    for k, (rel, sign) in sorted(cls.items()):
        print(f"sub-pixel class {k}: rel rms {rel:.3e} (/ 3e-2 = {rel / 3e-2:.3f}), sign agreement {sign:.5f}")
    assert all(rel < 3e-2 and sign > 0.99 for rel, sign in cls.values())
    # negative control: i' and j' swapped inside every 2 x 2 sub-block of the GPU output must fail at least one class
    swapped = low.view(4, 3, 64, 2, 2, 64, 2, 2).permute(0, 1, 2, 3, 7, 5, 6, 4).reshape(4, 3, 256, 256)
    bad = _subpixel_classes(swapped, ref)
    print("swapped i'/j': worst class rel rms", max(r for r, _ in bad.values()))
    assert any(rel >= 3e-2 or sign <= 0.99 for rel, sign in bad.values())


def _tok2img_ref(Q, K, V, B, T, L, shared):
    """fp64 8-head x 16 attention of the prompt tokens over the image tokens -> (out, bound) (B,T,128)"""
    Bk = 1 if shared else B
    qh = Q.double().view(B, T, 8, 16).permute(0, 2, 1, 3)
    kh = K.double().view(Bk, L, 8, 16).permute(0, 2, 1, 3)
    vh = V.double().view(Bk, L, 8, 16).permute(0, 2, 1, 3)
    s = qh @ kh.transpose(-1, -2) * 0.25
    o, pv, xr = _softmax_terms(s, vh)
    # logits: q / 4 (exact) then a 16-term fp32 fma chain -> |ds| <= 16 u sum |q||k| / 4; the row max moves by as much
    d = 16 * U * ((qh.abs() @ kh.abs().transpose(-1, -2)) * 0.25).amax(-1)
    eta = 2 * d + _exp_err(xr)
    # numerator: ceil(L/16)-term chains then 16 partial sums; denominator: ceil(L/256)-term chains, warp tree, 8 partials; one division
    n = math.ceil(L / 16) + 16 + math.ceil(L / 256) + 13 + 1
    bound = pv * (2 * eta + n * U)[..., None] * 1.01
    return o.permute(0, 2, 1, 3).reshape(B, T, 128), bound.permute(0, 2, 1, 3).reshape(B, T, 128)


def _run_tok2img(lib, B, T, L, shared, seed):
    g = _g(seed)
    Bk = 1 if shared else B
    Q = (torch.randn(B, T, 128, generator=g) * 8).cuda()          # logits of about +-30: the max subtraction matters
    K = torch.randn(Bk, L, 128, generator=g).bfloat16().cuda()
    V = torch.randn(Bk, L, 128, generator=g).bfloat16().cuda()
    out = torch.full((B, T, 128), float("nan"), device="cuda")
    lib.call("sam6d_sam_tok2img_attn", Q, K, V, 0 if shared else L * 128, B, T, L, out)
    return out, _tok2img_ref(Q, K, V, B, T, L, shared)


@pytest.mark.parametrize("B", [1, 3, 64])
@pytest.mark.parametrize("shared", [True, False])
@pytest.mark.parametrize("L", [4096, 1000, 33])
@pytest.mark.parametrize("T", [1, 7, 8])
def test_sam_tok2img_attn(lib, B, T, L, shared):
    out, (ref, bound) = _run_tok2img(lib, B, T, L, shared, seed=T * 1000 + L + B)
    _check(f"sam_tok2img_attn B={B} T={T} L={L} shared={shared}", (out.double() - ref).abs(), bound)


def test_sam_tok2img_attn_smem_limit(lib):
    """T * L fp32 scores live in shared memory: exactly 200 KB (T = 8, L = 6400) is accepted, one more key is refused"""
    out, (ref, bound) = _run_tok2img(lib, 1, 8, 6400, True, seed=6400)
    _check("sam_tok2img_attn T=8 L=6400", (out.double() - ref).abs(), bound)
    Q = torch.zeros(1, 8, 128, device="cuda")
    KV = torch.zeros(6401, 128, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(lib.Sam6dError, match="invalid argument"):
        lib.call("sam6d_sam_tok2img_attn", Q, KV, KV, 0, 1, 8, 6401, Q)


@pytest.mark.parametrize("shared", [True, False])
@pytest.mark.parametrize("L", [4096, 1000, 33])
@pytest.mark.parametrize("T", [1, 7, 8])
def test_sam_img2tok_attn(lib, T, L, shared):
    """image tokens attend to the prompt tokens; L is not a multiple of the 32-pixel CTA at 1000 and 33"""
    B = 3
    g = _g(2000 + T * 10 + L)
    Bq = 1 if shared else B
    Q = torch.randn(Bq, L, 128, generator=g).bfloat16().cuda()
    Kt = (torch.randn(B, T, 128, generator=g) * 5).cuda()
    Vt = torch.randn(B, T, 128, generator=g).cuda()
    out = torch.full((B, L, 128), float("nan"), dtype=torch.bfloat16, device="cuda")
    lib.call("sam6d_sam_img2tok_attn", Q, 0 if shared else L * 128, Kt, Vt, B, T, L, out)
    qh = Q.double().view(Bq, L, 8, 16).permute(0, 2, 1, 3)
    kh = Kt.double().view(B, T, 8, 16).permute(0, 2, 1, 3)
    vh = Vt.double().view(B, T, 8, 16).permute(0, 2, 1, 3)
    s = qh @ kh.transpose(-1, -2) * 0.25
    o, pv, xr = _softmax_terms(s, vh)
    d = 16 * U * ((qh.abs() @ kh.abs().transpose(-1, -2)) * 0.25).amax(-1)
    # fp32: logits as in tok2img, T-term chains for the sum and the products, 1 / den and one product; then one bf16 rounding
    e32 = pv * (2 * (2 * d + _exp_err(xr)) + (2 * T + 3) * U)[..., None] * 1.01
    bound = UB * (o.abs() + e32) + e32
    to = lambda t: t.permute(0, 2, 1, 3).reshape(B, L, 128)      # noqa: E731
    _check(f"sam_img2tok_attn T={T} L={L} shared={shared}", (out.double() - to(o)).abs(), to(bound))


@pytest.mark.parametrize("T", [1, 2, 7, 8])
@pytest.mark.parametrize("B", [1, 3, 64, 65])
def test_sam_self_attn(lib, B, T):
    """prompt-token self attention, 8 heads x 32, one warp per (prompt, head): 65 prompts leave a ragged last CTA"""
    g = _g(3000 + 10 * B + T)
    q, k, v = ((torch.randn(B, T, 256, generator=g) * 1.5).cuda() for _ in range(3))
    out = torch.full((B, T, 256), float("nan"), device="cuda")
    lib.call("sam6d_sam_self_attn", q, k, v, B, T, out)
    sep = lambda t: t.double().view(B, T, 8, 32).permute(0, 2, 1, 3)      # noqa: E731
    qh, kh, vh = sep(q), sep(k), sep(v)
    scale = 1 / math.sqrt(32)
    s = qh @ kh.transpose(-1, -2) * scale
    o, pv, xr = _softmax_terms(s, vh)
    # logits: 32 products reduced by a 5-level warp tree (gamma_6), times the fp32 constant 1/sqrt(32) (two roundings)
    d = (6 * U * ((qh.abs() @ kh.abs().transpose(-1, -2)) * scale) + 2 * U * s.abs()).amax(-1)
    bound = pv * (2 * (2 * d + _exp_err(xr)) + (2 * T + 2) * U)[..., None] * 1.01
    to = lambda t: t.permute(0, 2, 1, 3).reshape(B, T, 256)       # noqa: E731
    _check(f"sam_self_attn B={B} T={T}", (out.double() - to(o)).abs(), to(bound))


@pytest.mark.parametrize("rows,mean,std", [(1, 0.0, 1.0), (7, 0.0, 1.0), (8, 0.0, 1.0), (9, 0.0, 1.0), (3 * 4096 * 4, 0.0, 1.0),
                                           (1000, 50.0, 0.05), (1000, 50.0, 0.5), (1000, -3.0, 0.02)])
def test_sam_ln2d_gelu(lib, rows, mean, std):
    """LayerNorm2d (eps 1e-6) + erf-GELU over 64-channel bf16 pixel rows, including rows with a large mean and a small spread"""
    g = _g(4000 + rows + int(mean))
    x = (torch.randn(rows, 64, generator=g) * std + mean).bfloat16().cuda()
    gam = (1 + 0.2 * torch.randn(64, generator=g)).cuda()
    bet = (0.3 * torch.randn(64, generator=g)).cuda()
    y = torch.full((rows, 64), float("nan"), dtype=torch.bfloat16, device="cuda")
    lib.call("sam6d_sam_ln2d_gelu", x, gam, bet, rows, y)
    xd, gd, bd = x.double(), gam.double(), bet.double()
    mu = xd.mean(1, keepdim=True)
    dv = xd - mu
    var = dv.pow(2).mean(1, keepdim=True)
    r = 1 / torch.sqrt(var + 1e-6)
    z = gd * dv * r + bd
    ref = 0.5 * z * (1 + torch.erf(z / math.sqrt(2)))
    # mean: 64 terms summed pairwise then by a 5-level warp tree (gamma_6, charged 7u); x - mean: one more rounding
    e_mu = 7 * U * xd.abs().mean(1, keepdim=True)
    e_d = e_mu + U * dv.abs()
    # variance: the error of every deviation enters twice, products and tree (gamma_7, charged 8u)
    e_var = 2 * dv.abs().mean(1, keepdim=True) * e_mu + e_mu ** 2 + 8 * U * var
    # rsqrtf 2 ulp (4u relative), var + eps one rounding; half the relative error of the variance
    e_r = 0.5 * e_var / (var + 1e-6) + 6 * U
    # z = gamma (d rstd) + beta: two products and one sum
    e_z = gd.abs() * r * (e_d + dv.abs() * (e_r + 2 * U)) + U * z.abs()
    # GELU: slope <= 1.13, erff 2 ulp (<= 2^-22 absolute), three roundings; then one bf16 rounding of the result
    e_y = 1.13 * e_z + 0.5 * z.abs() * 2.0 ** -22 + 4 * U * ref.abs()
    bound = UB * (ref.abs() + e_y) + e_y
    _check(f"sam_ln2d_gelu rows={rows} mean={mean} std={std}", (y.double() - ref).abs(), bound)


@pytest.mark.parametrize("rows", [1, 4096])
def test_sam_pe_encode(lib, rows):
    """random-Fourier positional encoding: sin / cos of 2 pi ((2c - 1) G) with G drawn like the checkpoint's Gaussian matrix"""
    g = _g(5000 + rows)
    Gm = torch.randn(2, 128, generator=g)
    c = torch.rand(rows, 2, generator=g)
    corners = torch.tensor([[0.0, 1.0], [1.0, 0.0], [0.0, 0.0], [1.0, 1.0]])
    c[:min(rows, 4)] = corners[:min(rows, 4)]
    c_d, G_d = c.cuda(), Gm.cuda()
    out = torch.full((rows, 256), float("nan"), device="cuda")
    lib.call("sam6d_sam_pe_encode", c_d, G_d, rows, out)
    cd = 2 * c.double() - 1
    v = 2 * math.pi * (cd @ Gm.double())
    ref = torch.cat([torch.sin(v), torch.cos(v)], dim=1)
    # argument: 2c - 1 (<= u), the 2-term dot (two roundings), the fp32 2 pi (0.5 u) and its product: <= 5u of
    # 2 pi (|cx G0| + |cy G1|), |v| up to about 2 pi * 2 |G|; sin / cos are 1-Lipschitz; sinf / cosf 2 ulp (<= 2^-22)
    arg = 2 * math.pi * (cd.abs() @ Gm.double().abs())
    bound = (5 * U * arg + 2.0 ** -22).repeat(1, 2)
    print(f"sam_pe_encode: largest |argument| {v.abs().max().item():.1f}")
    _check(f"sam_pe_encode rows={rows}", (out.cpu().double() - ref).abs(), bound)
    # negative control: x and y exchanged
    if rows > 1:
        vw = 2 * math.pi * (cd.flip(1) @ Gm.double())
        assert _ratio((out.cpu().double() - torch.cat([torch.sin(vw), torch.cos(vw)], dim=1)).abs(), bound) > 1.0


# ================================================================================================== B. GEMM epilogues
def _gemm_bound(absdot, K, alpha, x, y, o, act, has_res, bf16_out, tc_acc=True):
    """fp32 accumulation of K bf16 products (2u each on the tensor cores), alpha * acc + bias (one fma), activation, residual add,
    optional bf16 rounding of the result"""
    e = 2 * K * U * abs(alpha) * absdot + U * x.abs()
    if act == 2:
        e = 1.13 * e + 0.5 * x.abs() * 2.0 ** -22 + 4 * U * y.abs()      # erf-GELU: slope <= 1.13, erff 2 ulp, three roundings
    if has_res:
        e = e + U * o.abs()
    if bf16_out:
        e = e + UB * (o.abs() + e)
    return e


def _act(x, act):
    if act == 1:
        return torch.relu(x)
    if act == 2:
        return 0.5 * x * (1 + torch.erf(x / math.sqrt(2)))
    return x


@pytest.mark.parametrize("odt", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("has_res", [False, True])
@pytest.mark.parametrize("has_bias", [False, True])
@pytest.mark.parametrize("act", [0, 1, 2])
@pytest.mark.parametrize("M,N,K", [(200, 130, 72), (4096, 256, 8), (333, 129, 200)])
def test_gemm_tma_epilogue_matrix(ops, M, N, K, act, has_bias, has_res, odt):
    """every EPI_DISPATCH instantiation of sam6d_gemm_tma.  K = 72 and 8 end in a partial (zero-filled) 64-wide k-block; N = 129
    makes ldc odd, which forces the single-element store path"""
    g = _g(M + N + K)
    alpha = 0.75
    A = torch.randn(M, K, generator=g).bfloat16().cuda()
    W = (torch.randn(N, K, generator=g) / math.sqrt(K)).bfloat16().cuda()
    bias = torch.randn(N, generator=g).cuda() if has_bias else None
    R = torch.randn(M, N, generator=g).to(odt).cuda() if has_res else None
    got = ops.gemm_tma(A, W, bias, residual=R, act=act, alpha=alpha, out_dtype=odt).double()
    Ad, Wd = A.double(), W.double()

    def ref_of(kk):
        x = alpha * (Ad[:, :kk] @ Wd[:, :kk].t()) + (bias.double() if has_bias else 0)
        y = _act(x, act)
        return x, y, y + (R.double() if has_res else 0)

    x, y, o = ref_of(K)
    bound = _gemm_bound(Ad.abs() @ Wd.abs().t(), K, alpha, x, y, o, act, has_res, odt == torch.bfloat16)
    _check(f"gemm_tma M={M} N={N} K={K} act={act} bias={has_bias} res={has_res} {odt}", (got - o).abs(), bound)
    # negative control: the product without its last, partial k-block
    assert _ratio((got - ref_of(K // 64 * 64)[2]).abs(), bound) > 1.0


@pytest.mark.parametrize("B,M,shared_res", [(1, 4096, True), (3, 4096, True), (3, 4096, False), (3, 1000, True), (2, 1000, False)])
def test_gemm_tma_batched_img_proj_views(ops, B, M, shared_res):
    """sam6d_gemm_tma_batched as the decoder's _img_proj calls it: one W shared by every problem (w_rpb = 0), a bias and a bf16
    residual shared by every problem (r_bs = 0) or per problem, bf16 out.  At M = 1000 a 128-row tile straddles two problems.
    C has 8 padding columns and one padding row per problem, which must keep their sentinel."""
    N, K, ldc = 128, 256, 136
    g = _g(6000 + B * 10 + M)
    A = torch.randn(B, M, K, generator=g).bfloat16().cuda()
    W = (torch.randn(N, K, generator=g) / 16).bfloat16().cuda()
    bias = torch.randn(N, generator=g).cuda()
    R = torch.randn(*((M, N) if shared_res else (B, M, N)), generator=g).bfloat16().cuda()
    out = torch.full((B, M + 1, ldc), 7.0, dtype=torch.bfloat16, device="cuda")
    ops.gemm_tma_batched(A, W, out[:, :M, :N], bias=bias, residual=R.expand(B, M, N))
    Ad, Wd = A.double(), W.double()
    x = Ad @ Wd.t() + bias.double()
    o = x + R.double()
    bound = _gemm_bound(Ad.abs() @ Wd.abs().t(), K, 1.0, x, x, o, 0, True, True)
    _check(f"gemm_tma_batched B={B} M={M} shared_res={shared_res}", (out[:, :M, :N].double() - o).abs(), bound)
    assert (out[:, :M, N:] == 7.0).all() and (out[:, M, :] == 7.0).all()


@pytest.mark.parametrize("C", [384, 768, 1024, 1536])
def test_gemm_bf16_dinov2_patch_embedding_views(ops, C):
    """sam6d_gemm_bf16 as DINOv2's patch embedding calls it: fp32 patches (K = 588 zero-padded to 592, rounded to bf16 in the
    kernel), bf16 W shared by the batch (sW = 0), a positional residual shared by the batch (sR = 0), C written from row 1 of a
    (B, 257, C) token buffer (sC = 257 C); row 0 (the class token) keeps its sentinel"""
    B, L, K, Kp = 6, 256, 588, 592
    g = _g(7000 + C)
    patches = torch.zeros(B * L, Kp)
    patches[:, :K] = torch.randn(B * L, K, generator=g)
    pw = torch.zeros(C, Kp)
    pw[:, :K] = torch.randn(C, K, generator=g) / math.sqrt(K)
    a, w = patches.cuda(), pw.bfloat16().cuda()
    pb, pos = torch.randn(C, generator=g).cuda(), torch.randn(L, C, generator=g).cuda()
    tok = torch.full((B, L + 1, C), 3.25, device="cuda")
    ops.gemm_tc(a.view(B, L, Kp), w, pb, residual=pos.expand(B, L, C), out=tok[:, 1:, :])
    Ad, Wd = a.bfloat16().double().view(B, L, Kp), w.double()
    x = Ad @ Wd.t() + pb.double()
    o = x + pos.double()
    bound = _gemm_bound(Ad.abs() @ Wd.abs().t(), Kp, 1.0, x, x, o, 0, True, False)
    _check(f"gemm_bf16 patch embedding C={C}", (tok[:, 1:].double() - o).abs(), bound)
    assert (tok[:, 0] == 3.25).all()


_DTC = {"f32": torch.float32, "bf16": torch.bfloat16}


@pytest.mark.parametrize("K", [8, 72])
@pytest.mark.parametrize("adt,wdt,odt", [("f32", "f32", "bf16"), ("f32", "bf16", "bf16"), ("bf16", "f32", "f32"), ("bf16", "f32", "bf16"),
                                         ("bf16", "bf16", "f32")])
def test_gemm_bf16_dtype_codes_and_k_tail(ops, adt, wdt, odt, K):
    """the operand / output dtype codes of sam6d_gemm_bf16 not covered elsewhere, with K inside one partial k-block"""
    M, N, alpha = 200, 300, 0.75
    g = _g(8000 + K)
    A = torch.randn(M, K, generator=g).cuda().to(_DTC[adt])
    W = (torch.randn(N, K, generator=g) / math.sqrt(K)).cuda().to(_DTC[wdt])
    bias, R = torch.randn(N, generator=g).cuda(), torch.randn(M, N, generator=g).cuda()
    got = ops.gemm_tc(A, W, bias, residual=R, relu=True, alpha=alpha, out_dtype=_DTC[odt]).double()
    Ad, Wd = A.bfloat16().double(), W.bfloat16().double()      # fp32 operands are rounded to bf16 (nearest) while staged
    x = alpha * (Ad @ Wd.t()) + bias.double()
    y = torch.relu(x)
    o = y + R.double()
    bound = _gemm_bound(Ad.abs() @ Wd.abs().t(), K, alpha, x, y, o, 1, True, odt == "bf16")
    _check(f"gemm_bf16 A={adt} W={wdt} C={odt} K={K}", (got - o).abs(), bound)
    # negative control (fp32 output, where the bound is not dominated by a bf16 rounding): fp32 W truncated to bf16 instead of
    # rounded to nearest
    if wdt == "f32" and odt == "f32":
        Wt = (W.view(torch.int32) & -65536).view(torch.float32).double()
        wrong = torch.relu(alpha * (Ad @ Wt.t()) + bias.double()) + R.double()
        assert _ratio((got - wrong).abs(), bound) > 1.0


# ================================================================================================== C. DINOv2 descriptor tail
def _attn_operands(B, H, S, seed, peaked=True):
    g = _g(seed)
    C = 64 * H
    q, k, v = (torch.randn(B, S, C, generator=g) for _ in range(3))
    if peaked:
        q[:, ::16] *= 6.0                                         # every 16th query: peaked softmax rows
    qk = torch.cat([q, k], dim=-1).view(B * S, 2 * C).bfloat16().cuda()
    vb = v.bfloat16().cuda()
    sep = lambda t: t.double().view(B, S, H, 64).permute(0, 2, 1, 3)      # noqa: E731
    return qk, vb, sep(qk.view(B, S, 2 * C)[..., :C]), sep(qk.view(B, S, 2 * C)[..., C:]), sep(vb)


def _attn_bounds(qh, kh, vh, scale, nkeys):
    """fp64 attention over the first `nkeys` keys + the bounds of attn_tc_ex's bf16 output and fp32 lse"""
    s = qh @ kh[:, :, :nkeys].transpose(-1, -2) * scale
    o, pv, xr = _softmax_terms(s, vh[:, :, :nkeys])
    lse = torch.logsumexp(s, dim=-1)
    # logits: 64 bf16 products on the tensor cores (2u each), scale = 1/8 exact; the row max carries the same error
    d = (128 * U * (qh.abs() @ kh[:, :, :nkeys].abs().transpose(-1, -2)) * scale).amax(-1)
    eta = 2 * d + _exp_err(xr)
    # lse = max + __logf(sum): the max's error, the sum's relative error (exp, a 64-term chain + 2 quad levels), __logf 3 ulp
    # (<= 2^-19 absolute for a sum below 256), one final rounding
    e_lse = d + eta + 66 * U + 2.0 ** -19 + U * lse.abs()
    # out: P is rounded to bf16 for the P V product (ub relative per weight), logit / exp error, fp32 row sum (66 terms) and
    # the P V accumulation on the tensor cores (2u x keys), 1 / sum; then one bf16 rounding
    e32 = pv * (UB + 2 * eta + (2 * 66 + 2 * nkeys + 2) * U)[..., None]
    e_out = e32 + UB * (o.abs() + e32)
    return s, o, lse, e_out, e_lse


@pytest.mark.parametrize("B", [1, 7])
@pytest.mark.parametrize("H", [6, 12, 16, 24])
def test_dinov2_attention_split(ops, H, B):
    """the 257-token attention of DINOv2 (ViT-S / B / L / g: 6 / 12 / 16 / 24 heads of 64): attn_tc_ex over keys 0..255 with
    its log-sum-exp, then attn_merge_key folds in key 256"""
    S, C, scale = 257, 64 * H, 0.125
    qk, vb, qh, kh, vh = _attn_operands(B, H, S, seed=9000 + 10 * H + B)
    vt = torch.zeros(B * H * 64, 272, dtype=torch.bfloat16, device="cuda")
    vt[:, :S] = vb.view(B, S, H, 64).permute(0, 2, 3, 1).reshape(B * H * 64, S)
    out, lse = ops.attn_tc_ex(qk, 0, qk, C, vt, B, H, S, S - 1, 64, scale, k_brows=S, k_row0=0, v_col0=0, want_lse=True)
    s256, o256, lse_ref, e_out, e_lse = _attn_bounds(qh, kh, vh, scale, S - 1)
    to = lambda t: t.permute(0, 2, 1, 3).reshape(B * S, C)        # noqa: E731
    _check(f"attn_tc_ex lse H={H} B={B}", (lse.double() - lse_ref).abs(), e_lse)
    _check(f"attn_tc_ex out (256 keys) H={H} B={B}", (out.double() - to(o256)).abs(), to(e_out))
    ops.attn_merge_key(qk, 0, qk, C, S, S - 1, vt, S - 1, lse, B, H, S, scale, out)
    s_all = qh @ kh.transpose(-1, -2) * scale
    o257 = torch.softmax(s_all, dim=-1) @ vh
    vc, sc = vh[:, :, S - 1], s_all[..., S - 1]                  # (B,H,64), (B,H,S)
    # merge: the 257th logit (64 products, 5-level warp tree: gamma_7, charged 8u), two __expf, one division, three products /
    # sums; the weight a = w_p / (w_p + w_c) moves by at most its logits' error; the bf16 input o_256 enters with weight a <= 1
    d_c = 8 * U * (qh.abs() * kh[:, :, S - 1:].abs()).sum(-1) * scale
    eps = e_lse + d_c + 2 * _exp_err((lse_ref - sc).abs()) + 6 * U
    e32 = e_out + (o256.abs() + vc[:, :, None].abs()) * eps[..., None]
    bound = e32 + UB * (o257.abs() + e32)
    _check(f"attn_merge_key out (257 keys) H={H} B={B}", (out.double() - to(o257)).abs(), to(bound))
    # negative control: the 257th key left out
    assert _ratio((out.double() - to(o256)).abs(), to(bound)) > 1.0


def test_attn_tc_ex_key_window(ops):
    """attn_tc_ex over a window of keys that starts inside the batch: K rows [b * k_brows + k_row0, + Sk), V^T columns
    [v_col0, + Sk); v_col0 % 8 == 0 (a TMA box starts on a 16-byte boundary), k_brows >= k_row0 + Sk"""
    B, H, S, Sk, k_row0, v_col0, scale = 3, 6, 257, 200, 5, 40, 0.125
    C = 64 * H
    qk, vb, qh, kh, vh = _attn_operands(B, H, S, seed=9500)
    g = _g(9501)
    vt = torch.randn(B * H * 64, 256, generator=g).bfloat16().cuda()         # finite everywhere, padding keys included
    out, lse = ops.attn_tc_ex(qk, 0, qk, C, vt, B, H, S, Sk, 64, scale, k_brows=S, k_row0=k_row0, v_col0=v_col0, want_lse=True)
    kw = kh[:, :, k_row0:k_row0 + Sk]
    vw = vt.double().view(B, H, 64, 256)[..., v_col0:v_col0 + Sk].transpose(-1, -2)
    _, o, lse_ref, e_out, e_lse = _attn_bounds(qh, kw, vw, scale, Sk)
    to = lambda t: t.permute(0, 2, 1, 3).reshape(B * S, C)        # noqa: E731
    _check("attn_tc_ex window lse", (lse.double() - lse_ref).abs(), e_lse)
    _check("attn_tc_ex window out", (out.double() - to(o)).abs(), to(e_out))
    # negative control: the window taken from key 0
    _, o0, _, _, _ = _attn_bounds(qh, kh[:, :, :Sk], vw, scale, Sk)
    assert _ratio((out.double() - to(o0)).abs(), to(e_out)) > 1.0


def _patch_mask(counts, P, G, patch, g):
    """(P, G*patch, G*patch) 0/1 mask whose (gy, gx) block has exactly counts[p, gy*G + gx] pixels set, at random places"""
    n = patch * patch
    rank = torch.rand(P, G * G, n, generator=g).argsort(-1).argsort(-1)
    blk = (rank < counts[..., None]).float().view(P, G, G, patch, patch)
    return blk.permute(0, 1, 3, 2, 4).reshape(P, G * patch, G * patch).contiguous()


@pytest.mark.parametrize("C", [384, 768, 1024, 1536])
def test_masked_patch_normalize(lib, C):
    """patch tokens read with the model's strides (row C, batch 257 C, base one row in: the class token is skipped); a token
    survives when more than half of its 14 x 14 mask pixels are set; survivors are L2-normalised with a 1e-12 floor"""
    P, G, patch, S = 3, 16, 14, 257
    g = _g(10000 + C)
    tok = torch.randn(P, S, C, generator=g)
    tok[:, 0] = float("nan")                                     # the class token must not be read
    counts = torch.randint(0, 197, (P, G * G), generator=g)
    counts[0, :4] = torch.tensor([98, 99, 98, 99])               # mean exactly 0.5: dropped; 99 / 196: kept
    counts[1, :4] = torch.tensor([0, 196, 97, 100])
    counts[2, :2] = torch.tensor([99, 196])
    tok[2, 1:3] = 0.0                                            # kept tokens with all-zero features -> zeros, not NaN
    pmask = _patch_mask(counts, P, G, patch, g)
    keep = counts > 98
    x = tok[:, 1:].double()
    ref = torch.where(keep[..., None], torch.nn.functional.normalize(x, dim=-1, eps=1e-12), torch.zeros_like(x))
    # f32: sum of squares over C/32-term fma chains + a 5-level warp tree, sqrtf, 1 / n and one product (IEEE, 3 roundings);
    # the square root halves the relative error of the sum
    e32 = ref.abs() * (((C / 32 + 5) / 2 + 3) * U) * 1.01
    tok_d, pm_d = tok.cuda(), pmask.cuda()
    base = tok_d[:, 1:]
    for want_f32, want_bf16, want_valid in itertools.product([True, False], repeat=3):
        f32 = torch.full((P, G * G, C), float("nan"), device="cuda") if want_f32 else None
        b16 = torch.full((P, G * G, C), float("nan"), dtype=torch.bfloat16, device="cuda") if want_bf16 else None
        val = torch.full((P, G * G), 7, dtype=torch.uint8, device="cuda") if want_valid else None
        args = (base, C, S * C, pm_d, P, G, patch, C, 0.5, f32, b16,
                val)
        if not (want_f32 or want_bf16):
            with pytest.raises(lib.Sam6dError, match="invalid argument"):
                lib.call("sam6d_masked_patch_normalize", *args)
            continue
        lib.call("sam6d_masked_patch_normalize", *args)
        tag = f"masked_patch_normalize C={C} f32={want_f32} bf16={want_bf16} valid={want_valid}"
        if want_f32:
            _check(tag + " f32", (f32.cpu().double() - ref).abs(), e32)
        if want_bf16:
            _check(tag + " bf16", (b16.cpu().double() - ref).abs(), e32 + UB * (ref.abs() + e32))
        if want_valid:
            assert torch.equal(val.cpu(), keep.to(torch.uint8))


def _appearance_ref(sim, qvalid, thred):
    """MaskedPatch_MatrixSimilarity.compute_straight / compute_visible_ratio (ism_oracle) restated on a given similarity matrix:
    appe = clamp(sum_q max_r sim / (#valid queries + 1e-6), 0, 1); vis = #(max_q sim > thred, != 0) / (#(max_q sim != 0) + 1e-6)"""
    rmax = sim.amax(-1)
    A = rmax.sum(-1)
    Q = qvalid.double().sum(-1)
    appe = (A / (Q + 1e-6)).clamp(0, 1)
    cmax = sim.amax(1)
    vis = ((cmax > thred) & (cmax != 0)).double().sum(-1) / ((cmax != 0).double().sum(-1) + 1e-6)
    return appe, vis, rmax.abs().sum(-1), Q


def test_appearance_restatement_matches_oracle():
    """the restated formulas equal ism_oracle's on similarity matrices built from masked patch descriptors"""
    g = _g(11000)
    qp, rp = torch.randn(3, 40, 16, generator=g, dtype=F64), torch.randn(3, 40, 16, generator=g, dtype=F64)
    qp[:, ::5] = 0
    rp[:, ::3] = 0
    qp, rp = torch.nn.functional.normalize(qp, dim=-1), torch.nn.functional.normalize(rp, dim=-1)
    appe, vis, _, _ = _appearance_ref(qp @ rp.transpose(1, 2), qp.abs().amax(-1) > 0, 0.5)
    # the oracle's count_nonzero(...) + 1e-6 are float32 tensors: one fp32 rounding of each denominator (and of the ratio)
    torch.testing.assert_close(appe, io.appearance_score(qp, rp), rtol=2 * U, atol=0)
    torch.testing.assert_close(vis, io.visible_ratio(qp, rp, 0.5).double(), rtol=4 * U, atol=0)


@pytest.mark.parametrize("N", [100, 255, 256])
def test_appearance_reduce(lib, N):
    """appearance score and visible ratio over a strided similarity stack (sim_ld > N, sim_bs > N sim_ld): rows whose every
    similarity is negative, reference columns that are exactly zero, a proposal without a valid query patch"""
    P, ld, thred = 6, N + 5, 0.5
    g = _g(12000 + N)
    body = torch.rand(P, N, N, generator=g) * 2 - 1
    qvalid = (torch.rand(P, N, generator=g) < 0.8).to(torch.uint8)
    body[0, :10] = -torch.rand(10, N, generator=g) - 0.01          # all-negative query rows
    body[1] = -torch.rand(N, N, generator=g) - 0.01                # every similarity negative: the score clamps at 0
    qvalid[1] = 1
    body[2, :, ::7] = 0.0                                          # reference columns that are exactly zero
    body[3] = 0.0
    qvalid[3] = 0                                                  # no valid query patch
    body[4] = 0.6 + 0.4 * torch.rand(N, N, generator=g)            # everything matches
    qvalid[4] = 1
    body = body * qvalid[..., None]                                # masked query patches are zero rows, as the model makes them
    body[(body - thred).abs() < 1e-4] = 0.25                       # nothing within fp32 noise of the threshold
    sim = torch.full((P, N + 3, ld), 5.0)                          # padding rows / columns hold a value that would win every max
    sim[:, :N, :N] = body
    sim_d, qv_d = sim.cuda(), qvalid.cuda()
    appe = torch.full((P,), float("nan"), device="cuda")
    vis = torch.full((P,), float("nan"), device="cuda")
    lib.call("sam6d_appearance_reduce", sim_d, ld, (N + 3) * ld, P, N, qv_d, thred, appe, vis)
    a_ref, v_ref, abs_sum, Q = _appearance_ref(body.double(), qvalid, thred)
    # appe: one row max per thread (exact), a 5-level warp tree and 8 partials (gamma_13), + 1e-6, one division; clamp is
    # 1-Lipschitz.  vis: integer counts, + 1e-6 and one division
    e_a = 13 * U * abs_sum / (Q + 1e-6) + 3 * U * a_ref.abs()
    e_v = 3 * U * v_ref.abs()
    _check(f"appearance_reduce N={N} appe", (appe.cpu().double() - a_ref).abs(), e_a)
    _check(f"appearance_reduce N={N} vis", (vis.cpu().double() - v_ref).abs(), e_v)
    print(f"N={N}: appe {[round(x, 4) for x in appe.tolist()]}, vis {[round(x, 4) for x in vis.tolist()]}")
    assert appe[1].item() == 0.0 and appe[3].item() == 0.0 and vis[3].item() == 0.0 and vis[1].item() == 0.0
