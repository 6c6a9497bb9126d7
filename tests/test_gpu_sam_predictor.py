"""GPU: SamPredictor and the kernels behind its prompt paths (sam6d_b200/sam_amg.py, csrc/sam_dec.cu): the mask-prompt embedding,
the attention kernels up to 32 tokens, the mask-token range of the hypernetwork product and the logit upscaling, each against a
float64 evaluation; then every case of tests/golden/sam_predictor.pt (outputs of the reference SamPredictor) end to end, and the
predictor against the automatic mask generator on the shapes they share.

Notation as tests/test_gpu_ism_kernels.py: u = 2^-24, ub = 2^-8, a chain of n fp32 roundings is charged n u."""
import ctypes
import math
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import sam_dec_oracle as so          # noqa: E402
from oracle import sam_predictor_oracle as sp    # noqa: E402
from sam6d_b200 import synth                     # noqa: E402

U = 2.0 ** -24
F64 = torch.float64


@pytest.fixture(scope="module")
def lib():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from sam6d_b200 import _lib
    return _lib


def _p(t):
    return ctypes.c_void_p(t.data_ptr() if t is not None else 0)


def _s():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _check(name, err, bound):
    err, bound = err.to(F64), bound.to(F64)
    assert torch.isfinite(err).all(), f"{name}: non-finite output"
    r = (err / bound.clamp_min(1e-300)).max().item()
    print(f"{name}: max error / bound = {r:.3g}  (max error {err.max().item():.3g})")
    assert r <= 1.0, f"{name}: error exceeds its bound by {r:.3g}x"


def _build_sam(seed=1):
    from sam6d_b200.sam_amg import MaskDecoder, PromptEncoder, Sam
    sd = so.make_state_dict(seed=seed)
    enc = torch.nn.Module()
    enc.img_size = 1024
    sam = Sam(enc, PromptEncoder(), MaskDecoder()).cuda().eval()
    sam.prompt_encoder.load_state_dict({k[len("prompt_encoder."):]: v for k, v in sd.items() if k.startswith("prompt_encoder.")}, strict=True)
    sam.mask_decoder.load_state_dict({k[len("mask_decoder."):]: v for k, v in sd.items() if k.startswith("mask_decoder.")}, strict=True)
    return sd, sam


# ================================================================================================== mask-prompt embedding
def _ln_gelu_f64(x, e, w, b):
    """LayerNorm2d (eps 1e-6) + GELU over dim 1 in fp64, with a first-order bound on the error of the fp32 kernel given an input
    error bound e (same shape as x): mean and variance of perturbed inputs, the division by sigma, the affine map, erf GELU
    (|GELU'| <= 1.13, erff 2 ulp and three roundings)"""
    n = x.shape[1]
    mu = x.mean(1, keepdim=True)
    d = x - mu
    var = d.pow(2).mean(1, keepdim=True)
    sig = torch.sqrt(var + 1e-6)
    z = d / sig
    E = e.amax(1, keepdim=True)
    e_mu = E + n * U * x.abs().amax(1, keepdim=True)
    e_var = 2 * d.abs().mean(1, keepdim=True) * (E + e_mu) + (n + 3) * U * var
    e_sig = e_var / (2 * sig * sig) * sig + 2 * U * sig
    e_z = (e + e_mu) / sig + z.abs() * e_sig / sig + 2 * U * z.abs()
    y = w[None, :, None, None] * z + b[None, :, None, None]
    e_y = w.abs()[None, :, None, None] * e_z + 2 * U * (w.abs()[None, :, None, None] * z.abs() + b.abs()[None, :, None, None])
    g = torch.nn.functional.gelu(y)
    return g, 1.13 * e_y + 8 * U * g.abs() + 4 * U * y.abs()


def _mask_embed_f64(sd, m):
    """mask_downscaling in fp64 -> (out (B,256,64,64), bound)"""
    p = {k[len("prompt_encoder.mask_downscaling."):]: v.double() for k, v in sd.items() if k.startswith("prompt_encoder.mask_downscaling.")}
    conv = torch.nn.functional.conv2d
    m = m.double()
    a = conv(m, p["0.weight"], p["0.bias"], stride=2)
    e_a = 5 * U * conv(m.abs(), p["0.weight"].abs(), p["0.bias"].abs(), stride=2)
    g1, e_g1 = _ln_gelu_f64(a, e_a, p["1.weight"], p["1.bias"])
    h = conv(g1, p["3.weight"], p["3.bias"], stride=2)
    e_h = conv(e_g1, p["3.weight"].abs(), stride=2) + 17 * U * conv(g1.abs(), p["3.weight"].abs(), p["3.bias"].abs(), stride=2)
    g2, e_g2 = _ln_gelu_f64(h, e_h, p["4.weight"], p["4.bias"])
    o = conv(g2, p["6.weight"], p["6.bias"])
    e_o = conv(e_g2, p["6.weight"].abs()) + 17 * U * conv(g2.abs(), p["6.weight"].abs(), p["6.bias"].abs())
    return o, 2 * e_o                                                     # x 2: the analysis is first order


@pytest.mark.parametrize("B", [1, 3])
def test_sam_mask_embed_against_fp64(lib, B):
    """sam6d_sam_mask_embed on random logits of +-20 (earlier predictions) and smooth ones, against mask_downscaling in fp64"""
    sd, sam = _build_sam()
    g = torch.Generator().manual_seed(70 + B)
    m = torch.cat([(torch.rand(B, 1, 256, 256, generator=g) * 40 - 20), sp.smooth_logits(B)], dim=0).contiguous()
    n = m.shape[0]
    got_view = sam.prompt_encoder.embed_masks(m.cuda())
    assert got_view.shape == (n, 256, 64, 64) and got_view.permute(0, 2, 3, 1).is_contiguous()      # a view of the token rows
    ref, bound = _mask_embed_f64(sd, m)
    _check(f"sam_mask_embed B={n}", (got_view.cpu().double() - ref).abs(), bound)
    # negative control: the two 2x2 convolutions with the kernel's row/column order swapped must fail the bound
    wrong, _ = _mask_embed_f64(sd, m.transpose(-1, -2))
    assert ((got_view.cpu().double() - wrong.transpose(-1, -2)).abs() / bound).max() > 1.0


# ================================================================================================== attention up to 32 tokens
def _softmax_terms(s, v):
    p = torch.softmax(s, dim=-1)
    return p @ v, p @ v.abs(), (s.amax(-1) - s.amin(-1))


def _exp_err(xr):
    return (2.0 + 1.173 * xr) * 2 * U + U * xr


TS = [5, 8, 9, 16, 27, 32]


@pytest.mark.parametrize("shared", [True, False])
@pytest.mark.parametrize("T", TS)
def test_sam_tok2img_attn_up_to_32_tokens(lib, T, shared):
    """tokens in CTAs of at most 8: the bound of tests/test_gpu_ism_kernels.py (per chunk the same arithmetic)"""
    B, L = 3, 4096
    g = torch.Generator().manual_seed(500 + T)
    Bk = 1 if shared else B
    Q = (torch.randn(B, T, 128, generator=g) * 8).cuda()
    K = torch.randn(Bk, L, 128, generator=g).bfloat16().cuda()
    V = torch.randn(Bk, L, 128, generator=g).bfloat16().cuda()
    out = torch.full((B, T, 128), float("nan"), device="cuda")
    lib.call("sam6d_sam_tok2img_attn", _p(Q), _p(K), _p(V), ctypes.c_longlong(0 if shared else L * 128), B, T, L, _p(out), _s())
    qh = Q.double().view(B, T, 8, 16).permute(0, 2, 1, 3)
    kh = K.double().view(Bk, L, 8, 16).permute(0, 2, 1, 3)
    vh = V.double().view(Bk, L, 8, 16).permute(0, 2, 1, 3)
    s = qh @ kh.transpose(-1, -2) * 0.25
    o, pv, xr = _softmax_terms(s, vh)
    d = 16 * U * ((qh.abs() @ kh.abs().transpose(-1, -2)) * 0.25).amax(-1)
    nn_ = math.ceil(L / 16) + 16 + math.ceil(L / 256) + 13 + 1
    bound = pv * (2 * (2 * d + _exp_err(xr)) + nn_ * U)[..., None] * 1.01
    to = lambda t: t.permute(0, 2, 1, 3).reshape(B, T, 128)       # noqa: E731
    _check(f"sam_tok2img_attn T={T} shared={shared}", (out.double() - to(o)).abs(), to(bound))


@pytest.mark.parametrize("T", TS)
def test_sam_img2tok_attn_up_to_32_tokens(lib, T):
    B, L = 3, 4096
    g = torch.Generator().manual_seed(600 + T)
    Q = torch.randn(B, L, 128, generator=g).bfloat16().cuda()
    Kt = (torch.randn(B, T, 128, generator=g) * 5).cuda()
    Vt = torch.randn(B, T, 128, generator=g).cuda()
    out = torch.full((B, L, 128), float("nan"), dtype=torch.bfloat16, device="cuda")
    lib.call("sam6d_sam_img2tok_attn", _p(Q), ctypes.c_longlong(L * 128), _p(Kt), _p(Vt), B, T, L, _p(out), _s())
    qh = Q.double().view(B, L, 8, 16).permute(0, 2, 1, 3)
    kh = Kt.double().view(B, T, 8, 16).permute(0, 2, 1, 3)
    vh = Vt.double().view(B, T, 8, 16).permute(0, 2, 1, 3)
    s = qh @ kh.transpose(-1, -2) * 0.25
    o, pv, xr = _softmax_terms(s, vh)
    d = 16 * U * ((qh.abs() @ kh.abs().transpose(-1, -2)) * 0.25).amax(-1)
    e32 = pv * (2 * (2 * d + _exp_err(xr)) + (2 * T + 3) * U)[..., None] * 1.01
    bound = 2.0 ** -8 * (o.abs() + e32) + e32
    to = lambda t: t.permute(0, 2, 1, 3).reshape(B, L, 128)      # noqa: E731
    _check(f"sam_img2tok_attn T={T}", (out.double() - to(o)).abs(), to(bound))


@pytest.mark.parametrize("T", TS)
def test_sam_self_attn_up_to_32_tokens(lib, T):
    B = 5
    g = torch.Generator().manual_seed(700 + T)
    q, k, v = ((torch.randn(B, T, 256, generator=g) * 1.5).cuda() for _ in range(3))
    out = torch.full((B, T, 256), float("nan"), device="cuda")
    lib.call("sam6d_sam_self_attn", _p(q), _p(k), _p(v), B, T, _p(out), _s())
    sep = lambda t: t.double().view(B, T, 8, 32).permute(0, 2, 1, 3)      # noqa: E731
    qh, kh, vh = sep(q), sep(k), sep(v)
    scale = 1 / math.sqrt(32)
    s = qh @ kh.transpose(-1, -2) * scale
    o, pv, xr = _softmax_terms(s, vh)
    d = (6 * U * ((qh.abs() @ kh.abs().transpose(-1, -2)) * scale) + 2 * U * s.abs()).amax(-1)
    bound = pv * (2 * (2 * d + _exp_err(xr)) + (2 * T + 2) * U)[..., None] * 1.01
    to = lambda t: t.permute(0, 2, 1, 3).reshape(B, T, 256)       # noqa: E731
    _check(f"sam_self_attn T={T}", (out.double() - to(o)).abs(), to(bound))


def test_attention_kernels_refuse_more_than_32_tokens(lib):
    q = torch.zeros(1, 33, 256, device="cuda")
    with pytest.raises(lib.Sam6dError, match="invalid argument"):
        lib.call("sam6d_sam_self_attn", _p(q), _p(q), _p(q), 1, 33, _p(q), _s())
    K = torch.zeros(4096, 128, dtype=torch.bfloat16, device="cuda")
    with pytest.raises(lib.Sam6dError, match="invalid argument"):
        lib.call("sam6d_sam_tok2img_attn", _p(q), _p(K), _p(K), ctypes.c_longlong(0), 1, 33, 4096, _p(q), _s())
    with pytest.raises(lib.Sam6dError, match="invalid argument"):
        lib.call("sam6d_sam_img2tok_attn", _p(K), ctypes.c_longlong(0), _p(q), _p(q), 1, 33, 4096, _p(K), _s())


# ================================================================================================== mask-token range, upscaling
def test_mask_dot_range_bit_identical(lib):
    B, G = 3, 64
    g = torch.Generator().manual_seed(9)
    up = torch.randn(B * G * G * 4, 128, generator=g).bfloat16().cuda()
    hyper = torch.randn(B, 4, 32, generator=g).cuda()
    S = 4 * G
    m3 = torch.empty(B, 3, S, S, device="cuda")
    lib.call("sam6d_sam_mask_dot", _p(up), _p(hyper), B, G, _p(m3), _s())
    r13 = torch.empty(B, 3, S, S, device="cuda")
    lib.call("sam6d_sam_mask_dot_range", _p(up), _p(hyper), B, G, 1, 3, _p(r13), _s())
    assert torch.equal(m3, r13)
    r04 = torch.empty(B, 4, S, S, device="cuda")
    lib.call("sam6d_sam_mask_dot_range", _p(up), _p(hyper), B, G, 0, 4, _p(r04), _s())
    r01 = torch.empty(B, 1, S, S, device="cuda")
    lib.call("sam6d_sam_mask_dot_range", _p(up), _p(hyper), B, G, 0, 1, _p(r01), _s())
    assert torch.equal(r01[:, 0], r04[:, 0]) and torch.equal(r13, r04[:, 1:])
    for m0, nm in ((0, 5), (3, 2), (-1, 1), (0, 0)):
        with pytest.raises(lib.Sam6dError, match="invalid argument"):
            lib.call("sam6d_sam_mask_dot_range", _p(up), _p(hyper), B, G, m0, nm, _p(r04), _s())


@pytest.mark.parametrize("size", [(480, 640), (640, 480), (37, 1000)])
def test_mask_upscale_against_postprocess_masks(lib, size):
    """sam6d_sam_mask_upscale against Sam.postprocess_masks in fp64.  Bound: each of the two bilinear stages computes its source
    coordinate (<= 256, <= 1024) with two fp32 roundings, which moves an interpolation weight by <= 3 u coord and the value by
    that times the 2 max|low| spread of the neighbours; plus 6 u max|low| per stage for the weighted sums"""
    _, sam = _build_sam()
    H, W = size
    ih, iw = so.preprocess_shape(H, W)
    low = torch.cat([sp.smooth_logits(11, 3), torch.rand(2, 1, 256, 256, generator=torch.Generator().manual_seed(3)) * 40 - 20])
    low = low.view(1, 5, 256, 256)
    ref = so.postprocess_masks(low.double(), (ih, iw), (H, W))
    got = sam.postprocess_masks(low.cuda(), (ih, iw), (H, W))
    assert got.shape == (1, 5, H, W)
    mx = low.abs().flatten(2).amax(-1).double()[..., None, None]
    bound = mx * U * (2 * 3 * 256 * 2 + 2 * 3 * 1024 * 2 + 12)
    _check(f"sam_mask_upscale {size}", (got.cpu().double() - ref).abs(), bound.expand_as(ref))
    bits = sam.binarize_masks(low.cuda(), (ih, iw), (H, W))
    assert bits.dtype == torch.bool and torch.equal(bits, got > sam.mask_threshold)


# ================================================================================================== the fixture's cases end to end
@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "sam_predictor.pt"), weights_only=False)


@pytest.fixture(scope="module")
def predictor(gold):
    from sam6d_b200.sam_amg import SamPredictor
    sd, sam = _build_sam(gold["meta"]["seed"])
    feat = synth.make_image_embedding(seed=gold["meta"]["seed"])
    assert feat.double().sum().item() == gold["feat_checksum"]
    p = SamPredictor(sam)
    p.features = feat.cuda()
    p.image_pe_rows = sam.prompt_encoder.dense_pe_rows()
    p.is_image_set = True
    return sd, feat, p


def _set_size(p, size):
    p.original_size, p.input_size = size, so.preprocess_shape(*size)


@pytest.mark.parametrize("size", [(480, 640), (640, 480)])
def test_predictor_cases_match_reference(gold, predictor, size):
    """low-res logits (rel rms < 3e-2, signs > 0.99) and IoU (|d| < 2e-2) against the reference's, the bars of
    test_gpu_sam_dec.py's decoder test; the thresholded full-size masks against the reference's at IoU >= 0.98.  The full-size
    masks (and case 5's mask input) come from the pinned oracle, recomputed here on the host CPU: it reproduces the fixture bit for
    bit on the CPU that made it (test_sam_predictor_cpu.py), and here within float rounding of another CPU's kernels."""
    sd, feat, p = predictor
    _set_size(p, size)
    ref_all = sp.run_cases(sd, feat, size)
    g = gold["sizes"][size]
    for name, c in sp.make_cases(size).items():
        rm, _, ro = ref_all[name]
        ri, rl = g[name]["iou"], g[name]["low_sub"]
        assert ((ro[..., ::8, ::8] - rl).pow(2).mean().sqrt() / rl.pow(2).mean().sqrt()).item() < 1e-4, name
        kw = sp.resolve_kwargs(name, c["kwargs"], ref_all["click"])
        if c["api"] == "predict_torch":
            b = p.transform.apply_boxes_torch(torch.as_tensor(kw["boxes"], dtype=torch.float, device="cuda"), size)
            m, i, l = (t.cpu() for t in p.predict_torch(None, None, boxes=b, multimask_output=kw["multimask_output"]))
        else:
            m, i, l = (torch.as_tensor(a) for a in p.predict(**kw))
        assert m.shape == rm.shape and i.shape == ri.shape and l.shape == ro.shape, name
        l = l[..., ::8, ::8]
        rel = ((l - rl).pow(2).mean().sqrt() / rl.pow(2).mean().sqrt()).item()
        sign = ((l > 0) == (rl > 0)).float().mean().item()
        ierr = (i - ri).abs().max().item()
        mb, rb = (m > 0, rm > 0) if kw.get("return_logits") else (m, rm)
        inter = (mb & rb).flatten(-2).sum(-1).double()
        union = (mb | rb).flatten(-2).sum(-1).double()
        miou = torch.where(union > 0, inter / union.clamp_min(1), torch.ones_like(union)).min().item()
        print(f"{size} {name:16s} rel rms {rel:.3e} sign {sign:.5f} max|iou - ref| {ierr:.3e} min mask IoU {miou:.4f}")
        assert rel < 3e-2 and sign > 0.99 and ierr < 2e-2 and miou >= 0.98, name


def test_one_click_matches_the_generator_bit_for_bit(gold, predictor):
    """one positive click: SamPredictor.predict_torch and CustomSamAutomaticMaskGenerator.process_batch run the same kernels at T = 7"""
    from sam6d_b200.sam_amg import CustomSamAutomaticMaskGenerator
    _, _, p = predictor
    size = (480, 640)
    _set_size(p, size)
    amg = CustomSamAutomaticMaskGenerator(p.model, points_per_side=8)
    amg.features, amg.image_pe_rows = p.features.clone(), p.image_pe_rows
    amg.original_size, amg.input_size = size, so.preprocess_shape(*size)
    pt = np.array([[333.0, 201.0]])
    _, _, _, low_g, iou_g, _ = amg.process_batch(pt)
    c = torch.as_tensor(p.transform.apply_coords(pt, size), dtype=torch.float, device="cuda")[None]
    _, iou_p, low_p = p.predict_torch(c, torch.ones(1, 1, dtype=torch.int, device="cuda"), multimask_output=True)
    assert torch.equal(low_p.reshape(3, 256, 256), low_g) and torch.equal(iou_p.reshape(-1), iou_g)


def test_image_embedding_same_as_generator_vit_b():
    """SamPredictor.set_image and the generator's set_image are one path: bit-identical features of a seeded ViT-B on 480 x 640"""
    from sam6d_b200.sam import VIT_CONFIGS
    from sam6d_b200.sam_amg import CustomSamAutomaticMaskGenerator, SamPredictor, sam_model_registry
    sam = sam_model_registry["vit_b"]("bf16").cuda().eval()
    sd = {"image_encoder." + k: v for k, v in synth.make_sam_state_dict(**VIT_CONFIGS["vit_b"], seed=1).items()}
    sd.update(synth.make_sam_decoder_state_dict(seed=1))
    sam.load_state_dict(sd, strict=True)
    frame = np.ascontiguousarray((synth.make_images(B=1, seed=3)[0, :, :480, :640].permute(1, 2, 0).clamp(-2, 2) * 60 + 128)
                                 .to(torch.uint8).numpy())
    amg = CustomSamAutomaticMaskGenerator(sam)
    f_g = amg.set_image(frame).clone()
    p = SamPredictor(sam)
    p.set_image(frame)
    assert p.is_image_set and p.original_size == (480, 640) and p.input_size == (768, 1024)
    assert torch.equal(p.get_image_embedding(), f_g)
    p.set_image(np.ascontiguousarray(frame[..., ::-1]), image_format="BGR")
    assert torch.equal(p.get_image_embedding(), f_g)
    masks, iou, low = p.predict(box=np.array([100, 80, 400, 300]), multimask_output=False)
    assert masks.shape == (1, 480, 640) and masks.dtype == np.bool_ and iou.shape == (1,) and low.shape == (1, 256, 256)
    p.reset_image()
    assert not p.is_image_set and p.features is None
