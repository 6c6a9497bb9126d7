"""GPU: the SAM image encoder's kernels (global and windowed rel-pos attention, the fp32 comparator attention, the encoder's
LayerNorms and row gathers) called directly, each against a float64 evaluation of the same operation in plain torch on the
operands rounded exactly as the kernel reads them; and the encoder's wiring, replayed stage by stage.

Every bound is derived from the kernel's arithmetic and written next to its check.  Notation: u = 2^-24 (fp32 unit roundoff),
ub = 2^-8 (bf16 unit roundoff: one round-to-nearest bf16 store moves a value by at most ub |x|), gamma_n ~ n u for a chain of n
fp32 roundings.  A tensor-core (wgmma) fp32 accumulation is charged 2u per added product: the accumulator may truncate rather
than round.  Documented accuracy of the math functions used: ex2.approx.f32 2 ulp of the result, __expf 2 + floor(|1.173 x|)
ulp, rsqrtf 2 ulp, erff 2 ulp; divisions are IEEE (nvcc's defaults).  An ulp of a result in [1, 2) is 2u, so "2 ulp" is a
relative error of at most 4u.

The attention kernels see logits s_j and values v_j; with p = softmax(s), pv = sum_j p_j |v_j| bounds every output channel's
sensitivity: a relative error eps_j on each weight p_j moves the output by at most 2 max_j |eps_j| pv (normalisation included),
and a relative error on every product of the P V sum by that error times pv.  A logit error ds_j is a relative weight error
of ds_j + max ds, which is the `2 * dlog` in every eta below.  Each check prints its largest error / bound ratio; where a bound
could hide a mistake, a deliberately wrong answer computed in torch must fail the same bound."""
import math
import types
from functools import partial

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

import _sam_encoder_ref as er                # noqa: E402
from oracle import sam_oracle as so          # noqa: E402
from sam6d_b200 import synth                 # noqa: E402

U = 2.0 ** -24          # fp32 unit roundoff
UB = 2.0 ** -8          # bf16 unit roundoff
F64 = torch.float64
EPS6 = float(np.float32(1e-6))     # the fp32 eps the encoder's LayerNorms receive
CONFIGS = [(80, 16), (64, 16), (64, 12)]     # (head dim, heads) of ViT-H, ViT-L, ViT-B
GRID, WS, WL, WN1 = 64, 14, 196, 208         # token grid, window size, tokens per window, keys rounded up to 16
SENT = -1232.0                               # a sentinel exactly representable in fp32 and bf16


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


def _f32(x):
    return float(np.float32(x))


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


class _Worst:
    """the largest error / bound ratio of one check over several chunks (heads, windows), reported once"""

    def __init__(self, name):
        self.name, self.r, self.e = name, 0.0, 0.0

    def add(self, err, bound):
        self.r = max(self.r, _ratio(err, bound))
        self.e = max(self.e, err.max().item())

    def check(self):
        print(f"{self.name}: max error / bound = {self.r:.3g}  (max error {self.e:.3g})")
        assert self.r <= 1.0, f"{self.name}: error exceeds its bound by {self.r:.3g}x"


class _Control:
    """a deliberately wrong answer: its largest |got - wrong| / bound over the chunks must exceed 1"""

    def __init__(self, name):
        self.name, self.r = name, 0.0

    def add(self, got, wrong, bound):
        self.r = max(self.r, ((got - wrong).abs() / bound.clamp_min(1e-300)).max().item())

    def check(self):
        print(f"  negative control {self.name}: max |got - wrong| / bound = {self.r:.3g}")
        assert self.r > 1.0, f"negative control {self.name} passes the bound ({self.r:.3g})"


def _maps(B, device="cuda"):
    from sam6d_b200.sam import ImageEncoderViT
    return ImageEncoderViT._index_maps(types.SimpleNamespace(_maps={}), B, GRID, WS, device)


# ================================================================================================== bounds of the attentions
def _out_bound(o, e32, odt):
    """the bound of a kernel whose fp32 result lies within e32 of o, stored as odt"""
    return e32 + UB * (o.abs() + e32) if odt == torch.bfloat16 else e32       # one output rounding


def _global_bound(s, mag, v, D):
    """sam6d_attn_global_tc_ex on logits s = scale q.k + q.Rh + q.Rw (float64, natural-log units), mag = the same sum over
    magnitudes, v the values -> (o, bound on the kernel's fp32 result)"""
    o, pv, xr = _softmax_terms(s, v)
    # logits, in natural-log units (the kernel works in log2 units: x = fmaf(S, sl2, th + tw), everything scaled by log2 e):
    #   S = q.k on the tensor cores (D products, 2u each); G_h = q.rel_h, G_w = q.rel_w the same (D-term wgmma of bf16 q against the
    #   bf16 tables); G * LOG2E one rounding each; sl2 = fp32(scale * LOG2E) one rounding; th + tw one; the fmaf one
    #   -> (2D + 4) u mag.  LOG2E itself is log2 e to within u: a common factor on all logits, i.e. a change of temperature that
    #   moves a weight by u |s - m| <= u xr relative.
    dlog = ((2 * D + 4) * U * mag).amax(-1)
    # p = ex2(x - m): the subtraction (u |x - m|, at most u xr in natural units) and ex2.approx (2 ulp = 4u).  ex2.approx.ftz flushes
    # results below 2^-126 to zero: at most 4096 * 2^-126 max|v| absolute in the output, charged below.
    eta = 2 * dlog + 2 * U * xr + 4 * U
    # online softmax: alpha = ex2(m_old - m_new) multiplies o and l by the SAME fp32 value, so its approximation error cancels in
    # o / l; the products o * alpha and fmaf(l, alpha, sum) round once per key tile each (32 tiles: 64u).  l sums the unrounded
    # p (16 pair sums of two roundings per tile and thread, then the quad sum of 4 partials: 34u), while P V reads P rounded to
    # bf16 (ub).  P V accumulates on the tensor cores over 4096 keys (2u each); 1 / l and o * inv one rounding each.
    return o, pv * (2 * eta + UB + (64 + 34 + 2 * 4096 + 2) * U)[..., None] + 4096 * 2.0 ** -126 * v.abs().amax()


def _window_bound(s, mag, v, D):
    """sam6d_attn_tc, BIAS_MODE 2 (up to 256 keys, single pass) -> (o, bound on the kernel's fp32 result)"""
    o, pv, xr = _softmax_terms(s, v)
    # logits: S on the tensor cores (2u per product), x = S * scale (one rounding), T_h / T_w two more D-term wgmmas over bf16
    # tables, th + tw and the final add one rounding each -> (2D + 3) u mag
    dlog = ((2 * D + 3) * U * mag).amax(-1)
    eta = 2 * dlog + _exp_err(xr)                 # p = __expf(x - max): one pass, no rescaling
    # row sum: 32 pair additions per thread (64 roundings; columns past Sk add exact zeros) and a quad sum (2); P rounded to
    # bf16 for P V; P V over N1 <= 208 keys on the tensor cores (2u each); 1 / sum and the product one rounding each
    return o, pv * (2 * eta + UB + (66 + 2 * WN1 + 2) * U)[..., None]


def _heads(m, rows, H, D, col0):
    """(rows, >= col0 + H*D) -> (H, rows, D) float64 of the head columns starting at col0"""
    return m[:, col0:col0 + H * D].to(F64).view(rows, H, D).transpose(0, 1)


# ================================================================================================== 1. global attention
def _global_operands(ops, D, H, B, seed):
    """q | k rows and V^T as the encoder makes them (gemm_tma_vt: q|k with ld = 2*H*D), with planted rows, and bf16-packed tables"""
    C, L = H * D, GRID * GRID
    g = _gc(seed)
    dev = "cuda"
    xw = torch.randn(B * L, C, generator=g, device=dev).bfloat16()
    W = (torch.randn(3 * C, C, generator=g, device=dev) * (1.2 / math.sqrt(C))).bfloat16()
    bias = torch.randn(3 * C, generator=g, device=dev) * 0.1
    qk, vt = ops.gemm_tma_vt(xw, W, bias, 2 * C, L, slot=2)
    vt = vt.clone()                                  # the V^T buffer is a reused cache slot
    scale = D ** -0.5
    s32 = _f32(scale)
    rh = torch.randn(2 * GRID - 1, D, generator=g, device=dev) * 0.15
    rw = torch.randn(2 * GRID - 1, D, generator=g, device=dev) * 0.15
    planted = []
    for b in range(B):
        for h in (0, H - 1):
            q = lambda r: qk[b * L + r, h * D:(h + 1) * D].float()          # noqa: E731
            kcol = slice(C + h * D, C + (h + 1) * D)
            # key m := c q_r so that the row's logit there is `target` above the scale of the rest
            for r, m, target in ((100, 7, 12.0),         # maximum in key tile 0
                                 (2000, 4000, 12.0),     # maximum in key tile 31: alpha rescales 31 tiles of real accumulators
                                 (3000, 2500, 120.0)):   # logit range > 100: ex2.approx.ftz flushes the rest to zero
                qr = q(r)
                qk[b * L + m, kcol] = (qr * (target / (s32 * qr.pow(2).sum()))).bfloat16()
            planted += [(b, h)]
    # maximum from the bias alone (image 0, head 0, query (19, 18)): rel_h row 68 and rel_w row 56 aligned with its q, so key
    # (14, 25) gets +8 from each table
    qd = qk[1234, :D].float()
    rh[63 + 5] = qd * (8.0 / qd.pow(2).sum())
    rw[63 - 7] = qd * (8.0 / qd.pow(2).sum())
    blob = ops.pack_rel_pos(rh, rw, slab_rows=128)
    return qk, vt, rh.bfloat16().to(F64), rw.bfloat16().to(F64), blob, scale, planted


def _global_ref(qk, vt, rhb, rwb, b, h, H, D, s32, v_image=None):
    """float64 logits, magnitudes and values of (image b, head h)"""
    C, L = H * D, GRID * GRID
    q = qk[b * L:(b + 1) * L, h * D:(h + 1) * D].to(F64)
    k = qk[b * L:(b + 1) * L, C + h * D:C + (h + 1) * D].to(F64)
    vb = b if v_image is None else v_image
    v = vt[(vb * H + h) * D:(vb * H + h + 1) * D, :L].to(F64).t()
    s = s32 * (q @ k.t()) + er.decomposed_bias(q, rhb, rwb, GRID, GRID)
    mag = s32 * (q.abs() @ k.abs().t()) + er.decomposed_bias(q.abs(), rhb.abs(), rwb.abs(), GRID, GRID)
    return q, k, v, s, mag


@pytest.mark.parametrize("D,H", CONFIGS)
@pytest.mark.parametrize("B", [1, 2])
def test_attn_global_tc(ops, lib, D, H, B):
    """sam6d_attn_global_tc_ex at the encoder's shapes: q|k straight from gemm_tma_vt (ld = 2*H*D, so the last head's second
    64-channel slab of K runs past the matrix at D = 80 and reads TMA zero fill), the 128-row packed tables, both output types;
    then through the C ABI with NaN in spare q|k columns and sentinel output columns"""
    C, L = H * D, GRID * GRID
    qk, vt, rhb, rwb, blob, scale, planted = _global_operands(ops, D, H, B, seed=1000 + 10 * D + H + B)
    s32 = _f32(scale)
    # wide operands: ld = 2C + 64 with NaN in [2C, ld) (only the first 16 channels of the last head's second K slab may enter an
    # MMA at D = 80); out_ld = C + 16 with sentinel columns
    ld = 2 * C + 64
    qk_wide = torch.full((B * L, ld), float("nan"), dtype=torch.bfloat16, device="cuda")
    qk_wide[:, :2 * C] = qk
    got = {}
    for odt in (torch.float32, torch.bfloat16):
        got[odt] = ops.attn_global_tc(qk, vt, blob, B, H, GRID, scale, out_dtype=odt, D=D)
        wide = torch.full((B * L, C + 16), SENT, dtype=odt, device="cuda")
        lib.call("sam6d_attn_global_tc_ex", qk_wide, ld, vt, vt.shape[1], blob, B, H, GRID, D, scale, wide, int(odt == torch.bfloat16),
                 C + 16)
        assert (wide[:, C:] == SENT).all(), "columns past H*D of the output were written"
        assert torch.equal(wide[:, :C], got[odt]), "spare q|k columns changed the result"
    worst = {odt: _Worst(f"attn_global_tc D={D} H={H} B={B} {str(odt)[6:]}") for odt in got}
    ctl = {n: _Control(n) for n in ("rel_h / rel_w swapped", "rel_h read transposed (kh - qh)", "bias times scale",
                                    "last key tile dropped")}
    if B == 2:
        ctl["image 0's V for image 1"] = _Control("image 0's V for image 1")
    ih, iw = er.rel_index(GRID, GRID, "cuda")
    for b in range(B):
        for h in range(H):
            q, k, v, s, mag = _global_ref(qk, vt, rhb, rwb, b, h, H, D, s32)
            o, bound = _global_bound(s, mag, v, D)
            for odt in got:
                gh = got[odt][b * L:(b + 1) * L, h * D:(h + 1) * D].to(F64)
                worst[odt].add((gh - o).abs(), _out_bound(o, bound, odt))
            if (b, h) not in planted:
                continue
            # the controls are measured on the fp32 output, which `bound` governs (no output rounding to absorb)
            gh = got[torch.float32][b * L:(b + 1) * L, h * D:(h + 1) * D].to(F64)
            qs = s32 * (q @ k.t())
            wrongs = {"rel_h / rel_w swapped": qs + er.decomposed_bias(q, rwb, rhb, GRID, GRID),
                      "rel_h read transposed (kh - qh)": qs + er.decomposed_bias(q, rhb, rwb, GRID, GRID, ih=2 * (GRID - 1) - ih),
                      "bias times scale": qs + s32 * er.decomposed_bias(q, rhb, rwb, GRID, GRID)}
            for n, sw in wrongs.items():
                ctl[n].add(gh, torch.softmax(sw, -1) @ v, bound)
            sd = s.clone()
            sd[:, L - 128:] = -math.inf
            ctl["last key tile dropped"].add(gh, torch.softmax(sd, -1) @ v, bound)
            if b == 1:
                v0 = vt[h * D:(h + 1) * D, :L].to(F64).t()
                ctl["image 0's V for image 1"].add(gh, torch.softmax(s, -1) @ v0, bound)
            del sd, wrongs, qs
    for w in worst.values():
        w.check()
    for c in ctl.values():
        c.check()


# ================================================================================================== 2. windowed attention
def _window_operands(ops, D, H, B, seed):
    """windows cut from a real 64 x 64 token grid by the encoder's partition map; q|k and V^T from gemm_tma_vt (S = 196)"""
    C = H * D
    g = _gc(seed)
    dev = "cuda"
    tok = torch.randn(B * GRID * GRID, C, generator=g, device=dev) + 0.3
    gam = 1.0 + 0.1 * torch.randn(C, generator=g, device=dev)
    bet = 0.1 * torch.randn(C, generator=g, device=dev)
    xn = ops.layernorm_bf16(tok, gam, bet, eps=1e-6)
    maps = _maps(B)
    xw = ops.gather_rows_bf16(xn.view(B, GRID * GRID, C), maps["part"]).view(-1, C)
    # the reference partition (F.pad AFTER norm1, image_encoder.py:243-264) of the same bf16 LayerNorm output, exactly
    ref_xw, pad_hw = so.window_partition(xn.view(B, GRID, GRID, C), WS)
    assert pad_hw == (70, 70)
    assert torch.equal(xw, ref_xw.reshape(-1, C))
    W = (torch.randn(3 * C, C, generator=g, device=dev) / math.sqrt(C)).bfloat16()
    # small q bias, so the padded tokens' queries are small; values with a positive mean, so that |o| ~ pv and a wrong
    # normalisation shows
    bias = torch.cat([0.02 * torch.randn(C, generator=g, device=dev), 0.1 * torch.randn(C, generator=g, device=dev),
                      2.0 + 0.3 * torch.randn(C, generator=g, device=dev)])
    qk, vt = ops.gemm_tma_vt(xw, W, bias, 2 * C, WL)
    vt = vt.clone()
    nW = B * 25
    assert vt.shape == (nW * C, WN1)
    # padded tokens are zero rows of xw: their q, k and v are the qkv bias rounded to bf16, exactly
    pad = maps["part"].view(-1) < 0
    assert int(pad.sum()) == B * (70 * 70 - 64 * 64)
    vtok = vt.view(nW, C, WN1)[:, :, :WL].transpose(1, 2).reshape(nW * WL, C)
    assert (qk[pad] == bias[:2 * C].bfloat16()).all() and (vtok[pad] == bias[2 * C:].bfloat16()).all()
    assert (vt.view(nW, C, WN1)[:, :, WL:] == 0).all()
    rh = torch.randn(2 * WS - 1, D, generator=g, device=dev) * 0.15
    rw = torch.randn(2 * WS - 1, D, generator=g, device=dev) * 0.15
    return qk, vt, rh, rw, pad.view(nW, WL), nW


def _attn_tc_call(lib, qk, vt, blob, nW, H, D, Hs, Ws, scale, odt, extra_rows=64):
    """sam6d_attn_tc (BIAS_MODE 2) into an output with sentinel columns past H*D and `extra_rows` sentinel rows past the end"""
    C, L = H * D, Hs * Ws
    out = torch.full((nW * L + extra_rows, C + 8), SENT, dtype=odt, device="cuda")
    lib.call("sam6d_attn_tc", qk, qk.shape[1], 0, qk, qk.shape[1], C, vt, vt.shape[1], nW, H, L, L, D, 2, 0, blob, 0, Hs, Ws, 0, scale, out,
             int(odt == torch.bfloat16), C + 8)
    assert (out[:, C:] == SENT).all(), "columns past H*D were written"
    assert (out[nW * L:] == SENT).all(), "rows past the last window were written (a query tile ran past m_lim)"
    return out[:nW * L, :C]


@pytest.mark.parametrize("D,H", CONFIGS)
@pytest.mark.parametrize("B", [1, 2])
def test_attn_tc_windows(ops, lib, D, H, B):
    """sam6d_attn_tc with the decomposed bias on the 25 windows per image of a padded 64 x 64 grid: the padded tokens are real
    keys (k, v = the qkv bias), the second 128-query tile of a window overruns into the next window's rows (and, for the last
    window, past the matrix) and must not write them; key-padding columns of V^T carry P = 0 exactly"""
    C = H * D
    qk, vt, rh, rw, pad, nW = _window_operands(ops, D, H, B, seed=2000 + 10 * D + H + B)
    scale = D ** -0.5
    s32 = _f32(scale)
    blob = ops.pack_rel_pos(rh, rw)
    rhb, rwb = rh.bfloat16().to(F64), rw.bfloat16().to(F64)
    got = {odt: _attn_tc_call(lib, qk, vt, blob, nW, H, D, WS, WS, scale, odt) for odt in (torch.float32, torch.bfloat16)}
    # the encoder's own call returns the same bits
    assert torch.equal(ops.attn_tc(qk, 0, qk, C, vt, nW, H, WL, WL, D, scale, rel=(blob, WS, WS), out_dtype=torch.bfloat16),
                       got[torch.bfloat16])
    # key padding: V^T columns 196..207 filled with large finite values change nothing, bit for bit (those keys have P = 0)
    vt_big = vt.clone()
    vt_big.view(nW, C, WN1)[:, :, WL:] = 1e30
    for odt in got:
        assert torch.equal(_attn_tc_call(lib, qk, vt_big, blob, nW, H, D, WS, WS, scale, odt), got[odt])
    del vt_big
    worst = {odt: _Worst(f"attn_tc windows D={D} H={H} nW={nW} {str(odt)[6:]}") for odt in got}
    ctl = {n: _Control(n) for n in ("rel_h / rel_w swapped", "qw - kw indexing rel_h", "padded keys masked out",
                                    "all 208 keys, logit 0 on the padding")}
    _, ih_w = er.rel_index(WS, WS, "cuda")                          # qw - kw + Hs - 1 (Hs == Ws)
    for w0 in range(0, nW, 5):
        ws_ = slice(w0, w0 + 5)
        rows = slice(w0 * WL, (w0 + 5) * WL)
        q = _heads(qk[rows], 5 * WL, H, D, 0).reshape(H, 5, WL, D).transpose(0, 1)          # (5, H, L, D)
        k = _heads(qk[rows], 5 * WL, H, D, C).reshape(H, 5, WL, D).transpose(0, 1)
        v = vt.view(nW, H, D, WN1)[ws_, :, :, :WL].to(F64).transpose(-1, -2)
        s = s32 * (q @ k.transpose(-1, -2)) + er.decomposed_bias(q, rhb, rwb, WS, WS)
        mag = s32 * (q.abs() @ k.abs().transpose(-1, -2)) + er.decomposed_bias(q.abs(), rhb.abs(), rwb.abs(), WS, WS)
        o, bound = _window_bound(s, mag, v, D)
        for odt in got:
            gw = got[odt][rows].to(F64).view(5, WL, H, D).transpose(1, 2)
            worst[odt].add((gw - o).abs(), _out_bound(o, bound, odt))
        gw = got[torch.float32][rows].to(F64).view(5, WL, H, D).transpose(1, 2)     # controls: the fp32 output, under `bound`
        qs = s32 * (q @ k.transpose(-1, -2))
        ctl["rel_h / rel_w swapped"].add(gw, torch.softmax(qs + er.decomposed_bias(q, rwb, rhb, WS, WS), -1) @ v, bound)
        ctl["qw - kw indexing rel_h"].add(gw, torch.softmax(qs + er.decomposed_bias(q, rhb, rwb, WS, WS, ih=ih_w), -1) @ v, bound)
        sm = s.masked_fill(pad[ws_][:, None, None, :], -math.inf)
        ctl["padded keys masked out"].add(gw, torch.softmax(sm, -1) @ v, bound)
        s208 = torch.cat([s, torch.zeros(*s.shape[:-1], WN1 - WL, dtype=F64, device="cuda")], -1)
        v208 = torch.cat([v, torch.zeros(*v.shape[:-2], WN1 - WL, D, dtype=F64, device="cuda")], -2)
        ctl["all 208 keys, logit 0 on the padding"].add(gw, torch.softmax(s208, -1) @ v208, bound)
        del s, mag, qs, sm, s208, v208
    for w in worst.values():
        w.check()
    for c in ctl.values():
        c.check()


@pytest.mark.parametrize("D,H", CONFIGS)
def test_attn_tc_nonsquare_window(ops, lib, D, H):
    """a 12 x 16 window (Sk = 192): Hs != Ws and tables of 23 and 31 rows, where mixing up the two grid sides shows"""
    C, Hs, Ws, nW = H * D, 12, 16, 3
    L = Hs * Ws
    g = _gc(3000 + D + H)
    xw = torch.randn(nW * L, C, generator=g, device="cuda").bfloat16()
    W = (torch.randn(3 * C, C, generator=g, device="cuda") / math.sqrt(C)).bfloat16()
    bias = torch.randn(3 * C, generator=g, device="cuda") * 0.1
    qk, vt = ops.gemm_tma_vt(xw, W, bias, 2 * C, L, slot=5)
    vt = vt.clone()
    rh = torch.randn(2 * Hs - 1, D, generator=g, device="cuda") * 0.3
    rw = torch.randn(2 * Ws - 1, D, generator=g, device="cuda") * 0.3
    scale = D ** -0.5
    s32 = _f32(scale)
    blob = ops.pack_rel_pos(rh, rw)
    rhb, rwb = rh.bfloat16().to(F64), rw.bfloat16().to(F64)
    got = {odt: _attn_tc_call(lib, qk, vt, blob, nW, H, D, Hs, Ws, scale, odt) for odt in (torch.float32, torch.bfloat16)}
    q = _heads(qk, nW * L, H, D, 0).reshape(H, nW, L, D).transpose(0, 1)
    k = _heads(qk, nW * L, H, D, C).reshape(H, nW, L, D).transpose(0, 1)
    v = vt.view(nW, H, D, L).to(F64).transpose(-1, -2)
    qs = s32 * (q @ k.transpose(-1, -2))
    s = qs + er.decomposed_bias(q, rhb, rwb, Hs, Ws)
    mag = s32 * (q.abs() @ k.abs().transpose(-1, -2)) + er.decomposed_bias(q.abs(), rhb.abs(), rwb.abs(), Hs, Ws)
    o, bound = _window_bound(s, mag, v, D)
    for odt in got:
        gw = got[odt].to(F64).view(nW, L, H, D).transpose(1, 2)
        _check(f"attn_tc 12x16 window D={D} H={H} {str(odt)[6:]}", (gw - o).abs(), _out_bound(o, bound, odt))
    gw = got[torch.float32].to(F64).view(nW, L, H, D).transpose(1, 2)         # controls: the fp32 output, under `bound`
    ih, _ = er.rel_index(Hs, Ws, "cuda")
    ctl = {n: _Control(n) for n in ("rel_h read transposed (kh - qh)", "the window read as 16 x 12")}
    ctl["rel_h read transposed (kh - qh)"].add(
        gw, torch.softmax(qs + er.decomposed_bias(q, rhb, rwb, Hs, Ws, ih=2 * (Hs - 1) - ih), -1) @ v, bound)
    # Hs and Ws exchanged (the tables exchanged with them, so that every row index stays in range)
    ctl["the window read as 16 x 12"].add(gw, torch.softmax(qs + er.decomposed_bias(q, rwb, rhb, Ws, Hs), -1) @ v, bound)
    for c in ctl.values():
        c.check()


# ================================================================================================== 3. fp32 comparator attention
@pytest.mark.parametrize("Hs,Ws,nW,D,H", [(14, 14, 3, 80, 2), (14, 14, 3, 64, 3), (9, 9, 4, 80, 2), (9, 9, 4, 64, 2),
                                          (9, 20, 2, 80, 2), (9, 20, 2, 64, 3), (64, 64, 1, 80, 16)])
def test_attn_relpos_fp32(ops, Hs, Ws, nW, D, H):
    """sam6d_attn_relpos (precision="fp32", and bf16 grids other than 14 and 64): 64-key tiles with an online softmax; the
    last tile of a 196- or 81-key window holds 4 or 17 keys and loads the rest clamped to key L - 1, which must not count"""
    C, L = H * D, Hs * Ws
    g = _gc(4000 + Hs * 7 + Ws + D + H)
    qkv = torch.randn(nW * L, 3 * C, generator=g, device="cuda") * 1.2
    rh = torch.randn(2 * Hs - 1, D, generator=g, device="cuda") * 0.3
    rw = torch.randn(2 * Ws - 1, D, generator=g, device="cuda") * 0.3
    scale = D ** -0.5
    s32 = _f32(scale)
    got = ops.attn_relpos(qkv, nW, Hs, Ws, H, rh, rw, scale)
    # the bf16 output is the fp32 output rounded once
    assert torch.equal(ops.attn_relpos(qkv, nW, Hs, Ws, H, rh, rw, scale, out_dtype=torch.bfloat16), got.bfloat16())
    rh64, rw64 = rh.to(F64), rw.to(F64)                  # this kernel reads the fp32 tables
    T = (L + 63) // 64
    worst = _Worst(f"attn_relpos fp32 {Hs}x{Ws} nW={nW} D={D} H={H}")
    dup = _Control("clamped duplicate of key L - 1 counted")
    for w, h in ((w, h) for w in range(nW) for h in range(H)):         # one (window, head) at a time: 64 x 64 is 4096 keys
        rows = slice(w * L, (w + 1) * L)
        q, k, v = (_heads(qkv[rows], L, H, D, i * C)[h] for i in range(3))
        s = s32 * (q @ k.transpose(-1, -2)) + er.decomposed_bias(q, rh64, rw64, Hs, Ws)
        mag = s32 * (q.abs() @ k.abs().transpose(-1, -2)) + er.decomposed_bias(q.abs(), rh64.abs(), rw64.abs(), Hs, Ws)
        o, pv, xr = _softmax_terms(s, v)
        # logits: q.k and the Hs + Ws table dot products are D-term fp32 fma chains (gamma_D); fmaf(dot, scale, h + w) and h + w
        # one rounding each -> (D + 3) u mag
        dlog = ((D + 3) * U * mag).amax(-1)
        eta = 2 * dlog + _exp_err(xr)
        # corr = __expf(m_old - m_new) multiplies o and l by the same fp32 value (its error cancels in o / l); the products
        # round once per tile each.  l: 2 additions per tile and lane, 5 warp-sum levels -> (3T + 5) u; o: an fma chain over
        # the L keys plus the T corrections -> (L + T) u; 1 / l and the product one rounding each.  fp32 output.
        bound = pv * (2 * eta + (L + T + 3 * T + 5 + 2) * U)[..., None]
        gw = got[rows, h * D:(h + 1) * D].to(F64)
        worst.add((gw - o).abs(), bound)
        if L % 64:
            s2 = torch.cat([s, s[..., L - 1:]], -1)
            v2 = torch.cat([v, v[L - 1:]], -2)
            dup.add(gw, torch.softmax(s2, -1) @ v2, bound)
    worst.check()
    if L % 64:
        dup.check()


# ================================================================================================== 4. row gathers
def test_gather_rows_partition_maps(ops):
    """gather_rows (fp32) and gather_rows_bf16 with the partition / unpartition / tap maps at B = 2: exact copies, and rows of
    exact zeros (all bits clear) at index -1"""
    B = 2
    maps = _maps(B)
    g = _gc(5000)
    src32 = torch.randn(B, GRID * GRID, 256, generator=g, device="cuda")
    src16 = torch.randn(B, GRID * GRID, 1280, generator=g, device="cuda").bfloat16()
    for name, idx in [("part", maps["part"]), ("unpart", maps["unpart"])] + [(f"tap {t}", m) for t, m in enumerate(maps["taps"])]:
        src16_ = src16 if name != "unpart" else torch.randn(B, 25 * WL, 1280, generator=g, device="cuda").bfloat16()
        src32_ = src32 if name != "unpart" else torch.randn(B, 25 * WL, 256, generator=g, device="cuda")
        for src, fn, ity in ((src32_, ops.gather_rows, torch.int32), (src16_, ops.gather_rows_bf16, torch.int16)):
            out = fn(src, idx)
            il = idx.long()
            ref = torch.where((il >= 0)[..., None], torch.gather(src, 1, il.clamp_min(0)[..., None].expand(-1, -1, src.shape[2])),
                              torch.zeros((), dtype=src.dtype, device="cuda"))
            assert torch.equal(out.view(ity), ref.view(ity)), f"{name} {src.dtype}"


# ================================================================================================== 5. LayerNorms
def _ln_rows(R, C, g):
    """ordinary rows; rows with a few channels near +-1e3 over an O(1) rest (ViT residual streams carry outliers); constant
    rows; rows at an offset of 50; tightly spread rows (sigma = 0.01, where eps matters)"""
    dev = "cuda"
    ordinary = torch.randn(R, C, generator=g, device=dev) * 2 + 0.5
    outl = torch.randn(R, C, generator=g, device=dev)
    for r in range(R):
        idx = torch.randint(0, C, (5,), generator=g, device=dev)
        outl[r, idx] = (torch.rand(5, generator=g, device=dev) * 200 + 900) * torch.sign(torch.randn(5, generator=g, device=dev))
    const = torch.full((R, C), 3.7, device=dev)
    offset = 50 + torch.randn(R, C, generator=g, device=dev)
    tight = 1 + 0.01 * torch.randn(R, C, generator=g, device=dev)
    return torch.cat([ordinary, outl, const, offset, tight]).contiguous()


def _ln_bound(x, g, b, eps, n_chain, odt):
    """the encoder's LayerNorm kernels (two-pass statistics, one warp per row, each lane owning C / 32 channels) -> (float64
    LayerNorm of x, bound).  n_chain = additions in one lane's sum: C / 128 float4 steps (vector kernel), C / 32 (generic)."""
    mu = x.mean(-1, keepdim=True)
    d = x - mu
    var = d.pow(2).mean(-1, keepdim=True)
    r = 1.0 / torch.sqrt(var + eps)
    out = d * r * g + b
    # mean: the lane's chain (n_chain, plus 2 pair sums inside a float4 in the vector kernel), 5 warp-sum levels, 1 / C one rounding
    e_mu = (n_chain + 8) * U * x.abs().mean(-1, keepdim=True)
    # variance on the computed mean: sum (x - mu - e)^2 = sum d^2 + C e^2 (the cross term vanishes); each d rounded once (2u on
    # d^2), the square and the pair sums (3), the lane chain, 5 levels, 1 / C; + eps one rounding
    e_var = (n_chain + 11) * U * var + e_mu ** 2 + U * (var + eps)
    e_r = 0.5 * e_var / (var + eps) + 4 * U             # rsqrtf 2 ulp; half the relative error of var + eps
    # (x - mean) one rounding, times rstd, times gamma, plus beta: one each; 1 % for second-order terms
    e = 1.01 * (g.abs() * r * (e_mu + 3 * U * d.abs() + d.abs() * e_r) + U * out.abs())
    if odt == torch.bfloat16:
        return out, e + UB * (out.abs() + e)            # one bf16 rounding
    return out, e


@pytest.mark.parametrize("C", [768, 1024, 1280])
def test_layernorm_bf16_vector(ops, C):
    """layernorm_bf16 (fp32 residual stream -> bf16 GEMM operand) at the three encoder widths: the vector kernel, whose NV = 10
    registers hold only 6, 8 or 10 float4 of a row"""
    g = _gc(6000 + C)
    x = _ln_rows(48, C, g)
    gam = 1.0 + 0.2 * torch.randn(C, generator=g, device="cuda")
    bet = 0.2 * torch.randn(C, generator=g, device="cuda")
    got = ops.layernorm_bf16(x, gam, bet, eps=1e-6)
    ref, bound = _ln_bound(x.to(F64), gam.to(F64), bet.to(F64), EPS6, C // 128, torch.bfloat16)
    _check(f"layernorm_bf16 vector C={C}", (got.to(F64) - ref).abs(), bound)


def test_layernorm_bf16_generic(lib):
    """layernorm_bf16 at C = 1280 through the generic kernel, reached with an x_ld that is not a multiple of 4"""
    C, ld = 1280, 1282
    g = _gc(6100)
    x = _ln_rows(48, C, g)
    rows = x.shape[0]
    xb = torch.full((rows, ld), float("nan"), device="cuda")
    xb[:, :C] = x
    gam = 1.0 + 0.2 * torch.randn(C, generator=g, device="cuda")
    bet = 0.2 * torch.randn(C, generator=g, device="cuda")
    y = torch.empty(rows, C, dtype=torch.bfloat16, device="cuda")
    lib.call("sam6d_layernorm_bf16", xb, rows, 0, ld, y, rows, 0, C, gam, bet, rows, C, 1e-6)
    ref, bound = _ln_bound(x.to(F64), gam.to(F64), bet.to(F64), EPS6, C // 32, torch.bfloat16)
    _check("layernorm_bf16 generic C=1280", (y.to(F64) - ref).abs(), bound)


def test_layernorm_neck_fp32(ops):
    """layernorm (fp32) at C = 256, eps = 1e-6: the neck's LayerNorm2d evaluated channel-last"""
    C = 256
    g = _gc(6200)
    x = _ln_rows(64, C, g)
    gam = 1.0 + 0.2 * torch.randn(C, generator=g, device="cuda")
    bet = 0.2 * torch.randn(C, generator=g, device="cuda")
    got = ops.layernorm(x, gam, bet, eps=1e-6)
    x64, g64, b64 = x.to(F64), gam.to(F64), bet.to(F64)
    ref, bound = _ln_bound(x64, g64, b64, EPS6, C // 32, torch.float32)
    _check("layernorm fp32 C=256 eps=1e-6", (got.to(F64) - ref).abs(), bound)
    wrong = er.layer_norm(x64, g64, b64, 10 * EPS6)
    r = _ratio((got.to(F64) - wrong).abs(), bound)
    print(f"  negative control eps x 10: {r:.3g}")
    assert r > 1.0


# ================================================================================================== 6. wiring
def _lin_bound(mag, K, extra=0.0):
    """a K-term tensor-core GEMM (2u per product) and its epilogue adds (bias, residual: one rounding each on `extra`)"""
    return 2 * K * U * mag + 2 * U * extra


def _bf_bound(ref, e):
    """a kernel value within e of ref, rounded once to bf16"""
    return e + UB * (ref.abs() + e)


@pytest.mark.parametrize("name", ["vit_h", "vit_l", "vit_b"])
def test_encoder_wiring_views(ops, name):
    """ImageEncoderViT (bf16) with one windowed and one global block: the module's forward replayed stage by stage with the
    same ops calls must give the same bits, and every stage is held to the reference formula (image_encoder.py) evaluated in
    float64 on the kernel's own output of the previous stage"""
    from sam6d_b200.sam import VIT_CONFIGS, ImageEncoderViT
    cfg = VIT_CONFIGS[name]
    C, H = cfg["embed_dim"], cfg["num_heads"]
    D = C // H
    sd = synth.make_sam_state_dict(embed_dim=C, depth=2, num_heads=H, global_attn_indexes=(1,))
    enc = ImageEncoderViT(depth=2, embed_dim=C, img_size=1024, mlp_ratio=4, norm_layer=partial(torch.nn.LayerNorm, eps=1e-6),
                          num_heads=H, patch_size=16, qkv_bias=True, use_rel_pos=True, global_attn_indexes=(1,), window_size=14,
                          out_chans=256).cuda().eval()
    enc.load_state_dict(sd, strict=True)
    img = synth.make_images(B=1).cuda()
    out = enc(img)
    # ---------------------------------------------------------------- replay (forward / _block_bf16 with the same calls)
    # The kernels run on the module's packed weights (enc._weights()); every reference below takes its weights, eps and scale
    # from the state dict and the reference's configuration instead, so a mis-packed weight fails its stage.
    w = enc._weights()
    maps = enc._index_maps(1, GRID, WS, img.device)
    P, L = 16, GRID * GRID
    eps = EPS6                                                       # build_sam.py: LayerNorm eps=1e-6, LayerNorm2d eps=1e-6
    scale = _f32(D ** -0.5)                                          # Attention.scale = head_dim ** -0.5

    def f64(key):
        return sd[key].cuda().to(F64)

    def wbf(key):
        """a reference weight as the tensor cores read it (rounded to bf16)"""
        return sd[key].cuda().bfloat16().to(F64)

    patches = img.float().reshape(1, 3, GRID, P, GRID, P).permute(0, 2, 4, 1, 3, 5).reshape(L, 3 * P * P).contiguous()
    tok = torch.empty(L, C, dtype=torch.float32, device="cuda")
    ops.gemm_tc(patches, w["pe_w"].bf16, w["pe_b"], residual=w["pos"], out=tok)
    # patch embed + pos: conv 16 x 16 / 16 == a 768-term GEMM over bf16 patches and weights; + bias, + pos one rounding each.
    # (The float64 conv itself is exact to within 768 * 2^-53 mag, 2^29 times below the charged 2 * 768 u mag.)
    pe_w = wbf("patch_embed.proj.weight")
    ref = (F.conv2d(img.bfloat16().to(F64), pe_w, f64("patch_embed.proj.bias"), stride=P).permute(0, 2, 3, 1).reshape(L, C)
           + f64("pos_embed").reshape(L, C))
    a64 = patches.bfloat16().to(F64)
    mag = a64.abs() @ pe_w.reshape(C, -1).abs().t()
    _check(f"{name} patch_embed", (tok.to(F64) - ref).abs(),
           _lin_bound(mag, 3 * P * P, ref.abs() + f64("patch_embed.proj.bias").abs()))
    del mag, a64
    for i, (blk, bw) in enumerate(zip(enc.blocks, w["blocks"])):
        p = f"blocks.{i}"
        windowed = i != 1                                            # global_attn_indexes=(1,)
        tag = f"{name} block {i} ({'windowed' if windowed else 'global'})"
        # LN1
        xn = ops.layernorm_bf16(tok, bw["n1w"], bw["n1b"], eps=bw["eps1"])
        r, b_ = _ln_bound(tok.to(F64), f64(p + ".norm1.weight"), f64(p + ".norm1.bias"), eps, C // 128, torch.bfloat16)
        _check(f"{tag} norm1", (xn.to(F64) - r).abs(), b_)
        if windowed:
            xw = ops.gather_rows_bf16(xn.view(1, L, C), maps["part"]).view(-1, C)
            ref_xw, _ = so.window_partition(xn.view(1, GRID, GRID, C), WS)
            assert torch.equal(xw, ref_xw.reshape(-1, C)), f"{tag}: window partition"
            nW, Hs = 25, WS
            qk, vt = ops.gemm_tma_vt(xw, bw["qkv"].bf16, bw["qkv_b"], 2 * C, Hs * Hs)
        else:
            xw, nW, Hs = xn, 1, GRID
            qk, vt = ops.gemm_tma_vt(xw, bw["qkv"].bf16, bw["qkv_b"], 2 * C, Hs * Hs, slot=2)
        S = Hs * Hs
        # qkv projection: C products on the tensor cores + bias, one bf16 rounding; V^T slot (window, head, channel) <- token
        Wq = wbf(p + ".attn.qkv.weight")
        R = xw.to(F64) @ Wq.t() + f64(p + ".attn.qkv.bias")
        eR = _lin_bound(xw.to(F64).abs() @ Wq.abs().t(), C, R.abs())
        n1 = vt.shape[1]
        vtok = vt[:nW * C].view(nW, C, n1)[:, :, :S].transpose(1, 2).reshape(nW * S, C)
        _check(f"{tag} qkv q|k", (qk.to(F64) - R[:, :2 * C]).abs(), _bf_bound(R[:, :2 * C], eR[:, :2 * C]))
        _check(f"{tag} qkv V^T", (vtok.to(F64) - R[:, 2 * C:]).abs(), _bf_bound(R[:, 2 * C:], eR[:, 2 * C:]))
        del R, eR, Wq
        rhb, rwb = wbf(p + ".attn.rel_pos_h"), wbf(p + ".attn.rel_pos_w")
        if windowed:
            att = ops.attn_tc(qk, 0, qk, C, vt, nW, H, S, S, D, blk.attn.scale, rel=(bw["rel_blob"], Hs, Hs), out_dtype=torch.bfloat16)
            q = _heads(qk, nW * S, H, D, 0).reshape(H, nW, S, D).transpose(0, 1)
            k = _heads(qk, nW * S, H, D, C).reshape(H, nW, S, D).transpose(0, 1)
            v = vt[:nW * C].view(nW, H, D, n1)[..., :S].to(F64).transpose(-1, -2)
            s = scale * (q @ k.transpose(-1, -2)) + er.decomposed_bias(q, rhb, rwb, Hs, Hs)
            mag = scale * (q.abs() @ k.abs().transpose(-1, -2)) + er.decomposed_bias(q.abs(), rhb.abs(), rwb.abs(), Hs, Hs)
            o, bound = _window_bound(s, mag, v, D)
            _check(f"{tag} attention", (att.to(F64).view(nW, S, H, D).transpose(1, 2) - o).abs(), _out_bound(o, bound, torch.bfloat16))
            del s, mag, o, bound
            att2 = ops.gather_rows_bf16(att.view(1, -1, C), maps["unpart"]).view(-1, C)
            ref_un = so.window_unpartition(att.view(nW, WS, WS, C), WS, (70, 70), (GRID, GRID)).reshape(L, C)
            assert torch.equal(att2, ref_un), f"{tag}: window unpartition"
        else:
            att = ops.attn_global_tc(qk, vt, bw["rel_blob"], 1, H, GRID, blk.attn.scale, D=D)
            wst = _Worst(f"{tag} attention")
            for h in range(H):
                _, _, v, s, mag = _global_ref(qk, vt, rhb, rwb, 0, h, H, D, scale)
                o, bound = _global_bound(s, mag, v, D)
                wst.add((att[:, h * D:(h + 1) * D].to(F64) - o).abs(), _out_bound(o, bound, torch.bfloat16))
                del s, mag, o, bound
            wst.check()
            att2 = att
        # proj + residual (fp32 residual stream): C products + bias + residual
        tok_in = tok
        tok = ops.gemm_tma(att2, bw["proj"].bf16, bw["proj_b"], residual=tok_in)
        Wp, bp = wbf(p + ".attn.proj.weight"), f64(p + ".attn.proj.bias")
        ref = att2.to(F64) @ Wp.t() + bp + tok_in.to(F64)
        _check(f"{tag} proj + residual", (tok.to(F64) - ref).abs(),
               _lin_bound(att2.to(F64).abs() @ Wp.abs().t(), C, ref.abs() + tok_in.to(F64).abs() + bp.abs()))
        # LN2
        xn = ops.layernorm_bf16(tok, bw["n2w"], bw["n2b"], eps=bw["eps2"])
        r, b_ = _ln_bound(tok.to(F64), f64(p + ".norm2.weight"), f64(p + ".norm2.bias"), eps, C // 128, torch.bfloat16)
        _check(f"{tag} norm2", (xn.to(F64) - r).abs(), b_)
        # MLP lin1 + GELU (erf) -> bf16
        h_ = ops.gemm_tma(xn, bw["l1"].bf16, bw["l1b"], act=2, out_dtype=torch.bfloat16)
        W1 = wbf(p + ".mlp.lin1.weight")
        a = xn.to(F64) @ W1.t() + f64(p + ".mlp.lin1.bias")
        ea = _lin_bound(xn.to(F64).abs() @ W1.abs().t(), C, a.abs())
        ref = F.gelu(a)
        # |gelu'| <= 1.13; own arithmetic 0.5 x (1 + erff(x / sqrt 2)): x / sqrt 2 (u, through erf' <= 1.13), erff 2 ulp, 1 + erf,
        # the products: <= (6 + |x|) u |x|
        e = 1.13 * ea + (6 + a.abs()) * U * a.abs()
        _check(f"{tag} lin1 + GELU", (h_.to(F64) - ref).abs(), _bf_bound(ref, e))
        del a, ea, e
        # lin2 + residual: 4C products
        tok_in = tok
        tok = ops.gemm_tma(h_, bw["l2"].bf16, bw["l2b"], residual=tok_in)
        W2, b2 = wbf(p + ".mlp.lin2.weight"), f64(p + ".mlp.lin2.bias")
        ref = h_.to(F64) @ W2.t() + b2 + tok_in.to(F64)
        _check(f"{tag} lin2 + residual", (tok.to(F64) - ref).abs(),
               _lin_bound(h_.to(F64).abs() @ W2.abs().t(), 4 * C, ref.abs() + tok_in.to(F64).abs() + b2.abs()))
        del ref, W1, W2
    # ---------------------------------------------------------------- neck (image_encoder.py:88-104)
    from sam6d_b200.pem import _gemm
    y = _gemm("bf16", tok, w["neck0"])
    A = tok.bfloat16().to(F64)                                       # the fp32 tokens are rounded to bf16 while staging
    W0 = wbf("neck.0.weight").reshape(256, C)
    ref = A @ W0.t()
    _check(f"{name} neck conv 1x1", (y.to(F64) - ref).abs(), _lin_bound(A.abs() @ W0.abs().t(), C))
    yl = ops.layernorm(y, w["ln1"][0], w["ln1"][1], eps=w["ln1"][2])
    r, b_ = _ln_bound(y.to(F64), f64("neck.1.weight"), f64("neck.1.bias"), eps, 256 // 32, torch.float32)
    _check(f"{name} neck LayerNorm2d 1", (yl.to(F64) - r).abs(), b_)
    acc = None
    y3 = yl.view(1, L, 256)
    for tap, Wt in zip(maps["taps"], w["neck2"]):
        shifted = ops.gather_rows(y3, tap).view(-1, 256)
        acc = _gemm("bf16", shifted, Wt, None, residual=acc)
    # 3 x 3 conv, padding 1, on the bf16-rounded LayerNorm output: 9 GEMMs of 256 products, each adding the previous partial
    # sum as its residual (one rounding each)
    x4 = yl.bfloat16().to(F64).t().reshape(1, 256, GRID, GRID)
    W3 = wbf("neck.2.weight")
    ref = F.conv2d(x4, W3, padding=1)[0].reshape(256, L).t()
    mag = F.conv2d(x4.abs(), W3.abs(), padding=1)[0].reshape(256, L).t()
    _check(f"{name} neck conv 3x3", (acc.to(F64) - ref).abs(), (2 * 9 * 256 + 9) * U * mag)
    fin = ops.layernorm(acc, w["ln2"][0], w["ln2"][1], eps=w["ln2"][2])
    r, b_ = _ln_bound(acc.to(F64), f64("neck.3.weight"), f64("neck.3.bias"), eps, 256 // 32, torch.float32)
    _check(f"{name} neck LayerNorm2d 2", (fin.to(F64) - r).abs(), b_)
    replay = fin.view(1, GRID, GRID, 256).permute(0, 3, 1, 2).contiguous()
    assert torch.equal(replay, out), "the stage-by-stage replay differs from the module's forward"
