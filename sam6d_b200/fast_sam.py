"""FastSAM segmentor of the ISM (ISM/model/fast_sam.py): YOLOv8x-seg or YOLOv8s-seg -- the ultralytics 8.0.135
`SegmentationModel` of `yolov8-seg.yaml` at scale x or s and nc = 1, what `FastSAM-x.pt` and `FastSAM-s.pt` hold -- on sm_90a
kernels, with the reference's `FastSAM` wrapper contract.

Network.  `YOLOv8Seg` has ultralytics' module tree and state_dict keys (`model.0.conv.weight`, `model.22.proto.upsample.bias`, ...),
so a real checkpoint loads with strict=True through `load_fastsam_checkpoint` (no ultralytics needed).  BatchNorm is folded into
each convolution in fp32 as ultralytics' fuse_conv_and_bn does (AutoBackend(fuse=True)), then rounded to bf16 once per parameter
version.  Activations are NHWC bf16 with fp32 accumulation:
  * every 1x1 / 3x3 convolution is one `sam6d_conv2d_tc` launch (implicit GEMM on wgmma, csrc/conv_tc.cu); the first layer
    (Cin = 3) is `sam6d_yolo_stem_c`, which also does the channel flip and /255 of the letterboxed u8 frame;
  * concatenation is free: C2f's chunk / cat, SPPF's four-way cat and the head's Concat layers are channel slices of one
    preallocated NHWC buffer that the producing layers write into;
  * the first 3x3 convolutions of the box, class and mask-coefficient branches of a level share their input and run as one
    launch (Cout 80 + 320 + 80 at x, 64 + 128 + 32 at s); their last 1x1 convolutions run as one block-diagonal launch
    (480 -> 97 at x, 224 -> 97 at s) that writes the level's
    rows of the fp32 head matrix (B, anchors, 64 DFL logits | class logit | 32 coefficients);
  * Proto's 2x2 stride-2 transposed convolution is four 1x1 launches, one per tap, written interleaved.

Post-processing (SegmentationPredictor.postprocess): `sam6d_yolo_decode` (DFL, dist2bbox, sigmoid, conf filter in anchor
order) -> stable sort by descending confidence (ties go to the lower anchor index; ultralytics' argsort is not stable, so its
order of exact ties is unspecified) -> `sam6d_sam_nms` (torchvision.ops.nms restated; class-aware NMS is plain NMS at nc = 1) ->
the first max_det -> `sam6d_yolo_masks` (process_mask with upsample=True) -> scale_boxes / clip_boxes -> postprocess_resize."""
import math
import pickle
from types import SimpleNamespace
from typing import Any, Dict, Optional

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _lib
from .layers import _Packed

bf = torch.bfloat16
REG_MAX, NM, NC = 16, 32, 1
HEAD_W = 4 * REG_MAX + NC + NM          # 97 columns per anchor
STRIDES = (8, 16, 32)

# yolov8-seg.yaml's scales that FastSAM publishes: (depth multiple, width multiple, max channels)
SCALES = {"x": (1.00, 1.25, 512), "s": (0.33, 0.50, 1024)}


def scale_layout(scale: str) -> SimpleNamespace:
    """the layer widths and C2f depths of a scale, by ultralytics' parse_model rules: width make_divisible(min(c, max_channels)
    * width, 8) of the yaml's 64 / 128 / 256 / 512 / 1024, depth max(round(n * depth), 1) of its 3 / 6 repeats.
    -> c (c0..c4), n3, n6 (the backbone's C2f depths; the head's are n3), npr (Proto width)"""
    if scale not in SCALES:
        raise ValueError(f"FastSAM scale must be one of {sorted(SCALES)}, got {scale!r}")
    depth, width, max_c = SCALES[scale]
    ch = lambda c: int(math.ceil(min(c, max_c) * width / 8) * 8)        # noqa: E731
    n = lambda k: max(round(k * depth), 1)                              # noqa: E731
    c = tuple(ch(v) for v in (64, 128, 256, 512, 1024))
    return SimpleNamespace(scale=scale, c=c, n3=n(3), n6=n(6), npr=c[2])


# =====================================================================================================================
# the module tree of ultralytics.nn.modules (8.0.135), parameters only
# =====================================================================================================================
class Conv(nn.Module):
    """Conv2d (no bias, padding k // 2) + BatchNorm2d (eps 1e-3) + SiLU"""

    def __init__(self, c1, c2, k=1, s=1):
        super().__init__()
        self.conv = nn.Conv2d(c1, c2, k, s, k // 2, bias=False)
        self.bn = nn.BatchNorm2d(c2, eps=1e-3, momentum=0.03)


class Bottleneck(nn.Module):
    def __init__(self, c, shortcut):
        super().__init__()
        self.cv1, self.cv2, self.add = Conv(c, c, 3), Conv(c, c, 3), shortcut


class C2f(nn.Module):
    def __init__(self, c1, c2, n, shortcut):
        super().__init__()
        self.c = c2 // 2
        self.cv1 = Conv(c1, 2 * self.c, 1)
        self.cv2 = Conv((2 + n) * self.c, c2, 1)
        self.m = nn.ModuleList(Bottleneck(self.c, shortcut) for _ in range(n))


class SPPF(nn.Module):
    def __init__(self, c1, c2):
        super().__init__()
        self.cv1, self.cv2 = Conv(c1, c1 // 2, 1), Conv(c1 // 2 * 4, c2, 1)


class Proto(nn.Module):
    def __init__(self, c1, c_, c2):
        super().__init__()
        self.cv1 = Conv(c1, c_, 3)
        self.upsample = nn.ConvTranspose2d(c_, c_, 2, 2, 0, bias=True)
        self.cv2 = Conv(c_, c_, 3)
        self.cv3 = Conv(c_, c2)


class DFL(nn.Module):
    def __init__(self, c1=REG_MAX):
        super().__init__()
        self.conv = nn.Conv2d(c1, 1, 1, bias=False).requires_grad_(False)
        self.conv.weight.data[:] = torch.arange(c1, dtype=torch.float).view(1, c1, 1, 1)


class Segment(nn.Module):
    def __init__(self, nc=NC, nm=NM, npr=320, ch=(320, 640, 640)):
        super().__init__()
        self.nc, self.nm, self.npr, self.nl, self.reg_max = nc, nm, npr, len(ch), REG_MAX
        c2, c3, c4 = max(16, ch[0] // 4, REG_MAX * 4), max(ch[0], min(nc, 100)), max(ch[0] // 4, nm)
        self.cv2 = nn.ModuleList(nn.Sequential(Conv(x, c2, 3), Conv(c2, c2, 3), nn.Conv2d(c2, 4 * REG_MAX, 1)) for x in ch)
        self.cv3 = nn.ModuleList(nn.Sequential(Conv(x, c3, 3), Conv(c3, c3, 3), nn.Conv2d(c3, nc, 1)) for x in ch)
        self.dfl = DFL(REG_MAX)
        self.proto = Proto(ch[0], npr, nm)
        self.cv4 = nn.ModuleList(nn.Sequential(Conv(x, c4, 3), Conv(c4, c4, 3), nn.Conv2d(c4, nm, 1)) for x in ch)


class _Layer(nn.Module):
    """Upsample / Concat entries of the layer list (no parameters)"""


# =====================================================================================================================
# weights in kernel form
# =====================================================================================================================
def fold_conv_bn(conv: nn.Conv2d, bn: nn.BatchNorm2d):
    """fuse_conv_and_bn (ultralytics/utils/torch_utils.py) in fp32 -> (weight (Cout,Cin,k,k), bias (Cout))"""
    w = conv.weight.detach().float()
    g, b = bn.weight.detach().float(), bn.bias.detach().float()
    mean, var = bn.running_mean.detach().float(), bn.running_var.detach().float()
    scale = g.div(torch.sqrt(bn.eps + var))
    bias = b - g.mul(mean).div(torch.sqrt(var + bn.eps))
    return w * scale.view(-1, 1, 1, 1), bias


class _CW:
    """one convolution ready for sam6d_conv2d_tc: w (Cout,k,k,Cin) bf16, bias (Cout) f32"""
    __slots__ = ("w", "b", "k", "cout", "cin")

    def __init__(self, w, b):
        self.cout, self.cin, self.k = w.shape[0], w.shape[1], w.shape[2]
        self.w = w.permute(0, 2, 3, 1).contiguous().to(bf)
        self.b = b.float().contiguous()


def _cw(m: Conv) -> _CW:
    return _CW(*fold_conv_bn(m.conv, m.bn))


# =====================================================================================================================
class YOLOv8Seg(nn.Module):
    """ultralytics SegmentationModel('yolov8{scale}-seg.yaml', nc=1), scale "x" (FastSAM-x: widths 80 / 160 / 320 / 640 / 640,
    C2f depths 3 / 6 / 6 / 3) or "s" (FastSAM-s: widths 32 / 64 / 128 / 256 / 512, depths 1 / 2 / 2 / 1).
    forward(frames (B,H,W,3) u8 letterboxed, H and W multiples of 32) -> head (B,A,97) f32, proto (B,H/4,W/4,32) f32."""

    def __init__(self, scale: str = "x"):
        super().__init__()
        lay = scale_layout(scale)
        c0, c1, c2, c3, c4 = lay.c
        n3, n6 = lay.n3, lay.n6
        L = [Conv(3, c0, 3, 2), Conv(c0, c1, 3, 2), C2f(c1, c1, n3, True), Conv(c1, c2, 3, 2), C2f(c2, c2, n6, True),
             Conv(c2, c3, 3, 2), C2f(c3, c3, n6, True), Conv(c3, c4, 3, 2), C2f(c4, c4, n3, True), SPPF(c4, c4),
             _Layer(), _Layer(), C2f(c4 + c3, c3, n3, False), _Layer(), _Layer(), C2f(c3 + c2, c2, n3, False),
             Conv(c2, c2, 3, 2), _Layer(), C2f(c2 + c3, c3, n3, False), Conv(c3, c3, 3, 2), _Layer(), C2f(c3 + c4, c4, n3, False),
             Segment(npr=lay.npr, ch=(c2, c3, c4))]
        self.model = nn.ModuleList(L)
        self.scale = scale
        self._packed = _Packed()

    # ---- packing ------------------------------------------------------------------------------------------------------
    def _weights(self):
        return self._packed.get(self._pack, self)

    def _pack(self):
        m = self.model
        w = {}
        sw, sb = fold_conv_bn(m[0].conv, m[0].bn)
        w["stem"] = (sw.permute(0, 2, 3, 1).contiguous(), sb.contiguous())        # fp32: the stem is a CUDA-core kernel
        for i in (1, 3, 5, 7, 16, 19):
            w[i] = _cw(m[i])
        for i in (2, 4, 6, 8, 12, 15, 18, 21):
            c = m[i]
            w[i] = SimpleNamespace(c=c.c, cv1=_cw(c.cv1), cv2=_cw(c.cv2), m=[(_cw(b.cv1), _cw(b.cv2), b.add) for b in c.m])
        w[9] = SimpleNamespace(cv1=_cw(m[9].cv1), cv2=_cw(m[9].cv2))
        seg = m[22]
        heads = []
        for l in range(seg.nl):
            br = (seg.cv2[l], seg.cv3[l], seg.cv4[l])
            f = [fold_conv_bn(b[0].conv, b[0].bn) for b in br]
            first = _CW(torch.cat([x[0] for x in f]), torch.cat([x[1] for x in f]))
            second = [_cw(b[1]) for b in br]
            widths = [b[1].conv.out_channels for b in br]
            lw = torch.zeros(HEAD_W, sum(widths), 1, 1, device=first.b.device)
            lb, r, c = [], 0, 0
            for b, wd in zip(br, widths):
                o = b[2].out_channels
                lw[r:r + o, c:c + wd] = b[2].weight.detach().float()
                lb.append(b[2].bias.detach().float())
                r, c = r + o, c + wd
            heads.append(SimpleNamespace(first=first, second=second, widths=widths, last=_CW(lw, torch.cat(lb))))
        w["head"] = heads
        p = seg.proto
        w["p1"], w["p2"], w["p3"] = _cw(p.cv1), _cw(p.cv2), _cw(p.cv3)
        up = p.upsample.weight.detach().float()                                     # (in, out, 2, 2)
        w["up"] = [[_CW(up[:, :, i, j].t().reshape(up.shape[1], up.shape[0], 1, 1), p.upsample.bias.detach().float()) for j in range(2)]
                   for i in range(2)]
        return w

    # ---- launches -----------------------------------------------------------------------------------------------------
    @staticmethod
    def _conv(x, cw: _CW, out, stride=1, silu=True, res=None, tap=None):
        """x (B,Hi,Wi,C) and out (B,Ho,Wo,C') NHWC views (channel slices allowed); tap (i, j): one tap of a 2x2 stride-2
        transposed convolution, out is then the (B,2Hi,2Wi,C') map"""
        B, Hi, Wi, Cin = x.shape
        if Cin != cw.cin or x.stride(3) != 1 or out.stride(3) != 1:
            raise ValueError("conv operand layout")
        sy, sx, oy, ox = (2, 2, tap[0], tap[1]) if tap is not None else (1, 1, 0, 0)
        _lib.call("sam6d_conv2d_tc", x, x.stride(2), B, Hi, Wi, Cin, cw.w, cw.k, stride, cw.cout, cw.b, int(silu), res,
                  res.stride(2) if res is not None else 0, res.stride(0) if res is not None else 0, out, int(out.dtype == torch.float32),
                  out.stride(2), out.stride(0), out.shape[2], sy, sx, oy, ox)
        return out

    def _c2f(self, x, cw, out):
        B, H, W, _ = x.shape
        c, n = cw.c, len(cw.m)
        buf = torch.empty(B, H, W, (2 + n) * c, dtype=bf, device=x.device)
        tmp = torch.empty(B, H, W, c, dtype=bf, device=x.device)
        self._conv(x, cw.cv1, buf[..., :2 * c])
        for i, (cv1, cv2, add) in enumerate(cw.m):
            inp = buf[..., (1 + i) * c:(2 + i) * c]
            self._conv(inp, cv1, tmp)
            self._conv(tmp, cv2, buf[..., (2 + i) * c:(3 + i) * c], res=inp if add else None)
        return self._conv(buf, cw.cv2, out)

    @staticmethod
    def _up(x, out):
        B, H, W, C = x.shape
        _lib.call("sam6d_yolo_upsample2x", x, x.stride(2), B, H, W, C, out, out.stride(2))

    @torch.no_grad()
    def forward(self, frames: torch.Tensor):
        if frames.dtype != torch.uint8 or frames.dim() != 4 or frames.shape[-1] != 3 or not frames.is_cuda:
            raise ValueError("frames: (B,H,W,3) uint8 CUDA tensor")
        B, H, W, _ = frames.shape
        if H % 32 or W % 32:
            raise ValueError(f"frame size {H}x{W}: letterbox to multiples of 32 first")
        w = self._weights()
        frames = frames.contiguous()
        dev = frames.device
        lay = scale_layout(self.scale)
        c0, c1, c2, c3, c4 = lay.c
        npr, conv = lay.npr, self._conv
        e = lambda h, ww, c, dt=bf: torch.empty(B, h, ww, c, dtype=dt, device=dev)   # noqa: E731
        s2, s4, s8, s16, s32 = (H // 2, W // 2), (H // 4, W // 4), (H // 8, W // 8), (H // 16, W // 16), (H // 32, W // 32)
        x0 = e(*s2, c0)
        _lib.call("sam6d_yolo_stem_c", frames, B, H, W, c0, w["stem"][0], w["stem"][1], x0)
        x1 = conv(x0, w[1], e(*s4, c1), stride=2)
        x2 = self._c2f(x1, w[2], e(*s4, c1))
        x3 = conv(x2, w[3], e(*s8, c2), stride=2)
        cat14 = e(*s8, c3 + c2)                                         # [up(12) | 4]
        self._c2f(x3, w[4], cat14[..., c3:])
        x5 = conv(cat14[..., c3:], w[5], e(*s16, c3), stride=2)
        cat11 = e(*s16, c4 + c3)                                        # [up(9) | 6]
        self._c2f(x5, w[6], cat11[..., c4:])
        x7 = conv(cat11[..., c4:], w[7], e(*s32, c4), stride=2)
        x8 = self._c2f(x7, w[8], e(*s32, c4))
        sppf = e(*s32, 2 * c4)                                          # [cv1 | 5x5 | 9x9 | 13x13], c4 / 2 each
        conv(x8, w[9].cv1, sppf[..., :c4 // 2])
        _lib.call("sam6d_yolo_sppf", sppf, 2 * c4, B, s32[0], s32[1], c4 // 2)
        cat20 = e(*s32, c3 + c4)                                        # [19 | 9]
        conv(sppf, w[9].cv2, cat20[..., c3:])
        self._up(cat20[..., c3:], cat11[..., :c4])
        cat17 = e(*s16, c2 + c3)                                        # [16 | 12]
        self._c2f(cat11, w[12], cat17[..., c2:])
        self._up(cat17[..., c2:], cat14[..., :c3])
        p3 = self._c2f(cat14, w[15], e(*s8, c2))
        conv(p3, w[16], cat17[..., :c2], stride=2)
        p4 = self._c2f(cat17, w[18], e(*s16, c3))
        conv(p4, w[19], cat20[..., :c3], stride=2)
        p5 = self._c2f(cat20, w[21], e(*s32, c4))
        # ---- Segment head: rows of all anchors, level after level
        sizes = (s8, s16, s32)
        A = sum(h * ww for h, ww in sizes)
        head = torch.empty(B, A, HEAD_W, dtype=torch.float32, device=dev)
        off = 0
        for hw, x, hc in zip(sizes, (p3, p4, p5), w["head"]):
            t1, t2 = e(*hw, sum(hc.widths)), e(*hw, sum(hc.widths))
            conv(x, hc.first, t1)
            c = 0
            for cw, wd in zip(hc.second, hc.widths):
                conv(t1[..., c:c + wd], cw, t2[..., c:c + wd])
                c += wd
            conv(t2, hc.last, head[:, off:off + hw[0] * hw[1]].unflatten(1, hw), silu=False)
            off += hw[0] * hw[1]
        pr1 = conv(p3, w["p1"], e(*s8, npr))
        up = e(*s4, npr)
        for i in range(2):
            for j in range(2):
                conv(pr1, w["up"][i][j], up, silu=False, tap=(i, j))
        pr2 = conv(up, w["p2"], e(*s4, npr))
        proto = conv(pr2, w["p3"], e(*s4, NM, torch.float32))
        return head, proto


# =====================================================================================================================
# checkpoint loading without ultralytics
# =====================================================================================================================
_ALLOWED_BUILTINS = {"object", "set", "frozenset", "dict", "list", "tuple", "slice", "bytearray", "complex", "float", "int", "str", "bool",
                     "range"}
_STUBS: Dict[tuple, type] = {}


class _FastSAMUnpickler(pickle.Unpickler):
    """maps every ultralytics.* global to an empty nn.Module subclass of the same name; resolves torch.*, collections.*,
    copyreg._reconstructor (how pickled modules are rebuilt) and plain builtins; anything else raises"""

    def find_class(self, module, name):
        root = module.split(".")[0]
        if root == "ultralytics":
            key = (module, name)
            if key not in _STUBS:
                _STUBS[key] = type(name, (nn.Module,), {"__module__": "sam6d_b200.fast_sam._ultralytics_stub"})
            return _STUBS[key]
        if root in ("torch", "collections") or (module == "copyreg" and name == "_reconstructor") or \
                (module in ("builtins", "__builtin__") and name in _ALLOWED_BUILTINS):
            return super().find_class(module, name)
        raise pickle.UnpicklingError(f"FastSAM checkpoint references a global outside the allowlist: {module}.{name}")


_pickle_module = SimpleNamespace(Unpickler=_FastSAMUnpickler, load=lambda f, **kw: _FastSAMUnpickler(f, **kw).load(),
                                 __name__="sam6d_b200.fast_sam._pickle")


def checkpoint_scale(sd: Dict[str, torch.Tensor]) -> Optional[str]:
    """the scale whose layout a state_dict's shapes announce -- model.0's output channels, the bottleneck counts of model.2 and
    model.4, model.9.cv2's output channels -- or None"""
    try:
        found = (sd["model.0.conv.weight"].shape[0], _bottlenecks(sd, "model.2"), _bottlenecks(sd, "model.4"), sd["model.9.cv2.conv.weight"].shape[0])
    except KeyError:
        return None
    for name in SCALES:
        lay = scale_layout(name)
        if found == (lay.c[0], lay.n3, lay.n6, lay.c[4]):
            return name
    return None


def _bottlenecks(sd, prefix):
    return len({k.split(".")[3] for k in sd if k.startswith(prefix + ".m.")})


def _found(sd):
    """what a state_dict holds, in the words of the rejection message"""
    def out_ch(k):
        return sd[k].shape[0] if k in sd and sd[k].dim() else "none"
    return (f"stem width {out_ch('model.0.conv.weight')}, SPPF width {out_ch('model.9.cv2.conv.weight')}, "
            f"C2f depths {_bottlenecks(sd, 'model.2')} / {_bottlenecks(sd, 'model.4')} in model.2 / model.4")


def load_fastsam_checkpoint(path) -> Dict[str, torch.Tensor]:
    """the ultralytics checkpoint `path` (FastSAM-x.pt or FastSAM-s.pt) -> fp32 state_dict with YOLOv8Seg's keys, checked
    against the layout of the scale its shapes announce (checkpoint_scale)"""
    ckpt = torch.load(path, map_location="cpu", weights_only=False, pickle_module=_pickle_module)
    model = (ckpt.get("ema") or ckpt["model"]) if isinstance(ckpt, dict) else None
    if not isinstance(model, nn.Module):
        raise ValueError(f"{path}: no 'ema' / 'model' module in the checkpoint")
    sd = {k: v.float() if v.is_floating_point() else v for k, v in model.float().state_dict().items()}
    scale = checkpoint_scale(sd)
    ref = YOLOv8Seg(scale or "x").state_dict()
    missing = sorted(set(ref) - set(sd))
    unexpected = sorted(set(sd) - set(ref))
    shapes = sorted(f"{k}: {tuple(sd[k].shape)} vs {tuple(ref[k].shape)}" for k in set(sd) & set(ref) if sd[k].shape != ref[k].shape)
    if scale is None:
        known = "; ".join(f"{n}: stem width {scale_layout(n).c[0]}, SPPF width {scale_layout(n).c[4]}, C2f depths "
                          f"{scale_layout(n).n3} / {scale_layout(n).n6}" for n in SCALES)
        raise ValueError(f"{path} is not a YOLOv8x-seg or YOLOv8s-seg (nc=1) checkpoint: found {_found(sd)} (known scales {known}); "
                         f"against YOLOv8x-seg: missing {missing}, unexpected {unexpected}, mis-shaped {shapes}")
    if missing or unexpected or shapes:
        raise ValueError(f"{path} is not a YOLOv8{scale}-seg (nc=1) checkpoint: found {_found(sd)}; missing {missing}, "
                         f"unexpected {unexpected}, mis-shaped {shapes}")
    return sd


def conv_shapes(scale: str, H: int, W: int):
    """every convolution of the network at an H x W frame, in forward order: dicts (name, Cin, Cout, k, s, H, W, Ho, Wo); the
    Proto upsample is listed once as its four 1 x 1 taps' combined Cout"""
    lay = scale_layout(scale)
    c0, c1, c2, c3, c4 = lay.c
    n3, n6, npr = lay.n3, lay.n6, lay.npr
    out = []

    def add(name, cin, cout, k, s, h, w):
        ho, wo = (h + 2 * (k // 2) - k) // s + 1, (w + 2 * (k // 2) - k) // s + 1
        out.append(dict(name=name, Cin=cin, Cout=cout, k=k, s=s, H=h, W=w, Ho=ho, Wo=wo))
        return ho, wo

    def c2f(name, ci, co, n, h, w):
        c = co // 2
        add(name + ".cv1", ci, 2 * c, 1, 1, h, w)
        for i in range(n):
            add(f"{name}.m.{i}.cv1", c, c, 3, 1, h, w)
            add(f"{name}.m.{i}.cv2", c, c, 3, 1, h, w)
        add(name + ".cv2", (2 + n) * c, co, 1, 1, h, w)

    h2 = add("model.0", 3, c0, 3, 2, H, W)
    h4 = add("model.1", c0, c1, 3, 2, *h2); c2f("model.2", c1, c1, n3, *h4)
    h8 = add("model.3", c1, c2, 3, 2, *h4); c2f("model.4", c2, c2, n6, *h8)
    h16 = add("model.5", c2, c3, 3, 2, *h8); c2f("model.6", c3, c3, n6, *h16)
    h32 = add("model.7", c3, c4, 3, 2, *h16); c2f("model.8", c4, c4, n3, *h32)
    add("model.9.cv1", c4, c4 // 2, 1, 1, *h32); add("model.9.cv2", 2 * c4, c4, 1, 1, *h32)
    c2f("model.12", c4 + c3, c3, n3, *h16); c2f("model.15", c3 + c2, c2, n3, *h8)
    add("model.16", c2, c2, 3, 2, *h8); c2f("model.18", c2 + c3, c3, n3, *h16)
    add("model.19", c3, c3, 3, 2, *h16); c2f("model.21", c3 + c4, c4, n3, *h32)
    seg = Segment(npr=npr, ch=(c2, c3, c4))
    widths = [seg.cv2[0][0].conv.out_channels, seg.cv3[0][0].conv.out_channels, seg.cv4[0][0].conv.out_channels]
    for i, (ch, hw) in enumerate(((c2, h8), (c3, h16), (c4, h32))):
        add(f"model.22.head.{i}.first", ch, sum(widths), 3, 1, *hw)
        for name, wd in zip(("cv2", "cv3", "cv4"), widths):
            add(f"model.22.{name}.{i}.1", wd, wd, 3, 1, *hw)
        add(f"model.22.head.{i}.last", sum(widths), HEAD_W, 1, 1, *hw)
    add("model.22.proto.cv1", c2, npr, 3, 1, *h8)
    add("model.22.proto.upsample", npr, 4 * npr, 1, 1, *h8)
    add("model.22.proto.cv2", npr, npr, 3, 1, h8[0] * 2, h8[1] * 2)
    add("model.22.proto.cv3", npr, NM, 1, 1, h8[0] * 2, h8[1] * 2)
    return out


# =====================================================================================================================
# host-side geometry of the predictor (LetterBox, scale_boxes, clip_boxes)
# =====================================================================================================================
def letterbox(image: np.ndarray, size: int = 640, stride: int = 32, pad_value: int = 114):
    """LetterBox(new_shape=(size,size), auto=True, stride) -> (padded image, (top, left))"""
    import cv2
    h, w = image.shape[:2]
    r = min(size / h, size / w)
    new_unpad = int(round(w * r)), int(round(h * r))
    dw, dh = np.mod(size - new_unpad[0], stride) / 2, np.mod(size - new_unpad[1], stride) / 2
    if (w, h) != new_unpad:
        image = cv2.resize(image, new_unpad, interpolation=cv2.INTER_LINEAR)
    top, bottom = int(round(dh - 0.1)), int(round(dh + 0.1))
    left, right = int(round(dw - 0.1)), int(round(dw + 0.1))
    image = cv2.copyMakeBorder(image, top, bottom, left, right, cv2.BORDER_CONSTANT, value=(pad_value,) * 3)
    return np.ascontiguousarray(image), (top, left)


def scale_boxes(img1_shape, boxes: torch.Tensor, img0_shape) -> torch.Tensor:
    """xyxy boxes in the letterboxed frame img1_shape -> the original frame img0_shape, clipped (in place)"""
    gain = min(img1_shape[0] / img0_shape[0], img1_shape[1] / img0_shape[1])
    pad = round((img1_shape[1] - img0_shape[1] * gain) / 2 - 0.1), round((img1_shape[0] - img0_shape[0] * gain) / 2 - 0.1)
    boxes[..., [0, 2]] -= pad[0]
    boxes[..., [1, 3]] -= pad[1]
    boxes[..., :4] /= gain
    boxes[..., 0].clamp_(0, img0_shape[1])
    boxes[..., 1].clamp_(0, img0_shape[0])
    boxes[..., 2].clamp_(0, img0_shape[1])
    boxes[..., 3].clamp_(0, img0_shape[0])
    return boxes


# =====================================================================================================================
class FastSAM:
    """ISM/model/fast_sam.py:FastSAM.  generate_masks(image (H,W,3) u8 RGB) -> {"masks": (N,H,W) float, "boxes": (N,4) float xyxy}.

    Behaviours of the reference kept on purpose:
      * conf is 0.25 whatever the config says: CustomYOLO sets the config's conf_threshold (0.05) and then overwrites it
        (fast_sam.py:34,39); iou = config.iou_threshold (0.9), max_det = config.max_det (200), class-aware NMS with nc = 1,
        retina_masks = False;
      * ultralytics treats a numpy frame as BGR and flips it; the reference passes RGB, so the network sees the channels reversed;
      * LetterBox to segmentor_width_size with auto=True (stride 32, pad 114); the resize is cv2 INTER_LINEAR on the host;
      * masks come out at the letterboxed shape, padding included, and postprocess_resize resamples them bilinearly to the
        original size (float masks); boxes are scale_boxes + clip_boxes in original pixels.
    Where the reference fails (no detection: `masks.data` of None), empty tensors are returned."""

    def __init__(self, checkpoint_path=None, config=None, segmentor_width_size=640, device=None, scale: Optional[str] = None):
        """scale: "x" or "s".  With a checkpoint the network is the scale the checkpoint holds (a different `scale` raises);
        without one it is `scale`, default "x"."""
        cfg = config if config is not None else SimpleNamespace(iou_threshold=0.9, conf_threshold=0.05, max_det=200)
        get = (lambda k: cfg[k]) if isinstance(cfg, dict) else (lambda k: getattr(cfg, k))
        self.iou, self.max_det = float(get("iou_threshold")), int(get("max_det"))
        self.conf = 0.25                                 # fast_sam.py:39 overrides the config's conf_threshold
        self.segmentor_width_size = segmentor_width_size
        self.current_device = torch.device(device) if device is not None else torch.device("cuda")
        sd = load_fastsam_checkpoint(checkpoint_path) if checkpoint_path is not None else None
        if sd is not None:
            held = checkpoint_scale(sd)
            if scale is not None and scale != held:
                raise ValueError(f"scale={scale!r} but {checkpoint_path} holds YOLOv8{held}-seg")
            scale = held
        self.model = YOLOv8Seg(scale or "x").to(self.current_device).eval()
        if sd is not None:
            self.model.load_state_dict(sd, strict=True)

    @torch.no_grad()
    def postprocess(self, head: torch.Tensor, proto: torch.Tensor, shape) -> Dict[str, torch.Tensor]:
        """one frame: head (A,97) f32, proto (mh,mw,32) f32, letterboxed shape (ih,iw) -> kept candidate rows (N,38) (x1,y1,x2,y2,
        conf,cls,32 coefficients; letterboxed pixels) and masks (N,ih,iw) u8"""
        ih, iw = shape
        mh, mw = proto.shape[:2]
        sizes = [(ih // s, iw // s) for s in STRIDES]
        A = head.shape[0]
        cand = torch.empty(A, 6 + NM, dtype=torch.float32, device=head.device)
        count = torch.empty(1, dtype=torch.int32, device=head.device)
        _lib.call("sam6d_yolo_decode", head, head.stride(0), A * head.stride(0), 1, *[v for hw in sizes for v in hw], self.conf, cand,
                  count)
        rows = cand[:int(count.item())]
        order = torch.argsort(rows[:, 4], descending=True, stable=True)
        rows = rows[order]
        keep = torch.empty(rows.shape[0], dtype=torch.uint8, device=rows.device)
        if rows.shape[0]:
            boxes = rows[:, :4].contiguous()
            _lib.call("sam6d_sam_nms", boxes, None, rows.shape[0], self.iou, keep)
        rows = rows[keep.bool()][:self.max_det].contiguous()
        masks = torch.empty(rows.shape[0], ih, iw, dtype=torch.uint8, device=rows.device)
        if rows.shape[0]:
            low = torch.empty(rows.shape[0], mh, mw, dtype=torch.float32, device=rows.device)
            _lib.call("sam6d_yolo_masks", proto.contiguous(), mh, mw, rows, rows.stride(0), rows.shape[0], ih, iw, mw / iw, mh / ih, low,
                      masks)
        return {"rows": rows, "masks": masks}

    def postprocess_resize(self, detections, orig_size):
        """fast_sam.py:94-113 (update_boxes=False)"""
        if detections["masks"].shape[0] and tuple(detections["masks"].shape[-2:]) != tuple(orig_size):
            detections["masks"] = F.interpolate(detections["masks"].unsqueeze(1).float(), size=(orig_size[0], orig_size[1]), mode="bilinear",
                                                align_corners=False)[:, 0, :, :]
        return detections

    @torch.no_grad()
    def generate_masks(self, image: np.ndarray) -> Dict[str, Any]:
        orig_size = image.shape[:2]
        lb, _ = letterbox(image, self.segmentor_width_size)
        frames = torch.from_numpy(lb).to(self.current_device).unsqueeze(0)
        head, proto = self.model(frames)
        d = self.postprocess(head[0], proto[0], lb.shape[:2])
        boxes = scale_boxes(lb.shape[:2], d["rows"][:, :4].clone(), orig_size)
        return self.postprocess_resize({"masks": d["masks"].float(), "boxes": boxes}, orig_size)
