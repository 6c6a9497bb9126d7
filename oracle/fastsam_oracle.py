"""CPU fp32 restatement of FastSAM-x (ISM/model/fast_sam.py over ultralytics 8.0.135): the YOLOv8x-seg SegmentationModel at nc=1,
fused as AutoBackend(fuse=True) fuses it, and the SegmentationPredictor steps -- LetterBox and the BGR flip, non_max_suppression
(with torchvision.ops.nms), process_mask, scale_boxes / clip_boxes -- and FastSAM.generate_masks / postprocess_resize.

ultralytics is not installed, so this is a restatement from the 8.0.135 sources as published, not checked against them
(DESIGN.md section 3 lists the rules restated).  It works on a state_dict with ultralytics' keys and plain torch functions only."""

import numpy as np
import torch
import torch.nn.functional as F

REG_MAX, NM = 16, 32
STRIDES = (8.0, 16.0, 32.0)


# ---------------------------------------------------------------------------------------------------------------- network
def fuse_conv_and_bn(w, bn_w, bn_b, mean, var, eps=1e-3):
    """ultralytics.utils.torch_utils.fuse_conv_and_bn (conv without bias)"""
    w_conv = w.clone().view(w.shape[0], -1)
    w_bn = torch.diag(bn_w.div(torch.sqrt(eps + var)))
    fw = torch.mm(w_bn, w_conv).view(w.shape)
    b_conv = torch.zeros(w.shape[0])
    fb = torch.mm(w_bn, b_conv.reshape(-1, 1)).reshape(-1) + (bn_b - bn_w.mul(mean).div(torch.sqrt(var + eps)))
    return fw, fb


class Net:
    def __init__(self, sd):
        self.sd = {k: v.float() for k, v in sd.items()}

    def conv(self, x, p, s=1, act=True):
        sd = self.sd
        w, b = fuse_conv_and_bn(sd[p + ".conv.weight"], sd[p + ".bn.weight"], sd[p + ".bn.bias"], sd[p + ".bn.running_mean"],
                                sd[p + ".bn.running_var"])
        k = w.shape[-1]
        y = F.conv2d(x, w, b, s, k // 2)
        return F.silu(y) if act else y

    def c2f(self, x, p, shortcut):
        y = list(self.conv(x, p + ".cv1").chunk(2, 1))
        n = len({k.split(".")[3] for k in self.sd if k.startswith(p + ".m.")})
        for i in range(n):
            z = self.conv(self.conv(y[-1], f"{p}.m.{i}.cv1"), f"{p}.m.{i}.cv2")
            y.append(y[-1] + z if shortcut else z)
        return self.conv(torch.cat(y, 1), p + ".cv2")

    def sppf(self, x, p):
        x = self.conv(x, p + ".cv1")
        y1 = F.max_pool2d(x, 5, 1, 2)
        y2 = F.max_pool2d(y1, 5, 1, 2)
        return self.conv(torch.cat((x, y1, y2, F.max_pool2d(y2, 5, 1, 2)), 1), p + ".cv2")

    def forward(self, x):
        """x (B,3,H,W) fp32 network input -> dict(raw (B,A,97) = per anchor [64 DFL logits | class logit | 32 coefficients],
        pred (B,37,A) = Segment's output [xywh | sigmoid(class) | coefficients], proto (B,32,H/4,W/4), sizes of the levels)"""
        c, up = self.conv, (lambda t: F.interpolate(t, scale_factor=2.0, mode="nearest"))
        y = {}
        x = c(x, "model.0", 2); x = c(x, "model.1", 2); x = self.c2f(x, "model.2", True); x = c(x, "model.3", 2)
        y[4] = x = self.c2f(x, "model.4", True); x = c(x, "model.5", 2); y[6] = x = self.c2f(x, "model.6", True)
        x = c(x, "model.7", 2); x = self.c2f(x, "model.8", True); y[9] = x = self.sppf(x, "model.9")
        x = torch.cat((up(x), y[6]), 1); y[12] = x = self.c2f(x, "model.12", False)
        x = torch.cat((up(x), y[4]), 1); p3 = x = self.c2f(x, "model.15", False)
        x = torch.cat((c(x, "model.16", 2), y[12]), 1); p4 = x = self.c2f(x, "model.18", False)
        x = torch.cat((c(x, "model.19", 2), y[9]), 1); p5 = self.c2f(x, "model.21", False)
        sd, B = self.sd, p3.shape[0]

        def branch(t, name, i):
            t = c(c(t, f"model.22.{name}.{i}.0"), f"model.22.{name}.{i}.1")
            return F.conv2d(t, sd[f"model.22.{name}.{i}.2.weight"], sd[f"model.22.{name}.{i}.2.bias"])

        feats = (p3, p4, p5)
        raw = torch.cat([torch.cat([branch(f, "cv2", i), branch(f, "cv3", i), branch(f, "cv4", i)], 1).flatten(2) for i, f in enumerate(feats)], 2)
        pr = c(p3, "model.22.proto.cv1")
        pr = F.conv_transpose2d(pr, sd["model.22.proto.upsample.weight"], sd["model.22.proto.upsample.bias"], stride=2)
        proto = c(c(pr, "model.22.proto.cv2"), "model.22.proto.cv3")
        sizes = [tuple(f.shape[2:]) for f in feats]
        return dict(raw=raw.transpose(1, 2).contiguous(), pred=decode(raw, sizes, sd["model.22.dfl.conv.weight"]), proto=proto, sizes=sizes)


def make_anchors(sizes, offset=0.5):
    pts, st = [], []
    for (h, w), s in zip(sizes, STRIDES):
        sy, sx = torch.meshgrid(torch.arange(h, dtype=torch.float32) + offset, torch.arange(w, dtype=torch.float32) + offset, indexing="ij")
        pts.append(torch.stack((sx, sy), -1).view(-1, 2))
        st.append(torch.full((h * w, 1), s))
    return torch.cat(pts), torch.cat(st)


def decode(raw, sizes, dfl_w):
    """Detect's inference tail + Segment's concatenation: raw (B,97,A) -> (B,37,A)"""
    B, _, A = raw.shape
    anchors, strides = (t.transpose(0, 1).to(raw.device, raw.dtype) for t in make_anchors(sizes))
    box, cls, mc = raw.split((4 * REG_MAX, 1, NM), 1)
    d = F.conv2d(box.view(B, 4, REG_MAX, A).transpose(2, 1).softmax(1), dfl_w).view(B, 4, A)     # DFL
    lt, rb = d.chunk(2, 1)
    x1y1, x2y2 = anchors.unsqueeze(0) - lt, anchors.unsqueeze(0) + rb
    dbox = torch.cat(((x1y1 + x2y2) / 2, x2y2 - x1y1), 1) * strides                                 # dist2bbox(xywh=True)
    return torch.cat((dbox, cls.sigmoid(), mc), 1)


# ---------------------------------------------------------------------------------------------------------------- predictor
def letterbox(img, new_shape=(640, 640), stride=32, color=(114, 114, 114)):
    """LetterBox(auto=True, center=True) -> (image, ratio, (dw, dh))"""
    import cv2
    shape = img.shape[:2]
    r = min(new_shape[0] / shape[0], new_shape[1] / shape[1])
    new_unpad = int(round(shape[1] * r)), int(round(shape[0] * r))
    dw, dh = new_shape[1] - new_unpad[0], new_shape[0] - new_unpad[1]
    dw, dh = np.mod(dw, stride), np.mod(dh, stride)
    dw /= 2
    dh /= 2
    if shape[::-1] != new_unpad:
        img = cv2.resize(img, new_unpad, interpolation=cv2.INTER_LINEAR)
    top, bottom = int(round(dh - 0.1)), int(round(dh + 0.1))
    left, right = int(round(dw - 0.1)), int(round(dw + 0.1))
    img = cv2.copyMakeBorder(img, top, bottom, left, right, cv2.BORDER_CONSTANT, value=color)
    return img, (r, r), (dw, dh)


def preprocess(imgs):
    """BasePredictor.preprocess for a list of letterboxed numpy frames: BGR -> RGB flip, HWC -> CHW, /255"""
    im = np.stack(imgs)[..., ::-1].transpose((0, 3, 1, 2))
    return torch.from_numpy(np.ascontiguousarray(im)).float() / 255


def xywh2xyxy(x):
    y = x.clone()
    y[..., 0] = x[..., 0] - x[..., 2] / 2
    y[..., 1] = x[..., 1] - x[..., 3] / 2
    y[..., 2] = x[..., 0] + x[..., 2] / 2
    y[..., 3] = x[..., 1] + x[..., 3] / 2
    return y


def non_max_suppression(prediction, conf_thres=0.25, iou_thres=0.9, max_det=200, nc=1, max_nm=30000, max_wh=7680, stable=True):
    """ultralytics.utils.ops.non_max_suppression (classes=None, agnostic=False, multi_label=False).  The confidence sort is
    stable here (ultralytics' argsort is not: the order of exact ties is unspecified there)."""
    import torchvision
    bs = prediction.shape[0]
    nm = prediction.shape[1] - nc - 4
    mi = 4 + nc
    xc = prediction[:, 4:mi].amax(1) > conf_thres
    output = [torch.zeros((0, 6 + nm))] * bs
    for xi, x in enumerate(prediction):
        x = x.transpose(0, -1)[xc[xi]]
        if not x.shape[0]:
            continue
        box, cls, mask = x.split((4, nc, nm), 1)
        box = xywh2xyxy(box)
        conf, j = cls.max(1, keepdim=True)
        x = torch.cat((box, conf, j.float(), mask), 1)[conf.view(-1) > conf_thres]
        if not x.shape[0]:
            continue
        x = x[x[:, 4].argsort(descending=True, stable=stable)[:max_nm]]
        c = x[:, 5:6] * max_wh
        boxes, scores = x[:, :4] + c, x[:, 4]
        i = torchvision.ops.nms(boxes, scores, iou_thres)[:max_det]
        output[xi] = x[i]
    return output


def crop_mask(masks, boxes):
    n, h, w = masks.shape
    x1, y1, x2, y2 = torch.chunk(boxes[:, :, None], 4, 1)
    r = torch.arange(w, dtype=x1.dtype)[None, None, :]
    c = torch.arange(h, dtype=x1.dtype)[None, :, None]
    return masks * ((r >= x1) * (r < x2) * (c >= y1) * (c < y2))


def process_mask(protos, masks_in, bboxes, shape, upsample=True, return_prob=False):
    """protos (32,mh,mw) -> (N,ih,iw) float 0/1 (and the pre-threshold probabilities when return_prob)"""
    c, mh, mw = protos.shape
    ih, iw = shape
    masks = (masks_in @ protos.float().view(c, -1)).sigmoid().view(-1, mh, mw)
    db = bboxes.clone()
    db[:, 0] *= mw / iw
    db[:, 2] *= mw / iw
    db[:, 3] *= mh / ih
    db[:, 1] *= mh / ih
    masks = crop_mask(masks, db)
    if upsample:
        masks = F.interpolate(masks[None], shape, mode="bilinear", align_corners=False)[0]
    return (masks.gt(0.5).float(), masks) if return_prob else masks.gt_(0.5)


def clip_boxes(boxes, shape):
    boxes[..., 0].clamp_(0, shape[1])
    boxes[..., 1].clamp_(0, shape[0])
    boxes[..., 2].clamp_(0, shape[1])
    boxes[..., 3].clamp_(0, shape[0])
    return boxes


def scale_boxes(img1_shape, boxes, img0_shape):
    gain = min(img1_shape[0] / img0_shape[0], img1_shape[1] / img0_shape[1])
    pad = round((img1_shape[1] - img0_shape[1] * gain) / 2 - 0.1), round((img1_shape[0] - img0_shape[0] * gain) / 2 - 0.1)
    boxes[..., [0, 2]] -= pad[0]
    boxes[..., [1, 3]] -= pad[1]
    boxes[..., :4] /= gain
    return clip_boxes(boxes, img0_shape)


def generate_masks(sd, image, size=640, conf=0.25, iou=0.9, max_det=200, net=None):
    """FastSAM.generate_masks on one RGB frame -> {"masks": (N,H,W) float, "boxes": (N,4), "scores": (N), "lb_shape", "out": forward}"""
    net = net or Net(sd)
    lb, _, _ = letterbox(image, (size, size))
    x = preprocess([lb])
    with torch.no_grad():
        out = net.forward(x)
    det = non_max_suppression(out["pred"], conf, iou, max_det=max_det)[0]
    shape = x.shape[2:]
    masks = process_mask(out["proto"][0], det[:, 6:], det[:, :4], shape, upsample=True) if det.shape[0] else torch.zeros(0, *shape)
    boxes = scale_boxes(shape, det[:, :4].clone(), image.shape[:2])
    if masks.shape[0]:
        masks = F.interpolate(masks.unsqueeze(1).float(), size=image.shape[:2], mode="bilinear", align_corners=False)[:, 0]
    return {"masks": masks, "boxes": boxes, "scores": det[:, 4], "det": det, "lb_shape": tuple(shape), "out": out}


def param_count(sd):
    """learnable parameters (BatchNorm running statistics and counters are buffers)"""
    return sum(v.numel() for k, v in sd.items() if not k.endswith(("num_batches_tracked", "running_mean", "running_var")))


def flops(sizes_hw=(480, 640)):
    """algorithmic GFLOP of one frame (2 x MACs of every convolution), from the layer shapes"""
    return sum(2.0 * l["Cout"] * l["Cin"] * l["k"] * l["k"] * l["Ho"] * l["Wo"] for l in conv_shapes(*sizes_hw)) / 1e9


def conv_shapes(H, W):
    """(name, Cin, Cout, k, stride, Hin, Win, Ho, Wo) of every convolution of the network at an H x W frame, from the layer table"""
    out = []

    def add(name, cin, cout, k, s, h, w):
        ho, wo = (h + 2 * (k // 2) - k) // s + 1, (w + 2 * (k // 2) - k) // s + 1
        out.append(dict(name=name, Cin=cin, Cout=cout, k=k, s=s, H=h, W=w, Ho=ho, Wo=wo))
        return ho, wo

    def c2f(name, c1, c2, n, h, w):
        c = c2 // 2
        add(name + ".cv1", c1, 2 * c, 1, 1, h, w)
        for i in range(n):
            add(f"{name}.m.{i}.cv1", c, c, 3, 1, h, w)
            add(f"{name}.m.{i}.cv2", c, c, 3, 1, h, w)
        add(name + ".cv2", (2 + n) * c, c2, 1, 1, h, w)

    h, w = add("model.0", 3, 80, 3, 2, H, W)
    h, w = add("model.1", 80, 160, 3, 2, h, w); c2f("model.2", 160, 160, 3, h, w)
    h8 = add("model.3", 160, 320, 3, 2, h, w); c2f("model.4", 320, 320, 6, *h8)
    h16 = add("model.5", 320, 640, 3, 2, *h8); c2f("model.6", 640, 640, 6, *h16)
    h32 = add("model.7", 640, 640, 3, 2, *h16); c2f("model.8", 640, 640, 3, *h32)
    add("model.9.cv1", 640, 320, 1, 1, *h32); add("model.9.cv2", 1280, 640, 1, 1, *h32)
    c2f("model.12", 1280, 640, 3, *h16); c2f("model.15", 960, 320, 3, *h8)
    add("model.16", 320, 320, 3, 2, *h8); c2f("model.18", 960, 640, 3, *h16)
    add("model.19", 640, 640, 3, 2, *h16); c2f("model.21", 1280, 640, 3, *h32)
    for i, (ch, hw) in enumerate(((320, h8), (640, h16), (640, h32))):
        for name, width, o in (("cv2", 80, 64), ("cv3", 320, 1), ("cv4", 80, 32)):
            add(f"model.22.{name}.{i}.0", ch, width, 3, 1, *hw)
            add(f"model.22.{name}.{i}.1", width, width, 3, 1, *hw)
            add(f"model.22.{name}.{i}.2", width, o, 1, 1, *hw)
    add("model.22.proto.cv1", 320, 320, 3, 1, *h8)
    add("model.22.proto.upsample", 320, 320 * 4, 1, 1, *h8)          # 2x2 stride-2 transposed conv: 4 taps of a 1x1
    add("model.22.proto.cv2", 320, 320, 3, 1, h8[0] * 2, h8[1] * 2)
    add("model.22.proto.cv3", 320, 32, 1, 1, h8[0] * 2, h8[1] * 2)
    return out
