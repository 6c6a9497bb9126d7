"""Times the FastSAM segmentor on one GPU and prints one JSON line: the YOLOv8x-seg or YOLOv8s-seg (--scale x / s) forward on
a 480 x 640 frame at B = 1 and B = 8 (CUDA events, GFLOP of the executed convolutions over time); FastSAM.generate_masks end
to end per frame; every distinct convolution shape alone at B = 1 and B = 8 with achieved TFLOP/s; and two yardsticks measured in the same run: torch /
cuDNN bf16 channels_last convolutions of the same network (the oracle's fused layers), and the SAM path's
CustomSamAutomaticMaskGenerator.generate_masks on the same frame.  Seeded weights (speed does not depend on their values).
The card's name, power limit and maximum SM clock are read with nvidia-smi in the same run.

    python tools/fastsam_bench.py [--scale x] [--iters 20]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _time(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", default="x", choices=("x", "s"))
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    from oracle import fastsam_oracle as fo
    from sam6d_b200 import synth
    from sam6d_b200.fast_sam import FastSAM, YOLOv8Seg, _CW, conv_shapes

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    dev = torch.device("cuda")
    sd = synth.make_fastsam_state_dict(1, args.scale)
    frame = synth.make_fastsam_frame(480, 640, 0)
    shapes = conv_shapes(args.scale, 480, 640)
    gflop = sum(2.0 * l["Cout"] * l["Cin"] * l["k"] ** 2 * l["Ho"] * l["Wo"] for l in shapes) / 1e9
    res = dict(card=card, scale=args.scale, frame="480x640", gflop_per_frame=round(gflop, 2))

    net = YOLOv8Seg(args.scale).to(dev).eval()
    net.load_state_dict(sd, strict=True)
    for B in (1, 8):
        x = torch.from_numpy(np.stack([frame] * B)).to(dev)
        ms = _time(lambda: net(x), args.iters)
        res[f"forward_b{B}_ms"] = round(ms, 3)
        res[f"forward_b{B}_tflops"] = round(gflop * B / ms, 1)

    seg = FastSAM(None, dict(iou_threshold=0.9, conf_threshold=0.05, max_det=200), device=dev, scale=args.scale)
    seg.model.load_state_dict(sd, strict=True)
    res["generate_masks_ms"] = round(_time(lambda: seg.generate_masks(frame), args.iters), 3)
    res["generate_masks_detections"] = int(seg.generate_masks(frame)["masks"].shape[0])

    # every distinct convolution shape alone (the Cin = 3 stem is its own kernel; the Proto upsample runs as 1 x 1 taps)
    seen, layers = set(), []
    g = torch.Generator(device=dev).manual_seed(0)
    for l in shapes:
        key = (l["H"], l["W"], l["Cin"], l["Cout"], l["k"], l["s"])
        if l["Cin"] == 3 or "upsample" in l["name"] or key in seen:
            continue
        seen.add(key)
        cw = _CW(torch.randn(l["Cout"], l["Cin"], l["k"], l["k"], device=dev, generator=g) * 0.05, torch.zeros(l["Cout"], device=dev))
        row = dict(layer=l["name"], shape=f"{l['Cin']}->{l['Cout']} k{l['k']} s{l['s']} {l['H']}x{l['W']}")
        for B in (1, 8):
            x = torch.randn(B, l["H"], l["W"], l["Cin"], device=dev, generator=g).to(torch.bfloat16)
            y = torch.empty(B, l["Ho"], l["Wo"], l["Cout"], device=dev, dtype=torch.bfloat16)
            fl = 2.0 * B * l["Cout"] * l["Cin"] * l["k"] ** 2 * l["Ho"] * l["Wo"]
            ms = _time(lambda: YOLOv8Seg._conv(x, cw, y, stride=l["s"]), 4 * args.iters)
            row[f"b{B}_us"] = round(ms * 1e3, 1)
            row[f"b{B}_tflops"] = round(fl / ms / 1e9, 1)
        layers.append(row)
    res["layers"] = layers

    # yardstick 1: the oracle's network (fused as ultralytics fuses it) in torch / cuDNN, bf16 channels_last
    class _Cudnn(fo.Net):
        def __init__(self, sd):
            self.sd, self.fused = sd, {}

        def conv(self, x, p, s=1, act=True):
            if p not in self.fused:
                w, b = fo.fuse_conv_and_bn(*(self.sd[p + k].float().cpu() for k in (".conv.weight", ".bn.weight", ".bn.bias", ".bn.running_mean",
                                                                                   ".bn.running_var")))
                self.fused[p] = (w.to(dev, torch.bfloat16).contiguous(memory_format=torch.channels_last), b.to(dev, torch.bfloat16))
            w, b = self.fused[p]
            y = F.conv2d(x, w, b, s, w.shape[-1] // 2)
            return F.silu(y) if act else y

    plain = lambda k: (".conv." not in k and ".bn." not in k) or k.endswith("dfl.conv.weight")   # noqa: E731  (not folded)
    ref = _Cudnn({k: (v.to(dev, torch.bfloat16) if plain(k) and v.is_floating_point() else v) for k, v in sd.items()})
    xin = fo.preprocess([frame]).to(dev, torch.bfloat16).contiguous(memory_format=torch.channels_last)
    with torch.no_grad():
        res["cudnn_bf16_forward_b1_ms"] = round(_time(lambda: ref.forward(xin), args.iters), 3)

    # yardstick 2: the SAM path on the same frame
    from sam6d_b200.sam_amg import CustomSamAutomaticMaskGenerator, build_sam_vit_h
    sam = build_sam_vit_h("bf16").to(dev).eval()
    s_sd = {"image_encoder." + k: v for k, v in synth.make_sam_state_dict(embed_dim=1280, depth=32, num_heads=16, global_attn_indexes=(7, 15, 23, 31),
                                                                           seed=1).items()}
    s_sd.update(synth.make_sam_decoder_state_dict(seed=1))
    sam.load_state_dict(s_sd, strict=True)
    amg = CustomSamAutomaticMaskGenerator(sam, points_per_batch=64, stability_score_thresh=0.97, box_nms_thresh=0.7, segmentor_width_size=640)
    res["sam_generate_masks_ms"] = round(_time(lambda: amg.generate_masks(frame), 3, warmup=1), 1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
