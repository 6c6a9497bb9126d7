"""Times SamPredictor (sam6d_b200/sam_amg.py) on one GPU in one process and prints one JSON line, for a seeded ViT-B and ViT-H:
  * set_image on one 480 x 640 frame (resize, normalise, image encoder, dense positional encoding);
  * predict_torch for 1, 16, 64 and 200 boxes, with and without a (B,1,256,256) mask_input, multimask_output on and off
    (thresholded masks at 480 x 640, what a box-prompted caller gets); the peak device memory of the 200-box calls;
  * per launch: sam6d_sam_mask_embed at 200 prompts (bytes written over kernel time, against the H100 SXM's 3.35 TB/s) and
    sam6d_sam_tok2img_attn at T = 32 against T = 8 (64 prompts, 4096 keys, per-prompt K / V);
  * CustomSamAutomaticMaskGenerator.generate_masks on the same frame (32 x 32 point grid), the yardstick.
CUDA events after warm-up.  Seeded weights (speed does not depend on their values).  The card's name and power limit are read
with nvidia-smi in the same run.

    python tools/sam_predictor_bench.py [--iters 10] [--types vit_b,vit_h]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_TBS = 3.35                  # H100 SXM5 80 GB peak DRAM bandwidth


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


def _kernel_us(lib, name, fn, iters):
    """mean time per launch of C-ABI function `name` inside fn, from the events _lib brackets it with"""
    fn()
    torch.cuda.synchronize()
    lib.time_kernel(name)
    for _ in range(iters):
        fn()
    torch.cuda.synchronize()
    ev = lib.timed_events(name)
    lib.time_kernel(name, False)
    return 1e3 * sum(a.elapsed_time(b) for a, b in ev) / len(ev)


def _boxes(n, H, W, g):
    xy = torch.rand(n, 2, generator=g) * torch.tensor([0.6 * W, 0.6 * H])
    wh = 40 + torch.rand(n, 2, generator=g) * torch.tensor([0.35 * W, 0.35 * H])
    return torch.cat([xy, xy + wh], dim=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--types", default="vit_b,vit_h")
    args = ap.parse_args()
    from sam6d_b200 import _lib, synth
    from sam6d_b200.sam import VIT_CONFIGS
    from sam6d_b200.sam_amg import CustomSamAutomaticMaskGenerator, SamPredictor, sam_model_registry

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    dev = torch.device("cuda")
    res = dict(card=card)
    H, W = 480, 640
    frame = (synth.make_images(B=1, seed=3)[0, :, :H, :W].permute(1, 2, 0).clamp(-2, 2) * 60 + 128).to(torch.uint8).numpy()
    frame = np.ascontiguousarray(frame)
    g = torch.Generator().manual_seed(0)

    for t in args.types.split(","):
        r = {}
        sam = sam_model_registry[t]("bf16").to(dev).eval()
        sd = {"image_encoder." + k: v for k, v in synth.make_sam_state_dict(**VIT_CONFIGS[t], seed=1).items()}
        sd.update(synth.make_sam_decoder_state_dict(seed=1))
        sam.load_state_dict(sd, strict=True)
        del sd
        p = SamPredictor(sam)
        r["set_image_ms"] = round(_time(lambda: p.set_image(frame), args.iters), 2)
        for n in (1, 16, 64, 200):
            boxes = p.transform.apply_boxes_torch(_boxes(n, H, W, g).to(dev), (H, W))
            mask_in = synth.make_images(B=n, size=256, seed=n)[:, :1].mul(8).to(dev).contiguous()
            for use_mask in (False, True):
                for multi in (True, False):
                    key = f"predict_torch_{n}box{'_mask' if use_mask else ''}_{'multi' if multi else 'single'}_ms"
                    fn = lambda: p.predict_torch(None, None, boxes=boxes, mask_input=mask_in if use_mask else None,  # noqa: E731
                                                 multimask_output=multi)
                    if n == 200:
                        torch.cuda.synchronize()
                        torch.cuda.reset_peak_memory_stats()
                    r[key] = round(_time(fn, max(2, args.iters // (1 + n // 64)), warmup=2), 2)
                    if n == 200:
                        r[key[:-3] + "_peak_gib"] = round(torch.cuda.max_memory_allocated() / 2 ** 30, 2)
        if t == args.types.split(",")[0]:
            # per launch: the mask-prompt embedding at 200 prompts, tok2img at T = 32 and T = 8
            m = synth.make_images(B=200, size=256, seed=1)[:, :1].mul(8).to(dev).contiguous()
            us = _kernel_us(_lib, "sam6d_sam_mask_embed", lambda: sam.prompt_encoder.embed_masks(m), args.iters)
            nbytes = 200 * 4096 * 256 * 4
            r["mask_embed_200_us"] = round(us, 1)
            r["mask_embed_200_tbs"] = round(nbytes / us / 1e6, 2)
            r["mask_embed_200_frac_of_peak"] = round(nbytes / us / 1e6 / HBM_TBS, 3)
            B, L = 64, 4096
            K = torch.randn(B, L, 128, device=dev).to(torch.bfloat16)
            V = torch.randn(B, L, 128, device=dev).to(torch.bfloat16)
            for T in (8, 32):
                Q = torch.randn(B, T, 128, device=dev)
                O = torch.empty_like(Q)
                call = lambda: _lib.call("sam6d_sam_tok2img_attn", ctypes.c_void_p(Q.data_ptr()), ctypes.c_void_p(K.data_ptr()),  # noqa: E731
                                         ctypes.c_void_p(V.data_ptr()), ctypes.c_longlong(L * 128), B, T, L, ctypes.c_void_p(O.data_ptr()),
                                         ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
                r[f"tok2img_b64_T{T}_us"] = round(_kernel_us(_lib, "sam6d_sam_tok2img_attn", call, args.iters), 1)
            del K, V, m
        amg = CustomSamAutomaticMaskGenerator(sam, points_per_batch=64, stability_score_thresh=0.97, box_nms_thresh=0.7,
                                              segmentor_width_size=640)
        r["generate_masks_480x640_ms"] = round(_time(lambda: amg.generate_masks(frame), 3, warmup=1), 1)
        res[t] = r
        del sam, p, amg
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
