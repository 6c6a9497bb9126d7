"""Times the three SAM backbones of the ISM segmentor (vit_b, vit_l, vit_h) on one GPU in one process and prints one JSON line:
  * the image encoder (bf16) at B = 1 and B = 8 on 1024 x 1024 inputs: CUDA events after warm-up, algorithmic GFLOP per frame
    from the shapes (encoder_gflop below) over the measured time;
  * sam6d_attn_global_tc_ex alone, per launch, at head dim 64 (vit_b: 12 heads, vit_l: 16 heads) and 80 (vit_h: 16 heads) for
    B = 1 and B = 8 images, with the QK^T + PV FLOPs (4 B H L^2 D, L = 4096) over kernel time;
  * CustomSamAutomaticMaskGenerator.generate_masks on one 480 x 640 frame (32 x 32 point grid, the CLI's settings).
Seeded weights (speed does not depend on their values).  The card's name, power limit and maximum SM clock are read with
nvidia-smi in the same run.

    python tools/sam_encoder_bench.py [--iters 10]"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TYPES = ("vit_b", "vit_l", "vit_h")


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


def encoder_gflop(embed_dim, depth, num_heads, global_attn_indexes, img=1024, patch=16, window=14, out_chans=256):
    """multiply-adds x 2 of one frame through ImageEncoderViT as the reference formulates it: patch embed; per block qkv over
    the tokens the attention sees (the 64 x 64 grid padded to 70 x 70 for the 25 windows of 14 x 14), QK^T and PV per window
    (or over the 4096 tokens), the two rel-pos tables (q . rel per key row and column), proj over the same tokens, the MLP
    over the 4096 tokens; the neck (1x1 conv, 3x3 conv).  LayerNorm, softmax, GELU are not counted."""
    C, G = embed_dim, img // patch
    L = G * G
    Gp = -(-G // window) * window
    f = 2 * L * C * 3 * patch * patch
    for i in range(depth):
        if i in global_attn_indexes:
            T, n, S = L, L, G
        else:
            T, n, S = Gp * Gp, window * window, window
        f += 2 * T * C * 3 * C                      # qkv
        f += 2 * 2 * (T // n) * n * n * C           # QK^T and PV over all heads
        f += 2 * 2 * T * S * C                      # q . rel_h, q . rel_w
        f += 2 * T * C * C                          # proj
        f += 2 * 2 * L * C * 4 * C                  # MLP
    f += 2 * L * C * out_chans + 2 * L * out_chans * out_chans * 9
    return f / 1e9


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    from sam6d_b200 import ops, synth
    from sam6d_b200.sam import VIT_CONFIGS
    from sam6d_b200.sam_amg import CustomSamAutomaticMaskGenerator, sam_model_registry

    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()[0]
    dev = torch.device("cuda")
    res = dict(card=card)
    frame = (synth.make_images(B=1, seed=3)[0, :, :480, :640].permute(1, 2, 0).clamp(-2, 2) * 60 + 128).to(torch.uint8).numpy()
    frame = np.ascontiguousarray(frame)

    for t in TYPES:
        cfg = VIT_CONFIGS[t]
        r = dict(gflop_per_frame=round(encoder_gflop(**cfg), 1))
        sam = sam_model_registry[t]("bf16").to(dev).eval()
        sd = {"image_encoder." + k: v for k, v in synth.make_sam_state_dict(**cfg, seed=1).items()}
        sd.update(synth.make_sam_decoder_state_dict(seed=1))
        sam.load_state_dict(sd, strict=True)
        del sd
        enc = sam.image_encoder
        for B in (1, 8):
            x = synth.make_images(B=B, seed=1).to(dev)
            ms = _time(lambda: enc(x), args.iters)
            r[f"encoder_b{B}_ms"] = round(ms, 2)
            r[f"encoder_b{B}_tflops"] = round(r["gflop_per_frame"] * B / ms, 1)
            del x
        # the global attention kernel alone at this backbone's head dim
        H, D, S = cfg["num_heads"], cfg["embed_dim"] // cfg["num_heads"], 64
        L = S * S
        blk = enc.blocks[cfg["global_attn_indexes"][0]]
        blob = ops.pack_rel_pos(blk.attn.rel_pos_h.detach().float().contiguous(), blk.attn.rel_pos_w.detach().float().contiguous(),
                                slab_rows=128)
        for B in (1, 8):
            g = torch.Generator(device=dev).manual_seed(B)
            qkv = torch.randn(B * L, 3 * H * D, device=dev, generator=g).to(torch.bfloat16)
            vt = ops.transpose_tokens(qkv, 2 * H * D, H * D, B, L)
            ms = _time(lambda: ops.attn_global_tc(qkv, vt, blob, B, H, S, D ** -0.5, D=D), 5 * args.iters)
            r[f"attn_global_D{D}_H{H}_b{B}_us"] = round(ms * 1e3, 1)
            r[f"attn_global_D{D}_H{H}_b{B}_tflops"] = round(4.0 * B * H * L * L * D / ms / 1e9, 1)
            del qkv, vt
        amg = CustomSamAutomaticMaskGenerator(sam, points_per_batch=64, stability_score_thresh=0.97, box_nms_thresh=0.7,
                                              segmentor_width_size=640)
        r["generate_masks_480x640_ms"] = round(_time(lambda: amg.generate_masks(frame), 3, warmup=1), 1)
        enc_share = r["encoder_b1_ms"] / r["generate_masks_480x640_ms"]
        r["encoder_b1_over_generate_masks"] = round(enc_share, 3)
        res[t] = r
        del amg, sam, enc, blk, blob
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
