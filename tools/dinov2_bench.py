"""Times the four DINOv2 descriptor backbones of the ISM (dinov2_vits14, vitb14, vitl14, vitg14) on one GPU in one process and
prints one JSON line:
  * CustomDINOv2.compute_cls_and_patch_features on P = 42 (the templates of one object), 100 and 200 (FastSAM's max_det)
    224 x 224 proposal crops: CUDA events after warm-up, algorithmic TFLOP/s from descriptor_gflop below over the measured time;
  * ViT-g's FFN input GEMM at P = 200 crops (M = 200 * 257 rows, K = 1536, w12 of 2 x 4096 rows): the fused SwiGLU epilogue
    (gemm_tma act=3, (M, 4096) bf16 out) against the same product as a plain GEMM ((M, 8192) bf16 out) followed by a separate
    silu(x1) * x2 pass in torch, and against the plain GEMM alone.
Seeded weights (speed does not depend on their values).  The card's name, power limit and current / maximum SM clock are read
with nvidia-smi in the same run, before and after the timed work.

    python tools/dinov2_bench.py [--iters 5] [--models dinov2_vits14,...]"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MODELS = ("dinov2_vits14", "dinov2_vitb14", "dinov2_vitl14", "dinov2_vitg14")
SIZES = (42, 100, 200)
S = 257                   # tokens per 224 x 224 crop: class token + 16 x 16 patches


def descriptor_gflop(C, depth, S=S):
    """per crop: 24 S C^2 for the qkv, proj and FFN GEMMs (the SwiGLU FFN of ViT-g, hidden 8C/3, costs the same 16 S C^2 as the
    Mlp's hidden 4C) plus 4 S^2 C for QK^T and PV, per block.  Patch embedding, LayerNorm, softmax and activations not counted."""
    return depth * (24 * S * C * C + 4 * S * S * C) / 1e9


def _card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()[0]


def _time(fn, iters, warmup=2):
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
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--models", default=",".join(MODELS))
    args = ap.parse_args()
    from sam6d_b200 import ops, synth
    from sam6d_b200.dinov2 import CustomDINOv2

    if not torch.cuda.is_available():
        raise SystemExit("dinov2_bench needs a CUDA device")
    dev = torch.device("cuda")
    res = dict(card_before=_card())
    g = torch.Generator(device=dev).manual_seed(0)
    images = torch.randn(max(SIZES), 3, 224, 224, device=dev, generator=g)
    masks = (torch.rand(max(SIZES), 224, 224, device=dev, generator=g) > 0.3).float()
    for name in args.models.split(","):
        with torch.device("cuda"):
            d = CustomDINOv2(name).eval()
        m = d.model
        d.model.load_state_dict(synth.make_dinov2_state_dict(embed_dim=m.embed_dim, depth=m.depth, num_heads=m.num_heads, seed=1,
                                                             ffn_layer=m.ffn_layer), strict=True)
        gf = descriptor_gflop(m.embed_dim, m.depth)
        r = dict(gflop_per_crop=round(gf, 1))
        for P in SIZES:
            ms = _time(lambda: d.compute_cls_and_patch_features(images[:P], masks[:P]), args.iters)
            r[f"P{P}_ms"] = round(ms, 2)
            r[f"P{P}_tflops"] = round(gf * P / ms, 1)
        res[name] = r
        del d, m
        torch.cuda.empty_cache()

    # ViT-g's SwiGLU FFN input GEMM, fused epilogue vs plain GEMM + separate elementwise pass
    M, K, H = 200 * S, 1536, 4096
    x = torch.randn(M, K, device=dev, generator=g).bfloat16()
    w12 = torch.randn(2 * H, K, device=dev, generator=g) / K ** 0.5
    b12 = 0.1 * torch.randn(2 * H, device=dev, generator=g)
    wp, bp, wb = ops.pack_swiglu_rows(w12).bfloat16(), ops.pack_swiglu_rows(b12), w12.bfloat16()

    def unfused():
        x1, x2 = ops.gemm_tma(x, wb, b12, out_dtype=torch.bfloat16).chunk(2, dim=-1)
        return F.silu(x1) * x2

    fused = ops.gemm_tma(x, wp, bp, act=ops.ACT_SWIGLU)
    diff = (fused.float() - unfused().float()).abs().max().item()
    tf = 2.0 * M * K * 2 * H / 1e9
    n = 10 * args.iters
    t_fused = _time(lambda: ops.gemm_tma(x, wp, bp, act=ops.ACT_SWIGLU), n)
    t_unfused = _time(unfused, n)
    t_plain = _time(lambda: ops.gemm_tma(x, wb, b12, out_dtype=torch.bfloat16), n)
    res["swiglu_gemm_M51400_K1536_N8192"] = dict(fused_ms=round(t_fused, 3), fused_tflops=round(tf / t_fused, 1), gemm_plus_elementwise_ms=round(t_unfused, 3),
                                                 plain_gemm_ms=round(t_plain, 3), plain_gemm_tflops=round(tf / t_plain, 1),
                                                 max_abs_diff_fused_vs_unfused=diff)
    res["card_after"] = _card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
