"""Per-entry-point GPU time of one 16-frame SAM ViT-H encoder pass (CUDA events around every C-ABI call).  Run on the GPU box."""
import os, sys, collections
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from sam6d_b200 import _lib
from sam6d_b200.sam import build_image_encoder

F = int(sys.argv[1]) if len(sys.argv) > 1 else 16
enc = build_image_encoder("vit_h", precision="bf16").cuda().eval()
img = torch.randn(F, 3, 1024, 1024, device="cuda")
with torch.no_grad():
    enc(img); enc(img)
    torch.cuda.synchronize()
    names = [n for n in dir(_lib.lib()) if n.startswith("sam6d_")] if hasattr(_lib.lib(), "__dir__") else []
    names = ["sam6d_gemm_tma", "sam6d_gemm_tma_vt", "sam6d_attn_tc", "sam6d_attn_global_tc_ex", "sam6d_layernorm_bf16", "sam6d_layernorm",
             "sam6d_gather_rows", "sam6d_gemm_bf16", "sam6d_transpose_tokens_bf16", "sam6d_gemm_f32", "sam6d_attn_relpos"]
    for n in names:
        _lib.time_kernel(n, True)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); enc(img); e1.record()
    torch.cuda.synchronize()
tot = e0.elapsed_time(e1)
print(f"{F} frames: {tot:.1f} ms")
for n in names:
    ev = _lib.timed_events(n)
    if ev:
        ms = sum(a.elapsed_time(b) for a, b in ev)
        print(f"  {n:32s} {len(ev):4d} calls {ms:8.2f} ms  {100 * ms / tot:5.1f}%")
