"""micro-benchmark: wgmma GEMM vs CUDA-core GEMM on the shapes of the matching path (GPU box)"""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sam6d_b200 import ops

def timeit(fn, n=20):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n): fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n

for (M, N, K) in [(6304, 1792, 256), (6304, 256, 256), (6304, 512, 256), (6304, 256, 512), (65536, 256, 256), (65536, 512, 256), (65536, 256, 512)]:
    A = torch.randn(M, K, device="cuda"); W = torch.randn(N, K, device="cuda"); Wb = W.bfloat16(); b = torch.randn(N, device="cuda")
    Ab = A.bfloat16()
    t0 = timeit(lambda: ops.gemm(A, W, b))
    t1 = timeit(lambda: ops.gemm_tc(A, Wb, b))
    t2 = timeit(lambda: ops.gemm_tc(Ab, Wb, b, out_dtype=torch.bfloat16))
    fl = 2.0 * M * N * K
    print(f"M={M:6d} N={N:5d} K={K:4d}  simt {t0*1e3:8.1f} us ({fl/t0/1e9:7.1f} TF)  tc(f32 A, f32 C) {t1*1e3:8.1f} us ({fl/t1/1e9:7.1f} TF)  tc(bf16 A, bf16 C) {t2*1e3:8.1f} us ({fl/t2/1e9:7.1f} TF)")
# batched score matrix 32 x (2049 x 2049 x 256)
B, S, C = 32, 2049, 256
f1 = torch.randn(B, S, C, device="cuda"); f2 = torch.randn(B, S, C, device="cuda"); out = torch.empty(B, S, S, device="cuda")
t0 = timeit(lambda: ops.gemm(f1, f2, out=out, alpha=10.0), n=5)
t1 = timeit(lambda: ops.gemm_tc(f1, f2, out=out, alpha=10.0), n=5)
fl = 2.0 * B * S * S * C
print(f"fine score 32x2049x2049x256: simt {t0:.3f} ms ({fl/t0/1e9:.1f} TF)  tc {t1:.3f} ms ({fl/t1/1e9:.1f} TF; output write {B*S*S*4/t1/1e6:.0f} GB/s)")

print("--- persistent TMA GEMM (bf16 in, bf16 out) vs staged wgmma GEMM")
for (M, N, K) in [(65536, 3840, 1280), (65536, 1280, 1280), (65536, 5120, 1280), (65536, 1280, 5120), (78400, 3840, 1280), (65536, 256, 256), (6304, 1792, 256), (65536, 512, 256)]:
    Ab = torch.randn(M, K, device="cuda").bfloat16(); Wb = torch.randn(N, K, device="cuda").bfloat16(); b = torch.randn(N, device="cuda")
    t1 = timeit(lambda: ops.gemm_tc(Ab, Wb, b, out_dtype=torch.bfloat16), n=5)
    t2 = timeit(lambda: ops.gemm_tma(Ab, Wb, b, out_dtype=torch.bfloat16), n=5)
    t3 = timeit(lambda: ops.gemm_tma(Ab, Wb, b, out_dtype=torch.float32), n=5)
    t4 = timeit(lambda: torch.nn.functional.linear(Ab, Wb), n=5)
    fl = 2.0 * M * N * K
    print(f"M={M:6d} N={N:5d} K={K:4d}  staged {t1*1e3:8.1f} us ({fl/t1/1e9:7.1f} TF)  tma->bf16 {t2*1e3:8.1f} us ({fl/t2/1e9:7.1f} TF)  tma->f32 {t3*1e3:8.1f} us ({fl/t3/1e9:7.1f} TF)  cuBLAS {t4*1e3:8.1f} us ({fl/t4/1e9:7.1f} TF)")
