"""Time the two geo_embed_tc passes at the bench size (64 clouds x 197^2 pairs).  Run on the GPU box."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from sam6d_b200 import ops, _lib

torch.manual_seed(0)
B, n = 64, 197
npairs = B * n * n
T = torch.rand(npairs, 4, device="cuda") * 3.0
div = torch.exp(torch.arange(0, 256, 2, device="cuda").float() * (-9.210340371976184 / 256))
Wa = (torch.randn(256, 256, device="cuda") / 16).to(torch.bfloat16)
Wd = (torch.randn(256, 256, device="cuda") / 16).to(torch.bfloat16)
bias = torch.randn(256, device="cuda")
for dt in (torch.bfloat16, torch.float32):
    E = torch.empty(npairs, 256, device="cuda", dtype=dt)
    def run():
        _lib.call("sam6d_geo_embed_tc", T, npairs, div, Wa, Wd, bias, E, 1 if dt == torch.bfloat16 else 0)
    for _ in range(3): run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10): run()
    e1.record(); torch.cuda.synchronize()
    print(f"geo_embed_tc {dt}: {e0.elapsed_time(e1) / 10 * 1e3:.1f} us (both passes)")
