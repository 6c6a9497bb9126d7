"""CPU study behind csrc/geo_lut.cu: error of the table-interpolated geometric embedding against the float64 embedding, next to the
error of the bf16-operand tensor-core product (csrc/geo_tc.cu), with the arithmetic of each kernel emulated in torch
(bf16 roundings where the kernels round).  Uses the module's own table builder (GeometricStructureEmbedding._tables).

    python tools/geo_lut_error.py"""
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import pem_oracle as po                      # noqa: E402
from sam6d_b200 import pem                               # noqa: E402


def bf(t):
    return t.float().to(torch.bfloat16).double()


def main():
    sd = po.make_state_dict(seed=1)
    geo = pem.GeometricStructureEmbedding(pem.DEFAULT_MODEL_CFG["geo_embedding"])
    geo.load_state_dict({k[len("geo_embedding."):]: v for k, v in sd.items() if k.startswith("geo_embedding.")})
    Wa, Wd = geo.proj_a.weight.detach().double(), geo.proj_d.weight.detach().double()
    bias = (geo.proj_a.bias + geo.proj_d.bias).detach().double()
    div = geo.embedding.div_term.double()

    def emb(x):
        om = x[..., None].double() * div
        return torch.stack([torch.sin(om), torch.cos(om)], dim=-1).reshape(*x.shape, 256)

    torch.manual_seed(0)
    n = 20000
    xa, xd = torch.rand(n, 3) * 12.0, torch.rand(n) * 12.0
    exact = emb(xd) @ Wd.T + bias + (emb(xa) @ Wa.T).max(dim=1).values

    def tensor_core(x, W):                                # bf16 sin/cos x bf16 weights, fp32 accumulation
        return (bf(emb(x).float()) @ bf(W).T).float().double()

    e_tc = bf(bf(tensor_core(xd, Wd) + bias.float().double()) + bf(tensor_core(xa.reshape(-1), Wa).reshape(n, 3, 256)).max(dim=1).values)

    rows = []
    for inv_h in (4.0, 8.0, 16.0):
        pem.GEO_LUT_INV_H = inv_h
        t = geo._tables(dict(div=geo.embedding.div_term, bias=bias.float()))

        def lerp32(tab, x):                               # the kernel: fp32 interpolation of the bf16 table, one rounding at the store
            tab = tab.double()
            u = x.float() * inv_h
            i = u.floor().clamp(0, tab.shape[0] - 2).long()
            tt = (u - i.float()).double()
            return (tab[i] + tt[..., None] * (tab[i + 1] - tab[i])).float().double()

        e_p = bf(lerp32(t["tab_d"], xd) + lerp32(t["tab_a"], xa.reshape(-1)).reshape(n, 3, 256).max(dim=1).values)
        rows.append((inv_h, t["tab_a"].shape[0], t["tab_d"].shape[0], (e_p - exact).pow(2).mean().sqrt().item(),
                     (e_p - exact).abs().max().item()))
    print(f"|E| rms {exact.pow(2).mean().sqrt():.3f}; bf16 rounding of the exact E alone: rms {(bf(exact) - exact).pow(2).mean().sqrt():.2e}")
    print(f"tensor-core product (geo_tc.cu arithmetic): rms {(e_tc - exact).pow(2).mean().sqrt():.2e} max {(e_tc - exact).abs().max():.2e}")
    for inv_h, na, nd, rms_p, mx_p in rows:
        print(f"table step 1/{inv_h:g} ({na} + {nd} rows, {(na + nd) * 512 / 1024:.0f} KB): fp32 interpolation rms {rms_p:.2e} max {mx_p:.2e}")


if __name__ == "__main__":
    main()
