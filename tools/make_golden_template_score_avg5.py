"""tools/make_golden_template_score_avg5.py -- GPU (H100).

Records what the template-scoring kernel (csrc/ism.cu) outputs with the 'avg_5' aggregation, so that later versions of the
kernel can be held to those outputs bit for bit.  It was run with the one-CTA-per-proposal kernel that preceded the
proposal-tiled one, and its output is committed as tests/golden/template_score_avg5.pt (checked by
tests/test_gpu_ism_aggregation.py).

Shapes: P in {1, 200} proposals x O in {1, 8, 21, 33} objects x T in {42, 162, 642} templates (the level-0 / 1 / 2 view
sets), C = 1024 (DINOv2 ViT-L).  P = 0 has nothing to record: that kernel's entry point rejected the empty query.  Inputs are synth.make_descriptors, regenerated from the seed by the test.  Stored per shape:
best object / score / template, the (P, O) object scores in full, and a SHA-256 of the (P, O, T) similarity tensor's bytes
(17 MB at the largest shape, too large to commit).

Usage: python tools/make_golden_template_score_avg5.py [out.pt]"""
import hashlib
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from sam6d_b200 import ops  # noqa: E402
from sam6d_b200.synth import make_descriptors  # noqa: E402

PS, OS, TS, C = (1, 200), (1, 8, 21, 33), (42, 162, 642), 1024


def seed_of(P, O, T):
    return 7 * P + 131 * O + T


def sha256(t):
    return hashlib.sha256(t.detach().cpu().contiguous().numpy().tobytes()).hexdigest()


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tests", "golden", "template_score_avg5.pt")
    cases = {}
    for O in OS:
        for T in TS:
            for P in PS:
                q, r = make_descriptors(P=P, O=O, T=T, C=C, seed=seed_of(P, O, T))
                qn = ops.l2norm_rows(q.cuda().contiguous())
                rn = ops.l2norm_rows(r.cuda().contiguous())
                sim, obj, bo, bs, bt = ops.template_score(qn, rn, want_sim=True)
                torch.cuda.synchronize()
                cases[(P, O, T)] = dict(seed=seed_of(P, O, T), input_checksum=dict(q=q.double().sum().item(), ref=r.double().sum().item()),
                                        sim_sha256=sha256(sim), obj_score=obj.cpu(), best_obj=bo.cpu(), best_score=bs.cpu(),
                                        best_tmpl=bt.cpu())
                print(f"P={P:3d} O={O:2d} T={T:3d}: sim {sim.sum().item():.6f}  best_score sum {bs.sum().item():.6f}")
    torch.save(dict(meta=dict(device=torch.cuda.get_device_name(0), torch=torch.__version__, C=C,
                              kernel="csrc/ism.cu template_score_kernel, one CTA per proposal"), cases=cases), out)
    print(f"wrote {out} ({os.path.getsize(out) / 1e6:.2f} MB)")


if __name__ == "__main__":
    main()
