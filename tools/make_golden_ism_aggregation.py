"""tools/make_golden_ism_aggregation.py -- DEV CONTAINER ONLY (needs the reference checkout).

Pins oracle/ism_agg_oracle.py (and, through the GPU tests, csrc/ism.cu) against the reference's OWN
Instance_Segmentation_Model.compute_semantic_score (ISM/model/detector.py:260-296) with every matching_config.aggregation_function
(mean, median, max, avg_5), imported unmodified through tools/ref_ism_import.py and called on a bare object carrying
`matching_config` and `ref_data`, as tools/make_golden_ism.py does for avg_5.
Writes tests/golden/ism_aggregation.pt: P = 16 proposals, C = 256, T in {42, 162, 642} x O in {1, 8, 21}, plus T = 3 (O = 8)
and T = 1 (O = 4); the descriptors carry exact ties (ism_agg_oracle.make_tied_descriptors).  The reference's avg_5 calls
topk(k=5), which raises when T < 5; there the oracle's k = min(5, T) rule is recorded, marked `reference=False`.

Usage: python tools/make_golden_ism_aggregation.py"""
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from oracle import ism_agg_oracle as ia  # noqa: E402
from ref_ism_import import import_reference_ism, STUBBED  # noqa: E402

P, C, THRESH = 16, 256, 0.2
SHAPES = [(O, T) for T in (42, 162, 642) for O in (1, 8, 21)] + [(8, 3), (4, 1)]


def main():
    loss, detector = import_reference_ism()
    ISMModel = detector.Instance_Segmentation_Model
    cases = {}
    for O, T in SHAPES:
        seed = 1000 + 37 * O + T
        q, ref = ia.make_tied_descriptors(P, O, T, C, seed)
        case = dict(P=P, O=O, T=T, C=C, seed=seed, input_checksum=dict(q=q.double().sum().item(), ref=ref.double().sum().item()))
        for agg in ia.AGGREGATIONS:
            o_idx, o_obj, o_sem, o_bt, o_sim, o_per = ia.compute_semantic_score(q, ref, agg, THRESH)
            host = types.SimpleNamespace(
                matching_config=types.SimpleNamespace(metric=loss.PairwiseSimilarity(), aggregation_function=agg, confidence_thresh=THRESH),
                ref_data={"descriptors": ref})
            host.best_template_pose = types.MethodType(ISMModel.best_template_pose, host)
            pinned = True
            try:
                with torch.no_grad():
                    idx_sel, pred_obj, sem, best_t = ISMModel.compute_semantic_score(host, q)
            except RuntimeError:
                assert agg == "avg_5" and T < 5, (agg, T)
                pinned = False
            if pinned:
                assert torch.equal(o_idx, idx_sel) and torch.equal(o_obj, pred_obj) and torch.equal(o_bt, best_t), (O, T, agg)
                assert torch.equal(o_sem, sem), (O, T, agg)
            case[agg] = dict(idx_selected=o_idx, pred_idx_objects=o_obj, semantic_score=o_sem, best_template=o_bt, per_obj=o_per,
                             reference=pinned)
            print(f"  O={O:2d} T={T:3d} {agg:6s}: {len(o_idx)} above {THRESH}; "
                  + ("oracle == reference bit for bit" if pinned else "reference raises (topk k=5 > T): oracle's rule recorded"))
        cases[(O, T)] = case
    out = os.path.join(ROOT, "tests", "golden", "ism_aggregation.pt")
    torch.save(dict(meta=dict(source="ISM/model/loss.py PairwiseSimilarity + ISM/model/detector.py compute_semantic_score / "
                              "best_template_pose of the reference (CPU, fp32)", torch=torch.__version__, confidence_thresh=THRESH,
                              stubbed_imports=list(STUBBED)), cases=cases), out)
    print(f"wrote {out} ({os.path.getsize(out) / 1e6:.2f} MB)")


if __name__ == "__main__":
    main()
