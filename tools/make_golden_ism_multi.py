"""tools/make_golden_ism_multi.py -- DEV CONTAINER ONLY (needs /root/reference).

Pins the multi-object restatement of oracle/ism_multi_oracle.py against the reference's OWN code:
    Detections.remove_very_small_detections / apply_nms_per_object_id / filter     ISM/model/utils.py:80-191
    Instance_Segmentation_Model.compute_semantic_score, compute_appearance_score, project_template_to_image,
    compute_geometric_score and the final score of test_step                      ISM/model/detector.py:260-383
imported unmodified (tools/ref_ism_import.py stubs the absent third-party imports) and called on a bare object carrying
`ref_data`, `matching_config` and `visible_thred`, in test_step's order.  Cases: seeded frames at O = 3 and O = 8, one with an
object that no proposal matches and one with every proposal on one object, each with a duplicated proposal (a tie of final
scores) and proposals too small to keep; plus per-object NMS on clustered boxes with quantised (tied) scores.  The reference
holds one pose set for all objects, so the oracle runs each frame twice: with the shared (T,4,4) poses and with them repeated
per object as (O,T,4,4), and both must equal the reference.  Writes tests/golden/ism_multi.pt: the case parameters (the inputs
are regenerated from them) and the reference's outputs.

Usage: python tools/make_golden_ism_multi.py"""
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from oracle import ism_multi_oracle as imo  # noqa: E402
from ref_ism_import import import_reference_ism, STUBBED  # noqa: E402

FRAMES = dict(o3_spread=dict(N=40, O=3, seed=0, mode="spread"), o3_one=dict(N=40, O=3, seed=1, mode="one"),
              o8_spread=dict(N=64, O=8, seed=2, mode="spread"), o8_empty=dict(N=64, O=8, seed=3, mode="empty"))
NMS_CASES = dict(o3=dict(N=120, O=3, seed=10), o8=dict(N=300, O=8, seed=11), o8_two_used=dict(N=200, O=8, seed=12, n_obj_used=2),
                 one=dict(N=150, O=1, seed=13))


def input_checksum(inp):
    return float(sum(inp[k].double().sum() for k in ("masks", "depth", "desc", "ref_desc", "q_patch", "ref_patch", "poses", "pointcloud")))


def reference_frame(loss, detector, utils, inp):
    """test_step from the Detections of the proposals to apply_nms_per_object_id"""
    ISMModel = detector.Instance_Segmentation_Model
    host = types.SimpleNamespace(
        matching_config=types.SimpleNamespace(metric=loss.PairwiseSimilarity(), aggregation_function="avg_5", confidence_thresh=0.2),
        ref_data={"descriptors": inp["ref_desc"], "appe_descriptors": inp["ref_patch"], "poses": inp["poses"],
                  "pointcloud": inp["pointcloud"]},
        visible_thred=0.5)
    for name in ("best_template_pose", "Calculate_the_query_translation"):
        setattr(host, name, types.MethodType(getattr(ISMModel, name), host))
    batch = {"depth": inp["depth"].unsqueeze(0), "cam_intrinsic": inp["K"].unsqueeze(0), "depth_scale": inp["depth_scale"]}
    N = inp["masks"].shape[0]
    det = utils.Detections({"masks": inp["masks"].clone(), "boxes": inp["boxes"].clone(), "index": torch.arange(N)})
    det.remove_very_small_detections(types.SimpleNamespace(min_box_size=0.05, min_mask_size=3e-4))
    after_small = det.index.clone()
    q, qp = inp["desc"][after_small], inp["q_patch"][after_small]
    with torch.no_grad():
        idx_sel, pred_obj, sem, best_t = ISMModel.compute_semantic_score(host, q)
        det.filter(idx_sel)
        qp = qp[idx_sel, :]
        appe, ref_aux = ISMModel.compute_appearance_score(host, best_t, pred_obj, qp)
        uv = ISMModel.project_template_to_image(host, best_t, pred_obj, batch, det.masks)
        geo, vis = ISMModel.compute_geometric_score(host, uv, det, qp, ref_aux, visible_thred=host.visible_thred)
        score = (sem + appe + geo * vis) / (1 + 1 + vis)
    det.add_attribute("scores", score)
    det.add_attribute("object_ids", pred_obj)
    det.apply_nms_per_object_id(nms_thresh=0.25)
    return dict(after_small=after_small, idx_sel=after_small[idx_sel], pred_obj=pred_obj, best_t=best_t, score=score,
                geometric_zero=not torch.is_tensor(geo), final_index=det.index, final_object=det.object_ids, final_score=det.scores)


def oracle_frame(inp, per_object_poses):
    keep = imo.remove_very_small_detections(inp["masks"], inp["boxes"])
    after_small = torch.nonzero(keep).flatten()
    O = inp["ref_desc"].shape[0]
    poses = inp["poses"].unsqueeze(0).repeat(O, 1, 1, 1) if per_object_poses else inp["poses"]
    s = imo.score_objects(inp["desc"][after_small], inp["ref_desc"], inp["q_patch"][after_small], inp["ref_patch"], inp["masks"][after_small],
                          inp["depth"], inp["K"], inp["depth_scale"], inp["boxes"][after_small], poses, inp["pointcloud"])
    idx_sel = after_small[s["idx_sel"]]
    k = imo.nms_per_object(inp["boxes"][idx_sel], s["score"], s["pred_obj"])
    return dict(after_small=after_small, idx_sel=idx_sel, pred_obj=s["pred_obj"], best_t=s["best_t"], score=s["score"],
                final_index=idx_sel[k], final_object=s["pred_obj"][k], final_score=s["score"][k])


def main():
    loss, detector = import_reference_ism()
    from model import utils
    frames = {}
    for tag, kw in FRAMES.items():
        inp = imo.make_multi_inputs(**kw)
        ref = reference_frame(loss, detector, utils, inp)
        for per_object in (False, True):
            ora = oracle_frame(inp, per_object)
            for k, v in ora.items():
                assert torch.equal(v, ref[k]), f"{tag} (per-object poses {per_object}): {k} differs"
        used = sorted(set(ref["pred_obj"].tolist()))
        print(f"  {tag}: {kw['N']} proposals, {len(ref['after_small'])} after the size filter, {len(ref['idx_sel'])} above the "
              f"semantic threshold on objects {used}, {len(ref['final_index'])} after NMS; geometric score zeroed: "
              f"{ref['geometric_zero']}; oracle == reference bit for bit")
        ref.pop("geometric_zero")
        frames[tag] = dict(kw=kw, input_checksum=input_checksum(inp), **ref)
    nms_cases = {}
    for tag, kw in NMS_CASES.items():
        boxes, scores, obj = imo.make_nms_case(**kw)
        det = utils.Detections({"boxes": boxes.clone(), "scores": scores.clone(), "object_ids": obj.clone(), "index": torch.arange(len(boxes))})
        det.apply_nms_per_object_id(nms_thresh=0.25)
        assert torch.equal(imo.nms_per_object(boxes, scores, obj), det.index), f"nms {tag} differs"
        print(f"  nms {tag}: {len(boxes)} boxes, {len(det.index)} kept; oracle == reference")
        nms_cases[tag] = dict(kw=kw, boxes=boxes, scores=scores, object_ids=obj, keep=det.index)
    out = os.path.join(ROOT, "tests", "golden", "ism_multi.pt")
    torch.save(dict(meta=dict(source="ISM/model/utils.py Detections + ISM/model/detector.py Instance_Segmentation_Model methods "
                              "imported from the reference (CPU)", torch=torch.__version__, stubbed_imports=list(STUBBED)),
                    frames=frames, nms=nms_cases), out)
    print(f"wrote {out} ({os.path.getsize(out) / 1e3:.1f} KB)")


if __name__ == "__main__":
    main()
