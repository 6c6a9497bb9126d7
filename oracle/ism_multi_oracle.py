"""oracle/ism_multi_oracle.py -- TEST INFRASTRUCTURE ONLY.

CPU restatement of the multi-object post-processing of Instance_Segmentation_Model.test_step (ISM/model/detector.py:324-391):
    remove_very_small_detections   ISM/model/utils.py:96-105   (Detections.remove_very_small_detections)
    nms_per_object                 ISM/model/utils.py:107-119  (Detections.apply_nms_per_object_id)
    score_objects                  detector.py:358-383: semantic, appearance and geometric score over O objects, final score,
                                   with per-object template poses (O,T,4,4) indexed as obj*T + t
Parity status: PINNED.  tools/make_golden_ism_multi.py runs the reference's own Detections and Instance_Segmentation_Model
methods on seeded inputs at O = 3 and O = 8 (score ties, an object without proposals, every proposal on one object) and finds
this restatement bit-identical; tests/golden/ism_multi.pt.  The reference holds one pose set for all objects, so the pinned
cases give every object the same poses; per-object poses are checked against this oracle only.
"""
from typing import Dict

import torch

from oracle import ism_oracle as io
from oracle.sam_dec_oracle import nms

MIN_BOX_SIZE, MIN_MASK_SIZE, NMS_THRESH = 0.05, 3e-4, 0.25      # ISM/configs/model/ISM_sam.yaml


def remove_very_small_detections(masks: torch.Tensor, boxes: torch.Tensor, min_box_size: float = MIN_BOX_SIZE,
                                 min_mask_size: float = MIN_MASK_SIZE) -> torch.Tensor:
    """masks (N,H,W) f32, boxes (N,4) int64 xyxy -> keep (N,) bool"""
    img_area = masks.shape[1] * masks.shape[2]
    box_areas = (boxes[:, 2] - boxes[:, 0]) * (boxes[:, 3] - boxes[:, 1]) / img_area
    mask_areas = masks.sum(dim=(1, 2)) / img_area
    return torch.logical_and(box_areas > min_box_size ** 2, mask_areas > min_mask_size)


def nms_per_object(boxes: torch.Tensor, scores: torch.Tensor, object_ids: torch.Tensor, thr: float = NMS_THRESH) -> torch.Tensor:
    """-> kept indices: object ids ascending, within an object torchvision.ops.nms's order (decreasing score)"""
    out = [torch.zeros(0, dtype=torch.long)]
    for o in torch.unique(object_ids).tolist():
        idx = torch.nonzero(object_ids == o).flatten()
        out.append(idx[nms(boxes[idx], scores[idx], thr)])
    return torch.cat(out)


def score_objects(desc: torch.Tensor, ref_desc: torch.Tensor, q_patch: torch.Tensor, ref_patch: torch.Tensor, masks: torch.Tensor,
                  depth: torch.Tensor, K: torch.Tensor, depth_scale: torch.Tensor, boxes: torch.Tensor, poses: torch.Tensor,
                  pointcloud: torch.Tensor, confidence_thresh: float = 0.2, visible_thred: float = 0.5) -> Dict[str, torch.Tensor]:
    """test_step from compute_semantic_score to the final score.  desc (P,C), ref_desc (O,T,C), q_patch (P,Np,C), ref_patch
    (O,T,Np,C), masks (P,H,W), boxes (P,4), poses (O,T,4,4) or (T,4,4) shared by all objects, pointcloud (O,npc,3)
    -> dict(idx_sel, pred_obj, best_t, semantic, appearance, visible, geometric, score) of the selected proposals"""
    idx_sel, pred_obj, sem, best_t, _, _ = io.compute_semantic_score(desc, ref_desc, confidence_thresh)
    qp = q_patch[idx_sel]
    ref_aux = ref_patch[pred_obj, best_t]
    appe = io.appearance_score(qp, ref_aux)
    vis = io.visible_ratio(qp, ref_aux, visible_thred)
    m, b = masks[idx_sel], boxes[idx_sel]
    T = ref_desc.shape[1]
    if poses.dim() == 4:
        poses, pose_idx = poses.reshape(-1, 4, 4), pred_obj * T + best_t
    else:
        pose_idx = best_t
    tr = io.query_translation(m, depth, K, depth_scale)
    vu = io.project_template_to_image(poses, pointcloud, pose_idx, pred_obj, tr, K, masks.shape[1], masks.shape[2])
    _, geo = io.geometric_iou(vu, b)
    score = (sem + appe + geo * vis) / (1 + 1 + vis)
    return dict(idx_sel=idx_sel, pred_obj=pred_obj, best_t=best_t, semantic=sem, appearance=appe, visible=vis,
                geometric=geo if torch.is_tensor(geo) else torch.zeros_like(sem), score=score)


def _unit_rows(x: torch.Tensor, g: torch.Generator, p_zero: float = 0.25) -> torch.Tensor:
    """L2-normalised rows with a share of all-zero rows (masked-out patches)"""
    x = torch.nn.functional.normalize(x, dim=-1)
    return x * (torch.rand(x.shape[:-1], generator=g) >= p_zero).float()[..., None]


def make_multi_inputs(N: int = 40, O: int = 3, T: int = 42, H: int = 240, W: int = 320, C: int = 64, Np: int = 16, Cp: int = 32,
                      seed: int = 0, mode: str = "spread"):
    """a seeded multi-object ISM frame: N proposals (elliptic masks over a depth ramp, the last four too small for
    remove_very_small_detections, proposal 1 a duplicate of proposal 0 so that two final scores tie), descriptors planted on
    the objects (with clutter proposals in mode "spread"), patch tokens, one template pose set shared by all objects (the reference's ref_data["poses"]) and per-object
    clouds.  mode: "spread" plants proposal p on object p % O, "empty" leaves object O-1 without proposals, "one" puts every
    proposal on object 0."""
    inp = io.make_geometric_inputs(N=N, H=H, W=W, T=T, O=O, seed=seed)
    g = torch.Generator().manual_seed(1000 + seed)
    masks, boxes = inp["masks"], inp["boxes"]
    yy, xx = torch.meshgrid(torch.arange(H), torch.arange(W), indexing="ij")
    for k, (cy, cx, ry, rx) in enumerate([(30, 40, 1.5, 1.5), (100, 200, 2, 2), (50, 60, 1, 30), (180, 250, 2.5, 1)]):
        i = N - 4 + k
        m = (((xx - cx) / rx) ** 2 + ((yy - cy) / ry) ** 2) <= 1.0
        masks[i] = m.float()
        ys, xs = torch.nonzero(m, as_tuple=True)
        boxes[i] = torch.stack([xs.min(), ys.min(), xs.max(), ys.max()])
    masks[1], boxes[1] = masks[0], boxes[0]
    ref = torch.randn(O, T, C, generator=g) + 1.5 * torch.randn(O, 1, C, generator=g)
    plant = {"spread": lambda p: p % O, "empty": lambda p: p % max(O - 1, 1), "one": lambda p: 0}[mode]
    clutter = (lambda p: p % 5 == 4) if mode == "spread" else (lambda p: False)     # a clutter proposal may match any object
    q = torch.stack([torch.randn(C, generator=g) if clutter(p) else ref[plant(p), (3 * p) % T] + 0.6 * torch.randn(C, generator=g)
                     for p in range(N)])
    q[1] = q[0]
    q_patch = _unit_rows(torch.randn(N, Np, Cp, generator=g), g)
    q_patch[1] = q_patch[0]
    ref_patch = _unit_rows(torch.randn(O, T, Np, Cp, generator=g), g)
    inp.update(desc=q, ref_desc=ref, q_patch=q_patch, ref_patch=ref_patch, masks=masks, boxes=boxes)
    return inp


def make_nms_case(N: int = 300, O: int = 8, seed: int = 0, n_obj_used=None):
    """boxes (N,4) f32 in clusters, scores quantised to quarters (exact ties), object ids among the first n_obj_used of O"""
    g = torch.Generator().manual_seed(seed)
    centre = torch.rand(12, 2, generator=g) * 400
    c = centre[torch.randint(0, 12, (N,), generator=g)] + torch.randn(N, 2, generator=g) * 12
    wh = 20 + torch.rand(N, 2, generator=g) * 60
    boxes = torch.cat([c - wh / 2, c + wh / 2], dim=1).round()
    scores = torch.randint(0, 4, (N,), generator=g).float() / 4
    obj = torch.randint(0, n_obj_used or O, (N,), generator=g)
    return boxes, scores, obj
