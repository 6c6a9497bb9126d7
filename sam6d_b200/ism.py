"""Instance Segmentation Model pieces on the hot path: per-proposal template scoring.

Mirrors  PairwiseSimilarity                         ISM/model/loss.py:21-44
         Instance_Segmentation_Model.compute_semantic_score / best_template_pose
                                                    ISM/model/detector.py:198-207, 260-296
with the same call signatures and return values.  One fused sm_90a kernel (csrc/ism.cu) computes the clamped cosine
matrix, the template aggregation (mean, median, max or avg-5) and the best-template argmax, and a second one the object
argmax; the reference's P-fold replication of the reference descriptors is never formed.

Geometric score (csrc/ism_geo.cu):
         Calculate_the_query_translation            ISM/model/detector.py:237-250, ISM/utils/trimesh_utils.py:77-105
         project_template_to_image                  ISM/model/detector.py:209-235
         compute_geometric_score (IoU part)         ISM/model/detector.py:311-323, ISM/utils/bbox_utils.py:197-221

Multi-object post-processing of Instance_Segmentation_Model.test_step (ISM/model/detector.py:324-391):
         Detections.remove_very_small_detections    ISM/model/utils.py:96-105
         Detections.apply_nms_per_object_id         ISM/model/utils.py:107-119 (csrc/sam_dec.cu: sam_nms_kernel with object ids)
"""
from types import SimpleNamespace

import torch
import torch.nn as nn

from . import _lib, ops


class PairwiseSimilarity(nn.Module):
    """forward(query (P,C), reference (O,T,C)) -> (P,O,T) clamped cosine similarity."""

    def __init__(self, metric="cosine", chunk_size=64):
        super().__init__()
        self.metric = metric
        self.chunk_size = chunk_size

    @torch.no_grad()
    def forward(self, query, reference):
        qn = ops.l2norm_rows(query.float().contiguous())
        rn = ops.l2norm_rows(reference.float().contiguous())
        sim, _, _, _, _ = ops.template_score(qn, rn, want_sim=True)
        return sim


def _normalized(x):
    x = x.float().contiguous()
    return ops.l2norm_rows(x) if x.numel() else x


def compute_semantic_score(proposal_descriptors, ref_descriptors, aggregation_function="avg_5", confidence_thresh=0.2):
    """detector.py:260-296 -> (idx_selected_proposals, pred_idx_objects, semantic_score, best_template), all int64/f32
    like the reference.  aggregation_function (matching_config): 'mean', 'median' (the lower median, as torch.median),
    'max' or 'avg_5' (ISM/configs/model/ISM_sam.yaml), all in the one fused kernel."""
    if aggregation_function not in ops.TEMPLATE_AGGREGATIONS:
        raise NotImplementedError(f"aggregation_function {aggregation_function!r}: one of {sorted(ops.TEMPLATE_AGGREGATIONS)}")
    qn = _normalized(proposal_descriptors)
    rn = ops.l2norm_rows(ref_descriptors.float().contiguous())
    _, _, best_obj, best_score, best_tmpl = ops.template_score(qn, rn, want_sim=False, aggregation=aggregation_function)
    keep = best_score > confidence_thresh
    idx_selected = torch.arange(best_score.shape[0], device=best_score.device)[keep]
    return idx_selected, best_obj[keep].long(), best_score[keep], best_tmpl[keep].long()


class SemanticScorer(nn.Module):
    """Holds `ref_data["descriptors"]` and `matching_config` like Instance_Segmentation_Model does, exposing
    compute_semantic_score(proposal_descriptors) with the reference signature."""

    def __init__(self, ref_descriptors, aggregation_function="avg_5", confidence_thresh=0.2):
        super().__init__()
        self.ref_data = {"descriptors": ref_descriptors}
        self.matching_config = SimpleNamespace(metric=PairwiseSimilarity(), aggregation_function=aggregation_function,
                                               confidence_thresh=confidence_thresh)

    def compute_semantic_score(self, proposal_decriptors):
        return compute_semantic_score(proposal_decriptors, self.ref_data["descriptors"],
                                      self.matching_config.aggregation_function, self.matching_config.confidence_thresh)


# ---------------------------------------------------------------------------------------------- geometric score
def _k64(cam_intrinsic: torch.Tensor, device) -> torch.Tensor:
    K = cam_intrinsic.reshape(3, 3) if cam_intrinsic.numel() == 9 else None
    if K is None:
        raise RuntimeError("cam_intrinsic must hold a 3x3 matrix")
    return K.to(device=device, dtype=torch.float64).contiguous()


@torch.no_grad()
def calculate_the_query_translation(proposal, depth, cam_intrinsic, depth_scale):
    """Instance_Segmentation_Model.Calculate_the_query_translation: proposal (N,H,W) masks, depth (H,W) integer depth image,
    cam_intrinsic (3,3), depth_scale (number or one-element tensor) -> (N,3) f32, the mean back-projected point of every
    proposal's masked depth.  One pass over mask x depth per proposal with float64 sums (the reference's input dtypes make its
    own computation float64); the reference's N x H x W float64 coordinate images are never formed."""
    m = proposal.reshape(-1, proposal.shape[-2], proposal.shape[-1]).to(torch.float32).contiguous()
    N, H, W = m.shape
    d = depth.reshape(H, W).to(device=m.device, dtype=torch.int32).contiguous()
    K = _k64(cam_intrinsic, m.device)
    out = torch.empty(N, 3, dtype=torch.float32, device=m.device)
    _lib.call("sam6d_query_translation", m, d, N, H, W, K, float(depth_scale), out)
    return out


@torch.no_grad()
def project_template_iou(poses, pointcloud, best_pose, pred_object_idx, translate, cam_intrinsic, image_hw, boxes, want_image_vu=False):
    """project_template_to_image + the box / IoU of compute_geometric_score in one launch.  poses (T,4,4), pointcloud (O,Np,3),
    best_pose / pred_object_idx (N,), translate (N,3), boxes (N,4) xyxy -> dict(xyxy (N,4) i32, iou (N,) f32, ok (N,) bool[,
    image_vu (N,Np,2) i32])."""
    H, W = image_hw
    dev = translate.device
    poses = poses.to(device=dev, dtype=torch.float32).contiguous()
    pc = pointcloud.to(device=dev, dtype=torch.float32).contiguous()
    if pc.dim() == 2:
        pc = pc.unsqueeze(0)
    bp = best_pose.to(device=dev, dtype=torch.int64).contiguous()
    po = pred_object_idx.to(device=dev, dtype=torch.int64).contiguous()
    bx = boxes.to(device=dev, dtype=torch.int64).contiguous()
    N, npc = bp.shape[0], pc.shape[1]
    if po.shape[0] != N or bx.shape != (N, 4) or translate.shape != (N, 3) or poses.shape[1:] != (4, 4):
        raise RuntimeError("project_template_iou: shape mismatch")
    if N and (int(bp.max()) >= poses.shape[0] or int(po.max()) >= pc.shape[0] or int(bp.min()) < 0 or int(po.min()) < 0):
        raise IndexError("project_template_iou: template / object index out of range")
    K = _k64(cam_intrinsic, dev)
    vu = torch.empty(N, npc, 2, dtype=torch.int32, device=dev) if want_image_vu else None
    xyxy = torch.empty(N, 4, dtype=torch.int32, device=dev)
    iou = torch.empty(N, dtype=torch.float32, device=dev)
    ok = torch.empty(N, dtype=torch.uint8, device=dev)
    tr = translate.to(torch.float32).contiguous()      # a named tensor: a temporary inside the argument list would be freed before the launch
    _lib.call("sam6d_project_template_iou", poses, poses.shape[0], pc, pc.shape[0], npc, bp, po, tr, K, N, H, W, bx, vu, xyxy, iou, ok)
    out = dict(xyxy=xyxy, iou=iou, ok=ok.bool())
    if want_image_vu:
        out["image_vu"] = vu
    return out


@torch.no_grad()
def compute_geometric_iou(poses, pointcloud, best_pose, pred_object_idx, masks, depth, cam_intrinsic, depth_scale, boxes):
    """the IoU half of the geometric score for all proposals of a frame: translation + projection + box + IoU (two launches).
    Follows the reference's batch-wide rule (bbox_utils.py:214-220): unless EVERY proposal's projected box meets its proposal box
    the score is 0 for the whole batch.  -> (iou (N,) f32, xyxy (N,4) i32, translate (N,3) f32)"""
    tr = calculate_the_query_translation(masks, depth, cam_intrinsic, depth_scale)
    H, W = masks.shape[-2], masks.shape[-1]
    r = project_template_iou(poses, pointcloud, best_pose, pred_object_idx, tr, cam_intrinsic, (H, W), boxes)
    iou = torch.where(r["ok"].all(), r["iou"], torch.zeros_like(r["iou"]))
    return iou, r["xyxy"], tr


# ---------------------------------------------------------------------------------------------- multi-object post-processing
MIN_BOX_SIZE, MIN_MASK_SIZE, NMS_THRESH = 0.05, 3e-4, 0.25      # ISM/configs/model/ISM_sam.yaml post_processing_config


@torch.no_grad()
def remove_very_small_detections(masks, boxes, min_box_size=MIN_BOX_SIZE, min_mask_size=MIN_MASK_SIZE):
    """Detections.remove_very_small_detections: masks (N,H,W), boxes (N,4) int64 xyxy -> keep (N,) bool on their device: box
    and mask area relative to the image above min_box_size^2 and min_mask_size.  The areas are reduced where the masks are."""
    img_area = masks.shape[1] * masks.shape[2]
    box_areas = (boxes[:, 2] - boxes[:, 0]) * (boxes[:, 3] - boxes[:, 1]) / img_area        # torchvision box_area
    mask_areas = masks.sum(dim=(1, 2)) / img_area
    return torch.logical_and(box_areas > min_box_size ** 2, mask_areas > min_mask_size)


@torch.no_grad()
def nms_per_object(boxes, scores, object_ids, nms_thresh=NMS_THRESH):
    """Detections.apply_nms_per_object_id: one torchvision.ops.nms per object id, as one launch over the boxes sorted by
    (object, decreasing score) -> kept indices (K,) int64 in the reference's order: object ids ascending, within an object
    by decreasing score (ties in proposal order)"""
    if boxes.shape[0] == 0:
        return torch.zeros(0, dtype=torch.long, device=boxes.device)
    order = torch.argsort(scores.float(), descending=True, stable=True)
    order = order[torch.argsort(object_ids[order], stable=True)]
    b = boxes[order].float().contiguous()
    obj = object_ids[order].to(torch.int32).contiguous()
    keep = torch.empty(b.shape[0], dtype=torch.uint8, device=b.device)
    _lib.call("sam6d_sam_nms", b, obj, b.shape[0], nms_thresh, keep)
    return order[keep.bool()]
