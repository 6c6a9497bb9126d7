"""SAM-6D in one process: the stages of the three template / ISM / PEM CLIs as functions on arrays and tensors, and `SAM6D`,
which keeps the models resident, onboards an object once and runs one RGB-D frame per call.

    from sam6d_b200.pipeline import SAM6D
    sam6d = SAM6D(segmentor="sam", checkpoint_dir="checkpoints", checkpoint="checkpoints/sam-6d-pem-base.pth")
    obj = sam6d.onboard("obj_000005.ply")                   # 42 templates rendered on the GPU, ISM + PEM template banks
    # denser ISM view sets and other aggregations: SAM6D(..., level_templates=2, pose_distribution="upper", aggregation_function="median")
    # ISM references from a BOP PBR split (rendering_type: pbr): SAM6D(..., rendering_type="pbr", pbr_root="datasets/ycbv")
    #   obj = sam6d.onboard("obj_000005.ply", obj_id=5)
    res = sam6d(rgb_u8, depth_u16, cam_K, depth_scale, obj)  # res.ism / res.pem: the CLIs' BOP-23 records; res.R, res.t

Several known objects in a frame (Instance_Segmentation_Model.test_step for the ISM, one PEM batch across the objects):

    objs = sam6d.onboard_objects(["obj_000001.ply", "obj_000005.ply"], obj_ids=[1, 5])
    res = sam6d.detect_objects(rgb_u8, depth_u16, cam_K, depth_scale, objs)   # records carry category_id = obj_ids[object]

The CLIs (sam6d_b200.cli.{render_custom_templates, ism_run_inference_custom, pem_run_inference_custom}) are file I/O around
the same stage functions, so one `SAM6D` frame computes what the chained CLIs compute from the same inputs and seeds.  Between
the ISM and the PEM the proposal masks stay on the device: their RLE is built by a kernel (ops.mask_rle) and only the run
ends come to the host, instead of every (H,W) float mask."""
import json
import os
import time
from dataclasses import dataclass
from types import SimpleNamespace
from typing import NamedTuple, Optional

import numpy as np
import torch

from . import bop, bop_eval, inputs, ism, meshio, ops, pbr, render, symmetry
from .cli import ism_run_inference_custom as ism_cli
from .cli import pem_run_inference_custom as pem_cli
from .cli import render_custom_templates as render_cli
from .pem import check_hypotheses, first_best

N_ISM_CLOUD = 2048                     # points of the geometric score's template cloud (ISM/run_inference_custom.py:196)
ICP_SAMPLES = 4096                     # surface samples per object for the ICP refinement (icp_iters > 0; not in the reference)
ICP_SEED = 6                           # their draws come from this seed, never from the caller's rng
RENDERING_TYPES = ("pyrender", "pbr")  # onboarding_config.rendering_type: the ISM references are renders, or BOP PBR frames


# ---- render + framing (Render/render_custom_templates.py) -----------------------------------------------------------------
def template_distance(mesh: meshio.Mesh, normalize: bool = True) -> float:
    """the template camera's distance from the origin: 4r with --normalize (r = max |bbox corner|), else 2"""
    if normalize:
        r = max(np.linalg.norm(mesh.vertices.max(axis=0)), np.linalg.norm(mesh.vertices.min(axis=0)))
        return 4.0 * float(r)
    return 2.0


def render_templates(mesh: meshio.Mesh, size: int = 512, normalize: bool = True, colorize: bool = False, base_color: float = 0.05,
                     poses_file: Optional[str] = None, level_templates: int = 0, pose_distribution: str = "all"):
    """the template views of one numpy mesh (mm) -> (render.render()'s dict for one object, poses (T,4,4) float64 in model units):
    the views of render.template_view_set(level_templates, pose_distribution), the 42 level-0 views first (the defaults: those
    42 only), or poses_file's.  Framing: camera 4r away with --normalize (r = max |bbox corner|), else 2; colours: base_color
    with colorize, else the mesh's texture / vertex colours / Blender's default grey."""
    distance = template_distance(mesh, normalize)
    if colorize:
        mesh.colors = mesh.uv = mesh.texture = None
        grey = float(base_color)
    else:
        grey = render_cli.BLENDER_DEFAULT_GREY
    poses, _ = render_cli.view_set(distance, poses_file, level_templates, pose_distribution)
    out = render_cli.render_views([render.upload(mesh)], poses[None], size, [[grey] * 3])
    return out, poses


def template_arrays(out, o: int = 0):
    """views of object o of render()'s output -> host arrays as the template files hold them: rgb (T,H,W,3) u8, mask (T,H,W) u8
    (255 = object), xyz (T,H,W,3) f16 in mm"""
    return out["rgb"][o].cpu().numpy(), out["mask"][o].cpu().numpy(), out["xyz"][o].cpu().numpy()


# ---- ISM template references (ISM/run_inference_custom.py:129-165) ----------------------------------------------------------
def ism_reference_features(desc, rgbs: np.ndarray, masks: np.ndarray, device):
    """template views rgb (T,H,W,3) u8 and mask (T,H,W) u8 -> (cls (T,C), masked patch tokens (T,256,C)) of the descriptor model"""
    boxes, templates, masks_t = [], [], []
    for rgb, mask in zip(rgbs, masks):
        ys, xs = np.nonzero(mask)
        boxes.append((xs.min(), ys.min(), xs.max() + 1, ys.max() + 1))                # PIL Image.getbbox of the mask file
        image = torch.from_numpy(rgb / 255).float()
        m = torch.from_numpy(mask / 255).float()
        templates.append(image * m[:, :, None])
        masks_t.append(m.unsqueeze(-1))
    templates = torch.stack(templates).permute(0, 3, 1, 2)
    masks_t = torch.stack(masks_t).permute(0, 3, 1, 2)
    boxes = torch.tensor(np.array(boxes))
    templates = ism_cli.crop_resize_pad_images(templates, boxes).to(device)
    masks_cropped = ism_cli.crop_resize_pad_images(masks_t, boxes).to(device)
    return desc.compute_cls_and_patch_features(templates, masks_cropped[:, 0, :, :].contiguous())


@dataclass
class IsmGeometry:
    """what the geometric score needs: template poses (T,4,4) f32 (metres), template cloud (npc,3) f32 (metres), depth (H,W) i32,
    K (3,3) as read, depth scale -- all on the device but the scale.  Several objects: poses (O,T,4,4) and cloud (O,npc,3)."""
    poses: torch.Tensor
    cloud: torch.Tensor
    depth: torch.Tensor
    K: torch.Tensor
    depth_scale: float


def ism_geometry(poses_m, cloud_m, depth_raw, cam_K, depth_scale, device) -> IsmGeometry:
    """the ISM CLI's conversions: poses and cloud to f32, depth to i32, K as np.array(cam_K) gives it, depth scale to a float"""
    return IsmGeometry(poses=torch.tensor(poses_m).float().to(device), cloud=torch.from_numpy(cloud_m).float().to(device),
                       depth=torch.from_numpy(np.asarray(depth_raw).astype(np.int32)).to(device),
                       K=torch.tensor(np.array(cam_K).reshape(3, 3), device=device), depth_scale=float(np.array(depth_scale)))


# ---- segment -> describe -> score (ISM/run_inference_custom.py:167-209) -------------------------------------------------------
def ism_detect(seg, desc, ref_cls, ref_patch, rgb_u8: np.ndarray, confidence_thresh: float, geometry: Optional[IsmGeometry] = None,
               mark=None, remove_small: bool = False, aggregation_function: str = "avg_5"):
    """-> SimpleNamespace(masks (N,H,W) f32, boxes (N,4) i64 xyxy, scores (N) f32, obj (N) i64, n_proposals, reason): the
    proposals above the semantic-score threshold with their final scores ((semantic + appearance + geometric x visible) /
    (2 + visible), or (semantic + appearance) / 2 without geometry) and the object each is assigned to.  ref_cls (T,C) and
    ref_patch (T,256,C) of one object, or (O,T,C) and (O,T,256,C) of several (geometry then holds every object's poses and
    cloud).  remove_small: Detections.remove_very_small_detections after the segmentor, as Instance_Segmentation_Model.test_step
    does.  aggregation_function: how the semantic score reduces each object's template similarities (ism.compute_semantic_score).
    reason is None, or why there is no detection.  mark(stage) is called after the segmentor, the descriptors and the
    scores (stage timing)."""
    from .dinov2 import MaskedPatch_MatrixSimilarity
    mark = mark or (lambda stage: None)
    if ref_cls.dim() == 2:
        ref_cls, ref_patch = ref_cls.unsqueeze(0), ref_patch.unsqueeze(0)
    det = seg.generate_masks(rgb_u8)
    det = SimpleNamespace(masks=det["masks"], boxes=det["boxes"].long(), scores=None, obj=None, n_proposals=int(det["masks"].shape[0]),
                          reason=None)
    if remove_small and det.n_proposals:
        keep = ism.remove_very_small_detections(det.masks, det.boxes).nonzero().flatten()
        det.masks, det.boxes = det.masks[keep], det.boxes[keep]
    mark("segmentor")
    if det.masks.shape[0] == 0:
        det.reason = "no mask proposal survived the filters"
        return det
    q_cls, q_patch = desc(rgb_u8, det)
    mark("descriptors")
    idx_sel, pred_obj, sem, best_t = ism.compute_semantic_score(q_cls, ref_cls, aggregation_function, confidence_thresh)
    det.masks, det.boxes, det.obj, q_patch = det.masks[idx_sel], det.boxes[idx_sel], pred_obj, q_patch[idx_sel]
    if idx_sel.numel() == 0:
        det.reason = "no proposal above the semantic-score threshold"
        mark("scores")
        return det
    ref_aux = ref_patch[pred_obj, best_t, ...]
    appe, vis = MaskedPatch_MatrixSimilarity().scores(q_patch, ref_aux, ism_cli.VISIBLE_THRED)
    if geometry is not None:
        g = geometry
        # each proposal's template pose among all objects' poses (O*T,4,4): row obj*T + t
        geo, _, _ = ism.compute_geometric_iou(g.poses.reshape(-1, 4, 4), g.cloud, pred_obj * ref_cls.shape[1] + best_t, pred_obj, det.masks,
                                              g.depth, g.K, g.depth_scale, det.boxes)
        det.scores = (sem + appe + geo * vis) / (1 + 1 + vis)
    else:
        det.scores = (sem + appe) / 2
    mark("scores")
    return det


# ---- BOP-23 records (ISM/model/utils.py:153-216) ----------------------------------------------------------------------------
def rle_counts(rle_cum: np.ndarray, rle_off: np.ndarray):
    """cumulative run ends + offsets (ops.mask_rle, inputs.pack_rle) -> every mask's uncompressed COCO RLE counts as int lists,
    exactly mask_to_rle's (a mask whose pixel (0,0) is set starts with the zero-length run: its first run end is 0)"""
    return [np.diff(rle_cum[rle_off[i]:rle_off[i + 1]], prepend=0).tolist() for i in range(len(rle_off) - 1)]


def ism_records(boxes_xyxy: np.ndarray, scores: np.ndarray, counts, hw, runtime: float, category_ids=None):
    """ISM detections -> the ISM CLI's JSON records (scene 0, image 0, category 1 or category_ids[i], bbox xywh)"""
    b = boxes_xyxy
    cats = [1] * len(b) if category_ids is None else [int(c) for c in category_ids]
    return [dict(scene_id=0, image_id=0, category_id=cats[i], bbox=[int(b[i, 0]), int(b[i, 1]), int(b[i, 2] - b[i, 0]), int(b[i, 3] - b[i, 1])],
                 score=float(scores[i]), time=float(runtime), segmentation={"counts": counts[i], "size": [int(hw[0]), int(hw[1])]})
            for i in range(len(b))]


def ism_records_from_masks(det, runtime: float):
    """records of ism_detect's detections, RLE on the device: one host copy of the run ends, none of the masks"""
    cum, off = ops.mask_rle(det.masks.contiguous())
    return ism_records(det.boxes.cpu().numpy(), det.scores.cpu().numpy(), rle_counts(cum.cpu().numpy(), off.cpu().numpy()),
                       det.masks.shape[1:], runtime)


# ---- PEM template bank (PEM/run_inference_custom.py:117-162) -----------------------------------------------------------------
def pem_template_bank(model, rgbs, masks, xyzs_mm, rng=None, device=None):
    """template views (uint8 rgb, uint8 mask 255 = object, float32 xyz in mm) -> (template points, template features) of the
    PEM's ViT-B branch"""
    cfg = pem_cli.TEST_DATASET
    all_tem, all_tem_pts, all_tem_choose = inputs.get_templates_from_arrays(rgbs, masks, xyzs_mm, cfg["n_sample_template_point"],
                                                                            cfg["img_size"], cfg["rgb_mask_flag"], rng=rng, device=device)
    with torch.no_grad():
        return model.feature_extraction.get_obj_feats(all_tem, all_tem_pts, all_tem_choose)


# ---- the per-object inputs of the steps after Net.forward (not in the reference) ----------------------------------------------
class PoseInputs(NamedTuple):
    """what finish_poses and symmetry_inputs need of O objects, each None when its step is off: icp (samples, normals) (O,M,3)
    f32 on the device (icp_model), meshes the O device meshes in mm that verification renders (verify_mesh), radii (O,) each
    object's max |model point| in metres (object_radii), symmetries their packed symmetry.SymmetrySet (object_symmetries)"""
    icp: Optional[tuple] = None
    meshes: Optional[list] = None
    radii: Optional[np.ndarray] = None
    symmetries: Optional["symmetry.SymmetrySet"] = None


def build_pose_inputs(meshes, model_points_m, device, icp: bool = False, verify: bool = False, symmetries=None,
                      obj_ids=None) -> PoseInputs:
    """O numpy meshes in mm (meshio.Mesh) and their model points (O,n,3) -> their PoseInputs: the ICP samples with icp, the
    device meshes and radii with verify, and unless None the packed symmetries of a check_symmetries value for obj_ids.  No
    draw from any caller's RNG: the ICP samples and "auto" symmetries draw from their own seeds, mesh by mesh."""
    samples = icp_tensors(*(np.stack(a) for a in zip(*[icp_model(m.vertices, m.faces) for m in meshes])), device) if icp else None
    return PoseInputs(icp=samples, meshes=[verify_mesh(m.vertices, m.faces, device) for m in meshes] if verify else None,
                      radii=object_radii(model_points_m) if verify else None,
                      symmetries=object_symmetries(symmetries, meshes, obj_ids, device))


# ---- PEM inputs + Net.forward (PEM/run_inference_custom.py:165-307) -------------------------------------------------------------
def pem_step(model, data: dict, bank, pose: PoseInputs, rand, rows, cam_K, icp_iters: int = 0, verify_tau: float = 0.1) -> dict:
    """Net.forward on the instances of `data` (get_test_data's or bop.pem_instances' dict; data["obj"] (P) the object index of
    each) and the steps after it -> Net.forward's outputs.  Each instance gets its object's template bank (O,2048,3),
    (O,2048,256); with several PEM hypotheses (Net.set_hypotheses) and pose.symmetries, hypotheses distinct up to its
    object's symmetries (symmetry_inputs).  rand: the coarse stage's uniforms (None: torch's global CUDA generator, the
    reference's torch.rand).  Then finish_poses with pose's ICP samples (icp_iters > 0), and with pose.meshes verification
    against rows, the frame's device depth and masks (inputs.FrameInputs.rows), with tolerance verify_tau x the object's radius."""
    data["dense_po"], data["dense_fo"] = bank[0][data["obj"]], bank[1][data["obj"]]
    if pose.symmetries is not None and model.hypotheses[0] > 1:
        symmetry_inputs(data, pose.symmetries, data["obj"])
    with torch.no_grad():
        out = model(data, rand=rand)
        return finish_poses(out, data["pts"], data["model"], data["obj"], pose.icp, icp_iters, pose.meshes, pose.radii, rows, cam_K,
                            verify_tau)


def pem_frame(model, bank, dets, rgb_u8, depth_raw, cam_K, depth_scale, model_points_m, det_obj, det_score_thresh: float, rng=None,
              generator: Optional[torch.Generator] = None, device=None, mark=None, pose: PoseInputs = PoseInputs(), icp_iters: int = 0,
              verify_tau: float = 0.1):
    """ISM records of O objects -> SimpleNamespace(dets, out, img, model_points, obj, choose_idx, rand): the detections the PEM
    keeps (above det_score_thresh with enough valid depth) as copies of their records, Net.forward's outputs (None when none is
    kept), the frame image and the model points (O,n,3) as get_test_data returns them, the object index obj (P) int64 and the
    sample indices choose_idx (P,2048) of every kept detection, and rand, the coarse stage's uniforms.  bank (O,2048,3),
    (O,2048,256), model_points_m (O,n,3) and det_obj the object index of every record (one object: model_points_m[None] and
    zeros); each detection gets its object's radius filter, model points and template bank, and all run as one batch
    (pem_step, with the objects' PoseInputs `pose`, default none).  The coarse stage's uniforms are drawn from `generator` when
    one is given, else from torch's global CUDA generator.  mark(stage) after the inputs and after the forward."""
    cfg = pem_cli.TEST_DATASET
    mark = mark or (lambda stage: None)
    got = inputs.get_test_data(
        [dict(d) for d in dets], rgb_u8, depth_raw, cam_K, depth_scale, model_points_m, det_score_thresh,
        cfg["n_sample_observed_point"], cfg["img_size"], cfg["rgb_mask_flag"], rng=rng, device=device, det_obj=det_obj,
        frame_rows=pose.meshes is not None)
    data, img, _, model_points, kept = got[:5]
    n = data["pts"].size(0)
    mark("pem_inputs")
    out = rand = None
    if n:
        if generator is not None:
            rand = torch.rand(n, model.coarse_point_matching.cfg.nproposal1 * 3, device=data["pts"].device, generator=generator)
        out = pem_step(model, data, bank, pose, rand, got[5] if pose.meshes is not None else None, cam_K, icp_iters, verify_tau)
    mark("forward")
    return SimpleNamespace(dets=kept, out=out, img=img, model_points=model_points, obj=data["obj"].cpu().numpy(),
                           choose_idx=data["choose_idx"], rand=rand)


def reported_scores(out: dict, det_score: torch.Tensor) -> torch.Tensor:
    """the score a pose is reported with: pred_pose_score x its detection's score, x verify when the poses were verified"""
    score = out["pred_pose_score"] * det_score
    return score * out["verify"] if "verify" in out else score


def pem_records(frame):
    """pem_frame's result -> the PEM CLI's records: the kept ISM records with the pose score (reported_scores), R and t (mm).
    The host arrays behind them are kept on `frame` as pose_scores, pred_rot, pred_trans (mm) for the visualisation.  When the
    poses were verified (verify_out) each record also carries "verify".  With several PEM hypotheses each record also carries
    "hypothesis", the index of the one it reports."""
    if frame.out is None:
        return []
    out = frame.out
    verified = "verify" in out
    frame.pose_scores = reported_scores(out, out["score"]).detach().cpu().numpy()
    if verified:
        verify = out["verify"].cpu().numpy()
    frame.pred_rot = out["pred_R"].detach().cpu().numpy()
    frame.pred_trans = out["pred_t"].detach().cpu().numpy() * 1000
    hyp = out["hyp_index"].cpu().numpy() if "hyp_index" in out else None
    records = frame.dets
    for idx in range(len(records)):
        records[idx]["score"] = float(frame.pose_scores[idx])
        records[idx]["R"] = list(frame.pred_rot[idx].tolist())
        records[idx]["t"] = list(frame.pred_trans[idx].tolist())
        if verified:
            records[idx]["verify"] = float(verify[idx])
        if hyp is not None:
            records[idx]["hypothesis"] = int(hyp[idx])
    return records


# ---- depth refinement of the PEM poses (not in the reference) ---------------------------------------------------------------
def icp_model(verts_mm: np.ndarray, faces: np.ndarray):
    """a CAD model in mm -> (ICP_SAMPLES surface points (M,3) f32 in metres, their unit face normals (M,3) f32), drawn from
    np.random.default_rng(ICP_SEED): the same samples for the same mesh, and no draw from any caller's RNG"""
    pts, nrm = meshio.sample_surface(verts_mm, faces, ICP_SAMPLES, np.random.default_rng(ICP_SEED), return_normals=True)
    return pts / np.float32(1000.0), nrm


def icp_tensors(points_m, normals, device):
    """icp_model arrays of one object (M,3) or of O objects (O,M,3) -> (samples, normals) (O,M,3) f32 on the device"""
    m = np.asarray(points_m).shape[-2]
    return tuple(torch.from_numpy(np.ascontiguousarray(np.asarray(a, dtype=np.float32).reshape(-1, m, 3))).to(device)
                 for a in (points_m, normals))


def icp_refine_out(out: dict, pts: torch.Tensor, model: torch.Tensor, obj: torch.Tensor, icp, iters: int):
    """refine Net.forward's poses against the observed points pts (P,N,3) in place: out["pred_R"], out["pred_t"] become the
    refined pose, the PEM's stays in out["pem_R"], out["pem_t"]; out["icp_inliers"] (P) i32 and out["icp_rms"] (P) f32 (metres)
    are the last iteration's inlier count and point-to-plane RMS.  model (P,n,3): each instance's model points, whose max norm
    is its object radius; obj (P): its object index into icp = (samples, normals) (O,M,3)."""
    radius = model.norm(dim=2).amax(dim=1).contiguous()
    R, t, inliers, rms, _ = ops.icp_refine(out["pred_R"].contiguous(), out["pred_t"].contiguous(), pts.contiguous(), icp[0], icp[1],
                                           obj.to(torch.int32).contiguous(), radius, iters)
    out.update(pem_R=out["pred_R"], pem_t=out["pred_t"], pred_R=R, pred_t=t, icp_inliers=inliers, icp_rms=rms)
    return out


# ---- depth verification of the reported poses (not in the reference) ----------------------------------------------------------
def verify_mesh(verts_mm: np.ndarray, faces: np.ndarray, device) -> meshio.Mesh:
    """a CAD model in mm -> its vertices and faces on the device, the mesh ops.verify_poses renders (no colours)"""
    faces = np.asarray(faces)
    if faces.ndim != 2 or faces.shape[0] == 0:
        raise ValueError("pose verification renders the object: its mesh needs faces")
    return render.upload(meshio.Mesh(vertices=np.asarray(verts_mm, np.float32), faces=faces), device)


def object_radii(model_points_m) -> np.ndarray:
    """model points (n,3) or (O,n,3) -> (O,) each object's max |model point| in metres, as ObjectSet.radii"""
    mp = np.asarray(model_points_m, dtype=np.float32)
    return np.asarray([np.max(np.linalg.norm(m, axis=1)) for m in mp.reshape((-1,) + mp.shape[-2:])])


def verify_out(out: dict, meshes, obj: np.ndarray, radii: np.ndarray, rows, cam_K, verify_tau: float):
    """check Net.forward's (or the ICP's) poses against the frame in place: out["verify_counts"] (P,6) i32 and out["verify"]
    (P,) f32 of ops.verify_poses.  meshes: the objects' device meshes in mm; obj (P) each pose's object; radii (O,) metres;
    rows: inputs.FrameInputs.rows of the kept detections (depth, mask, mrow); tau = verify_tau x the object's radius."""
    obj = np.asarray(obj, dtype=np.int64)
    tau = float(verify_tau) * np.asarray(radii, dtype=np.float64)[obj]
    counts, v = ops.verify_poses(out["pred_R"].contiguous(), out["pred_t"].contiguous(), obj, meshes, rows.depth, rows.mask, rows.mrow,
                                 np.asarray(cam_K, dtype=np.float64).reshape(3, 3), tau)
    out.update(verify_counts=counts, verify=v)
    return out


# ---- several PEM hypotheses per detection (not in the reference) ----------------------------------------------------------------
def finish_poses(out: dict, pts: torch.Tensor, model: torch.Tensor, obj: torch.Tensor, icp=None, icp_iters: int = 0, verify=None,
                 radii=None, rows=None, cam_K=None, verify_tau: float = 0.1):
    """the steps after Net.forward, in place: ICP (icp_iters > 0, icp_refine_out), then verification (verify, the objects'
    device meshes: verify_out with radii (O,) and the frame's rows), and with several hypotheses (out["hyp_R"] (B,K,3,3),
    Net.set_hypotheses) the choice of each detection's pose.  pts (B,N,3) observed points, model (B,n,3) model points, obj (B)
    object index of each detection.
    - One hypothesis, or verification off: Net's choice stands; ICP refines the reported poses only.
    - Several hypotheses and verification on: ICP refines all B K poses and verify_out checks all of them, each against its
      detection's mask row; the reported pose is the first valid k with the largest hyp_pose_score x verify.  out then also
      holds hyp_verify (B,K) and, with ICP, hyp_icp_R (B,K,3,3), hyp_icp_t (B,K,3); pred_*, verify, verify_counts, pem_*,
      icp_* and hyp_index are the chosen hypothesis's."""
    K = out["hyp_R"].shape[1] if "hyp_R" in out else 1
    if K == 1 or verify is None:
        if icp_iters > 0:
            icp_refine_out(out, pts, model, obj, icp, icp_iters)
        if verify is not None:
            verify_out(out, verify, obj.cpu().numpy(), radii, rows, cam_K, verify_tau)
        return out
    B = out["hyp_R"].shape[0]
    hyp = dict(pred_R=out["hyp_R"].reshape(B * K, 3, 3), pred_t=out["hyp_t"].reshape(B * K, 3))
    if icp_iters > 0:
        icp_refine_out(hyp, *(x.repeat_interleave(K, dim=0) for x in (pts, model, obj)), icp, icp_iters)
    verify_out(hyp, verify, np.repeat(obj.cpu().numpy(), K), radii,
               SimpleNamespace(depth=rows.depth, mask=rows.mask, mrow=np.repeat(np.asarray(rows.mrow), K)), cam_K, verify_tau)
    v = hyp["verify"].view(B, K)
    idx = first_best(out["hyp_pose_score"] * v, out["hyp_valid"])
    sel = idx + torch.arange(B, device=idx.device) * K
    keys = ("pred_R", "pred_t", "verify", "verify_counts") + (("pem_R", "pem_t", "icp_inliers", "icp_rms") if icp_iters > 0 else ())
    out.update({k: hyp[k][sel] for k in keys})
    out.update(hyp_index=idx, pred_pose_score=out["hyp_pose_score"].reshape(-1)[sel], hyp_verify=v)
    if icp_iters > 0:
        out.update(hyp_icp_R=hyp["pred_R"].view(B, K, 3, 3), hyp_icp_t=hyp["pred_t"].view(B, K, 3))
    return out


# ---- hypotheses distinct up to the objects' symmetries (not in the reference) ---------------------------------------------------
SYMMETRY_SOURCES = ("auto",)           # besides None and {obj_id: models_info entry}; run_bop_pem also takes "models_info"


def symmetry_inputs(data: dict, symmetries: "symmetry.SymmetrySet", obj: torch.Tensor) -> dict:
    """fill Net.forward's hyp_sym_R, hyp_sym_t and hyp_sym_range (pem.SYM_KEYS) in place: every object's packed set, and each
    detection's range in it by its object index obj (B)"""
    obj = obj.to(symmetries.range.device)
    data.update(hyp_sym_R=symmetries.R, hyp_sym_t=symmetries.t, hyp_sym_range=symmetries.range[obj].contiguous())
    return data


def check_symmetries(symmetries, obj_ids, sources=SYMMETRY_SOURCES):
    """ValueError unless symmetries is None, one of `sources`, or a dict holding a models_info entry for every id of obj_ids"""
    if symmetries is None or (isinstance(symmetries, str) and symmetries in sources):
        return
    if isinstance(symmetries, dict):
        missing = [i for i in obj_ids if int(i) not in symmetries]
        if missing:
            raise ValueError(f"symmetries: no models_info entry for obj_ids {missing}")
        bad = [i for i in obj_ids if not isinstance(symmetries[int(i)], dict)]
        if bad:
            raise ValueError(f"symmetries: the entries of obj_ids {bad} are not models_info dicts")
        return
    raise ValueError(f"symmetries must be None, one of {sources} or {{obj_id: models_info entry}}, got {symmetries!r}")


def object_symmetries(symmetries, meshes, obj_ids, device) -> Optional["symmetry.SymmetrySet"]:
    """a checked `symmetries` value -> the objects' packed symmetry sets (symmetry.pack_sets), or None.  "auto":
    symmetry.find_symmetries of every meshio.Mesh"""
    if symmetries is None:
        return None
    if isinstance(symmetries, str):
        infos = [symmetry.find_symmetries(m, backend=symmetry.GpuBackend(device)) for m in meshes]
    else:
        infos = [symmetries[int(i)] for i in obj_ids]
    return symmetry.pack_sets(infos, device)


# ---- the whole pipeline ----------------------------------------------------------------------------------------------------
@dataclass
class Onboarded:
    """one object after SAM6D.onboard: ISM references, template poses, geometric-score cloud, PEM template bank (1,2048,3),
    (1,2048,256), model points; pose_inputs, the object's PoseInputs (O = 1) for the SAM6D's icp_iters and verify and the
    symmetries it was onboarded with"""
    ref_cls: torch.Tensor
    ref_patch: torch.Tensor
    poses_m: np.ndarray
    cloud_m: np.ndarray
    bank: tuple
    model_points_m: np.ndarray
    pose_inputs: PoseInputs = PoseInputs()


class SAM6D:
    """the SAM-6D models, built once (through the ISM and PEM CLIs' build_models / build_fastsam / build_model, so checkpoint
    names, seeded weights and thresholds are theirs).  onboard() an object, then call the instance once per RGB-D frame.

    The ISM settings of the reference's configuration: level_templates (0 / 1 / 2 = 42 / 162 / 642 views) and pose_distribution
    ("all", or "upper": cameras with z >= 0) choose the views the ISM matches against (onboarding_config); aggregation_function
    ("mean", "median", "max", "avg_5") how each object's template similarities become its semantic score (matching_config).
    The PEM always uses the 42 level-0 views.  fastsam_model ("FastSAM-x" or "FastSAM-s") picks the FastSAM checkpoint and
    network when segmentor is "fastsam".

    rendering_type (onboarding_config): "pyrender", the ISM references are GPU renders of the CAD model; "pbr", they are
    frames of the BOP split pbr_root/pbr_split (sam6d_b200/pbr.py: for each view the frame whose object pose is nearest it,
    cut out with its visible mask), which needs each object's BOP id and pose_distribution "all".  The split is scanned once,
    at the first onboarding.  The geometric-score poses, the template cloud, the PEM bank and the model points come from the
    mesh either way.

    icp_iters (not in the reference; default 0, off): refine every PEM pose with that many point-to-plane ICP iterations
    against the frame's observed points (icp_refine_out).  Records then carry the refined R and t; scores are unchanged.

    verify (not in the reference; default False, off): render every reported pose, after any ICP, and count its agreement with
    the frame's depth and its detection's mask (verify_out, with tolerance verify_tau x the object's radius).  Each record's
    score is then pred_pose_score x ISM score x verify, and the record carries "verify"; R and t are unchanged.  Onboarding
    keeps each object's mesh on the device for it.

    pem_hypotheses (not in the reference; default 1, off): run the PEM's fine stage from that many mutually distinct coarse
    hypotheses, at least hyp_min_angle degrees or hyp_min_dist object radii apart (Net.set_hypotheses), and report one pose
    per detection: the one with the best pose score, or with verify on the best pose score x verify over all of them
    (finish_poses; with ICP every hypothesis is refined before it is verified).  Records then carry "hypothesis".  Objects
    onboarded with symmetries (onboard_objects) get hypotheses that are distinct up to their symmetries."""
    rendering_type = "pyrender"

    def __init__(self, segmentor: str = "sam", sam_model_type: str = "vit_h", dinov2_model: str = "dinov2_vitl14",
                 checkpoint_dir: Optional[str] = None, checkpoint: Optional[str] = None, random_weights: bool = False,
                 stability_score_thresh: float = 0.97, pred_iou_thresh: float = 0.88, points_per_side: int = 32,
                 confidence_thresh: float = ism_cli.CONFIDENCE_THRESH, det_score_thresh: float = 0.2, precision: str = "bf16",
                 device=None, level_templates: int = 0, pose_distribution: str = "all", aggregation_function: str = "avg_5",
                 fastsam_model: str = "FastSAM-x", rendering_type: str = "pyrender", pbr_root: Optional[str] = None,
                 pbr_split: str = "train_pbr", icp_iters: int = 0, verify: bool = False, verify_tau: float = 0.1,
                 pem_hypotheses: int = 1, hyp_min_angle: float = 30.0, hyp_min_dist: float = 0.2):
        if segmentor not in ("sam", "fastsam"):
            raise ValueError(f"The segmentor_model {segmentor} is not supported")
        if fastsam_model not in ism_cli.FASTSAM_MODELS:
            raise ValueError(f"fastsam_model must be one of {sorted(ism_cli.FASTSAM_MODELS)}, got {fastsam_model!r}")
        render.template_view_set(level_templates, pose_distribution)          # ValueError on an unknown view set
        if aggregation_function not in ops.TEMPLATE_AGGREGATIONS:
            raise ValueError(f"aggregation_function must be one of {sorted(ops.TEMPLATE_AGGREGATIONS)}, got {aggregation_function!r}")
        if rendering_type not in RENDERING_TYPES:
            raise ValueError(f"rendering_type must be one of {RENDERING_TYPES}, got {rendering_type!r}")
        if rendering_type == "pbr":
            if pbr_root is None:
                raise ValueError('rendering_type "pbr" needs pbr_root, the BOP dataset directory that holds the pbr_split')
            if pose_distribution != "all":
                raise NotImplementedError(f'rendering_type "pbr" selects references for pose_distribution "all" only, got {pose_distribution!r}')
            pbr.list_scenes(pbr_root, pbr_split)                              # FileNotFoundError without the split
        if int(icp_iters) < 0:
            raise ValueError(f"icp_iters must be >= 0, got {icp_iters}")
        self.icp_iters = int(icp_iters)
        if not (np.isfinite(verify_tau) and verify_tau > 0):
            raise ValueError(f"verify_tau must be a finite number > 0, got {verify_tau}")
        self.verify, self.verify_tau = bool(verify), float(verify_tau)
        hypotheses = check_hypotheses(pem_hypotheses, hyp_min_angle, hyp_min_dist)
        self.rendering_type, self.pbr_root, self.pbr_split, self._pbr_rows = rendering_type, pbr_root, pbr_split, None
        self.level_templates, self.pose_distribution = int(level_templates), pose_distribution
        self.aggregation_function = aggregation_function
        self.device = torch.device(device if device is not None else "cuda")
        self.confidence_thresh = float(confidence_thresh)
        self.det_score_thresh = float(det_score_thresh)
        ism_args = SimpleNamespace(segmentor_model=segmentor, sam_model_type=sam_model_type, fastsam_model=fastsam_model, dinov2_model=dinov2_model,
                                   checkpoint_dir=checkpoint_dir, random_weights=random_weights,
                                   stability_score_thresh=stability_score_thresh, pred_iou_thresh=pred_iou_thresh,
                                   points_per_side=points_per_side)
        self.seg, self.desc = ism_cli.build_models(ism_args, self.device)
        self.pem = pem_cli.build_model(SimpleNamespace(precision=precision, checkpoint=checkpoint, random_weights=random_weights), self.device)
        if hypotheses[0] > 1:
            self.pem.set_hypotheses(*hypotheses)

    def onboard(self, mesh_or_ply_path, template_size: int = 512, rng=None, obj_id: Optional[int] = None, symmetries=None) -> Onboarded:
        """render the templates of a CAD model in mm (a PLY path or a numpy meshio.Mesh) with render_custom_templates' framing
        and colours, and build everything a frame needs from them without touching a file: every view of
        render.template_view_set(level_templates, pose_distribution) is rendered once; the ISM references and the
        geometric-score poses come from the ISM's views, the PEM template bank from the 42 level-0 views.  Random draws, from
        `rng` (default numpy's global RNG), in the order the chained CLIs make them: the ISM template cloud, the PEM template
        samples, the PEM model points.

        rendering_type "pbr": obj_id, the object's BOP id, is required; the ISM references are the split's frames chosen by
        pbr.select_references, whose draws come first from `rng`, then the draws above; only the 42 level-0 views are rendered.

        symmetries (not in the reference; used with pem_hypotheses > 1): None, "auto" or the object's models_info entry, kept
        in Onboarded.pose_inputs (onboard_objects)."""
        if isinstance(symmetries, dict):
            symmetries = {0: symmetries}
        check_symmetries(symmetries, [0])
        refs = None
        if self.rendering_type == "pbr":
            if obj_id is None:
                raise ValueError('rendering_type "pbr" needs the BOP object id: onboard(..., obj_id=)')
            ref_cls, ref_patch = self._pbr_references([obj_id], rng)
            refs = (ref_cls[0], ref_patch[0])
        mesh = meshio.load_ply_mesh(mesh_or_ply_path) if isinstance(mesh_or_ply_path, str) else mesh_or_ply_path
        ob = self._onboard_mesh(mesh, template_size, rng, refs)
        ob.pose_inputs = build_pose_inputs([mesh], ob.model_points_m, self.device, icp=self.icp_iters > 0, verify=self.verify,
                                           symmetries=symmetries, obj_ids=[0])
        return ob

    def _pbr_references(self, obj_ids, rng):
        """the PBR references of every object of obj_ids -> (ref_cls (O,T,C), ref_patch (O,T,256,C)) for the ISM's views"""
        if self._pbr_rows is None:
            self._pbr_rows = pbr.scan_split(self.pbr_root, self.pbr_split)
        union, index = render.template_view_set(self.level_templates, "all")
        sel = pbr.select_references(self._pbr_rows, obj_ids, union[index], rng)
        return pbr.reference_features(self.desc, self._pbr_rows, sel, self.device)

    def _onboard_mesh(self, mesh: meshio.Mesh, template_size, rng, refs=None) -> Onboarded:
        """onboard() from the numpy mesh but for its pose inputs, with the ISM references `refs` (ref_cls, ref_patch) when they
        are given"""
        verts, faces = mesh.vertices, mesh.faces
        if refs is None:
            out, poses = render_templates(mesh, template_size, level_templates=self.level_templates, pose_distribution=self.pose_distribution)
            ism_index = render.template_view_set(self.level_templates, self.pose_distribution)[1]
            rgbs, masks, xyzs = template_arrays(out)
            del out
            ref_cls, ref_patch = ism_reference_features(self.desc, rgbs[ism_index], masks[ism_index], self.device)
        else:
            out, _ = render_templates(mesh, template_size)                    # the PEM's 42 level-0 views
            rgbs, masks, xyzs = template_arrays(out)
            del out
            ref_cls, ref_patch = refs
            poses, ism_index = render_cli.view_set(template_distance(mesh), None, self.level_templates, "all")
        cloud = meshio.sample_surface(verts, faces, N_ISM_CLOUD, rng) / 1000.0
        n0 = pem_cli.TEST_DATASET["n_template_view"]
        bank = pem_template_bank(self.pem, list(rgbs[:n0]), list(masks[:n0]), [x.astype(np.float32) for x in xyzs[:n0]], rng=rng,
                                 device=self.device)
        model_points = meshio.sample_surface(verts, faces, pem_cli.TEST_DATASET["n_sample_model_point"], rng) / 1000.0
        return Onboarded(ref_cls, ref_patch, render_cli.to_metres(poses[ism_index]), cloud, bank, model_points)

    def onboard_objects(self, meshes, obj_ids=None, template_size: int = 512, rng=None, symmetries=None) -> "ObjectSet":
        """onboard() every mesh in turn (random draws from `rng`, object after object) and stack the results into an ObjectSet,
        whose pose inputs are built once for all of them.  obj_ids: the category id of every object (distinct ints), default
        1..O.  The fp32 patch tokens (44 MB per object at C = 1024) are copied into the stack as each object is built, so only
        one object's extra copy is alive at a time.

        rendering_type "pbr": obj_ids are required and are the objects' BOP ids.  The references of all objects are selected
        first (pbr.select_references' draws, object after object, as the reference's load_processed_metaData makes them), then
        built in one pass over the split's frames straight into the stacks; then each mesh is onboarded with its draws.

        symmetries (not in the reference; used with pem_hypotheses > 1): None (default), "auto" (symmetry.find_symmetries of
        every mesh, whose samples draw from their own seed, not from `rng`) or {obj_id: models_info entry}; kept packed on the
        device in ObjectSet.pose_inputs (symmetry.pack_sets), so that detect_objects' hypotheses are distinct up to them."""
        meshes = list(meshes)
        n = len(meshes)
        if self.rendering_type == "pbr" and obj_ids is None:
            raise ValueError('rendering_type "pbr" needs the BOP id of every object: onboard_objects(meshes, obj_ids)')
        obj_ids = list(range(1, n + 1)) if obj_ids is None else [int(i) for i in obj_ids]
        if n == 0 or len(obj_ids) != n or len(set(obj_ids)) != n:
            raise ValueError(f"onboard_objects: {n} meshes need {n} distinct obj_ids, got {obj_ids}")
        check_symmetries(symmetries, obj_ids)
        meshes = [meshio.load_ply_mesh(m) if isinstance(m, str) else m for m in meshes]
        if self.rendering_type == "pbr":
            ref_cls, ref_patch = self._pbr_references(obj_ids, rng)
            parts = [self._onboard_mesh(mesh, template_size, rng, (ref_cls[o], None)) for o, mesh in enumerate(meshes)]
        else:
            parts, ref_patch = [], None
            for o, mesh in enumerate(meshes):
                ob = self._onboard_mesh(mesh, template_size, rng)
                if ref_patch is None:
                    ref_patch = ob.ref_patch.new_empty((n,) + tuple(ob.ref_patch.shape))
                ref_patch[o] = ob.ref_patch
                ob.ref_patch = None
                parts.append(ob)
        objs = ObjectSet.stack(parts, ref_patch, obj_ids)
        objs.pose_inputs = build_pose_inputs(meshes, objs.model_points_m, self.device, icp=self.icp_iters > 0, verify=self.verify,
                                             symmetries=symmetries, obj_ids=obj_ids)
        return objs

    def __call__(self, rgb_u8: np.ndarray, depth_raw: np.ndarray, cam_K, depth_scale, obj: Onboarded, rng=None, mark=None):
        """one RGB-D frame: rgb (H,W,3) u8, depth (H,W) raw u16, cam_K (9 values) and depth_scale as camera.json holds them.
        -> SimpleNamespace(ism, pem: the CLIs' records; masks (N,H,W) f32, boxes (N,4) i64, scores (N) f32 of the ISM detections;
        R (P,3,3), t (P,3) metres of the PEM's, on the device).  `rng` draws the observed-point samples (default numpy's global
        RNG); the coarse stage's uniforms come from a fresh torch generator seeded with the PEM's RD_SEED, so a frame's poses
        do not depend on earlier frames.  mark(stage), when given, is called after each stage (stage timing)."""
        return self._frame(rgb_u8, depth_raw, cam_K, depth_scale, obj, None, rng, mark)

    def detect_objects(self, rgb_u8: np.ndarray, depth_raw: np.ndarray, cam_K, depth_scale, objects: "ObjectSet", rng=None, mark=None,
                       pem: bool = True):
        """one RGB-D frame with several onboarded objects, the fields of __call__ plus obj (N) i64, the object index of every ISM
        detection.  The ISM follows Instance_Segmentation_Model.test_step: proposals, remove_very_small_detections, descriptors,
        semantic score over all objects, appearance score against the assigned object's best template, geometric score with
        that object's cloud and template pose, final score, apply_nms_per_object_id (records ordered by object, then by
        decreasing score; category_id = obj_ids[object]).  The PEM runs every kept detection in one Net.forward batch, each
        with its object's radius filter, model points and template bank; sample indices are drawn in detection order.
        mark(stage) as for __call__, plus "nms".  pem=False stops after the ISM records (pem [], R and t None).  The result's
        ism_time is the host seconds from the segmentor to the end of the NMS, test_step's proposal + matching time."""
        return self._frame(rgb_u8, depth_raw, cam_K, depth_scale, objects, objects.obj_ids, rng, mark, pem)

    # ---- a BOP test split (ISM/run_inference.py, PEM/test_bop.py; sam6d_b200/bop.py) ------------------------------------------
    def onboard_bop(self, bop_root: str, dataset_name: str, template_size: int = 512, rng=None) -> "ObjectSet":
        """onboard_objects() of every object of the dataset (bop.load_objects: sorted model ids, the ids passed as obj_ids)"""
        objs = bop.load_objects(bop_root, dataset_name)
        return self.onboard_objects(objs.ply_paths, obj_ids=objs.ids, template_size=template_size, rng=rng)

    def run_bop_ism(self, bop_root: str, dataset_name: str, objects: "ObjectSet", out_path: Optional[str] = None,
                    max_frames: Optional[int] = None, mark=None):
        """Instance_Segmentation_Model.test_step over every frame of bop.scan_test_split (the first max_frames), then
        test_epoch_end's result file: detect_objects (ISM only) on the image test_step segments (bop.round_trip of the decoded
        frame), records with scene_id, image_id = frame id, category_id = bop.category_ids of the object index (the objects in
        onboarding order, which is load_objects' order for onboard_bop) and time = proposal + matching seconds.  Frames in scan
        order.  Writes the list to out_path with a plain json.dump (save_json_bop23) and returns it.  mark(stage) is called
        after "decode" and after each stage of detect_objects."""
        mark = mark or (lambda stage: None)
        cats = bop.category_ids(dataset_name, len(objects.obj_ids))
        records = []
        for f in bop.scan_test_split(bop_root, dataset_name)[:max_frames]:
            rgb = bop.round_trip(bop.decode_rgb(f.rgb_path))
            depth = bop.decode_depth(f.depth_path)
            mark("decode")
            res = self.detect_objects(rgb, depth, f.cam_K, f.depth_scale, objects, mark=mark, pem=False)
            for r, o in zip(res.ism, res.obj.tolist() if res.ism else []):
                r.update(scene_id=f.scene_id, image_id=f.frame_id, category_id=cats[o], time=float(res.ism_time))
            records += res.ism
        if out_path is not None:
            with open(out_path, "w") as fh:
                json.dump(records, fh)
        return records

    def run_bop_pem(self, detections_path: str, bop_root: str, dataset_name: str, template_dir: str, out_path: Optional[str] = None,
                    rng=None, max_frames: Optional[int] = None, mark=None, symmetries=None):
        """test_bop.py over a detection file (ours or the reference ISM's; uncompressed RLE): per image of the file (bop.
        group_detections, the first max_frames), bop.pem_instances, then Net.forward on all of the image's instances with the
        coarse-stage uniforms of test_bop.py (bop.pem_rand: one CUDA generator seeded RD_SEED for the run, one torch.rand per
        chunk of 16).  Random draws from `rng` (default numpy's global RNG): the model points of every object, each object's
        42 template samples, then the observed points in detection order.  An image none of whose detections survives is
        skipped (the reference fails there).  Writes the CSV lines to out_path and returns them.  mark(stage) after
        "onboard", and per image after "decode", "pem_inputs" and "forward".  icp_iters > 0: each image's poses are refined (icp_refine_out) before its rows are built.
        verify: each image's poses are then verified (verify_out, the dataset's meshes) and each row's score is
        pred_pose_score x detection score x verify.  symmetries, with pem_hypotheses > 1: as onboard_objects', or "models_info",
        the dataset's own models_info.json next to its models."""
        mark = mark or (lambda stage: None)
        rng = rng if rng is not None else np.random
        cfg = pem_cli.TEST_DATASET
        objs = bop.load_objects(bop_root, dataset_name)
        check_symmetries(symmetries, objs.ids, SYMMETRY_SOURCES + ("models_info",))
        if symmetries == "models_info":
            symmetries = bop_eval.load_models_info(os.path.join(bop_root, dataset_name, bop.model_dir(dataset_name), "models_info.json"))
            check_symmetries(symmetries, objs.ids)
        meshes = [meshio.load_ply_mesh(p) for p in objs.ply_paths]
        model_points = np.stack([meshio.sample_surface(m.vertices, m.faces, bop.N_SAMPLE_MODEL_POINT, rng) / 1000.0 for m in meshes])
        model_points = model_points.astype(np.float32)
        banks = [pem_template_bank(self.pem, *bop.load_templates(template_dir, dataset_name, i, cfg["n_template_view"]), rng=rng,
                                   device=self.device) for i in objs.ids]
        bank = tuple(torch.stack([b[k].reshape(b[k].shape[-2:]) for b in banks]) for k in range(2))
        del banks
        pose = build_pose_inputs(meshes, model_points, self.device, icp=self.icp_iters > 0, verify=self.verify,
                                 symmetries=symmetries if self.pem.hypotheses[0] > 1 else None, obj_ids=objs.ids)
        mark("onboard")
        with open(detections_path) as fh:
            groups = bop.group_detections(json.load(fh))
        g = torch.Generator(device=self.device)
        g.manual_seed(pem_cli.RD_SEED)
        n_rand = self.pem.coarse_point_matching.cfg.nproposal1 * 3
        lines = []
        for (scene_id, image_id), dets in groups[:max_frames]:
            rgb_path, depth_path, cam_K, depth_scale = bop.frame_paths(bop_root, dataset_name, scene_id, image_id)
            image, raw = bop.decode_pem_image(rgb_path), bop.decode_depth(depth_path)
            mark("decode")
            torch.cuda.synchronize(self.device)
            t0 = time.time()
            got = bop.pem_instances(dets, image, raw, cam_K, depth_scale, objs, model_points, rng=rng, n_sample=cfg["n_sample_observed_point"],
                                    img_size=cfg["img_size"], device=self.device, frame_rows=self.verify)
            data, kept = got[:2]
            mark("pem_inputs")
            n = len(kept)
            if n == 0:
                continue
            rand = bop.pem_rand(g, n, n_rand, self.device)
            out = pem_step(self.pem, data, bank, pose, rand, got[3] if self.verify else None, cam_K, self.icp_iters, self.verify_tau)
            scores = reported_scores(out, data["score"]).cpu().numpy()
            R = out["pred_R"].reshape(-1, 9).cpu().numpy()
            t = out["pred_t"].cpu().numpy() * 1000
            image_time = time.time() - t0 + float(np.float32(dets[0]["time"]))
            mark("forward")
            lines += bop.csv_rows(scene_id, image_id, [d["category_id"] for d in kept], scores, R, t, image_time)
        if out_path is not None:
            with open(out_path, "w+") as fh:
                fh.writelines(lines)
        return lines

    def _frame(self, rgb_u8, depth_raw, cam_K, depth_scale, obj, obj_ids, rng, mark, pem=True):
        multi = obj_ids is not None
        mark = mark or (lambda stage: None)
        t0 = time.time()
        geometry = ism_geometry(obj.poses_m, obj.cloud_m, depth_raw, cam_K, depth_scale, self.device)
        t_ism = time.time()
        det = ism_detect(self.seg, self.desc, obj.ref_cls, obj.ref_patch, rgb_u8, self.confidence_thresh, geometry, mark, remove_small=multi,
                         aggregation_function=self.aggregation_function)
        if multi and det.reason is None:
            keep = ism.nms_per_object(det.boxes, det.scores, det.obj)
            det.masks, det.boxes, det.scores, det.obj = det.masks[keep], det.boxes[keep], det.scores[keep], det.obj[keep]
            mark("nms")
        ism_time = time.time() - t_ism
        if det.reason is not None:
            mark("rle")
            mark("ism_records")
            return SimpleNamespace(ism=[], pem=[], masks=det.masks, boxes=det.boxes, scores=det.scores, R=None, t=None, frame=None,
                                   n_proposals=det.n_proposals, reason=det.reason, ism_time=ism_time, **({"obj": det.obj} if multi else {}))
        cum, off = ops.mask_rle(det.masks.contiguous())
        mark("rle")
        counts = rle_counts(cum.cpu().numpy(), off.cpu().numpy())
        det_obj = det.obj.cpu().numpy()
        records = ism_records(det.boxes.cpu().numpy(), det.scores.cpu().numpy(), counts, det.masks.shape[1:], time.time() - t0,
                              category_ids=np.asarray(obj_ids)[det_obj] if multi else None)
        mark("ism_records")
        if not pem:
            return SimpleNamespace(ism=records, pem=[], masks=det.masks, boxes=det.boxes, scores=det.scores, R=None, t=None, frame=None,
                                   n_proposals=det.n_proposals, reason=None, ism_time=ism_time, **({"obj": det.obj} if multi else {}))
        pose = obj.pose_inputs if self.verify else obj.pose_inputs._replace(meshes=None)       # pem_step verifies given meshes
        if (self.icp_iters > 0 and pose.icp is None) or (self.verify and pose.meshes is None):
            raise ValueError("ICP and pose verification need the objects' ICP samples and device meshes: onboard them with a SAM6D "
                             "of this icp_iters and verify")
        g = torch.Generator(device=self.device)
        g.manual_seed(pem_cli.RD_SEED)
        mp = np.asarray(obj.model_points_m)
        frame = pem_frame(self.pem, obj.bank, records, rgb_u8, depth_raw, cam_K, depth_scale, mp.reshape((-1,) + mp.shape[-2:]), det_obj,
                          self.det_score_thresh, rng=rng, generator=g, device=self.device, mark=mark, pose=pose, icp_iters=self.icp_iters,
                          verify_tau=self.verify_tau)
        pem_recs = pem_records(frame)
        mark("pem_records")
        R = frame.out["pred_R"] if frame.out is not None else None
        t = frame.out["pred_t"] if frame.out is not None else None
        return SimpleNamespace(ism=records, pem=pem_recs, masks=det.masks, boxes=det.boxes, scores=det.scores, R=R, t=t, frame=frame,
                               n_proposals=det.n_proposals, reason=None, ism_time=ism_time, **({"obj": det.obj} if multi else {}))


@dataclass
class ObjectSet:
    """several objects after SAM6D.onboard_objects, stacked along a leading object axis O: ISM references ref_cls (O,T,C) and
    ref_patch (O,T,256,C), template poses poses_m (O,T,4,4) (the framing distance depends on the mesh), geometric-score clouds
    cloud_m (O,2048,3), PEM template banks (O,2048,3) and (O,2048,256), model points model_points_m (O,Nm,3), each object's
    radius (O,) (the PEM's max |model point|) and category ids obj_ids; pose_inputs, the objects' PoseInputs for the SAM6D's
    icp_iters and verify and the symmetries they were onboarded with"""
    ref_cls: torch.Tensor
    ref_patch: torch.Tensor
    poses_m: np.ndarray
    cloud_m: np.ndarray
    bank: tuple
    model_points_m: np.ndarray
    radii: np.ndarray
    obj_ids: list
    pose_inputs: PoseInputs = PoseInputs()

    @staticmethod
    def stack(parts, ref_patch, obj_ids) -> "ObjectSet":
        """Onboarded objects (their ref_patch already stacked into `ref_patch`) -> ObjectSet, without pose inputs"""
        mp = np.stack([np.asarray(p.model_points_m, dtype=np.float32) for p in parts])
        return ObjectSet(ref_cls=torch.stack([p.ref_cls for p in parts]), ref_patch=ref_patch,
                         poses_m=np.stack([p.poses_m for p in parts]), cloud_m=np.stack([p.cloud_m for p in parts]),
                         bank=tuple(torch.stack([p.bank[i].reshape(p.bank[i].shape[-2:]) for p in parts]) for i in range(2)),
                         model_points_m=mp, radii=object_radii(mp), obj_ids=list(obj_ids))
