"""Drop-in for SAM-6D/Instance_Segmentation_Model/run_inference_custom.py (SURVEY.md 8b, CLI row): same arguments, same inputs
(`$OUT/templates/{rgb,mask}_i.png`, rgb / depth PNGs, camera.json, CAD PLY), same outputs
(`$OUT/sam6d_results/detection_ism.{json,npz}`: BOP-23 records `{scene_id, image_id, category_id, bbox[xywh], score, time,
segmentation{counts,size}}`, ISM/model/utils.py:153-216).

    python -m sam6d_b200.cli.ism_run_inference_custom --segmentor_model sam --output_dir OUT --cad_path obj.ply \\
        --rgb_path rgb.png --depth_path depth.png --cam_path camera.json [--stability_score_thresh 0.97]

Pipeline (ISM/run_inference_custom.py:97-209): template descriptors (DINOv2 cls + masked patch tokens of the 42 views) -> SAM
automatic mask generation (ViT-H / -L / -B encoder, prompt encoder, mask decoder, filters, NMS) -> proposal descriptors -> semantic score
(avg-5 template cosine) -> appearance score -> geometric score (template pose projection IoU x visible ratio) -> final score.
All model compute runs through the C ABI (sam6d_b200/{sam,sam_amg,dinov2,ism}.py).  The geometric score needs the camera pose of
every template view: `templates/template_poses.npy` (42 x 4 x 4, written by render_point_templates; for BlenderProc renders pass the
reference's predefined level-0 poses with --template_poses); without it the final score is (semantic + appearance) / 2.

`--sam_model_type {vit_h,vit_l,vit_b}` picks the SAM backbone (the reference's hydra `model.segmentor_model.sam.model_type`,
default vit_h) and its checkpoint `{checkpoint_dir}/segment-anything/sam_vit_{h_4b8939,l_0b3195,b_01ec64}.pth` through
sam_amg.load_sam.

`--segmentor_model fastsam` (ISM_fastsam.yaml) replaces SAM by FastSAM (sam6d_b200/fast_sam.py: YOLOv8x-seg or YOLOv8s-seg, conf
0.25, iou 0.9, max_det 200) built from `{checkpoint_dir}/FastSAM/<--fastsam_model>.pt` or the reference's
`./checkpoints/FastSAM/<--fastsam_model>.pt` (`--fastsam_model {FastSAM-x,FastSAM-s}`, default FastSAM-x; the reference's hydra
`model.segmentor_model.checkpoint_path`); it needs only the DINOv2 checkpoint besides.  The rest of the pipeline and the output
files are the same.

`--dinov2_model {dinov2_vits14,dinov2_vitb14,dinov2_vitl14,dinov2_vitg14}` picks the descriptor backbone (the reference's hydra
`model.descriptor_model.model_name`, default dinov2_vitl14) and its checkpoint `{checkpoint_dir}/dinov2/<name>_pretrain.pth`.
dinov2_vitg14 is built with the SwiGLU FFN its published checkpoint holds (sam6d_b200/dinov2.py: FFN_OF_MODEL).

`--aggregation_function {mean,median,max,avg_5}` (the reference's matching_config, default avg_5) reduces each object's template
similarities to its semantic score.  `--level_templates {0,1,2}` and `--pose_distribution {all,upper}` (onboarding_config) pick
the ISM's views among templates rendered by render_custom_templates with the same two flags (render.template_view_set's
layout: the 42 level-0 views first); the defaults use every view in the directory, as before."""
import argparse
import glob
import json
import os
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

VISIBLE_THRED = 0.5            # ISM/configs/model/ISM_sam.yaml
CONFIDENCE_THRESH = 0.2
FASTSAM_MODELS = {"FastSAM-x": "x", "FastSAM-s": "s"}          # checkpoint name -> YOLOv8-seg scale


def get_parser():
    ap = argparse.ArgumentParser()
    ap.add_argument("--segmentor_model", default="sam", help="The segmentor model in ISM")
    ap.add_argument("--output_dir", nargs="?", help="Path to root directory of the output")
    ap.add_argument("--cad_path", nargs="?", help="Path to CAD(mm)")
    ap.add_argument("--rgb_path", nargs="?", help="Path to RGB image")
    ap.add_argument("--depth_path", nargs="?", help="Path to Depth image(mm)")
    ap.add_argument("--cam_path", nargs="?", help="Path to camera information")
    ap.add_argument("--stability_score_thresh", default=0.97, type=float, help="stability_score_thresh of SAM")
    # not in the reference: where weights / template poses come from
    ap.add_argument("--checkpoint_dir", default=None,
                    help="directory with segment-anything/sam_vit_h_4b8939.pth (or the --sam_model_type's file, or FastSAM/<--fastsam_model>.pt) "
                         "and dinov2/<--dinov2_model>_pretrain.pth")
    ap.add_argument("--sam_model_type", default="vit_h", choices=("vit_h", "vit_l", "vit_b"),
                    help="not in the reference: the hydra `model.segmentor_model.sam.model_type` (SAM backbone)")
    ap.add_argument("--fastsam_model", default="FastSAM-x", choices=FASTSAM_MODELS,
                    help="not in the reference: the FastSAM checkpoint of --segmentor_model fastsam (FastSAM-x: YOLOv8x-seg, FastSAM-s: YOLOv8s-seg)")
    ap.add_argument("--dinov2_model", default="dinov2_vitl14", choices=("dinov2_vits14", "dinov2_vitb14", "dinov2_vitl14", "dinov2_vitg14"),
                    help="not in the reference: the hydra `model.descriptor_model.model_name` (DINOv2 descriptor backbone)")
    ap.add_argument("--random_weights", action="store_true", help="seeded random weights when no checkpoints exist (plumbing runs)")
    ap.add_argument("--template_poses", default=None, help="(T,4,4) .npy of the template camera poses (default: templates/template_poses.npy)")
    ap.add_argument("--points_per_side", default=32, type=int)
    ap.add_argument("--pred_iou_thresh", default=0.88, type=float)
    ap.add_argument("--confidence_thresh", default=CONFIDENCE_THRESH, type=float, help="semantic-score threshold (ISM_sam.yaml: 0.2)")
    ap.add_argument("--aggregation_function", default="avg_5", choices=("mean", "median", "max", "avg_5"),
                    help="matching_config.aggregation_function: how an object's template similarities become its semantic score")
    ap.add_argument("--level_templates", default=0, type=int, choices=(0, 1, 2),
                    help="onboarding_config.level_templates: the ISM's views, 0 / 1 / 2 = 42 / 162 / 642")
    ap.add_argument("--pose_distribution", default="all", choices=("all", "upper"),
                    help="onboarding_config.pose_distribution: all, or upper (cameras with z >= 0)")
    return ap


def crop_resize_pad_images(images: torch.Tensor, boxes: torch.Tensor, target: int = 224) -> torch.Tensor:
    """CropResizePad (ISM/utils/bbox_utils.py:89-126) for per-item images (the 42 template views, once per object)"""
    sizes = boxes[:, 2:] - boxes[:, :2]
    scale = target / torch.max(sizes, dim=-1)[0]
    out = []
    for image, box, s in zip(images, boxes, scale):
        image = image[:, box[1]:box[3], box[0]:box[2]]
        image = F.interpolate(image.unsqueeze(0), scale_factor=s.item())[0]
        oh, ow = image.shape[1:]
        if 1.0 != ow / oh:
            pt, pl = max((target - oh) // 2, 0), max((target - ow) // 2, 0)
            image = F.pad(image, (pl, target - ow - pl, pt, target - oh - pt))
        image = F.interpolate(image.unsqueeze(0), scale_factor=target / image.shape[1])[0]
        out.append(image)
    return torch.stack(out)


def mask_to_rle(binary_mask: np.ndarray):
    """ISM/model/utils.py:25-43"""
    flat = np.asarray(binary_mask).ravel(order="F").astype(np.uint8)
    change = np.flatnonzero(np.diff(flat)) + 1
    counts = np.diff(np.concatenate([[0], change, [flat.size]])).tolist()
    if flat.size and flat[0] == 1:
        counts = [0] + counts
    return {"counts": counts, "size": list(binary_mask.shape)}


def _new_desc(args, device):
    from ..dinov2 import CustomDINOv2
    return CustomDINOv2(args.dinov2_model, "x_norm_clstoken", image_size=224, chunk_size=16, descriptor_width_size=640).to(device).eval()


def _dino_checkpoint(args):
    return os.path.join(args.checkpoint_dir, "dinov2", f"{args.dinov2_model}_pretrain.pth") if args.checkpoint_dir else None


def _seeded_dino_state_dict(vit):
    """seed-1 weights for the built backbone (the defaults are ViT-L/14's: the same draw as before the backbone was selectable)"""
    from .. import synth
    return synth.make_dinov2_state_dict(embed_dim=vit.embed_dim, depth=vit.depth, num_heads=vit.num_heads, seed=1, ffn_layer=vit.ffn_layer)


def build_fastsam(args, device):
    """FastSAM (ISM/configs/model/segmentor_model/fast_sam.yaml) + DINOv2"""
    from ..fast_sam import FastSAM
    desc = _new_desc(args, device)
    ck = args.checkpoint_dir
    name = getattr(args, "fastsam_model", "FastSAM-x")
    if name not in FASTSAM_MODELS:
        raise ValueError(f"fastsam_model must be one of {sorted(FASTSAM_MODELS)}, got {name!r}")
    scale = FASTSAM_MODELS[name]
    cands = ([os.path.join(ck, "FastSAM", name + ".pt")] if ck else []) + [os.path.join(".", "checkpoints", "FastSAM", name + ".pt")]
    fs_ck = next((c for c in cands if os.path.exists(c)), None)
    dino_ck = _dino_checkpoint(args)
    cfg = dict(iou_threshold=0.9, conf_threshold=0.05, max_det=200)
    if fs_ck and dino_ck and os.path.exists(dino_ck):
        seg = FastSAM(fs_ck, cfg, segmentor_width_size=640, device=device, scale=scale)
        desc.model.load_state_dict(torch.load(dino_ck, map_location="cpu"), strict=True)
    elif args.random_weights:
        from .. import synth
        print("=> WARNING: no checkpoints, seeded random weights (detections are meaningless; plumbing run)", file=sys.stderr)
        seg = FastSAM(None, cfg, segmentor_width_size=640, device=device, scale=scale)
        seg.model.load_state_dict(synth.make_fastsam_state_dict(seed=1, scale=scale), strict=True)
        desc.model.load_state_dict(_seeded_dino_state_dict(desc.model), strict=True)
    else:
        raise FileNotFoundError("FastSAM / DINOv2 checkpoints not found (pass --checkpoint_dir, or --random_weights for a plumbing run)")
    return seg, desc


def build_models(args, device):
    from ..sam import VIT_CONFIGS
    from ..sam_amg import CustomSamAutomaticMaskGenerator, load_sam, pretrained_weight_dict, sam_model_registry
    if args.segmentor_model == "fastsam":
        return build_fastsam(args, device)
    mt = args.sam_model_type

    def new_desc():            # built after SAM: module construction keeps drawing torch's global RNG in the same order
        return _new_desc(args, device)

    ck = args.checkpoint_dir
    sam_dir = os.path.join(ck, "segment-anything") if ck else None
    sam_ck = os.path.join(sam_dir, pretrained_weight_dict[mt]) if ck else None
    dino_ck = _dino_checkpoint(args)
    if sam_ck and os.path.exists(sam_ck) and os.path.exists(dino_ck):
        sam = load_sam(mt, sam_dir, "bf16").to(device).eval()
        desc = new_desc()
        desc.model.load_state_dict(torch.load(dino_ck, map_location="cpu"), strict=True)
    elif args.random_weights:
        from .. import synth
        print("=> WARNING: no checkpoints, seeded random weights (detections are meaningless; plumbing run)", file=sys.stderr)
        sam = sam_model_registry[mt]("bf16").to(device).eval()
        desc = new_desc()
        sd = {"image_encoder." + k: v for k, v in synth.make_sam_state_dict(**VIT_CONFIGS[mt], seed=1).items()}
        sd.update(synth.make_sam_decoder_state_dict(seed=1))
        sam.load_state_dict(sd, strict=True)
        desc.model.load_state_dict(_seeded_dino_state_dict(desc.model), strict=True)
    else:
        raise FileNotFoundError("SAM / DINOv2 checkpoints not found (pass --checkpoint_dir, or --random_weights for a plumbing run)")
    seg = CustomSamAutomaticMaskGenerator(sam, points_per_batch=64, stability_score_thresh=args.stability_score_thresh, box_nms_thresh=0.7,
                                          segmentor_width_size=640, pred_iou_thresh=args.pred_iou_thresh, points_per_side=args.points_per_side)
    return seg, desc


def ism_views(n_files: int, level_templates: int = 0, pose_distribution: str = "all") -> np.ndarray:
    """indices of the ISM's template files among the n_files views of a template directory: all of them for the default
    view set, else render.template_view_set(level_templates, pose_distribution)'s ISM views, whose layout the directory
    must have"""
    from .. import render
    if (level_templates, pose_distribution) == (0, "all"):
        return np.arange(n_files)
    union, index = render.template_view_set(level_templates, pose_distribution)
    if n_files != len(union):
        raise ValueError(f"--level_templates {level_templates} --pose_distribution {pose_distribution} needs the {len(union)} views "
                         f"render_custom_templates writes with the same flags; the template directory holds {n_files}")
    return index


def main(argv=None):
    args = get_parser().parse_args(argv)
    if args.segmentor_model not in ("sam", "fastsam"):
        raise ValueError(f"The segmentor_model {args.segmentor_model} is not supported")
    from PIL import Image
    from .. import meshio, pipeline
    device = torch.device("cuda")
    os.makedirs(f"{args.output_dir}/sam6d_results", exist_ok=True)
    t_start = time.time()
    seg, desc = build_models(args, device)
    # ---- templates (run_inference_custom.py:129-165) ---------------------------------------------------------------------
    tdir = os.path.join(args.output_dir, "templates")
    n_t = len(glob.glob(f"{tdir}/*.npy")) - int(os.path.exists(os.path.join(tdir, "template_poses.npy")))
    views = ism_views(n_t, args.level_templates, args.pose_distribution)
    rgbs = np.stack([np.array(Image.open(os.path.join(tdir, f"rgb_{i}.png")).convert("RGB")) for i in views])
    masks = np.stack([np.array(Image.open(os.path.join(tdir, f"mask_{i}.png")).convert("L")) for i in views])
    ref_cls, ref_patch = pipeline.ism_reference_features(desc, rgbs, masks, device)
    pose_path = args.template_poses or os.path.join(tdir, "template_poses.npy")
    geometry = None
    if os.path.exists(pose_path):
        cam = json.load(open(args.cam_path))
        verts, faces, _ = meshio.load_ply(args.cad_path)
        geometry = pipeline.ism_geometry(np.load(pose_path)[views], meshio.sample_surface(verts, faces, pipeline.N_ISM_CLOUD) / 1000.0,
                                         np.array(Image.open(args.depth_path)), cam["cam_K"], cam["depth_scale"], device)
    else:
        print("=> no template poses: final score = (semantic + appearance) / 2", file=sys.stderr)
    # ---- proposals + descriptors + scores (:167-209) ----------------------------------------------------------------------------
    rgb = np.array(Image.open(args.rgb_path).convert("RGB"))
    det = pipeline.ism_detect(seg, desc, ref_cls, ref_patch, rgb, args.confidence_thresh, geometry,
                              aggregation_function=args.aggregation_function)
    out_json = f"{args.output_dir}/sam6d_results/detection_ism.json"
    if det.reason is not None:
        json.dump([], open(out_json, "w"))
        print(f"=> {det.reason}")
        return 0
    # ---- BOP-23 records (ISM/model/utils.py:153-216) --------------------------------------------------------------------------
    results = pipeline.ism_records_from_masks(det, time.time() - t_start)
    b = det.boxes.cpu().numpy()
    np.savez(f"{args.output_dir}/sam6d_results/detection_ism.npz", scene_id=0, image_id=0, category_id=np.ones(len(b), dtype=np.int64),
             score=det.scores.cpu().numpy(), bbox=np.stack([b[:, 0], b[:, 1], b[:, 2] - b[:, 0], b[:, 3] - b[:, 1]], axis=1),
             time=results[0]["time"], segmentation=det.masks.cpu().numpy())
    json.dump(results, open(out_json, "w"))
    print(f"=> {len(results)} detections written to {out_json}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
