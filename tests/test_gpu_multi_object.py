"""GPU: SAM-6D on several objects per frame (SAM6D.onboard_objects / detect_objects).

- The NMS kernel with object ids (csrc/sam_dec.cu) against tests/golden/ism_multi.pt, index for index and in the reference's
  order; with one object it equals the single-category NMS.
- PEM input stage A with a radius threshold per detection against oracle/input_oracle.py.
- detect_objects on a three-mesh scene with seeded weights against the oracle composed from the stage functions.
- Each object's poses in the multi-object PEM batch against pem_frame on that object's detections alone.
- onboard_objects([m]) + detect_objects against a hand composition of test_step on the single-object stages."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "ism_multi.pt"), weights_only=False)


@pytest.mark.parametrize("tag", ["o3", "o8", "o8_two_used", "one"])
def test_nms_per_object_matches_reference(gold, tag):
    from sam6d_b200 import ism
    from sam6d_b200.sam_amg import CustomSamAutomaticMaskGenerator as SamAutomaticMaskGenerator
    c = gold["nms"][tag]
    keep = ism.nms_per_object(c["boxes"].cuda(), c["scores"].cuda(), c["object_ids"].cuda())
    assert torch.equal(keep.cpu(), c["keep"])
    if tag == "one":
        assert torch.equal(keep, SamAutomaticMaskGenerator.nms(c["boxes"].cuda(), c["scores"].cuda(), 0.25))
    # every box on one object: the single-category NMS
    zero = torch.zeros_like(c["object_ids"]).cuda()
    assert torch.equal(ism.nms_per_object(c["boxes"].cuda(), c["scores"].cuda(), zero),
                       SamAutomaticMaskGenerator.nms(c["boxes"].cuda(), c["scores"].cuda(), 0.25))


def test_nms_per_object_frames(gold):
    """the final NMS of the pinned multi-object frames, from the reference's own scores"""
    from oracle import ism_multi_oracle as imo
    from sam6d_b200 import ism
    for tag, c in gold["frames"].items():
        boxes = imo.make_multi_inputs(**c["kw"])["boxes"][c["idx_sel"]]
        keep = ism.nms_per_object(boxes.cuda(), c["score"].cuda(), c["pred_obj"].cuda())
        assert torch.equal(c["idx_sel"][keep.cpu()], c["final_index"]), tag


def test_stage_a_per_detection_radius(golden_dir):
    from oracle import input_oracle as io
    from sam6d_b200 import inputs
    g = torch.load(os.path.join(golden_dir, "pem_input.pt"), weights_only=False)
    rgb, depth = g["rgb"].numpy(), g["depth"].numpy().astype(np.uint16)
    dets = [d for d in g["dets"] if d["score"] > 0.2]
    radii = (np.float32(g["radius"]) * np.array([1.0, 0.3, 0.6, 2.0, 0.15, 1.3] * len(dets), dtype=np.float32))[:len(dets)]
    frame = inputs.FrameInputs(dets, rgb, depth, g["cam_K"], g["depth_scale"], radii)
    same = inputs.FrameInputs(dets, rgb, depth, g["cam_K"], g["depth_scale"], np.full(len(dets), np.float32(g["radius"])))
    scalar = inputs.FrameInputs(dets, rgb, depth, g["cam_K"], g["depth_scale"], g["radius"])
    # one radius for every detection, as an array or as a number: the same stage-A outputs.  choose2 / cloud2 are (P, cap)
    # scratch of which stage A writes the first n_valid rows of each detection; the rest is never initialised
    assert np.array_equal(same.stats_host, scalar.stats_host)
    for p, n in enumerate(scalar.n_valid().tolist()):
        assert torch.equal(same.choose2[p, :n], scalar.choose2[p, :n]) and torch.equal(same.cloud2[p, :n], scalar.cloud2[p, :n]), p
    K = np.array(g["cam_K"]).reshape(3, 3)
    whole_depth = depth.astype(np.float32) * g["depth_scale"] / 1000.0
    whole_pts = io.get_point_cloud_from_depth(whole_depth, K)
    n_changed = 0
    for p, d in enumerate(dets):
        ci = np.arange(2048) % 4
        r = io.build_instance(d["segmentation"], whole_depth, whole_pts, rgb, radii[p], 2048, 224, True, ci)
        nv = int(frame.n_valid()[p]) if p in frame.kept() else None
        assert (r is None) == (nv is None), p
        if r is None:
            continue
        assert nv == r["n_valid"] and frame.bbox()[p].tolist() == list(r["bbox"]), p
        pts = frame.sample(np.array([p]), ci[None], 224, True)[0]
        torch.testing.assert_close(pts[0].cpu(), torch.from_numpy(r["pts"]), atol=0, rtol=2e-7)
        n_changed += nv != int(scalar.n_valid()[p])
    assert n_changed >= 1, "the per-detection radii should change some filtered point counts"


# ---- whole frames ---------------------------------------------------------------------------------------------------------------
def _scene(golden_dir, tmp):
    """the example frame and three CADs: the convex hull of its object's samples at three scales (three radii)"""
    from scipy.spatial import ConvexHull
    from sam6d_b200 import meshio
    g = torch.load(os.path.join(golden_dir, "pem_input.pt"), weights_only=False)
    pts = g["model_points"].numpy().astype(np.float64) * 1000.0
    hull = ConvexHull(pts)
    remap = {v: i for i, v in enumerate(hull.vertices)}
    faces = np.array([[remap[a] for a in s] for s in hull.simplices], dtype=np.int64)
    cols = np.random.RandomState(0).randint(40, 255, (len(hull.vertices), 3)).astype(np.uint8)
    meshes = [meshio.Mesh(vertices=(pts[hull.vertices] * s).astype(np.float32), faces=faces, colors=cols) for s in (1.0, 0.7, 1.4)]
    frame = (g["rgb"].numpy().astype(np.uint8), g["depth"].numpy().astype(np.uint16), g["cam_K"], g["depth_scale"])
    return meshes, frame


_MODEL = {}


def _sam6d():
    from sam6d_b200.pipeline import SAM6D
    if "m" not in _MODEL:
        # FastSAM: with seeded weights it keeps its max_det proposals, where the seeded SAM's NMS leaves a single mask
        _MODEL["m"] = SAM6D(segmentor="fastsam", random_weights=True, confidence_thresh=-1, det_score_thresh=-1)
    return _MODEL["m"]


@pytest.fixture(scope="module")
def scene(golden_dir, tmp_path_factory):
    model = _sam6d()
    meshes, frame = _scene(golden_dir, str(tmp_path_factory.mktemp("scene")))
    objs = model.onboard_objects(meshes, obj_ids=[3, 7, 12], template_size=192, rng=np.random.RandomState(0))
    res = model.detect_objects(*frame, objs, rng=np.random.RandomState(5))
    return model, objs, frame, res


def test_detect_objects_against_oracle(scene):
    """the stages on the device (proposals, descriptors) feed the oracle's size filter, scores and per-object NMS.  The device
    computes the patch-token similarities in bf16 (dinov2.MaskedPatch_MatrixSimilarity), so the oracle gets the tokens rounded to
    bf16 and the final scores are held to 1e-5; the per-object NMS order is checked exactly on the device's scores."""
    from types import SimpleNamespace
    from oracle import ism_multi_oracle as imo
    from sam6d_b200.pipeline import ism_detect, ism_geometry
    model, objs, (rgb, depth, K, scale), res = scene
    assert res.reason is None and len(res.ism) >= 2
    d = model.seg.generate_masks(rgb)
    masks, boxes = d["masks"], d["boxes"].long()
    keep = torch.nonzero(imo.remove_very_small_detections(masks.cpu(), boxes.cpu())).flatten()
    sub = SimpleNamespace(masks=masks[keep.cuda()], boxes=boxes[keep.cuda()])
    q_cls, q_patch = model.desc(rgb, sub)
    bf = lambda x: x.cpu().bfloat16().float()                                   # noqa: E731
    s = imo.score_objects(q_cls.cpu(), objs.ref_cls.cpu(), bf(q_patch), bf(objs.ref_patch), sub.masks.cpu(),
                          torch.from_numpy(depth.astype(np.int32)), torch.tensor(np.array(K).reshape(3, 3)),
                          torch.tensor([float(scale)], dtype=torch.float64), sub.boxes.cpu(), torch.tensor(objs.poses_m).float(),
                          torch.from_numpy(objs.cloud_m).float(), confidence_thresh=-1)
    assert len(s["idx_sel"]) == len(keep)
    # detect_objects' ISM before its NMS: the same proposals, objects and (to bf16 rounding) scores as the oracle
    geometry = ism_geometry(objs.poses_m, objs.cloud_m, depth, K, scale, model.device)
    det = ism_detect(model.seg, model.desc, objs.ref_cls, objs.ref_patch, rgb, -1, geometry, remove_small=True)
    assert torch.equal(det.boxes.cpu(), sub.boxes.cpu()) and torch.equal(det.obj.cpu(), s["pred_obj"])
    torch.testing.assert_close(det.scores.cpu(), s["score"], atol=1e-5, rtol=0)
    order = imo.nms_per_object(det.boxes.cpu(), det.scores.cpu(), det.obj.cpu())
    print(f"detect_objects: {res.n_proposals} proposals, {len(keep)} after the size filter, {len(res.ism)} after NMS on objects "
          f"{sorted(set(s['pred_obj'].tolist()))}, {len(res.pem)} poses; max |score - oracle| "
          f"{float((det.scores.cpu() - s['score']).abs().max()):.2e}")
    assert len(order) < len(keep)
    assert torch.equal(res.obj.cpu(), det.obj.cpu()[order]) and torch.equal(res.boxes.cpu(), det.boxes.cpu()[order])
    assert torch.equal(res.scores.cpu(), det.scores.cpu()[order]) and torch.equal(res.masks, det.masks[order.cuda()])
    assert [r["category_id"] for r in res.ism] == [objs.obj_ids[o] for o in res.obj.tolist()]
    assert [r["category_id"] for r in res.pem] == [objs.obj_ids[o] for o in res.frame.obj.tolist()]
    assert res.R.shape == (len(res.pem), 3, 3)


def test_pem_rows_match_single_object_frames(scene):
    """every object's rows of the one multi-object Net.forward batch against pem_frame on that object's detections alone, with
    the same sample indices and coarse-stage uniforms: the rows of a batch do not depend on each other, so they are bit-equal"""
    from sam6d_b200.pipeline import pem_frame
    model, objs, (rgb, depth, K, scale), res = scene
    fr = res.frame
    assert fr.out is not None and len(set(fr.obj.tolist())) >= 2
    for o in sorted(set(fr.obj.tolist())):
        rows = np.flatnonzero(fr.obj == o)
        dets = [r for r in res.ism if r["category_id"] == objs.obj_ids[o]]
        bank = (objs.bank[0][o:o + 1], objs.bank[1][o:o + 1])
        alone = _pem_alone(model, bank, dets, rgb, depth, K, scale, objs.model_points_m[o], fr.choose_idx[rows], fr.rand[rows])
        for k in ("pred_R", "pred_t", "pred_pose_score"):
            assert torch.equal(fr.out[k][torch.from_numpy(rows).cuda()], alone[k]), (o, k)


def _pem_alone(model, bank, dets, rgb, depth, K, scale, model_points, choose_idx, rand):
    from sam6d_b200 import inputs
    from sam6d_b200.cli import pem_run_inference_custom as pem_cli
    cfg = pem_cli.TEST_DATASET
    data, _, _, _, kept = inputs.get_test_data([dict(d) for d in dets], rgb, depth, K, scale, model_points, model.det_score_thresh,
                                               cfg["n_sample_observed_point"], cfg["img_size"], cfg["rgb_mask_flag"], choose_idx=choose_idx)
    n = data["pts"].size(0)
    assert n == len(choose_idx)
    data["dense_po"], data["dense_fo"] = bank[0].repeat(n, 1, 1), bank[1].repeat(n, 1, 1)
    with torch.no_grad():
        return model.pem(data, rand=rand)


def test_one_object_against_test_step(golden_dir, tmp_path):
    """onboard_objects([m]) + detect_objects against test_step composed by hand from the single-object stages: proposals,
    size filter, descriptors, scores, NMS at 0.25; then the PEM frame of __call__ on the NMS survivors"""
    from types import SimpleNamespace
    from sam6d_b200 import ism, ops
    from sam6d_b200.pipeline import ism_detect, ism_geometry, ism_records, pem_frame, rle_counts
    from sam6d_b200.sam_amg import CustomSamAutomaticMaskGenerator as SamAutomaticMaskGenerator
    from sam6d_b200.cli import pem_run_inference_custom as pem_cli
    model = _sam6d()
    meshes, (rgb, depth, K, scale) = _scene(golden_dir, str(tmp_path))
    objs = model.onboard_objects(meshes[:1], template_size=192, rng=np.random.RandomState(0))
    res = model.detect_objects(rgb, depth, K, scale, objs, rng=np.random.RandomState(5))
    one = model.onboard(meshes[0], template_size=192, rng=np.random.RandomState(0))
    geometry = ism_geometry(one.poses_m, one.cloud_m, depth, K, scale, model.device)
    d = model.seg.generate_masks(rgb)
    small = ism.remove_very_small_detections(d["masks"], d["boxes"].long()).nonzero().flatten()

    class Seg:                                                      # the segmentor followed by the size filter
        def generate_masks(self, image):
            return {"masks": d["masks"][small], "boxes": d["boxes"][small]}
    det = ism_detect(Seg(), model.desc, one.ref_cls, one.ref_patch, rgb, model.confidence_thresh, geometry)
    keep = SamAutomaticMaskGenerator.nms(det.boxes, det.scores, 0.25)
    assert torch.equal(res.boxes, det.boxes[keep]) and torch.equal(res.scores, det.scores[keep])
    assert torch.equal(res.masks, det.masks[keep]) and res.obj.eq(0).all()
    cum, off = ops.mask_rle(det.masks[keep].contiguous())
    recs = ism_records(det.boxes[keep].cpu().numpy(), det.scores[keep].cpu().numpy(), rle_counts(cum.cpu().numpy(), off.cpu().numpy()),
                       det.masks.shape[1:], 0.0)
    strip = lambda rs: [{k: v for k, v in r.items() if k != "time"} for r in rs]   # noqa: E731
    assert strip(res.ism) == strip(recs)
    g = torch.Generator(device=model.device)
    g.manual_seed(pem_cli.RD_SEED)
    frame = pem_frame(model.pem, one.bank, recs, rgb, depth, K, scale, one.model_points_m[None], np.zeros(len(recs), np.int64),
                      model.det_score_thresh, rng=np.random.RandomState(5), generator=g, device=model.device)
    assert torch.equal(res.R, frame.out["pred_R"]) and torch.equal(res.t, frame.out["pred_t"])


def test_run_sam6d_several_cads(golden_dir, tmp_path):
    import cv2
    import json
    from sam6d_b200.cli import run_sam6d
    meshes, (rgb, depth, K, scale) = _scene(golden_dir, str(tmp_path))
    cads = []
    for i, m in enumerate(meshes[:2]):
        cads.append(str(tmp_path / f"obj{i}.ply"))
        with open(cads[-1], "w") as fh:
            fh.write("ply\nformat ascii 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\nproperty uchar red\n"
                     "property uchar green\nproperty uchar blue\nelement face %d\nproperty list uchar int vertex_indices\nend_header\n"
                     % (len(m.vertices), len(m.faces)))
            for v, c in zip(m.vertices, m.colors):
                fh.write("%f %f %f %d %d %d\n" % (v[0], v[1], v[2], c[0], c[1], c[2]))
            for f in m.faces:
                fh.write("3 %d %d %d\n" % tuple(f))
    cv2.imwrite(str(tmp_path / "rgb.png"), rgb[:, :, ::-1])
    cv2.imwrite(str(tmp_path / "depth.png"), depth)
    json.dump(dict(cam_K=K, depth_scale=scale), open(tmp_path / "camera.json", "w"))
    out = tmp_path / "out"
    assert run_sam6d.main(["--output_dir", str(out), "--cad_path", *cads, "--obj_ids", "4", "9", "--rgb_path", str(tmp_path / "rgb.png"),
                           "--depth_path", str(tmp_path / "depth.png"), "--cam_path", str(tmp_path / "camera.json"),
                           "--segmentor_model", "fastsam", "--random_weights", "--confidence_thresh", "-1", "--det_score_thresh", "-1",
                           "--template_size", "192"]) == 0
    r = out / "sam6d_results"
    ism_recs, pem_recs = json.load(open(r / "detection_ism.json")), json.load(open(r / "detection_pem.json"))
    cats = [x["category_id"] for x in ism_recs]
    print(f"run_sam6d with two CADs: {len(ism_recs)} ISM records (categories {sorted(set(cats))}), {len(pem_recs)} poses")
    assert ism_recs and set(cats) <= {4, 9} and cats == sorted(cats, key=[4, 9].index)
    assert pem_recs and {x["category_id"] for x in pem_recs} <= {4, 9} and (r / "vis_pem.png").exists()
