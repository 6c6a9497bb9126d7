"""GPU: ISM references from a BOP PBR split on the synthetic split of tests/golden/ism_pbr.pt.

- sam6d_pbr_reference_crops: every box and crop of every row of the split bit-equal to the numpy oracle (tests/_pbr_oracle.py)
  and, on the stored references, to the reference's own BOPTemplatePBR, across chunk boundaries and with frames shared
  between references.
- SAM6D(rendering_type="pbr").onboard_objects: references equal compute_cls_and_patch_features on the oracle's crops; PEM bank,
  cloud, model points and geometric-score poses equal a "pyrender" onboarding drawn after the same selection.
- detect_objects on that ObjectSet against the hand composition of the stage functions; run_sam6d --rendering_type pbr."""
import json
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _pbr_oracle as po   # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "ism_pbr.pt"), weights_only=False)


@pytest.fixture(scope="module")
def root(gold, tmp_path_factory):
    return po.write_split(gold["files"], str(tmp_path_factory.mktemp("bop")))


def _keys(rows, index):
    return [(str(rows.scene_id[i]), int(rows.frame_id[i]), int(rows.idx_obj[i])) for i in index]


@pytest.mark.parametrize("max_rows,budget", [(256, 1 << 28), (5, 20000)])
def test_crops_match_oracle_and_reference(gold, root, max_rows, budget):
    """every row of the split (every mask kind, frame size and format); the small chunks put rows of one frame in different
    calls and leave several frames per call"""
    from sam6d_b200 import pbr
    rows = pbr.scan_rows(root)
    index = np.arange(len(rows))
    got, calls = {}, 0
    for where, boxes, rgb, pmask in pbr.iter_crops(rows, index, max_rows=max_rows, frame_budget_bytes=budget):
        calls += 1
        for j, k in enumerate(where.tolist()):
            frame, mask = pbr.decode_rgb(rows.rgb_path[k]), pbr.decode_mask(rows.mask_path(k))
            box, want_rgb, want_mask = po.reference_crop(frame, mask)
            assert boxes[j].tolist() == box.tolist(), k
            assert torch.equal(rgb[j].cpu(), want_rgb), k
            assert torch.equal(pmask[j].cpu(), want_mask), k
            got[k] = (rgb[j].cpu(), pmask[j].cpu())
    assert sorted(got) == index.tolist()
    assert calls >= (len(rows) + max_rows - 1) // max_rows
    where_key = {k: i for i, k in enumerate(_keys(rows, index))}
    for c in gold["levels"][0]["crops"]:
        rgb, pmask = got[where_key[tuple(c["key"])]]
        assert torch.equal(rgb, po.unpack(c["templates"])) and torch.equal(pmask, po.unpack(c["template_masks"])), c["key"]


def test_crops_shared_frame():
    """one frame, several references of it, in a call with other frames; masks of every value"""
    from sam6d_b200 import pbr
    rs = np.random.RandomState(3)
    frames = rs.randint(0, 256, (3, 37, 53, 3)).astype(np.uint8)
    masks = np.zeros((5, 37, 53), np.uint8)
    masks[0, 3:20, 0:9] = 255
    masks[1, 10:37, 40:53] = rs.randint(0, 256, (27, 13))
    masks[2, 0:1, 0:53] = 7                                                  # a one-pixel-high box
    masks[3] = rs.randint(0, 2, (37, 53)) * 255
    masks[4, 36, 52] = 1
    fidx = np.array([1, 1, 0, 2, 1], np.int32)
    boxes, rgb, pmask = pbr.crop_frames(torch.from_numpy(frames).cuda(), torch.from_numpy(fidx).cuda(), torch.from_numpy(masks).cuda())
    for r in range(5):
        box, want_rgb, want_mask = po.reference_crop(frames[fidx[r]], masks[r])
        assert boxes[r].tolist() == box.tolist() and torch.equal(rgb[r].cpu(), want_rgb) and torch.equal(pmask[r].cpu(), want_mask), r


# ---- onboarding and frames -----------------------------------------------------------------------------------------------------
_MODEL = {}


def _sam6d(root):
    from sam6d_b200.pipeline import SAM6D
    if "m" not in _MODEL:
        _MODEL["m"] = SAM6D(segmentor="fastsam", random_weights=True, confidence_thresh=-1, det_score_thresh=-1, rendering_type="pbr",
                            pbr_root=root)
    return _MODEL["m"]


def _scene(golden_dir):
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


@pytest.fixture(scope="module")
def onboarded(root, golden_dir):
    model = _sam6d(root)
    meshes, frame = _scene(golden_dir)
    objs = model.onboard_objects(meshes, obj_ids=[1, 2, 5], template_size=192, rng=np.random.RandomState(0))
    return model, meshes, frame, objs


def test_onboard_objects_pbr_references(onboarded):
    from sam6d_b200 import pbr, render
    model, _, _, objs = onboarded
    rows = model._pbr_rows
    union, index = render.template_view_set(0, "all")
    sel = pbr.select_references(rows, [1, 2, 5], union[index], np.random.RandomState(0))
    crops = [po.reference_crop(pbr.decode_rgb(rows.rgb_path[k]), pbr.decode_mask(rows.mask_path(k))) for k in sel.reshape(-1)]
    rgb = torch.stack([c[1] for c in crops]).cuda()
    mask = torch.stack([c[2] for c in crops]).cuda()
    cls, patch = model.desc.compute_cls_and_patch_features(rgb, mask)
    O, T = sel.shape
    assert objs.ref_cls.shape == (O, T, cls.shape[-1]) and objs.ref_patch.shape == (O, T) + tuple(patch.shape[1:])
    d_cls = (objs.ref_cls.reshape(O * T, -1) - cls).abs().max().item()
    d_patch = (objs.ref_patch.reshape(O * T, *patch.shape[1:]) - patch).abs().max().item()
    print(f"pbr references: {len(np.unique(sel))} distinct rows for {O * T} templates; max |diff| cls {d_cls:.2e} patch {d_patch:.2e}")
    # the descriptors of a row do not depend on the other images of its batch up to the last bits of the GEMM tiling
    assert d_cls <= 1e-5 and d_patch <= 1e-5


def test_onboard_objects_pbr_mesh_parts(onboarded):
    """the PEM bank, cloud, model points and poses of the pbr onboarding equal a pyrender onboarding drawn after the selection"""
    from sam6d_b200 import pbr, render
    model, meshes, _, objs = onboarded
    rng = np.random.RandomState(0)
    union, index = render.template_view_set(0, "all")
    pbr.select_references(model._pbr_rows, [1, 2, 5], union[index], rng)
    model.rendering_type = "pyrender"
    try:
        pyr = model.onboard_objects(meshes, obj_ids=[1, 2, 5], template_size=192, rng=rng)
    finally:
        model.rendering_type = "pbr"
    assert np.array_equal(objs.cloud_m, pyr.cloud_m) and np.array_equal(objs.model_points_m, pyr.model_points_m)
    assert np.array_equal(objs.poses_m, pyr.poses_m) and np.array_equal(objs.radii, pyr.radii) and objs.obj_ids == pyr.obj_ids
    assert torch.equal(objs.bank[0], pyr.bank[0]) and torch.equal(objs.bank[1], pyr.bank[1])


def test_detect_objects_with_pbr_references(onboarded):
    from sam6d_b200 import ism
    from sam6d_b200.pipeline import ism_detect, ism_geometry
    model, _, (rgb, depth, K, scale), objs = onboarded
    res = model.detect_objects(rgb, depth, K, scale, objs, rng=np.random.RandomState(5))
    geometry = ism_geometry(objs.poses_m, objs.cloud_m, depth, K, scale, model.device)
    det = ism_detect(model.seg, model.desc, objs.ref_cls, objs.ref_patch, rgb, model.confidence_thresh, geometry, remove_small=True)
    keep = ism.nms_per_object(det.boxes, det.scores, det.obj)
    assert res.reason is None and len(res.ism) == len(keep) >= 1
    assert torch.equal(res.boxes, det.boxes[keep]) and torch.equal(res.scores, det.scores[keep]) and torch.equal(res.obj, det.obj[keep])
    assert [r["category_id"] for r in res.ism] == [objs.obj_ids[o] for o in res.obj.tolist()]
    print(f"detect_objects with pbr references: {res.n_proposals} proposals, {len(res.ism)} detections, {len(res.pem)} poses")


def test_run_sam6d_pbr(root, golden_dir, tmp_path):
    import cv2
    from sam6d_b200.cli import run_sam6d
    meshes, (rgb, depth, K, scale) = _scene(golden_dir)
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
    assert run_sam6d.main(["--output_dir", str(out), "--cad_path", *cads, "--obj_ids", "2", "5", "--rgb_path", str(tmp_path / "rgb.png"),
                           "--depth_path", str(tmp_path / "depth.png"), "--cam_path", str(tmp_path / "camera.json"),
                           "--segmentor_model", "fastsam", "--random_weights", "--confidence_thresh", "-1", "--det_score_thresh", "-1",
                           "--template_size", "192", "--rendering_type", "pbr", "--pbr_root", root]) == 0
    r = out / "sam6d_results"
    ism_recs, pem_recs = json.load(open(r / "detection_ism.json")), json.load(open(r / "detection_pem.json"))
    print(f"run_sam6d --rendering_type pbr: {len(ism_recs)} ISM records, {len(pem_recs)} poses")
    assert ism_recs and {x["category_id"] for x in ism_recs} <= {2, 5} and pem_recs
