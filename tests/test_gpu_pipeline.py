"""GPU: SAM-6D in one process (sam6d_b200/pipeline.py) and the mask -> RLE kernel behind its ISM -> PEM hand-off
(csrc/mask_rle.cu).

- ops.mask_rle against the ISM CLI's numpy mask_to_rle and inputs.pack_rle, exactly, on blob masks and edge cases.
- SAM6D.onboard + one frame against the chained CLIs (render_custom_templates -> ISM CLI -> PEM CLI) on the repository's
  example frame, for SAM ViT-B and FastSAM with seeded weights: both JSON files must be equal field by field except `time`.
  The one-process CLI (python -m sam6d_b200.cli.run_sam6d) is compared the same way.
- A resident SAM6D gives the same result for a frame before and after another frame."""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

H0, W0 = 480, 640


# ---- RLE kernel ----------------------------------------------------------------------------------------------------------------
def _blobs(n, H, W, seed):
    """n masks of 1-4 random ellipses each, 0/1 float32 (what the segmentors return)"""
    g = torch.Generator().manual_seed(seed)
    ys, xs = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing="ij")
    out = torch.zeros(n, H, W)
    for i in range(n):
        for _ in range(int(torch.randint(1, 5, (1,), generator=g))):
            cy, cx = float(torch.rand(1, generator=g)) * H, float(torch.rand(1, generator=g)) * W
            ry, rx = 2 + float(torch.rand(1, generator=g)) * H / 3, 2 + float(torch.rand(1, generator=g)) * W / 3
            out[i] = torch.maximum(out[i], (((ys - cy) / ry) ** 2 + ((xs - cx) / rx) ** 2 <= 1).float())
    return out


def _check_rle(masks_cpu):
    from sam6d_b200 import inputs, ops
    from sam6d_b200.cli.ism_run_inference_custom import mask_to_rle
    from sam6d_b200.pipeline import rle_counts
    n, H, W = masks_cpu.shape
    cum, off = ops.mask_rle(masks_cpu.cuda().contiguous())
    torch.cuda.synchronize()
    cum, off = cum.cpu().numpy(), off.cpu().numpy()
    m = masks_cpu.numpy()
    recs = [{"segmentation": mask_to_rle(m[i] > 0)} for i in range(n)]
    ref_cum, ref_off = inputs.pack_rle(recs, H, W)
    assert off.dtype == np.int32 and cum.dtype == np.int32
    assert np.array_equal(off, ref_off), "offsets differ from pack_rle"
    assert np.array_equal(cum, ref_cum), "run ends differ from pack_rle"
    assert rle_counts(cum, off) == [r["segmentation"]["counts"] for r in recs]
    return cum, off


@pytest.mark.parametrize("n", [1, 200])
def test_mask_rle_blobs(n):
    _check_rle(_blobs(n, H0, W0, seed=n))


def test_mask_rle_odd_size():
    _check_rle(_blobs(7, 37, 53, seed=3))


def test_mask_rle_edge_cases():
    H, W = 37, 53
    m = torch.zeros(8, H, W)
    m[1] = 1.0                                               # all one: counts [0, H*W]
    m[2, 0, 0] = 1.0                                         # only the first position
    m[3, H - 1, W - 1] = 1.0                                 # only the last position
    m[4, :, 0] = 1.0                                         # a full first column: counts [0, H, H*W - H]
    m[5] = ((torch.arange(H)[:, None] + torch.arange(W)[None, :]) % 2).float()             # checkerboard, (1,1) set
    m[6] = 1.0 - m[5]                                        # checkerboard, (0,0) set
    cum, off = _check_rle(m)
    assert np.diff(off).tolist() == [1, 2, 3, 2, 3, H * W, H * W + 1, 1]
    _check_rle(_blobs(3, 32, 64, seed=9))                    # W a multiple of the band width


def test_mask_rle_special_values():
    """set iff value > 0: NaN, -0.0 and negatives are unset, 1e-30 is set"""
    vals = torch.tensor([float("nan"), -0.0, 0.0, -1.0, -1e-30, 1e-30, 1.0, 3.5, float("inf"), float("-inf")])
    g = torch.Generator().manual_seed(0)
    m = vals[torch.randint(0, len(vals), (4, 41, 67), generator=g)]
    _check_rle(m)
    cum, off = _check_rle(torch.full((1, 5, 6), 1e-30))
    assert cum.tolist() == [0, 30]
    cum, off = _check_rle(torch.full((1, 5, 6), -0.0))
    assert cum.tolist() == [30]


def test_mask_rle_empty():
    from sam6d_b200 import ops
    cum, off = ops.mask_rle(torch.zeros(0, H0, W0, device="cuda"))
    assert cum.numel() == 0 and off.cpu().tolist() == [0]


# ---- the whole pipeline against the chained CLIs ----------------------------------------------------------------------------
def _write_ply(path, verts_mm, faces, colors):
    with open(path, "w") as fh:
        fh.write("ply\nformat ascii 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n"
                 "property uchar red\nproperty uchar green\nproperty uchar blue\nelement face %d\nproperty list uchar int vertex_indices\nend_header\n"
                 % (len(verts_mm), len(faces)))
        for v, c in zip(verts_mm, colors):
            fh.write("%f %f %f %d %d %d\n" % (v[0], v[1], v[2], c[0], c[1], c[2]))
        for f in faces:
            fh.write("3 %d %d %d\n" % tuple(f))


def _example(out, golden_dir):
    """the example frame of tests/golden/pem_input.pt and the convex hull of its object's samples as the CAD (as in test_gpu_cli)"""
    import cv2
    from scipy.spatial import ConvexHull
    gold = torch.load(os.path.join(golden_dir, "pem_input.pt"), weights_only=False)
    cv2.imwrite(os.path.join(out, "rgb.png"), gold["rgb"].numpy()[:, :, ::-1])
    cv2.imwrite(os.path.join(out, "depth.png"), gold["depth"].numpy().astype(np.uint16))
    json.dump(dict(cam_K=gold["cam_K"], depth_scale=gold["depth_scale"]), open(os.path.join(out, "camera.json"), "w"))
    pts_mm = gold["model_points"].numpy().astype(np.float64) * 1000.0
    hull = ConvexHull(pts_mm)
    remap = {v: i for i, v in enumerate(hull.vertices)}
    cad = os.path.join(out, "obj.ply")
    _write_ply(cad, pts_mm[hull.vertices], np.array([[remap[a] for a in s] for s in hull.simplices]),
               np.random.RandomState(0).randint(40, 255, (len(hull.vertices), 3)))
    common = ["--cad_path", cad, "--rgb_path", os.path.join(out, "rgb.png"), "--depth_path", os.path.join(out, "depth.png"),
              "--cam_path", os.path.join(out, "camera.json")]
    return gold, cad, common


# the permissive thresholds of test_gpu_cli.test_ism_cli_then_pem_cli: seeded weights give low scores, and every proposal
# should reach the PEM
CONFIGS = {
    "sam": dict(ism=["--sam_model_type", "vit_b", "--stability_score_thresh", "0.0", "--pred_iou_thresh", "-10", "--points_per_side", "8"],
                kw=dict(segmentor="sam", sam_model_type="vit_b", stability_score_thresh=0.0, pred_iou_thresh=-10, points_per_side=8)),
    "fastsam": dict(ism=["--segmentor_model", "fastsam"], kw=dict(segmentor="fastsam")),
}


def _strip_time(records):
    return [{k: v for k, v in r.items() if k != "time"} for r in records]


def _same_records(a, b, what):
    a, b = _strip_time(a), _strip_time(b)
    assert len(a) == len(b), f"{what}: {len(a)} vs {len(b)} records"
    for i, (x, y) in enumerate(zip(a, b)):
        assert x.keys() == y.keys(), (what, i)
        for k in x:
            assert x[k] == y[k], f"{what}: record {i} field {k} differs"


def _chain(out, cad, common, cfg):
    from sam6d_b200.cli import ism_run_inference_custom as ism_cli, pem_run_inference_custom as pem_cli, render_custom_templates as rct
    rct.main(["--cad_path", cad, "--output_dir", out, "--size", "192"])
    args = ["--output_dir", out] + common
    np.random.seed(0)
    assert ism_cli.main(args + cfg["ism"] + ["--random_weights", "--confidence_thresh", "-1"]) == 0
    assert pem_cli.main(args + ["--seg_path", os.path.join(out, "sam6d_results", "detection_ism.json"), "--random_weights",
                                "--det_score_thresh", "-1"]) == 0
    res = os.path.join(out, "sam6d_results")
    return json.load(open(os.path.join(res, "detection_ism.json"))), json.load(open(os.path.join(res, "detection_pem.json")))


_MODELS = {}


def _sam6d(seg):
    from sam6d_b200.pipeline import SAM6D
    if seg not in _MODELS:
        _MODELS[seg] = SAM6D(**CONFIGS[seg]["kw"], random_weights=True, confidence_thresh=-1, det_score_thresh=-1)
    return _MODELS[seg]


def _frame_inputs(gold):
    return gold["rgb"].numpy().astype(np.uint8), gold["depth"].numpy().astype(np.uint16), gold["cam_K"], gold["depth_scale"]


@pytest.mark.parametrize("seg", ["sam", "fastsam"])
def test_pipeline_matches_chained_clis(tmp_path, golden_dir, seg):
    out = str(tmp_path)
    gold, cad, common = _example(out, golden_dir)
    ism_ref, pem_ref = _chain(out, cad, common, CONFIGS[seg])
    print(f"{seg}: chained CLIs {len(ism_ref)} ISM / {len(pem_ref)} PEM records")
    assert len(ism_ref) >= 1 and len(pem_ref) >= 1
    model = _sam6d(seg)
    rng = np.random.RandomState(0)
    obj = model.onboard(cad, template_size=192, rng=rng)
    res = model(*_frame_inputs(gold), obj, rng=rng)
    # records as they would be read back from the JSON files (json round-trips Python floats and ints exactly)
    _same_records(ism_ref, json.loads(json.dumps(res.ism)), f"{seg} ISM")
    _same_records(pem_ref, json.loads(json.dumps(res.pem)), f"{seg} PEM")
    assert res.masks.shape[0] == len(ism_ref) and res.R.shape == (len(pem_ref), 3, 3)
    if seg == "sam":
        from sam6d_b200.cli import run_sam6d
        one = os.path.join(out, "one")
        np.random.seed(0)
        assert run_sam6d.main(["--output_dir", one] + common + CONFIGS[seg]["ism"] +
                              ["--random_weights", "--confidence_thresh", "-1", "--det_score_thresh", "-1", "--template_size", "192"]) == 0
        r = os.path.join(one, "sam6d_results")
        _same_records(ism_ref, json.load(open(os.path.join(r, "detection_ism.json"))), "run_sam6d ISM")
        _same_records(pem_ref, json.load(open(os.path.join(r, "detection_pem.json"))), "run_sam6d PEM")
        assert os.path.exists(os.path.join(r, "vis_pem.png"))
        assert not os.path.exists(os.path.join(one, "templates")) and not os.path.exists(os.path.join(r, "detection_ism.npz"))


def test_resident_state(tmp_path, golden_dir):
    """frame A, frame B, frame A through one SAM6D (each with a fresh RandomState(5)): both A results are identical"""
    gold, cad, _ = _example(str(tmp_path), golden_dir)
    model = _sam6d("sam")
    obj = model.onboard(cad, template_size=192, rng=np.random.RandomState(0))
    rgb, depth, K, scale = _frame_inputs(gold)
    noise = np.random.RandomState(1).randint(-25, 26, rgb.shape)
    rgb_b = np.ascontiguousarray(np.clip(rgb[:, ::-1].astype(np.int64) + noise, 0, 255).astype(np.uint8))
    depth_b = np.ascontiguousarray(depth[:, ::-1])
    a1 = model(rgb, depth, K, scale, obj, rng=np.random.RandomState(5))
    b = model(rgb_b, depth_b, K, scale, obj, rng=np.random.RandomState(5))
    a2 = model(rgb, depth, K, scale, obj, rng=np.random.RandomState(5))
    print(f"frame A: {len(a1.ism)} / {len(a1.pem)} records, frame B: {len(b.ism)} / {len(b.pem)}")
    assert len(a1.pem) >= 1
    assert _strip_time(a1.ism) != _strip_time(b.ism)
    _same_records(a1.ism, a2.ism, "A ISM")
    _same_records(a1.pem, a2.pem, "A PEM")
    for k in ("masks", "boxes", "scores", "R", "t"):
        assert torch.equal(getattr(a1, k), getattr(a2, k)), k
