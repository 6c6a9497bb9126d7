"""No GPU: the host logic of the one-process pipeline (sam6d_b200/pipeline.py, sam6d_b200/cli/run_sam6d.py) -- records from
RLE run ends, and the run_sam6d arguments."""
import numpy as np
import pytest


def _run_ends(mask):
    """the definition the mask_rle kernel implements: column-major positions k where the pixel differs from position k-1
    (k = 0 when pixel (0,0) is set), then H*W"""
    flat = (np.asarray(mask) > 0).ravel(order="F").astype(np.int8)
    prev = np.concatenate([[0], flat[:-1]])
    return np.concatenate([np.flatnonzero(flat != prev), [flat.size]]).astype(np.int32)


def _masks():
    rs = np.random.RandomState(0)
    H, W = 23, 31
    ms = [np.zeros((H, W)), np.ones((H, W)), rs.rand(H, W) - 0.5, (np.indices((H, W)).sum(0) % 2).astype(np.float64)]
    one = np.zeros((H, W))
    one[0, 0] = 1
    ms.append(one)
    last = np.zeros((H, W))
    last[-1, -1] = 1
    ms.append(last)
    blob = np.zeros((H, W))
    blob[5:12, 3:20] = 1
    ms.append(blob)
    ms.append(np.array([[np.nan, -0.0], [1e-30, -2.0]]))
    return ms


def test_run_ends_definition_matches_mask_to_rle_and_pack_rle():
    from sam6d_b200 import inputs
    from sam6d_b200.cli.ism_run_inference_custom import mask_to_rle
    from sam6d_b200.pipeline import rle_counts
    for m in _masks():
        ref = mask_to_rle(m > 0)
        cum, off = inputs.pack_rle([{"segmentation": ref}], *m.shape)
        ends = _run_ends(m)
        assert np.array_equal(ends, cum) and off.tolist() == [0, len(ends)]
        assert rle_counts(ends, off) == [ref["counts"]]


def test_records_from_run_ends():
    from sam6d_b200.cli.ism_run_inference_custom import mask_to_rle
    from sam6d_b200.pipeline import ism_records, rle_counts
    ms = [m for m in _masks() if m.shape == (23, 31)]
    ends = [_run_ends(m) for m in ms]
    off = np.concatenate([[0], np.cumsum([len(e) for e in ends])]).astype(np.int32)
    counts = rle_counts(np.concatenate(ends), off)
    boxes = np.array([[1, 2, 11, 22]] * len(ms), dtype=np.int64)
    scores = np.linspace(0.1, 0.9, len(ms)).astype(np.float32)
    recs = ism_records(boxes, scores, counts, (23, 31), 0.5)
    for r, m, s in zip(recs, ms, scores):
        assert r == dict(scene_id=0, image_id=0, category_id=1, bbox=[1, 2, 10, 20], score=float(s), time=0.5,
                         segmentation=mask_to_rle(m > 0))
        assert all(type(c) is int for c in r["segmentation"]["counts"]) and type(r["bbox"][0]) is int


def test_run_sam6d_arguments():
    from sam6d_b200.cli import ism_run_inference_custom as ism_cli, pem_run_inference_custom as pem_cli, run_sam6d
    req = ["--cad_path", "o.ply", "--rgb_path", "r.png", "--depth_path", "d.png", "--cam_path", "c.json", "--output_dir", "out"]
    a = run_sam6d.get_parser().parse_args(req)
    ism_d = ism_cli.get_parser().parse_args([])
    pem_d = pem_cli.get_parser().parse_args([])
    for k in ("segmentor_model", "stability_score_thresh", "checkpoint_dir", "sam_model_type", "dinov2_model", "points_per_side",
              "pred_iou_thresh", "confidence_thresh", "random_weights"):
        assert getattr(a, k) == getattr(ism_d, k), k
    for k in ("det_score_thresh", "checkpoint", "precision"):
        assert getattr(a, k) == getattr(pem_d, k), k
    assert a.template_size == 512 and a.output_dir == "out" and a.cad_path == "o.ply"
    a = run_sam6d.get_parser().parse_args(req + ["--segmentor_model", "fastsam", "--sam_model_type", "vit_b", "--template_size", "192",
                                                 "--precision", "fp32", "--random_weights", "--det_score_thresh", "-1"])
    assert (a.segmentor_model, a.sam_model_type, a.template_size, a.precision, a.random_weights, a.det_score_thresh) == \
        ("fastsam", "vit_b", 192, "fp32", True, -1.0)
    for bad in (["--segmentor_model", "mobile_sam"], ["--sam_model_type", "vit_x"], ["--precision", "fp16"]):
        with pytest.raises(SystemExit):
            run_sam6d.get_parser().parse_args(req + bad)
    with pytest.raises(SystemExit):
        run_sam6d.get_parser().parse_args(req[2:])                        # --cad_path is required
