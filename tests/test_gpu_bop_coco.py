"""GPU: BOP detection / segmentation scoring (sam6d_b200/bop_eval_coco.py, csrc/bop_eval.cu) against numpy and the float64 oracle
(oracle/bop_coco_oracle.py) on a split built here (tests/_bop_coco_split.py): two scenes, image sizes 96 x 128 and 30 x 41
(1230 pixels, not a multiple of 32), overlapping procedural masks (one touching pixel (0,0), one covering the last pixel, an
empty visible mask, an empty full mask), visib_fract around 0.1, and detections that are RLEs of perturbed GT masks.

The kernels give integers, so they must equal numpy exactly, and evaluate_bop22_coco must reproduce the oracle's precision and
recall arrays exactly (the same float64 operations on the same integers), and its stats within 1e-12 (summation order)."""
import json

import numpy as np
import pytest
import torch

from oracle import bop_coco_oracle as bco
from sam6d_b200 import bop_eval_coco as bc
from sam6d_b200 import ops, pipeline
from sam6d_b200.cli import eval_bop_coco
from sam6d_b200.cli.ism_run_inference_custom import mask_to_rle

import _bop_coco_split as sp

pytestmark = pytest.mark.gpu


def np_pack(mask, words):
    flat = np.zeros(words * 32, bool)
    f = (np.asarray(mask) > 0).ravel(order="F")
    flat[:len(f)] = f
    return np.packbits(flat.reshape(-1, 8), axis=1, bitorder="little").reshape(-1).view("<u4")


def _masks(rng, H, W, n):
    m = (rng.rand(n, H, W) < rng.uniform(0.05, 0.95, (n, 1, 1))).astype(np.uint8) * rng.randint(1, 256, (n, H, W)).astype(np.uint8)
    m[0] = 0                                          # empty
    if n > 1:
        m[1] = 1                                      # full
    if n > 2:
        m[2] = 0
        m[2, 0, 0] = 200                              # pixel (0,0) only
    if n > 3:
        m[3] = 0
        m[3, H - 1, W - 1] = 3                        # the last pixel only
    return m


def test_pack_and_pair_kernels_match_numpy():
    rng = np.random.RandomState(0)
    shapes = [(30, 41, 7), (96, 128, 6), (1, 1, 3), (7, 33, 5), (480, 640, 4), (960, 1280, 2)]
    masks, woff, total = [], [], 0
    for H, W, n in shapes:
        m = _masks(rng, H, W, n)
        for i in range(n):
            masks.append(m[i])
            woff.append(total)
            total += bc.mask_words(H, W)
    # u8 copies at offsets 0.., RLE copies after them: every mask twice in one buffer, filled with a sentinel first, since both
    # kernels must write every word of a mask (the padding words after it are the caller's)
    bits = torch.full((2 * total,), -1, dtype=torch.int32, device="cuda")
    k = 0
    for H, W, n in shapes:
        ms = np.stack(masks[k:k + n])
        area, box = bc.pack_u8(torch.from_numpy(ms).cuda(), woff[k:k + n], bits)
        area2, box2 = bc.pack_u8(torch.from_numpy(ms).cuda())
        assert torch.equal(area, area2) and torch.equal(box, box2)
        for i in range(n):
            on = ms[i] > 0
            assert int(area[i]) == int(on.sum())
            ys, xs = np.nonzero(on)
            want = [xs.min(), ys.min(), xs.max(), ys.max()] if len(xs) else [-1] * 4
            assert box[i].tolist() == [int(v) for v in want], (H, W, i)
        k += n
    rles = [mask_to_rle(m > 0) for m in masks]
    cums = [np.cumsum(r["counts"]).astype(np.int32) for r in rles]
    rle_off = np.concatenate([[0], np.cumsum([len(c) for c in cums])]).astype(np.int32)
    bc.pack_rle(np.concatenate(cums), rle_off, [m.shape for m in masks], [total + w for w in woff], bits)
    host = bits.cpu().numpy().view(np.uint32)
    pad = []
    for i, m in enumerate(masks):
        nw, real = bc.mask_words(*m.shape), (m.size + 31) // 32
        want = np_pack(m, nw)[:real]
        np.testing.assert_array_equal(host[woff[i]:woff[i] + real], want, err_msg=f"pack_u8 {m.shape} {i}")
        np.testing.assert_array_equal(host[total + woff[i]:total + woff[i] + real], want, err_msg=f"pack_rle {m.shape} {i}")
        pad += [w + j for w in (woff[i], total + woff[i]) for j in range(real, nw)]
    assert (host[pad] == 0xFFFFFFFF).all()                     # padding is not written
    bits[torch.tensor(pad, dtype=torch.long, device="cuda")] = 0
    # pairs of one size, both copies; the padding words between masks are 0
    off = np.array(woff + [total + w for w in woff] + [2 * total], np.int64)
    size_of = [m.shape for m in masks] * 2
    pa, pb = [], []
    for a in range(2 * len(masks)):
        for b in range(2 * len(masks)):
            if size_of[a] == size_of[b] and rng.rand() < 0.7:
                pa.append(a)
                pb.append(b)
    cnt = bc.mask_pair_counts(bits, off, pa, pb).cpu().numpy()
    for j, (a, b) in enumerate(zip(pa, pb)):
        assert cnt[j] == int(((masks[a % len(masks)] > 0) & (masks[b % len(masks)] > 0)).sum()), (a, b)
    assert len(pa) > 100


@pytest.fixture(scope="module")
def split(tmp_path_factory):
    root = tmp_path_factory.mktemp("bop_coco")
    gts = sp.write_split(str(root))
    res = sp.write_json(root / "result_toy.json", sp.perturbed_detections(gts))
    return str(root), gts, res


def _compare(got, want):
    for k in ("n_images", "n_detections", "n_gt", "n_ignored_gt", "n_pairs", "obj_ids"):
        assert got[k] == want[k], (k, got[k], want[k])
    np.testing.assert_array_equal(np.array(got["precision"]), want["precision"])
    np.testing.assert_array_equal(np.array(got["recall"]), want["recall"])
    for k in bco.STAT_NAMES:
        assert abs(got[k] - want[k]) <= 1e-12, (k, got[k], want[k])
    for o, v in want["ap_per_object"].items():
        assert abs(got["ap_per_object"][o] - v) <= 1e-12


@pytest.mark.parametrize("iou_type,bbox_type", [("segm", "amodal"), ("bbox", "amodal"), ("bbox", "modal")])
def test_evaluate_matches_oracle(split, iou_type, bbox_type):
    root, gts, res = split
    got = bc.evaluate_bop22_coco(root, "toy", res, iou_type=iou_type, bbox_type=bbox_type)
    want = bco.evaluate(root, "toy", res, iou_type=iou_type, bbox_type=bbox_type)
    _compare(got, want)
    n_inst = sum(len(v) for v in gts.values())
    assert got["n_gt"] == n_inst - 1 - (bbox_type == "amodal")        # the empty visible mask; with amodal the empty full mask
    assert got["n_ignored_gt"] == 3 and got["obj_ids"] == [1, 2, 3]
    assert 0.0 < got["AP"] < 1.0 and 0.0 < got["AR100"] < 1.0 and got["AP_small"] > -1 and got["AP_large"] > -1
    print(f"[bop_coco] {iou_type}/{bbox_type}: " + " ".join(f"{k} {got[k]:.4f}" for k in bco.STAT_NAMES))


def test_tiny_budget_gives_identical_results(split, monkeypatch):
    root, _, res = split
    full = bc.evaluate_bop22_coco(root, "toy", res)
    monkeypatch.setattr(bc, "MASK_BUDGET_BYTES", 1)
    tiny = bc.evaluate_bop22_coco(root, "toy", res)
    assert json.dumps(full) == json.dumps(tiny)


def test_gt_masks_as_ism_records_score_one(split, tmp_path):
    """the GT masks written the way run_bop writes detections (ops.mask_rle on the device, pipeline.ism_records)"""
    root, gts, _ = split
    recs = []
    for (s, im), insts in gts.items():
        keep = [(o, vis) for o, vis, full, _ in insts if vis.any() and full.any()]
        m = torch.from_numpy(np.stack([v for _, v in keep]).astype(np.float32)).cuda()
        cum, off = ops.mask_rle(m)
        counts = pipeline.rle_counts(cum.cpu().numpy(), off.cpu().numpy())
        boxes = np.array([[b[0], b[1], b[0] + b[2], b[1] + b[3]] for b in (sp.box_xywh(v) for _, v in keep)])
        for r in pipeline.ism_records(boxes, np.linspace(0.9, 0.5, len(keep)), counts, m.shape[1:], 0.25, [o for o, _ in keep]):
            recs.append(dict(r, scene_id=s, image_id=im))
    got = bc.evaluate_bop22_coco(root, "toy", sp.write_json(tmp_path / "gt.json", recs))
    assert got["AP"] == pytest.approx(1.0, abs=1e-12) and got["AR100"] == 1.0
    assert got["n_detections"] == got["n_gt"]


def test_cli_writes_json(split, tmp_path, capsys):
    root, _, res = split
    out = tmp_path / "out"
    assert eval_bop_coco.main(["--bop_root", root, "--dataset_name", "toy", "--result_json", res, "--output_dir", str(out),
                               "--iou_type", "bbox", "--bbox_type", "modal"]) == 0
    saved = json.load(open(out / "scores_bop22_coco_bbox_toy.json"))
    want = bc.evaluate_bop22_coco(root, "toy", res, iou_type="bbox", bbox_type="modal")
    assert saved["AP"] == want["AP"] and saved["n_pairs"] == want["n_pairs"]
    assert np.array(saved["precision"]).shape == (10, 101, 3, 4, 3)
    assert "AR_large:" in capsys.readouterr().out
