"""BOP detection / segmentation scoring (the BOP Challenge 2022 2D tasks) of an ISM result JSON against a BOP test split: COCO
average precision and recall as the BOP toolkit's eval_bop22_coco.py computes them through pycocotools' COCOeval.

    scores = evaluate_bop22_coco(bop_root, "ycbv", "out/result_ycbv.json")           # iou_type "segm"; or "bbox"
    scores["AP"], scores["AR100"], scores["ap_per_object"]

Definition (pycocotools' COCOeval.evaluate / accumulate / summarize with BOP's ground truth):

* images: the distinct (scene_id, im_id) of the targets file (default <dataset>/test_targets_bop19.json), in sorted order;
  detections on other images are dropped;
* GT instances: every instance of scene_gt.json of a target image, in file order (pbr.scan_rows on bop.split_name's split).  The
  visible mask is mask_visib/<im>_<idx>.png, set where > 0; an instance whose visible mask is empty is dropped, and with
  bbox_type "amodal" also one whose full mask mask/<im>_<idx>.png is empty.  area = the visible mask's pixel count (both iou
  types); box [x_min, y_min, x_max - x_min + 1, y_max - y_min + 1] of the full mask ("amodal", the toolkit's default) or the
  visible mask ("modal"); ignore = visib_fract < 0.1;
* categories: obj_id, sorted; the K categories are those of the kept GT instances.  Only (category, area range) cells with a GT
  instance that is not ignored count toward a mean; detections of other categories change no number;
* detections: within each (image, category) sorted by score, descending, stably (ties keep file order), and cut to the first
  MAX_DETS = 100.  segm: the mask of the record's uncompressed COCO RLE, area = its pixel count; bbox: the record's bbox
  (x, y, w, h floats), area = w h;
* IoU: segm |D & G| / (|D| + |G| - |D & G|) from integer counts, divided in float64; bbox pycocotools' bbIou: w = min(dx + dw,
  gx + gw) - max(dx, gx), h likewise, 0 when either is <= 0, then i / (dw dh + gw gh - i);
* matching, per (image, category, area range all [0, 1e10] / small [0, 32^2] / medium [32^2, 96^2] / large [96^2, 1e10]) and per
  IoU threshold t of linspace(0.5, 0.95, 10): a GT is ignored in the cell when it has ignore set or its area is outside the range
  (bounds inclusive); GT instances are ordered non-ignored first, stably; detections in score order each scan the unmatched GT
  instances, skip one whose IoU is below the running best (which starts at min(t, 1 - 1e-10)), else take it and raise the best
  to its IoU (so a tie goes to the later GT), and stop at the first ignored GT once they hold a non-ignored one.  A detection
  matched to an ignored GT is ignored, and so is an unmatched one whose area is outside the range.  Matching with 100
  detections and keeping the first maxDet of them is the same as matching with maxDet, since a match depends only on the
  detections before it;
* accumulation, per (threshold, category, area range, maxDet in 1 / 10 / 100) over the images in order: the first maxDet
  detections of each image merged by a stable descending sort of their scores; tp, fp running sums (ignored detections add to
  neither); rc = tp / n_non_ignored_gt, pr = tp / (tp + fp + np.spacing(1)), made non-increasing from the right; precision at
  the recall thresholds linspace(0, 1, 101) = pr at searchsorted(rc, r, "left"), 0 past the end; recall = the last rc, 0 with
  no detection; -1 in both for a cell without a non-ignored GT;
* stats: AP, AP50, AP75, AP_small, AP_medium, AP_large, AR1, AR10, AR100, AR_small, AR_medium, AR_large, each the mean of the
  cells > -1 (-1 when none), area "all" and maxDet 100 unless the name says otherwise; ap_per_object: AP of one category.

BOP's rule that a GT instance with visib_fract < 0.1 is ignored is applied as pycocotools' per-instance ignore flag: a detection
matched to such an instance is neither a true nor a false positive.

The per-pair work runs on the GPU (csrc/bop_eval.cu): GT masks are decoded on the host and bit-packed with their areas and
boxes by sam6d_bop_pack_u8, the detections that share an (image, category) with a kept GT instance are bit-packed from their run
ends by sam6d_bop_pack_rle, and sam6d_bop_mask_pair_counts counts |D & G| of every such pair.  The area of every detection is
the sum of its odd runs, on the host.  Images go through in chunks whose packed masks and staged u8 GT masks stay within
MASK_BUDGET_BYTES.  Matching (match) and accumulation (accumulate, summarize) are vectorised numpy on the host."""
import json
import math
import os
import sys
import time
from collections import OrderedDict

import numpy as np
import torch

from . import _lib, bop, pbr
from .bop_eval import _image_size, load_targets
from .pbr import _tick

IOU_TYPES = ("segm", "bbox")
BBOX_TYPES = ("amodal", "modal")
IOU_THRS = np.linspace(0.5, 0.95, int(np.round((0.95 - 0.5) / 0.05)) + 1)
REC_THRS = np.linspace(0.0, 1.00, int(np.round((1.00 - 0.0) / 0.01)) + 1)
AREA_NAMES = ("all", "small", "medium", "large")
AREA_RNGS = np.array([[0, 1e5 ** 2], [0, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]], np.float64)
MAX_DETS = (1, 10, 100)
MIN_VISIB_FRACT = 0.1
STAT_NAMES = ("AP", "AP50", "AP75", "AP_small", "AP_medium", "AP_large", "AR1", "AR10", "AR100", "AR_small", "AR_medium", "AR_large")
# packed masks of a chunk of images, plus the u8 GT masks staged for packing, stay within this many bytes on the device
MASK_BUDGET_BYTES = 1 << 30


# ---- readers -----------------------------------------------------------------------------------------------------------------
def load_detections(path: str):
    """an ISM result JSON (a list of records scene_id, image_id, category_id, score, bbox [x, y, w, h], segmentation {"counts":
    uncompressed run lengths, "size": [h, w]}; time is not read) -> dict of scene_id, im_id, obj_id (n,) i64, score (n,) f64,
    bbox (n,4) f64, size (n,2) i64 and counts (list of (m,) i64 run lengths), in file order.  A malformed record raises a
    ValueError naming its index; compressed RLE strings raise NotImplementedError"""
    with open(path) as fh:
        data = json.load(fh)
    if not isinstance(data, list):
        raise ValueError(f"{path}: expected a JSON list of detection records")
    cols = {k: [] for k in ("scene_id", "im_id", "obj_id", "score", "bbox", "size", "counts")}
    for i, d in enumerate(data):
        try:
            if not isinstance(d, dict):
                raise ValueError("not an object")
            for k in ("scene_id", "image_id", "category_id"):
                if isinstance(d.get(k), bool) or not isinstance(d.get(k), int):
                    raise ValueError(f"{k} must be an integer, got {d.get(k)!r}")
            score = d.get("score")
            if isinstance(score, bool) or not isinstance(score, (int, float)) or not math.isfinite(score):
                raise ValueError(f"score must be a finite number, got {score!r}")
            bb = d.get("bbox")
            if (not isinstance(bb, (list, tuple)) or len(bb) != 4
                    or any(isinstance(v, bool) or not isinstance(v, (int, float)) or not math.isfinite(v) for v in bb)):
                raise ValueError(f"bbox must be 4 finite numbers [x, y, w, h], got {bb!r}")
            seg = d.get("segmentation")
            if not isinstance(seg, dict) or "counts" not in seg or "size" not in seg:
                raise ValueError("segmentation must be {\"counts\": [...], \"size\": [h, w]}")
            size = seg["size"]
            if (not isinstance(size, (list, tuple)) or len(size) != 2
                    or any(isinstance(v, bool) or not isinstance(v, int) or v <= 0 for v in size)):
                raise ValueError(f"segmentation size must be [h, w] positive integers, got {size!r}")
            counts = seg["counts"]
            if isinstance(counts, (str, bytes)):
                raise NotImplementedError(f"{path}: record {i}: compressed COCO RLE strings: SAM-6D's ISM writes uncompressed "
                                          "counts (mask_to_rle)")
            if not isinstance(counts, (list, tuple)) or any(isinstance(v, bool) or not isinstance(v, int) for v in counts):
                raise ValueError("segmentation counts must be a list of integers")
            c = np.asarray(counts, np.int64)
            if (c < 0).any() or int(c.sum()) != size[0] * size[1]:
                raise ValueError(f"segmentation counts must be non-negative and sum to h * w = {size[0] * size[1]}")
        except ValueError as e:
            raise ValueError(f"{path}: record {i}: {e}") from None
        cols["scene_id"].append(d["scene_id"])
        cols["im_id"].append(d["image_id"])
        cols["obj_id"].append(d["category_id"])
        cols["score"].append(float(score))
        cols["bbox"].append([float(v) for v in bb])
        cols["size"].append([int(size[0]), int(size[1])])
        cols["counts"].append(c)
    n = len(cols["score"])
    return dict(scene_id=np.array(cols["scene_id"], np.int64), im_id=np.array(cols["im_id"], np.int64),
                obj_id=np.array(cols["obj_id"], np.int64), score=np.array(cols["score"], np.float64),
                bbox=np.array(cols["bbox"], np.float64).reshape(n, 4), size=np.array(cols["size"], np.int64).reshape(n, 2),
                counts=cols["counts"])


def rle_area(counts: np.ndarray) -> int:
    """pixel count of an uncompressed COCO RLE: the sum of its odd runs"""
    return int(np.asarray(counts, np.int64)[1::2].sum())


# ---- kernels ------------------------------------------------------------------------------------------------------------------
def mask_words(H: int, W: int) -> int:
    """32-bit words of one packed H x W mask, rounded up to a multiple of 4 (the pair kernel's 16-byte loads)"""
    return ((H * W + 31) // 32 + 3) // 4 * 4


def pack_u8(masks: torch.Tensor, word_off=None, bits: torch.Tensor = None):
    """masks (n,H,W) u8 CUDA (set where > 0) -> (area (n) i32, box (n,4) i32 x_min, y_min, x_max, y_max, -1 when empty), on the
    device; with bits (int32 CUDA) and word_off (n), each mask is also packed into bits at its offset (csrc/bop_eval.cu)"""
    if not isinstance(masks, torch.Tensor) or not masks.is_cuda or masks.dtype != torch.uint8 or masks.dim() != 3:
        raise RuntimeError("pack_u8: masks must be a CUDA uint8 (n,H,W) tensor")
    n, H, W = masks.shape
    dev = masks.device
    masks = masks.contiguous()
    area = torch.empty(n, dtype=torch.int32, device=dev)
    box = torch.empty(n, 4, dtype=torch.int32, device=dev)
    woff = None
    if bits is not None:
        woff_h = np.asarray(word_off, np.int64)
        if woff_h.shape != (n,):
            raise ValueError("pack_u8: one word offset per mask")
        _check_bits(bits, woff_h, mask_words(H, W))
        woff = torch.as_tensor(woff_h.astype(np.int32), device=dev)
    _lib.call("sam6d_bop_pack_u8", masks, n, H, W, woff, bits, area, box)
    return area, box


def pack_rle(rle_cum, rle_off, hw, word_off, bits: torch.Tensor):
    """uncompressed RLEs as cumulative run ends (rle_cum, rle_off (n+1): inputs.pack_rle's layout), hw (n,2) their H, W,
    word_off (n) -> packed into bits (int32 CUDA) at word_off (csrc/bop_eval.cu)"""
    dev = bits.device
    rle_off = np.asarray(rle_off, np.int32)
    hw = np.asarray(hw, np.int64).reshape(-1, 2)
    n = len(rle_off) - 1
    if len(hw) != n or len(word_off) != n:
        raise ValueError("pack_rle: hw (n,2) and word_off (n) for the n masks of rle_off (n+1)")
    if n == 0:
        return
    words = np.array([mask_words(int(h), int(w)) for h, w in hw])
    _check_bits(bits, np.asarray(word_off), words)
    cum = torch.as_tensor(np.asarray(rle_cum, np.int32), device=dev) if len(rle_cum) else torch.zeros(1, dtype=torch.int32, device=dev)
    off_d = torch.as_tensor(rle_off, device=dev)
    hw_d = torch.as_tensor(hw.astype(np.int32), device=dev)
    woff = torch.as_tensor(np.asarray(word_off, np.int32), device=dev)
    _lib.call("sam6d_bop_pack_rle", cum, off_d, hw_d, woff, n, bits)


def mask_pair_counts(bits: torch.Tensor, word_off, pair_a, pair_b) -> torch.Tensor:
    """|A & B| of P pairs of packed masks (word_off (n+1): the offsets of the n masks and the end; the masks of a pair share one
    size) -> (P) i32 on the device (csrc/bop_eval.cu)"""
    dev = bits.device
    woff = np.asarray(word_off, np.int64)
    a, b = np.asarray(pair_a, np.int64), np.asarray(pair_b, np.int64)
    P = len(a)
    if b.shape != (P,) or (P and (min(a.min(), b.min()) < 0 or max(a.max(), b.max()) >= len(woff) - 1)):
        raise ValueError(f"mask_pair_counts: pair indices must be (P,) in [0, {len(woff) - 1})")
    if (woff % 4).any() or (np.diff(woff) < 0).any() or woff[-1] > bits.numel():
        raise ValueError("mask_pair_counts: word offsets must be increasing multiples of 4 within bits")
    if P and (np.diff(woff)[a] != np.diff(woff)[b]).any():
        raise ValueError("mask_pair_counts: the masks of a pair must have the same size")
    if not bits.is_cuda or bits.dtype != torch.int32 or bits.data_ptr() % 16:
        raise RuntimeError("mask_pair_counts: bits must be a 16-byte aligned CUDA int32 tensor")
    out = torch.empty(P, dtype=torch.int32, device=dev)
    woff_d = torch.as_tensor(woff.astype(np.int32), device=dev)
    a_d, b_d = torch.as_tensor(a.astype(np.int32), device=dev), torch.as_tensor(b.astype(np.int32), device=dev)
    _lib.call("sam6d_bop_mask_pair_counts", bits, woff_d, a_d, b_d, P, out)
    return out


def _check_bits(bits, word_off, words):
    if not isinstance(bits, torch.Tensor) or not bits.is_cuda or bits.dtype != torch.int32 or not bits.is_contiguous():
        raise RuntimeError("bits must be a contiguous CUDA int32 tensor")
    end = np.asarray(word_off, np.int64) + words
    if len(end) and (np.asarray(word_off).min() < 0 or end.max() > bits.numel() or end.max() >= 2 ** 31):
        raise ValueError(f"packed masks must lie within bits ({bits.numel()} words)")


# ---- matching and accumulation ------------------------------------------------------------------------------------------------
def bbox_iou(det_xywh: np.ndarray, gt_xywh: np.ndarray) -> np.ndarray:
    """pycocotools' bbIou without crowd: (D,4) x (G,4) x, y, w, h -> (D,G) float64"""
    d, g = np.asarray(det_xywh, np.float64)[:, None, :], np.asarray(gt_xywh, np.float64)[None, :, :]
    w = np.minimum(d[..., 0] + d[..., 2], g[..., 0] + g[..., 2]) - np.maximum(d[..., 0], g[..., 0])
    h = np.minimum(d[..., 1] + d[..., 3], g[..., 1] + g[..., 3]) - np.maximum(d[..., 1], g[..., 1])
    i = w * h
    with np.errstate(divide="ignore", invalid="ignore"):
        o = i / (d[..., 2] * d[..., 3] + g[..., 2] * g[..., 3] - i)
    return np.where((w <= 0) | (h <= 0), 0.0, o)


def match(ious, gt_ignore, gt_area, det_area, det_valid=None, gt_valid=None):
    """the matching of N (image, category) groups at once (module docstring), padded to D detections and G GT instances.
    ious (N,D,G) float64 with each group's detections in score order; gt_ignore (N,G) bool; gt_area (N,G), det_area (N,D);
    det_valid (N,D), gt_valid (N,G) bool mark the real entries (default all) -> (gt_index (N,A,T,D) i64: the matched GT's
    index in the group's own order, -1 for none; det_ignore (N,A,T,D) bool; gt_ig (N,A,G) bool the GT ignored in each area
    range).  A = 4 area ranges, T = 10 IoU thresholds."""
    ious = np.asarray(ious, np.float64)
    N, D, G = ious.shape
    A, T = len(AREA_RNGS), len(IOU_THRS)
    gt_ignore, gt_area, det_area = np.asarray(gt_ignore, bool), np.asarray(gt_area, np.float64), np.asarray(det_area, np.float64)
    det_valid = np.ones((N, D), bool) if det_valid is None else np.asarray(det_valid, bool)
    gt_valid = np.ones((N, G), bool) if gt_valid is None else np.asarray(gt_valid, bool)
    lo, hi = AREA_RNGS[:, 0], AREA_RNGS[:, 1]
    gt_ig = gt_ignore[:, None, :] | (gt_area[:, None, :] < lo[None, :, None]) | (gt_area[:, None, :] > hi[None, :, None])
    ig = np.broadcast_to(gt_ig[:, :, None, :], (N, A, T, G))
    thr = np.minimum(IOU_THRS, 1 - 1e-10)[None, None, :, None]
    taken = np.broadcast_to(~gt_valid[:, None, None, :], (N, A, T, G)).copy()     # padding never matches
    gt_index = np.full((N, A, T, D), -1, np.int64)
    rev = np.arange(G)[::-1]
    for d in range(D):
        iou = ious[:, None, None, d, :]
        cand = ~taken & (iou >= thr) & det_valid[:, d, None, None, None]
        m = np.full((N, A, T), -1, np.int64)
        for group in (False, True):                 # the non-ignored GT first; the ignored ones only when none of those matched
            c = cand & (ig == group) & (m == -1)[..., None]
            v = np.where(c, iou, -np.inf)
            best = v.max(axis=-1, keepdims=True)
            last = c & (v == best)                  # every candidate at the best IoU; the scan keeps the last one
            has = last.any(axis=-1)
            idx = G - 1 - np.argmax(last[..., rev], axis=-1)
            m = np.where(has, idx, m)
        gt_index[..., d] = m
        n_, a_, t_ = np.nonzero(m >= 0)
        taken[n_, a_, t_, m[n_, a_, t_]] = True
    matched = gt_index >= 0
    ig_of_match = np.take_along_axis(np.broadcast_to(gt_ig[:, :, None, :], (N, A, T, G)), np.maximum(gt_index, 0), axis=-1) & matched
    out_of_range = (det_area[:, None, :] < lo[None, :, None]) | (det_area[:, None, :] > hi[None, :, None])    # (N,A,D)
    det_ignore = ig_of_match | (~matched & out_of_range[:, :, None, :])
    return gt_index, det_ignore, gt_ig


def accumulate(det_score, det_rank, det_cat, det_matched, det_ignore, gt_cat, gt_ig, K: int):
    """the accumulation of pycocotools (module docstring).  Detections of all groups concatenated image by image, each group in
    score order: det_score (n) f64, det_rank (n) their position in their (image, category) group, det_cat (n) category index in
    [0, K), det_matched / det_ignore (A,T,n) bool; gt_cat (g) category index of every GT instance, gt_ig (A,g) bool ->
    (precision (T,R,K,A,M), recall (T,K,A,M)) float64, -1 in the cells without a non-ignored GT"""
    A, T, R, M = len(AREA_RNGS), len(IOU_THRS), len(REC_THRS), len(MAX_DETS)
    det_score, det_rank, det_cat = np.asarray(det_score, np.float64), np.asarray(det_rank), np.asarray(det_cat)
    det_matched, det_ignore = np.asarray(det_matched, bool), np.asarray(det_ignore, bool)
    gt_cat, gt_ig = np.asarray(gt_cat), np.asarray(gt_ig, bool)
    precision = -np.ones((T, R, K, A, M))
    recall = -np.ones((T, K, A, M))
    for k in range(K):
        npig = (~gt_ig[:, gt_cat == k]).sum(axis=1)            # (A,)
        if not npig.any():
            continue
        in_k = det_cat == k
        for mi, max_det in enumerate(MAX_DETS):
            sel = np.flatnonzero(in_k & (det_rank < max_det))
            sel = sel[np.argsort(-det_score[sel], kind="stable")]
            dtm, dti = det_matched[:, :, sel], det_ignore[:, :, sel]
            tp = np.cumsum(dtm & ~dti, axis=2).astype(np.float64)
            fp = np.cumsum(~dtm & ~dti, axis=2).astype(np.float64)
            nd = len(sel)
            for a in range(A):
                if npig[a] == 0:
                    continue
                rc = tp[a] / npig[a]                              # (T, nd)
                pr = tp[a] / (fp[a] + tp[a] + np.spacing(1))
                pr = np.maximum.accumulate(pr[:, ::-1], axis=1)[:, ::-1]
                recall[:, k, a, mi] = rc[:, -1] if nd else 0.0
                for t in range(T):
                    inds = np.searchsorted(rc[t], REC_THRS, side="left")
                    q = np.zeros(R)
                    ok = inds < nd
                    q[ok] = pr[t, inds[ok]]
                    precision[t, :, k, a, mi] = q
    return precision, recall


def _mean_valid(s):
    s = s[s > -1]
    return float(np.mean(s)) if s.size else -1.0


def summarize(precision, recall) -> dict:
    """the 12 COCO stats of COCOeval.summarize from accumulate's arrays"""
    p, r = np.asarray(precision), np.asarray(recall)
    a = {n: i for i, n in enumerate(AREA_NAMES)}
    m100 = MAX_DETS.index(100)
    t50, t75 = int(np.flatnonzero(IOU_THRS == 0.5)[0]), int(np.flatnonzero(IOU_THRS == 0.75)[0])
    out = OrderedDict()
    out["AP"] = _mean_valid(p[:, :, :, a["all"], m100])
    out["AP50"] = _mean_valid(p[t50, :, :, a["all"], m100])
    out["AP75"] = _mean_valid(p[t75, :, :, a["all"], m100])
    for n in ("small", "medium", "large"):
        out[f"AP_{n}"] = _mean_valid(p[:, :, :, a[n], m100])
    for mi, md in enumerate(MAX_DETS):
        out[f"AR{md}"] = _mean_valid(r[:, :, a["all"], mi])
    for n in ("small", "medium", "large"):
        out[f"AR_{n}"] = _mean_valid(r[:, :, a[n], m100])
    return out


# ---- the split ----------------------------------------------------------------------------------------------------------------
def _full_mask_path(rows, k):
    p = rows.mask_path(k)
    return os.path.join(os.path.dirname(os.path.dirname(p)), "mask", os.path.basename(p))


def evaluate_bop22_coco(bop_root: str, dataset_name: str, result_json: str, targets=None, iou_type: str = "segm",
                        bbox_type: str = "amodal", device=None, timings=None) -> dict:
    """COCO scores of result_json on <bop_root>/<dataset_name> (module docstring).  targets: the targets file (default
    <dataset>/test_targets_bop19.json).  timings: a dict to which the seconds of "decode" (PNG masks), "pack", "pairs" (the
    pair-count kernel), "match" and "accumulate" are added (the device is synchronised for that).  -> dict: the 12 stats,
    ap_per_object {obj_id: AP}, obj_ids (the K axis), recall_thresholds, iou_thresholds, area_ranges, max_dets, precision
    (10,101,K,4,3) and recall (10,K,4,3) as lists, and the counts n_images, n_detections (detections scored: on a target image,
    of a GT category, within the first 100 of their group), n_gt (GT instances kept), n_ignored_gt (of those, with
    visib_fract < 0.1) and n_pairs (detection-GT pairs whose IoU was computed)"""
    if iou_type not in IOU_TYPES:
        raise ValueError(f"iou_type must be one of {IOU_TYPES}, got {iou_type!r}")
    if bbox_type not in BBOX_TYPES:
        raise ValueError(f"bbox_type must be one of {BBOX_TYPES}, got {bbox_type!r}")
    device = torch.device(device if device is not None else "cuda")
    budget = int(MASK_BUDGET_BYTES)
    ds_root = os.path.join(bop_root, dataset_name)
    targets = load_targets(targets if targets is not None else os.path.join(ds_root, "test_targets_bop19.json"))
    images = sorted({(s, i) for s, i, _, _ in targets})
    img_index = {k: j for j, k in enumerate(images)}
    dets = load_detections(result_json)

    split = bop.split_name(dataset_name)
    frames = {(f.scene_id, f.frame_id): f for f in bop.scan_test_split(bop_root, dataset_name)}
    rows = pbr.scan_rows(ds_root, split, max_num_scenes=None, max_num_frames=sys.maxsize)
    gt_rows = {k: [] for k in images}
    for r in range(len(rows)):
        key = (int(rows.scene_id[r]), int(rows.frame_id[r]))
        if key in gt_rows:
            gt_rows[key].append(r)
    sizes = {}
    for key in images:
        if key not in frames:
            raise ValueError(f"target scene {key[0]} image {key[1]} is not in {os.path.join(ds_root, split)}")
        sizes[key] = _image_size(frames[key].rgb_path)

    # detections of target images, grouped by (image, obj_id), each group in stable score order
    groups = OrderedDict()
    for r in range(len(dets["score"])):
        key = (int(dets["scene_id"][r]), int(dets["im_id"][r]))
        if key not in img_index:
            continue
        if tuple(dets["size"][r]) != sizes[key]:
            raise ValueError(f"{result_json}: record {r}: segmentation size {dets['size'][r].tolist()} does not match the size "
                             f"{list(sizes[key])} of scene {key[0]} image {key[1]}")
        groups.setdefault((key, int(dets["obj_id"][r])), []).append(r)
    for g, rs in groups.items():
        rs = np.asarray(rs, np.int64)
        groups[g] = rs[np.argsort(-dets["score"][rs], kind="stable")][:MAX_DETS[-1]]
    det_area_all = np.array([rle_area(c) for c in dets["counts"]], np.float64) if iou_type == "segm" else \
        dets["bbox"][:, 2] * dets["bbox"][:, 3]
    gt_objs = {key: {int(rows.obj_id[r]) for r in gt_rows[key]} for key in images}

    # per image: kept GT (row, area, box) and the IoU matrix of each (image, obj_id) with kept GT and detections
    gt_kept = {}                                    # image -> list of (row, area, box xywh)
    ious = {}                                       # (image, obj_id) -> (D,G) float64
    n_pairs = 0
    t0 = time.perf_counter()
    pos = 0
    while pos < len(images):
        # a chunk of images within the budget (at least one)
        chunk, nbytes = [], 0
        while pos < len(images):
            key = images[pos]
            H, W = sizes[key]
            nw = mask_words(H, W)
            n_gt = len(gt_rows[key])
            n_det = sum(len(groups.get((key, o), ())) for o in gt_objs[key]) if iou_type == "segm" else 0
            cost = n_gt * (H * W * (2 if bbox_type == "amodal" else 1) + nw * 4) + n_det * nw * 4
            if chunk and nbytes + cost > budget:
                break
            chunk.append(key)
            nbytes += cost
            pos += 1
        t0 = _process_chunk(chunk, rows, gt_rows, sizes, groups, dets, iou_type, bbox_type, device, gt_kept, ious, timings, t0)
    for (key, o), m in ious.items():
        n_pairs += m.size

    # K categories, groups with detections and kept GT
    obj_ids = sorted({int(rows.obj_id[r]) for key in images for r, _, _ in gt_kept[key]})
    cat = {o: k for k, o in enumerate(obj_ids)}
    K = len(obj_ids)
    t0 = time.perf_counter()
    g_keys = [(key, o) for key in images for o in obj_ids
              if any(int(rows.obj_id[r]) == o for r, _, _ in gt_kept[key]) or len(groups.get((key, o), ()))]
    n_det_total = sum(len(groups.get(g, ())) for g in g_keys)
    A, T = len(AREA_RNGS), len(IOU_THRS)
    det_score = np.zeros(n_det_total)
    det_rank = np.zeros(n_det_total, np.int64)
    det_cat = np.zeros(n_det_total, np.int64)
    det_m = np.zeros((A, T, n_det_total), bool)
    det_i = np.zeros((A, T, n_det_total), bool)
    gt_cat, gt_ig_cols, n_ign = [], [], 0
    both = []
    off = 0
    spans = {}
    for g in g_keys:
        key, o = g
        rs = groups.get(g, np.zeros(0, np.int64))
        n = len(rs)
        det_score[off:off + n] = dets["score"][rs]
        det_rank[off:off + n] = np.arange(n)
        det_cat[off:off + n] = cat[o]
        spans[g] = (off, n)
        gts = [(r, a, b) for r, a, b in gt_kept[key] if int(rows.obj_id[r]) == o]
        ign = np.array([rows.visib_fract[r] < MIN_VISIB_FRACT for r, _, _ in gts], bool)
        area = np.array([a for _, a, _ in gts], np.float64)
        n_ign += int(ign.sum())
        lo, hi = AREA_RNGS[:, 0], AREA_RNGS[:, 1]
        gt_cat += [cat[o]] * len(gts)
        gt_ig_cols.append(ign[None, :] | (area[None, :] < lo[:, None]) | (area[None, :] > hi[:, None]))
        if n and gts:
            both.append((g, ign, area))
        elif n:
            # no GT of this object in the image: every detection is unmatched, ignored only when its area is out of range
            da = det_area_all[rs]
            det_i[:, :, off:off + n] = ((da[None, :] < lo[:, None]) | (da[None, :] > hi[:, None]))[:, None, :]
        off += n
    if both:
        N = len(both)
        Dm = max(spans[g][1] for g, _, _ in both)
        Gm = max(len(i) for _, i, _ in both)
        I = np.zeros((N, Dm, Gm))
        gi, ga, da = np.zeros((N, Gm), bool), np.zeros((N, Gm)), np.zeros((N, Dm))
        dv, gv = np.zeros((N, Dm), bool), np.zeros((N, Gm), bool)
        for j, (g, ign, area) in enumerate(both):
            off, n = spans[g]
            m = ious[g]
            I[j, :n, :len(ign)] = m
            gi[j, :len(ign)], ga[j, :len(ign)], gv[j, :len(ign)] = ign, area, True
            da[j, :n], dv[j, :n] = det_area_all[groups[g]], True
        gidx, dig, _ = match(I, gi, ga, da, dv, gv)
        for j, (g, _, _) in enumerate(both):
            off, n = spans[g]
            det_m[:, :, off:off + n] = gidx[j, :, :, :n] >= 0
            det_i[:, :, off:off + n] = dig[j, :, :, :n]
    t0 = _tick(timings, "match", t0)
    gt_ig = np.concatenate(gt_ig_cols, axis=1) if gt_ig_cols else np.zeros((A, 0), bool)
    precision, recall = accumulate(det_score, det_rank, det_cat, det_m, det_i, np.asarray(gt_cat, np.int64), gt_ig, K)
    stats = summarize(precision, recall)
    m100 = MAX_DETS.index(100)
    ap_obj = {o: _mean_valid(precision[:, :, k, 0, m100]) for o, k in cat.items()}
    _tick(timings, "accumulate", t0)

    out = OrderedDict(stats)
    out.update(iou_type=iou_type, bbox_type=bbox_type, ap_per_object=ap_obj, obj_ids=obj_ids,
               recall_thresholds=REC_THRS.tolist(), iou_thresholds=IOU_THRS.tolist(), area_ranges=dict(zip(AREA_NAMES, AREA_RNGS.tolist())),
               max_dets=list(MAX_DETS), precision=precision.tolist(), recall=recall.tolist(), n_images=len(images),
               n_detections=int(n_det_total), n_gt=int(sum(len(v) for v in gt_kept.values())), n_ignored_gt=n_ign, n_pairs=int(n_pairs))
    return out


def _process_chunk(chunk, rows, gt_rows, sizes, groups, dets, iou_type, bbox_type, device, gt_kept, ious, timings, t0):
    """decode and pack the GT masks of a chunk of images, keep the non-empty instances, and compute the IoU matrices of the
    chunk's (image, obj_id) groups -> the time mark for the next stage"""
    # GT masks: visible (bits packed for segm), full (area and box only) with amodal
    vis, full = {}, {}
    for key in chunk:
        H, W = sizes[key]
        for r in gt_rows[key]:
            for store, path in ((vis, rows.mask_path(r)),) + (((full, _full_mask_path(rows, r)),) if bbox_type == "amodal" else ()):
                m = pbr.decode_mask(path)
                if m.shape != (H, W):
                    raise ValueError(f"{path}: mask {m.shape} does not match the image size {(H, W)}")
                store[r] = m
    t0 = _tick(timings, "decode", t0)
    # word offsets: GT visible masks first, then the detections that share an (image, obj_id) with a GT instance
    slots, woff, total = {}, [], 0
    if iou_type == "segm":
        for key in chunk:
            for r in gt_rows[key]:
                slots[("g", r)] = len(woff)
                woff.append(total)
                total += mask_words(*sizes[key])
        for key in chunk:
            for o in sorted({int(rows.obj_id[r]) for r in gt_rows[key]}):
                for d in groups.get((key, o), ()):
                    slots[("d", int(d))] = len(woff)
                    woff.append(total)
                    total += mask_words(*sizes[key])
    bits = torch.zeros(max(total, 4), dtype=torch.int32, device=device) if iou_type == "segm" else None
    # pack_u8 per image size
    info = {}
    for store, packed in ((vis, iou_type == "segm"), (full, False)):
        by_size = OrderedDict()
        for key in chunk:
            for r in gt_rows[key]:
                if r in store:
                    by_size.setdefault(sizes[key], []).append(r)
        for (H, W), rs in by_size.items():
            m = torch.from_numpy(np.stack([store[r] for r in rs])).to(device)
            if packed:
                area, box = pack_u8(m, [woff[slots[("g", r)]] for r in rs], bits)
            else:
                area, box = pack_u8(m)
            area, box = area.cpu().numpy(), box.cpu().numpy()
            for j, r in enumerate(rs):
                info[(store is full, r)] = (int(area[j]), box[j].astype(np.int64))
            del m
    del vis, full
    kept = {}
    for key in chunk:
        kept[key] = []
        for r in gt_rows[key]:
            area, vbox = info[(False, r)]
            if area == 0:
                continue
            if bbox_type == "amodal":
                farea, fbox = info[(True, r)]
                if farea == 0:
                    continue
                b = fbox
            else:
                b = vbox
            kept[key].append((r, area, [float(b[0]), float(b[1]), float(b[2] - b[0] + 1), float(b[3] - b[1] + 1)]))
        gt_kept[key] = kept[key]
    if iou_type == "bbox":
        t0 = _tick(timings, "pack", t0, sync=True)
        for key in chunk:
            for o in sorted({int(rows.obj_id[r]) for r, _, _ in kept[key]}):
                rs = groups.get((key, o), ())
                if len(rs):
                    gb = np.array([b for r, _, b in kept[key] if int(rows.obj_id[r]) == o], np.float64)
                    ious[(key, o)] = bbox_iou(dets["bbox"][rs], gb)
        return t0
    # detections of groups with a kept GT instance, packed from their run ends
    todo = []
    for key in chunk:
        for o in sorted({int(rows.obj_id[r]) for r, _, _ in kept[key]}):
            todo += [int(d) for d in groups.get((key, o), ())]
    if todo:
        cums = [np.cumsum(dets["counts"][d]).astype(np.int32) for d in todo]
        rle_off = np.concatenate([[0], np.cumsum([len(c) for c in cums])]).astype(np.int32)
        pack_rle(np.concatenate(cums), rle_off, dets["size"][todo], [woff[slots[("d", d)]] for d in todo], bits)
    t0 = _tick(timings, "pack", t0, sync=True)
    pa, pb, where = [], [], []
    for key in chunk:
        for o in sorted({int(rows.obj_id[r]) for r, _, _ in kept[key]}):
            rs = groups.get((key, o), ())
            gts = [(r, a) for r, a, _ in kept[key] if int(rows.obj_id[r]) == o]
            if not len(rs):
                continue
            where.append(((key, o), len(rs), len(gts), len(pa)))
            for d in rs:
                for r, _ in gts:
                    pa.append(slots[("d", int(d))])
                    pb.append(slots[("g", r)])
    if pa:
        cnt = mask_pair_counts(bits, np.asarray(woff + [total], np.int64), pa, pb).cpu().numpy().astype(np.int64)
    t0 = _tick(timings, "pairs", t0, sync=True)
    for g, nd, ng, start in where:
        inter = cnt[start:start + nd * ng].reshape(nd, ng)
        rs = groups[g]
        da = np.array([rle_area(dets["counts"][d]) for d in rs], np.int64)
        ga = np.array([a for r, a, _ in kept[g[0]] if int(rows.obj_id[r]) == g[1]], np.int64)
        ious[g] = inter / (da[:, None] + ga[None, :] - inter).astype(np.float64)
    del bits
    return t0
