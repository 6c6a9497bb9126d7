"""Pure-Python float64 restatement of the BOP detection / segmentation scoring (sam6d_b200/bop_eval_coco.py's module docstring
states the definition: pycocotools' COCOeval with BOP's ground truth, as the BOP toolkit's eval_bop22_coco.py runs it).  Test
infrastructure only: scalar loops over run-length lists and pixels, no GPU, none of the package's code.

    mask_runs(mask)                          (H,W) array, set where > 0 -> foreground runs [(start, end)) in column-major order
    rle_runs(counts)                         uncompressed COCO counts -> the same runs
    runs_area(runs), runs_intersection(a, b)
    segm_iou(d, g), bbox_iou(d, g)           one detection-GT pair
    evaluate_img(ious, gt_ignore, gt_area, det_area, area_rng)     pycocotools' evaluateImg for one (image, category, area)
    accumulate(evals, K)                     pycocotools' accumulate
    summarize(precision, recall)             the 12 stats
    evaluate(bop_root, dataset, result_json, targets=None, iou_type="segm", bbox_type="amodal")"""
import bisect
import json
import os

import numpy as np

IOU_THRS = [float(t) for t in np.linspace(0.5, 0.95, 10)]     # pycocotools' values (linspace rounding, not 0.5 + 0.05 k)
REC_THRS = [float(r) for r in np.linspace(0.0, 1.0, 101)]
AREA_RNGS = [(0.0, 1e10), (0.0, 1024.0), (1024.0, 9216.0), (9216.0, 1e10)]
MAX_DETS = [1, 10, 100]
EPS = 2.0 ** -52                                       # np.spacing(1)
STAT_NAMES = ["AP", "AP50", "AP75", "AP_small", "AP_medium", "AP_large", "AR1", "AR10", "AR100", "AR_small", "AR_medium", "AR_large"]


# ---- masks as run lists ---------------------------------------------------------------------------------------------------------
def mask_runs(mask):
    """-> (runs, (x_min, y_min, x_max, y_max) or None), runs in column-major pixel order k = x H + y"""
    H, W = len(mask), len(mask[0])
    runs, start, k = [], None, 0
    x0 = y0 = None
    x1 = y1 = -1
    for x in range(W):
        for y in range(H):
            on = mask[y][x] > 0
            if on:
                x0 = x if x0 is None else min(x0, x)
                y0 = y if y0 is None else min(y0, y)
                x1, y1 = max(x1, x), max(y1, y)
                if start is None:
                    start = k
            elif start is not None:
                runs.append((start, k))
                start = None
            k += 1
    if start is not None:
        runs.append((start, k))
    return runs, (None if x0 is None else (x0, y0, x1, y1))


def rle_runs(counts):
    runs, pos = [], 0
    for j, c in enumerate(counts):
        if j % 2 == 1 and c > 0:
            runs.append((pos, pos + c))
        pos += c
    return runs


def runs_area(runs):
    return sum(e - s for s, e in runs)


def runs_intersection(a, b):
    i = j = n = 0
    while i < len(a) and j < len(b):
        lo, hi = max(a[i][0], b[j][0]), min(a[i][1], b[j][1])
        if hi > lo:
            n += hi - lo
        if a[i][1] < b[j][1]:
            i += 1
        else:
            j += 1
    return n


def segm_iou(d_runs, g_runs):
    i = runs_intersection(d_runs, g_runs)
    u = runs_area(d_runs) + runs_area(g_runs) - i
    return float(i) / float(u) if u > 0 else 0.0


def bbox_iou(d, g):
    w = min(d[0] + d[2], g[0] + g[2]) - max(d[0], g[0])
    if w <= 0:
        return 0.0
    h = min(d[1] + d[3], g[1] + g[3]) - max(d[1], g[1])
    if h <= 0:
        return 0.0
    i = w * h
    return i / (d[2] * d[3] + g[2] * g[3] - i)


# ---- COCOeval -------------------------------------------------------------------------------------------------------------------
def evaluate_img(ious, gt_ignore, gt_area, det_area, area_rng):
    """one (image, category, area range): ious[d][g] with the detections in score order (already cut to 100), GT in their own
    order -> dict gt_index[t][d] (the matched GT's own index or -1), det_ignore[t][d], gt_ig[g]"""
    G, D = len(gt_ignore), len(det_area)
    gt_ig = [bool(gt_ignore[g]) or gt_area[g] < area_rng[0] or gt_area[g] > area_rng[1] for g in range(G)]
    order = sorted(range(G), key=lambda g: gt_ig[g])           # stable: non-ignored first
    gt_index = [[-1] * D for _ in IOU_THRS]
    det_ignore = [[False] * D for _ in IOU_THRS]
    for t, thr in enumerate(IOU_THRS):
        gtm = [False] * G
        for d in range(D):
            iou = min(thr, 1 - 1e-10)
            m = -1
            for gind in order:
                if gtm[gind]:
                    continue
                if m > -1 and not gt_ig[m] and gt_ig[gind]:
                    break
                if ious[d][gind] < iou:
                    continue
                iou = ious[d][gind]
                m = gind
            if m == -1:
                continue
            det_ignore[t][d] = gt_ig[m]
            gt_index[t][d] = m
            gtm[m] = True
        for d in range(D):
            if gt_index[t][d] == -1 and (det_area[d] < area_rng[0] or det_area[d] > area_rng[1]):
                det_ignore[t][d] = True
    return dict(gt_index=gt_index, det_ignore=det_ignore, gt_ig=gt_ig)


def accumulate(evals, K):
    """evals[k][a] = list over images (in order) of (det_scores in score order, evaluate_img's result) of category k, area a ->
    precision[t][r][k][a][m], recall[t][k][a][m]"""
    T, R, A, M = len(IOU_THRS), len(REC_THRS), len(AREA_RNGS), len(MAX_DETS)
    precision = [[[[[-1.0] * M for _ in range(A)] for _ in range(K)] for _ in range(R)] for _ in range(T)]
    recall = [[[[-1.0] * M for _ in range(A)] for _ in range(K)] for _ in range(T)]
    for k in range(K):
        for a in range(A):
            E = evals[k][a]
            npig = sum(1 for _, e in E for ig in e["gt_ig"] if not ig)
            if npig == 0:
                continue
            for mi, max_det in enumerate(MAX_DETS):
                entries = []                    # (score, image position, rank) -> a stable merge by descending score
                for ii, (scores, e) in enumerate(E):
                    for d in range(min(max_det, len(scores))):
                        entries.append((scores[d], ii, d))
                order = sorted(range(len(entries)), key=lambda j: -entries[j][0])
                for t in range(T):
                    tp = fp = 0
                    rc, pr = [], []
                    for j in order:
                        _, ii, d = entries[j]
                        e = E[ii][1]
                        matched = e["gt_index"][t][d] >= 0
                        ignored = e["det_ignore"][t][d]
                        if matched and not ignored:
                            tp += 1
                        elif not matched and not ignored:
                            fp += 1
                        rc.append(float(tp) / npig)
                        pr.append(float(tp) / (float(fp) + float(tp) + EPS))
                    nd = len(rc)
                    recall[t][k][a][mi] = rc[-1] if nd else 0.0
                    for i in range(nd - 1, 0, -1):
                        if pr[i] > pr[i - 1]:
                            pr[i - 1] = pr[i]
                    for r, thr in enumerate(REC_THRS):
                        pi = bisect.bisect_left(rc, thr)
                        precision[t][r][k][a][mi] = pr[pi] if pi < nd else 0.0
    return precision, recall


def _mean(values):
    v = [x for x in values if x > -1]
    return sum(v) / len(v) if v else -1.0


def summarize(precision, recall):
    T, R = len(precision), len(precision[0])
    K = len(precision[0][0])
    t50, t75 = IOU_THRS.index(0.5), IOU_THRS.index(0.75)

    def ap(ts, a):
        return _mean([precision[t][r][k][a][2] for t in ts for r in range(R) for k in range(K)])

    def ar(a, mi):
        return _mean([recall[t][k][a][mi] for t in range(T) for k in range(K)])
    s = [ap(range(T), 0), ap([t50], 0), ap([t75], 0), ap(range(T), 1), ap(range(T), 2), ap(range(T), 3),
         ar(0, 0), ar(0, 1), ar(0, 2), ar(1, 2), ar(2, 2), ar(3, 2)]
    return dict(zip(STAT_NAMES, s))


# ---- the split ------------------------------------------------------------------------------------------------------------------
def _png(path):
    from PIL import Image
    with Image.open(path) as im:
        return np.array(im).tolist()


def evaluate(bop_root, dataset, result_json, targets=None, iou_type="segm", bbox_type="amodal"):
    split = "test_primesense" if dataset in ("hb", "tless") else "test"
    ds = os.path.join(bop_root, dataset)
    with open(targets or os.path.join(ds, "test_targets_bop19.json")) as fh:
        images = sorted({(int(t["scene_id"]), int(t["im_id"])) for t in json.load(fh)})
    with open(result_json) as fh:
        records = json.load(fh)
    # GT: every instance of a target image in file order; drop empty visible (and, amodal, empty full) masks
    gts = {im: [] for im in images}
    for s, i in images:
        sdir = os.path.join(ds, split, f"{s:06d}")
        with open(os.path.join(sdir, "scene_gt.json")) as fh:
            insts = json.load(fh)[str(i)]
        with open(os.path.join(sdir, "scene_gt_info.json")) as fh:
            infos = json.load(fh)[str(i)]
        for idx, (inst, info) in enumerate(zip(insts, infos)):
            vis = _png(os.path.join(sdir, "mask_visib", f"{i:06d}_{idx:06d}.png"))
            runs, vbox = mask_runs(vis)
            if not runs:
                continue
            box = vbox
            if bbox_type == "amodal":
                _, box = mask_runs(_png(os.path.join(sdir, "mask", f"{i:06d}_{idx:06d}.png")))
                if box is None:
                    continue
            gts[(s, i)].append(dict(obj=int(inst["obj_id"]), runs=runs, area=runs_area(runs),
                                    box=[float(box[0]), float(box[1]), float(box[2] - box[0] + 1), float(box[3] - box[1] + 1)],
                                    ignore=info["visib_fract"] < 0.1))
    cats = sorted({g["obj"] for im in images for g in gts[im]})
    # detections per (image, category), stable score order, first 100
    dets = {}
    for rec in records:
        key = (rec["scene_id"], rec["image_id"])
        if key in gts and rec["category_id"] in cats:
            dets.setdefault((key, rec["category_id"]), []).append(rec)
    for g in dets:
        dets[g] = sorted(dets[g], key=lambda r: -r["score"])[:100]
    n_pairs = n_det = 0
    evals = [[[] for _ in AREA_RNGS] for _ in cats]
    for im in images:
        for k, c in enumerate(cats):
            gl = [g for g in gts[im] if g["obj"] == c]
            dl = dets.get((im, c), [])
            if not gl and not dl:
                continue
            n_det += len(dl)
            if iou_type == "segm":
                druns = [rle_runs(r["segmentation"]["counts"]) for r in dl]
                darea = [runs_area(r) for r in druns]
                ious = [[segm_iou(dr, g["runs"]) for g in gl] for dr in druns]
            else:
                darea = [r["bbox"][2] * r["bbox"][3] for r in dl]
                ious = [[bbox_iou(r["bbox"], g["box"]) for g in gl] for r in dl]
            n_pairs += len(dl) * len(gl)
            scores = [r["score"] for r in dl]
            for a, rng in enumerate(AREA_RNGS):
                evals[k][a].append((scores, evaluate_img(ious, [g["ignore"] for g in gl], [g["area"] for g in gl], darea, rng)))
    precision, recall = accumulate(evals, len(cats))
    out = summarize(precision, recall)
    out["ap_per_object"] = {c: _mean([precision[t][r][k][0][2] for t in range(len(IOU_THRS)) for r in range(len(REC_THRS))])
                            for k, c in enumerate(cats)}
    out.update(obj_ids=cats, precision=np.array(precision), recall=np.array(recall), n_images=len(images), n_detections=n_det,
               n_gt=sum(len(v) for v in gts.values()), n_ignored_gt=sum(g["ignore"] for v in gts.values() for g in v), n_pairs=n_pairs)
    return out
