"""float64 numpy restatement of the BOP19 pose-task scoring (sam6d_b200/bop_eval.py's module docstring states the definitions;
BOP Challenge 2020, Hodan et al., ECCVW 2020, sec. 2.2).  Test infrastructure only: straightforward loops, no GPU.

    symmetries(info)                       identity + discrete, continuous discretised, compositions
    mssd(R_e, t_e, R_g, t_g, X, syms)      max-over-vertices, min-over-symmetries 3D distance
    mspd(R_e, t_e, R_g, t_g, X, syms, K)   the same between projections
    vsd_counts(d_e, d_g, d_test, K, delta, diameter, taus)   |U|, |I|, per-tau cost counts from given depth images
    spheres_overlap(t_e, t_g, r)           the VSD shortcut
    match(errors, scores, valid, thr)      greedy matching of one (scene, image, object)
    evaluate(...)                          recalls and ARs of a split, with the depth renders supplied by the caller"""
import json
import math
import os

import numpy as np

TAUS = [0.05 * k for k in range(1, 11)]
THETAS = [0.05 * k for k in range(1, 11)]
MSSD_FRACS = [0.05 * k for k in range(1, 11)]
MSPD_PX = [5.0 * k for k in range(1, 11)]


def rotation(axis, angle):
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    c, s = math.cos(angle), math.sin(angle)
    x, y, z = a
    return np.array([[c + x * x * (1 - c), x * y * (1 - c) - z * s, x * z * (1 - c) + y * s],
                     [y * x * (1 - c) + z * s, c + y * y * (1 - c), y * z * (1 - c) - x * s],
                     [z * x * (1 - c) - y * s, z * y * (1 - c) + x * s, c + z * z * (1 - c)]])


def symmetries(info, step=0.01):
    """-> list of (R (3,3), t (3,)) float64"""
    disc = [(np.eye(3), np.zeros(3))]
    for m in info.get("symmetries_discrete", []):
        m = np.array(m, np.float64).reshape(4, 4)
        disc.append((m[:3, :3], m[:3, 3]))
    cont = []
    for sym in info.get("symmetries_continuous", []):
        off = np.array(sym["offset"], np.float64)
        n = int(math.ceil(math.pi / step))
        for i in range(1, n):
            R = rotation(sym["axis"], i * 2.0 * math.pi / n)
            cont.append((R, off - R @ off))
    if not cont:
        return disc
    out = []
    for Rd, td in disc:
        for Rc, tc in cont:
            out.append((Rc @ Rd, Rc @ td + tc))
    return out


def mssd(R_e, t_e, R_g, t_g, X, syms):
    X = np.asarray(X, np.float64)
    pe = X @ np.asarray(R_e, np.float64).T + t_e
    best = math.inf
    for Rs, ts in syms:
        pg = (X @ Rs.T + ts) @ np.asarray(R_g, np.float64).T + t_g
        best = min(best, float(np.linalg.norm(pe - pg, axis=1).max()))
    return best


def _project(P, K):
    return np.stack([K[0][0] * P[:, 0] / P[:, 2] + K[0][2], K[1][1] * P[:, 1] / P[:, 2] + K[1][2]], axis=1)


def mspd(R_e, t_e, R_g, t_g, X, syms, K):
    X = np.asarray(X, np.float64)
    K = np.asarray(K, np.float64)
    ue = _project(X @ np.asarray(R_e, np.float64).T + t_e, K)
    best = math.inf
    for Rs, ts in syms:
        ug = _project((X @ Rs.T + ts) @ np.asarray(R_g, np.float64).T + t_g, K)
        best = min(best, float(np.linalg.norm(ue - ug, axis=1).max()))
    return best


U32 = 2.0 ** -24


def mssd_band(t_e, t_g, X, syms):
    """an upper bound on |fp32 kernel - float64| of MSSD: the inputs rounded to fp32, A = R_e - R_g R_s and b = t_e - R_g t_s - t_g
    formed in fp32 (a few rounded operations on values of magnitude <= 3 and <= |t_e| + |t_g| + 3 |t_s|), A x + b and the norm:
    64 units of 2^-24 of the magnitudes involved, a wide factor over the operation count"""
    r = float(np.linalg.norm(np.asarray(X, np.float64), axis=1).max())
    ts = max(float(np.linalg.norm(t)) for _, t in syms)
    return 64 * U32 * (3 * r + float(np.linalg.norm(t_e)) + float(np.linalg.norm(t_g)) + 3 * ts)


def mspd_band(R_e, t_e, t_g, X, syms, K):
    """the same for MSPD: both camera-frame points carry at most E = mssd_band + 64 u (|x| + |t_e|) of absolute error, and
    f x / z moves by at most f E (1 / z + |x, y| / z^2) per point, at the smallest z of the estimate's points, doubled for the
    two points, plus the rounding of the projections"""
    X = np.asarray(X, np.float64)
    pe = X @ np.asarray(R_e, np.float64).T + t_e
    r = float(np.linalg.norm(X, axis=1).max())
    E = mssd_band(t_e, t_g, X, syms) + 64 * U32 * (r + float(np.linalg.norm(t_e)))
    zmin = min(float(pe[:, 2].min()), float(t_g[2]) - r) - 2 * E
    xy = max(float(np.abs(pe[:, :2]).max()), float(np.abs(t_g[:2]).max()) + r)
    f = max(abs(K[0][0]), abs(K[1][1]))
    return 2 * f * E * (1.0 / zmin + xy / zmin ** 2) + 16 * U32 * f * xy / zmin


def distance_image(depth, K):
    """dist(u,v) = depth sqrt(((u - cx) / fx)^2 + ((v - cy) / fy)^2 + 1) at integer pixel indices"""
    depth = np.asarray(depth, np.float64)
    H, W = depth.shape
    K = np.asarray(K, np.float64)
    u = (np.arange(W) - K[0, 2]) / K[0, 0]
    v = (np.arange(H) - K[1, 2]) / K[1, 1]
    return depth * np.sqrt(u[None, :] ** 2 + v[:, None] ** 2 + 1.0)


def vsd_masks(d_e, d_g, d_t, delta):
    """distance images -> (V_g, V_e)"""
    vg = (d_g > 0) & ((d_g - d_t <= delta) | (d_t == 0))
    ve = ((d_e > 0) & ((d_e - d_t <= delta) | (d_t == 0))) | (vg & (d_e > 0))
    return vg, ve


def vsd_counts(dep_e, dep_g, dep_t, K, delta, diameter, taus=TAUS):
    """-> [|U|, |I|, cost count per tau] (ints) from depth images (camera z; test depth in mm)"""
    d_e, d_g, d_t = distance_image(dep_e, K), distance_image(dep_g, K), distance_image(dep_t, K)
    vg, ve = vsd_masks(d_e, d_g, d_t, delta)
    inter = vg & ve
    r = np.abs(d_g - d_e)[inter] / diameter
    return [int((vg | ve).sum()), int(inter.sum())] + [int((r >= tau).sum()) for tau in taus]


def vsd_margin_pixels(dep_e, dep_g, dep_t, K, delta, diameter, taus=TAUS, rel=64 * 2.0 ** -24):
    """pixels at which a decision of vsd_counts flips under a relative perturbation `rel` of every distance: the visibility
    tests d - d_t <= delta and the cost tests |d_g - d_e| / diameter >= tau.  rel bounds fp32 rounding of the distance
    image (a handful of rounded operations, each 2^-24 relative) with a wide factor"""
    d_e, d_g, d_t = distance_image(dep_e, K), distance_image(dep_g, K), distance_image(dep_t, K)
    marg = np.zeros(d_e.shape, bool)
    for d in (d_e, d_g):
        slack = rel * (np.abs(d) + np.abs(d_t)) + 1e-9
        marg |= (d > 0) & (d_t > 0) & (np.abs(d - d_t - delta) <= slack)
    slack = rel * (np.abs(d_g) + np.abs(d_e)) / diameter + 1e-12
    r = np.abs(d_g - d_e) / diameter
    for tau in taus:
        marg |= (d_g > 0) & (d_e > 0) & (np.abs(r - tau) <= slack + rel * tau)
    return int(marg.sum())


def vsd_errors(counts):
    U, I = counts[0], counts[1]
    if U == 0:
        return [1.0] * (len(counts) - 2)
    return [(c + U - I) / U for c in counts[2:]]


def spheres_overlap(t_e, t_g, radius):
    t_e, t_g = np.asarray(t_e, np.float64), np.asarray(t_g, np.float64)
    d = math.hypot(t_e[0] / t_e[2] - t_g[0] / t_g[2], t_e[1] / t_e[2] - t_g[1] / t_g[2])
    return d < radius / t_e[2] + radius / t_g[2]


def match(errors, valid, thr):
    """errors[i][j] of estimate i (in decreasing score order) and GT j; valid[j]; thr -> true positives"""
    matched = set()
    tp = 0
    for row in errors:
        best, best_j = math.inf, -1
        for j, e in enumerate(row):
            if j in matched or not e < thr:
                continue
            if e < best:
                best, best_j = e, j
        if best_j >= 0:
            matched.add(best_j)
            tp += bool(valid[best_j])
    return tp


def _split_dir(root, dataset):
    return os.path.join(root, dataset, "test_primesense" if dataset in ("hb", "tless") else "test")


def vsd_error_range(counts, margin):
    """the range of e(tau) when every count may move by `margin` pixels: the numerator cost + |U| - |I| by 2 margin, |U| by margin"""
    U, I = counts[0], counts[1]
    lo, hi = [], []
    for c in counts[2:]:
        num = c + U - I
        lo.append(max(0.0, (num - 2 * margin) / (U + margin)) if U + margin > 0 else 1.0)
        hi.append(min(1.0, (num + 2 * margin) / (U - margin)) if U - margin > 0 else 1.0)
    if U - margin <= 0:
        hi = [1.0] * len(hi)
    return lo, hi


def evaluate(bop_root, dataset, result_csv, render_depth, targets=None, load_vertices=None):
    """recalls and ARs of a split.  render_depth(obj_id, R, t, K, H, W) -> (H,W) camera-z depth; load_vertices(path) -> (V,3);
    test depth = the stored image x depth_scale rounded to float32 (as the evaluator uploads it).
    -> dict recall_vsd (100, index tau * 10 + theta), recall_mssd (10), recall_mspd (10), ar_*, ar, n_gt, and ambiguous: the
    (pair, threshold) decisions that an fp32 evaluation may take the other way (mssd_band, mspd_band, vsd_margin_pixels)"""
    from PIL import Image
    root = os.path.join(bop_root, dataset)
    with open(targets or os.path.join(root, "test_targets_bop19.json")) as fh:
        tg = json.load(fh)
    mdir = os.path.join(root, "models_eval")
    with open(os.path.join(mdir, "models_info.json")) as fh:
        info = {int(k): v for k, v in json.load(fh).items()}
    ests = []
    with open(result_csv) as fh:
        for line in fh:
            f = line.strip().split(",")
            if len(f) != 7 or f[0] == "scene_id":
                continue
            ests.append(dict(scene=int(f[0]), im=int(f[1]), obj=int(f[2]), score=float(f[3]),
                             R=np.array([float(x) for x in f[4].split()]).reshape(3, 3), t=np.array([float(x) for x in f[5].split()])))
    delta = 5.0 if dataset == "itodd" else 15.0
    tp = dict(vsd=np.zeros(100, np.int64), mssd=np.zeros(10, np.int64), mspd=np.zeros(10, np.int64))
    n_gt = 0
    ambiguous = 0
    cache = {}
    for t in tg:
        s, im, o, cnt = int(t["scene_id"]), int(t["im_id"]), int(t["obj_id"]), int(t["inst_count"])
        sdir = os.path.join(_split_dir(bop_root, dataset), f"{s:06d}")
        if s not in cache:
            cache[s] = [json.load(open(os.path.join(sdir, n))) for n in ("scene_gt.json", "scene_gt_info.json", "scene_camera.json")]
        sgt, sinfo, scam = cache[s]
        K = np.array(scam[str(im)]["cam_K"], np.float64).reshape(3, 3)
        dpath = os.path.join(sdir, "depth", f"{im:06d}.png")
        dep_t = (np.array(Image.open(dpath)).astype(np.float64) * float(scam[str(im)]["depth_scale"])).astype(np.float32)
        H, W = dep_t.shape
        gts = [(g, gi) for g, gi in zip(sgt[str(im)], sinfo[str(im)]) if int(g["obj_id"]) == o]
        valid = [gi["visib_fract"] >= 0.1 for _, gi in gts]
        n_gt += sum(valid)
        mine = [e for e in ests if (e["scene"], e["im"], e["obj"]) == (s, im, o)]
        mine = sorted(mine, key=lambda e: -e["score"])[:cnt]          # sorted() is stable
        if not mine or not gts:
            continue
        X = load_vertices(os.path.join(mdir, f"obj_{o:06d}.ply"))
        syms = symmetries(info[o])
        diam = float(info[o]["diameter"])
        E = {k: [] for k in ("mssd", "mspd", "vsd")}
        for e in mine:
            row = {k: [] for k in E}
            for g, _ in gts:
                Rg, tgt = np.array(g["cam_R_m2c"], np.float64).reshape(3, 3), np.array(g["cam_t_m2c"], np.float64).reshape(3)
                row["mssd"].append(mssd(e["R"], e["t"], Rg, tgt, X, syms))
                row["mspd"].append(mspd(e["R"], e["t"], Rg, tgt, X, syms, K))
                b3, b2 = mssd_band(e["t"], tgt, X, syms), mspd_band(e["R"], e["t"], tgt, X, syms, K)
                ambiguous += sum(abs(row["mssd"][-1] - f * diam) <= b3 for f in MSSD_FRACS)
                ambiguous += sum(abs(row["mspd"][-1] - px * W / 640.0) <= b2 for px in MSPD_PX)
                if spheres_overlap(e["t"], tgt, diam / 2):
                    de, dg = render_depth(o, e["R"], e["t"], K, H, W), render_depth(o, Rg, tgt, K, H, W)
                    c = vsd_counts(de, dg, dep_t, K, delta, diam)
                    lo, hi = vsd_error_range(c, vsd_margin_pixels(de, dg, dep_t, K, delta, diam))
                    ambiguous += sum(lo[a] <= th + 1e-12 and th - 1e-12 <= hi[a] for a in range(10) for th in THETAS)
                    row["vsd"].append(vsd_errors(c))
                else:
                    row["vsd"].append([1.0] * 10)
            for k in E:
                E[k].append(row[k])
        for a, f in enumerate(MSSD_FRACS):
            tp["mssd"][a] += match(E["mssd"], valid, f * diam)
        for a, px in enumerate(MSPD_PX):
            tp["mspd"][a] += match(E["mspd"], valid, px * W / 640.0)
        for a in range(10):
            errs = [[v[a] for v in row] for row in E["vsd"]]
            for b, th in enumerate(THETAS):
                tp["vsd"][a * 10 + b] += match(errs, valid, th)
    out = dict(n_gt=n_gt, ambiguous=int(ambiguous))
    for k in tp:
        out[f"recall_{k}"] = tp[k] / n_gt if n_gt else np.zeros(len(tp[k]))
        out[f"ar_{k}"] = float(np.mean(out[f"recall_{k}"]))
    out["ar"] = (out["ar_vsd"] + out["ar_mssd"] + out["ar_mspd"]) / 3.0
    return out
