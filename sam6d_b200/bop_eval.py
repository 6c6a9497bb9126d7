"""BOP19 pose-task scoring (task 1, localisation with known instance counts) of a result CSV against a BOP test split.

    scores = evaluate_bop19(bop_root, "ycbv", "out/result_ycbv.csv")     # -> ar, ar_vsd, ar_mssd, ar_mspd, recalls, counts

The definitions are those of the BOP Challenge 2019/2020 (Hodan et al., "BOP Challenge 2020 on 6D Object Localization",
ECCVW 2020, sec. 2.2; VSD from Hodan et al., "On Evaluation of 6D Object Pose Estimation", ECCVW 2016), as the BOP toolkit
implements them (misc.get_symmetry_transformations, pose_error.vsd / mssd / mspd, pose_matching.match_poses):

* estimates per target: the inst_count estimates of a (scene, image, object) with the highest score, a stable sort (ties keep
  file order); estimates that match no target are ignored;
* symmetries (symmetry_transforms): the identity plus each symmetries_discrete entry; each continuous entry (axis, offset)
  becomes the rotations by i 2 pi / n about the axis, i = 1..n-1, n = ceil(pi / 0.01) = 315, with t = -R offset + offset; with
  continuous entries the set is every composition (R_c R_d, R_c t_d + t_c), so it holds no identity of its own;
* MSSD = min over symmetries S of max over model vertices x of |(R_e x + t_e) - (R_g S x + t_g)| (mm); MSPD the same between
  the projections through K (px); thresholds 0.05..0.50 x diameter and 5..50 x (image width / 640) px;
* VSD: depth of the model rendered at both poses (render.render), distance images dist = depth sqrt(((u - cx) / fx)^2 +
  ((v - cy) / fy)^2 + 1), V_g = d_g > 0 and (d_g - d_test <= delta or d_test = 0), V_e the same on d_e or-ed with (V_g and
  d_e > 0), e(tau) = (#{p in V_g & V_e : |d_g - d_e| / diameter >= tau} + |V_g | V_e| - |V_g & V_e|) / |V_g | V_e| (1 when
  empty); delta = 15 mm (5 mm on itodd), tau = 0.05..0.50, correctness thresholds theta = 0.05..0.50 for every tau; e = 1 for
  every tau when the projected bounding spheres (radius diameter / 2 about t) do not overlap, and such pairs are not rendered;
* matching per threshold within a (scene, image, object): estimates in decreasing score order each take the unmatched GT
  instance with the smallest error below the threshold; GT instances with visib_fract < 0.1 can be matched but count neither as
  true positives nor in the denominator; recall = sum of true positives / sum of valid GT instances over the split; AR_X = the
  mean recall over X's thresholds, AR = the mean of AR_VSD, AR_MSSD and AR_MSPD.

MSSD / MSPD and the VSD pixel counts run on the GPU (csrc/bop_eval.cu); reading, the sphere test, matching and the recalls stay
on the host.  Renders are batched per (object, K, image size) and chunked so render()'s outputs stay within
RENDER_BUDGET_BYTES.  The rasteriser drops a triangle with a vertex at z <= 1e-3 mm (no clipping), where OpenGL would clip it."""
import functools
import json
import math
import os
import sys
import warnings
from collections import OrderedDict

import numpy as np
import torch

from . import _lib, bop, meshio, pbr, render

ERROR_TYPES = ("vsd", "mssd", "mspd")
VSD_TAUS = np.arange(0.05, 0.51, 0.05)           # misfit tolerance, fraction of the diameter
VSD_THETAS = np.arange(0.05, 0.51, 0.05)         # correctness thresholds of e_VSD
MSSD_FRACS = np.arange(0.05, 0.51, 0.05)         # x diameter, mm
MSPD_PX = np.arange(5, 51, 5).astype(np.float64)  # x (image width / 640), px
VSD_DELTA = 15.0
VSD_DELTA_ITODD = 5.0
MIN_VISIB_FRACT = 0.1
MAX_SYM_DISC_STEP = 0.01
# render() keeps rgb, mask, xyz, tri, depth and the u64 visibility buffer of every view: 26 bytes per pixel
RENDER_BYTES_PER_PIXEL = 26
RENDER_BUDGET_BYTES = 1 << 30
MAX_VSD_PAIRS_PER_CALL = 65535


# ---- readers -----------------------------------------------------------------------------------------------------------------
def load_targets(path: str):
    """test_targets_bop19.json -> [(scene_id, im_id, obj_id, inst_count)] in file order"""
    with open(path) as fh:
        data = json.load(fh)
    try:
        return [(int(d["scene_id"]), int(d["im_id"]), int(d["obj_id"]), int(d["inst_count"])) for d in data]
    except (KeyError, TypeError) as e:
        raise ValueError(f"{path}: every target needs scene_id, im_id, obj_id and inst_count ({e})") from None


def load_results(path: str):
    """a BOP results CSV (bop.csv_rows: scene_id,im_id,obj_id,score,R,t,time; R row-major, t in mm; an optional header line)
    -> dict of scene_id, im_id, obj_id (n,) i64, score (n,) f64, R (n,3,3) f64, t (n,3) f64, in file order"""
    cols = {k: [] for k in ("scene_id", "im_id", "obj_id", "score", "R", "t")}
    with open(path) as fh:
        for ln, line in enumerate(fh, 1):
            line = line.strip()
            if not line or (ln == 1 and line.startswith("scene_id")):
                continue
            f = line.split(",")
            try:
                if len(f) != 7:
                    raise ValueError(f"{len(f)} fields")
                R = [float(v) for v in f[4].split()]
                t = [float(v) for v in f[5].split()]
                if len(R) != 9 or len(t) != 3:
                    raise ValueError(f"R has {len(R)} values and t {len(t)}")
                row = (int(f[0]), int(f[1]), int(f[2]), float(f[3]))
            except ValueError as e:
                raise ValueError(f"{path}:{ln}: expected scene_id,im_id,obj_id,score,R (9),t (3),time ({e})") from None
            for k, v in zip(("scene_id", "im_id", "obj_id", "score"), row):
                cols[k].append(v)
            cols["R"].append(R)
            cols["t"].append(t)
    n = len(cols["score"])
    return dict(scene_id=np.array(cols["scene_id"], np.int64), im_id=np.array(cols["im_id"], np.int64),
                obj_id=np.array(cols["obj_id"], np.int64), score=np.array(cols["score"], np.float64),
                R=np.array(cols["R"], np.float64).reshape(n, 3, 3), t=np.array(cols["t"], np.float64).reshape(n, 3))


def models_eval_dir(bop_root: str, dataset_name: str) -> str:
    """<dataset>/models_eval, or bop.model_dir()'s folder with a warning when the dataset has no models_eval"""
    d = os.path.join(bop_root, dataset_name, "models_eval")
    if os.path.isdir(d):
        return d
    fallback = os.path.join(bop_root, dataset_name, bop.model_dir(dataset_name))
    warnings.warn(f"{d} not found: scoring with the models of {fallback} instead")
    return fallback


def load_models_info(path: str):
    """models_info.json -> {obj_id: info dict}"""
    with open(path) as fh:
        return {int(k): v for k, v in json.load(fh).items()}


def symmetry_transforms(info, max_sym_disc_step: float = MAX_SYM_DISC_STEP):
    """the symmetry set of one models_info entry (module docstring) -> (R (S,3,3), t (S,3)) float64, t in mm"""
    disc = [(np.eye(3), np.zeros(3))]
    for m in info.get("symmetries_discrete", []):
        m = np.asarray(m, np.float64).reshape(4, 4)
        disc.append((m[:3, :3], m[:3, 3]))
    cont = []
    for sym in info.get("symmetries_continuous", []):
        axis = np.asarray(sym["axis"], np.float64)
        axis = axis / np.linalg.norm(axis)
        offset = np.asarray(sym["offset"], np.float64).reshape(3)
        n = int(math.ceil(math.pi / max_sym_disc_step))
        for i in range(1, n):
            R = _axis_angle(axis, i * 2.0 * math.pi / n)
            cont.append((R, -R @ offset + offset))
    if cont:
        pairs = [(Rc @ Rd, Rc @ td + tc) for Rd, td in disc for Rc, tc in cont]
    else:
        pairs = disc
    return np.stack([p[0] for p in pairs]), np.stack([p[1] for p in pairs])


def _axis_angle(axis, angle):
    """Rodrigues: rotation by angle about the unit axis"""
    x, y, z = axis
    K = np.array([[0.0, -z, y], [z, 0.0, -x], [-y, x, 0.0]])
    return np.eye(3) + math.sin(angle) * K + (1.0 - math.cos(angle)) * (K @ K)


# ---- kernels ------------------------------------------------------------------------------------------------------------------
def _dev(a, dtype, device):
    if isinstance(a, torch.Tensor):
        return a.to(device=device, dtype=dtype).contiguous()
    return torch.from_numpy(np.ascontiguousarray(a)).to(device=device, dtype=dtype).contiguous()


def mssd_mspd(est, gt, pair_obj, K, verts, syms, device="cuda") -> torch.Tensor:
    """MSSD (mm) and MSPD (px) of P pairs on the GPU (csrc/bop_eval.cu).  est, gt (P,12): R row-major then t (mm); pair_obj (P)
    object index; K (P,4) fx, fy, cx, cy of each pair's image; verts: per object (V,3) vertices (mm); syms: per object (S,12)
    symmetry transforms (R row-major, t), S >= 1.  Arrays or tensors, computed in fp32 -> (P,2) f32 on the device"""
    device = torch.device(device)
    O = len(verts)
    if O == 0 or len(syms) != O:
        raise ValueError("mssd_mspd: one vertex array and one symmetry set per object")
    est, gt, K = _dev(est, torch.float32, device), _dev(gt, torch.float32, device), _dev(K, torch.float32, device)
    pair_obj = _dev(pair_obj, torch.int32, device)
    P = est.shape[0]
    if est.shape != (P, 12) or gt.shape != (P, 12) or K.shape != (P, 4) or pair_obj.shape != (P,):
        raise ValueError("mssd_mspd: est, gt (P,12), K (P,4), pair_obj (P,)")
    if P and (int(pair_obj.min()) < 0 or int(pair_obj.max()) >= O):
        raise ValueError(f"mssd_mspd: pair_obj outside [0, {O})")
    nv = [int(v.shape[0]) for v in verts]
    ns = [int(s.shape[0]) for s in syms]
    if min(ns) < 1 or min(nv) < 1:
        raise ValueError("mssd_mspd: every object needs vertices and at least one symmetry (the identity)")
    V = torch.cat([_dev(v, torch.float32, device).reshape(-1, 3) for v in verts]).contiguous()
    S = torch.cat([_dev(s, torch.float32, device).reshape(-1, 12) for s in syms]).contiguous()
    voff = _dev(np.concatenate([[0], np.cumsum(nv)]), torch.int32, device)
    soff = _dev(np.concatenate([[0], np.cumsum(ns)]), torch.int32, device)
    out = torch.empty(P, 2, dtype=torch.float32, device=device)
    _lib.call("sam6d_bop_mssd_mspd", est, gt, pair_obj, K, P, V, voff, S, soff, O, max(ns), out)
    return out


def vsd_counts(depth_est, depth_gt, depth_test, pair_img, K, delta: float, diameter: float, taus=VSD_TAUS) -> torch.Tensor:
    """VSD pixel counts on the GPU (csrc/bop_eval.cu).  depth_est, depth_gt (P,H,W) f32 CUDA rendered camera z (0 = empty),
    depth_test (N,H,W) f32 CUDA test depth in mm, pair_img (P) its image; K (3,3) of all pairs; delta and diameter in mm, taus
    (10) fractions of the diameter -> (P,12) i32: |U|, |I|, then #{p in I : |d_g - d_e| / diameter >= tau} per tau"""
    for name, t in (("depth_est", depth_est), ("depth_gt", depth_gt), ("depth_test", depth_test)):
        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.float32 or t.dim() != 3:
            raise RuntimeError(f"vsd_counts: {name} must be a CUDA float32 (n,H,W) tensor")
    P, H, W = depth_est.shape
    if tuple(depth_gt.shape) != (P, H, W) or tuple(depth_test.shape[1:]) != (H, W):
        raise ValueError("vsd_counts: depth_est, depth_gt (P,H,W) and depth_test (N,H,W) must share H and W")
    if P > MAX_VSD_PAIRS_PER_CALL:
        raise ValueError(f"vsd_counts: at most {MAX_VSD_PAIRS_PER_CALL} pairs per call")
    dev = depth_est.device
    pair_img = _dev(pair_img, torch.int32, dev)
    if pair_img.shape != (P,) or (P and (int(pair_img.min()) < 0 or int(pair_img.max()) >= depth_test.shape[0])):
        raise ValueError(f"vsd_counts: pair_img must be (P,) indices into the {depth_test.shape[0]} test depths")
    taus = _dev(np.asarray(taus, np.float32).reshape(-1), torch.float32, dev)
    if taus.numel() != 10:
        raise ValueError("vsd_counts: 10 taus")
    K = np.asarray(K.cpu() if isinstance(K, torch.Tensor) else K, np.float64).reshape(3, 3)
    de, dg, dt = depth_est.contiguous(), depth_gt.contiguous(), depth_test.contiguous()
    out = torch.empty(P, 12, dtype=torch.int32, device=dev)
    _lib.call("sam6d_bop_vsd_counts", de, dg, dt, pair_img, P, H, W, float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]),
              float(delta), float(diameter), taus, out)
    return out


def vsd_errors(counts: np.ndarray) -> np.ndarray:
    """(n,12) counts -> (n,10) e(tau) = (cost + |U| - |I|) / |U|, 1 where |U| = 0"""
    counts = np.asarray(counts, np.int64)
    U, I, cost = counts[:, :1], counts[:, 1:2], counts[:, 2:]
    with np.errstate(divide="ignore", invalid="ignore"):
        e = (cost + U - I) / U.astype(np.float64)
    return np.where(U > 0, e, 1.0)


def spheres_overlap(t_est: np.ndarray, t_gt: np.ndarray, radius) -> np.ndarray:
    """the VSD shortcut: do the projections of the spheres of `radius` about t_est and t_gt (n,3) overlap?"""
    t_est, t_gt = np.asarray(t_est, np.float64), np.asarray(t_gt, np.float64)
    d = np.linalg.norm(t_est[:, :2] / t_est[:, 2:] - t_gt[:, :2] / t_gt[:, 2:], axis=1)
    return d < radius * (1.0 / t_est[:, 2] + 1.0 / t_gt[:, 2])


# ---- matching -----------------------------------------------------------------------------------------------------------------
def match_count(err: np.ndarray, thr: np.ndarray, valid: np.ndarray) -> np.ndarray:
    """greedy matching of one (scene, image, object) at n thresholds: err (n, n_est, n_gt) with the estimates in decreasing score
    order, thr (n,), valid (n_gt,) bool -> (n,) true positives: each estimate takes the unmatched GT with the smallest error
    below the threshold (the first on a tie); a match of an invalid GT counts nothing"""
    n, n_est, n_gt = err.shape
    tp = np.zeros(n, np.int64)
    if n_est == 0 or n_gt == 0:
        return tp
    err = np.where(np.isnan(err), np.inf, err)
    matched = np.zeros((n, n_gt), bool)
    rows = np.arange(n)
    for i in range(n_est):
        e = np.where(matched | (err[:, i, :] >= thr[:, None]), np.inf, err[:, i, :])
        j = np.argmin(e, axis=1)
        ok = np.isfinite(e[rows, j])
        matched[rows[ok], j[ok]] = True
        tp += ok & valid[j]
    return tp


# ---- the split ----------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=64)
def _test_depth_mm(path: str, depth_scale: float) -> np.ndarray:
    return (bop.decode_depth(path).astype(np.float64) * depth_scale).astype(np.float32)


def _image_size(path: str):
    from PIL import Image
    with Image.open(path) as im:
        return im.size[1], im.size[0]


def evaluate_bop19(bop_root: str, dataset_name: str, result_csv: str, targets=None, error_types=ERROR_TYPES, device=None) -> dict:
    """BOP19 scores of result_csv on <bop_root>/<dataset_name> (module docstring).  targets: the targets file (default
    <dataset>/test_targets_bop19.json).  error_types: any of "vsd", "mssd", "mspd"; "ar" is the mean of their ARs (BOP's AR
    with all three).  -> dict: ar, ar_<type>, recall_<type> (per threshold; VSD as a 10 x 10 list [tau][theta]), thresholds,
    n_targets (target entries), n_estimates (estimates kept for a target), n_gt (valid GT instances), n_pairs (estimate-GT
    pairs scored)"""
    error_types = tuple(error_types)
    if not error_types or any(e not in ERROR_TYPES for e in error_types):
        raise ValueError(f"error_types must be a non-empty subset of {ERROR_TYPES}, got {error_types}")
    device = torch.device(device if device is not None else "cuda")
    ds_root = os.path.join(bop_root, dataset_name)
    targets = load_targets(targets if targets is not None else os.path.join(ds_root, "test_targets_bop19.json"))
    res = load_results(result_csv)

    # ground truth and cameras of the split
    split = bop.split_name(dataset_name)
    frames = {(f.scene_id, f.frame_id): f for f in bop.scan_test_split(bop_root, dataset_name)}
    rows = pbr.scan_rows(ds_root, split, max_num_scenes=None, max_num_frames=sys.maxsize)
    gt_of = {}
    for k in range(len(rows)):
        gt_of.setdefault((int(rows.scene_id[k]), int(rows.frame_id[k]), int(rows.obj_id[k])), []).append(k)

    # estimates kept per target
    want = OrderedDict()
    for s, i, o, n in targets:
        want[(s, i, o)] = want.get((s, i, o), 0) + n
    cand = {}
    for r in range(len(res["score"])):
        key = (int(res["scene_id"][r]), int(res["im_id"][r]), int(res["obj_id"][r]))
        if key in want:
            cand.setdefault(key, []).append(r)
    kept = {}
    for key, rs in cand.items():
        rs = np.asarray(rs)
        kept[key] = rs[np.argsort(-res["score"][rs], kind="stable")][:want[key]]

    obj_ids = sorted({o for _, _, o in want})
    mdir = models_eval_dir(bop_root, dataset_name)
    info = load_models_info(os.path.join(mdir, "models_info.json"))
    for o in obj_ids:
        if o not in info:
            raise ValueError(f"object {o} has no entry in {os.path.join(mdir, 'models_info.json')}")
    diam = {o: float(info[o]["diameter"]) for o in obj_ids}

    # pairs: every kept estimate of a target with every GT instance of its object in the image
    pe, pg, pk, n_gt = [], [], [], 0
    images = {}
    for key in want:
        if (key[0], key[1]) not in frames:
            raise ValueError(f"target scene {key[0]} image {key[1]} is not in {os.path.join(ds_root, split)}")
        g = gt_of.get(key, [])
        n_gt += sum(rows.visib_fract[k] >= MIN_VISIB_FRACT for k in g)
        for r in kept.get(key, []):
            for k in g:
                pe.append(r)
                pg.append(k)
                pk.append(key)
        if (key[0], key[1]) not in images:
            f = frames[(key[0], key[1])]
            images[(key[0], key[1])] = (np.asarray(f.cam_K, np.float64).reshape(3, 3), _image_size(f.depth_path), f)
    pe, pg = np.asarray(pe, np.int64), np.asarray(pg, np.int64)
    P = len(pe)
    pair_obj_id = np.array([k[2] for k in pk], np.int64)
    R_e, t_e = res["R"][pe].reshape(P, 3, 3), res["t"][pe].reshape(P, 3)
    R_g, t_g = rows.poses[pg][:, :3, :3].reshape(P, 3, 3), rows.poses[pg][:, :3, 3].reshape(P, 3)

    models = {}
    if P:
        for o in sorted(set(pair_obj_id.tolist())):
            path = os.path.join(mdir, f"obj_{o:06d}.ply")
            if not os.path.exists(path):
                raise FileNotFoundError(f"no model {path}")
            v, f, _ = meshio.load_ply(path)
            models[o] = (v, f)

    err = {}
    if P and ("mssd" in error_types or "mspd" in error_types):
        objs = sorted(models)
        oidx = {o: i for i, o in enumerate(objs)}
        syms = []
        for o in objs:
            sR, st = symmetry_transforms(info[o])
            syms.append(np.concatenate([sR.reshape(-1, 9), st], axis=1))
        Kp = np.array([[*images[(k[0], k[1])][0][[0, 1, 0, 1], [0, 1, 2, 2]]] for k in pk], np.float64)
        out = mssd_mspd(np.concatenate([R_e.reshape(P, 9), t_e], 1), np.concatenate([R_g.reshape(P, 9), t_g], 1),
                        np.array([oidx[o] for o in pair_obj_id], np.int32), Kp, [models[o][0] for o in objs], syms, device)
        out = out.cpu().numpy().astype(np.float64)
        err["mssd"], err["mspd"] = out[:, 0], out[:, 1]
    if P and "vsd" in error_types:
        try:
            err["vsd"] = _vsd_errors(dataset_name, pk, pair_obj_id, R_e, t_e, R_g, t_g, images, models, diam, device)
        finally:
            _test_depth_mm.cache_clear()          # decoded test depth is kept only while one evaluation runs

    # matching per target and threshold
    thr_def = {"vsd": VSD_THETAS, "mssd": MSSD_FRACS, "mspd": MSPD_PX}
    tp = {e: np.zeros(100 if e == "vsd" else 10, np.int64) for e in error_types}
    by_key = {}
    for i, key in enumerate(pk):
        by_key.setdefault(key, []).append(i)
    n_est = 0
    for key in want:
        ests = kept.get(key, [])
        n_est += len(ests)
        g = gt_of.get(key, [])
        if not len(ests) or not g:
            continue
        idx = np.asarray(by_key[key]).reshape(len(ests), len(g))       # pairs were made estimate-major
        valid = rows.visib_fract[g] >= MIN_VISIB_FRACT
        width = images[(key[0], key[1])][1][1]
        for e in error_types:
            if e == "vsd":
                E = np.repeat(np.moveaxis(err["vsd"][idx], 2, 0), len(VSD_THETAS), axis=0)    # (tau x theta, est, gt)
                thr = np.tile(VSD_THETAS, len(VSD_TAUS))
            else:
                thr = MSSD_FRACS * diam[key[2]] if e == "mssd" else MSPD_PX * (width / 640.0)
                E = np.broadcast_to(err[e][idx], (len(thr),) + idx.shape)
            tp[e] += match_count(E, thr, valid)

    out = dict(n_targets=len(targets), n_estimates=int(n_est), n_gt=int(n_gt), n_pairs=int(P),
               thresholds=dict(vsd_tau=VSD_TAUS.tolist(), vsd_theta=VSD_THETAS.tolist(), mssd_diameter_fraction=MSSD_FRACS.tolist(),
                               mspd_px_at_640=MSPD_PX.tolist()))
    ars = []
    for e in error_types:
        rec = tp[e] / n_gt if n_gt else np.zeros_like(tp[e], np.float64)
        out[f"recall_{e}"] = rec.reshape(10, 10).tolist() if e == "vsd" else rec.tolist()
        out[f"ar_{e}"] = float(rec.mean())
        ars.append(out[f"ar_{e}"])
    out["ar"] = float(np.mean(ars))
    return out


def _vsd_errors(dataset_name, pk, pair_obj_id, R_e, t_e, R_g, t_g, images, models, diam, device):
    """(P,10) e_VSD of every pair: 1 where the sphere test fails, else from the rendered depths and the kernel's counts"""
    P = len(pk)
    e = np.ones((P, len(VSD_TAUS)))
    radius = np.array([diam[o] for o in pair_obj_id]) / 2.0
    live = np.flatnonzero(spheres_overlap(t_e, t_g, radius))
    delta = VSD_DELTA_ITODD if dataset_name == "itodd" else VSD_DELTA
    groups = OrderedDict()
    for i in live:
        K, (H, W), _ = images[(pk[i][0], pk[i][1])]
        groups.setdefault((int(pair_obj_id[i]), tuple(K.reshape(-1).tolist()), H, W), []).append(i)
    for (o, Kt, H, W), sel in groups.items():
        v, f = models[o]
        if len(f) == 0:
            raise ValueError(f"object {o}: the model has no faces, so VSD cannot render it")
        mesh = render.upload(meshio.Mesh(v, f.astype(np.int32)), device)
        K = np.asarray(Kt).reshape(3, 3)
        step = max(1, min(MAX_VSD_PAIRS_PER_CALL, RENDER_BUDGET_BYTES // (2 * H * W * RENDER_BYTES_PER_PIXEL)))
        for c0 in range(0, len(sel), step):
            ch = np.asarray(sel[c0:c0 + step])
            n = len(ch)
            poses = np.zeros((1, 2 * n, 4, 4), np.float32)
            poses[0, :n, :3, :3], poses[0, :n, :3, 3] = R_e[ch], t_e[ch]
            poses[0, n:, :3, :3], poses[0, n:, :3, 3] = R_g[ch], t_g[ch]
            poses[0, :, 3, 3] = 1.0
            depth = render.render([mesh], torch.from_numpy(poses).to(device), K, H, W)["depth"][0]
            imgs = list(OrderedDict.fromkeys((pk[i][0], pk[i][1]) for i in ch))
            slot = {k: j for j, k in enumerate(imgs)}
            test = []
            for k in imgs:
                fr = images[k][2]
                d = _test_depth_mm(fr.depth_path, float(fr.depth_scale))
                if d.shape != (H, W):
                    raise ValueError(f"{fr.depth_path}: depth {d.shape} does not match the image size {(H, W)}")
                test.append(d)
            dt = torch.from_numpy(np.stack(test)).to(device)
            counts = vsd_counts(depth[:n], depth[n:], dt, np.array([slot[(pk[i][0], pk[i][1])] for i in ch], np.int32), K, delta,
                                diam[o])
            e[ch] = vsd_errors(counts.cpu().numpy())
            del depth, dt
    return e
