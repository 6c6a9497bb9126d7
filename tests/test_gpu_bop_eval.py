"""GPU: BOP19 scoring (sam6d_b200/bop_eval.py, csrc/bop_eval.cu) against the float64 oracle (oracle/bop_eval_oracle.py) on a
synthetic split built here: three procedural meshes (an ellipsoid, a cylinder with a continuous symmetry about z, a box with a
discrete one), two scenes of different image sizes, test depth rendered at the GT poses, and result CSVs with perturbations of
known size.

Bounds (stated in the oracle): MSSD / MSPD of the kernel are within mssd_band / mspd_band of the float64 values computed from
the same fp32 inputs (a wide multiple of 2^-24 of the magnitudes the residual form and the projection handle).  VSD counts
differ from the oracle's at most by the pixels whose visibility or cost decision lies within 64 x 2^-24 (relative) of its
threshold.  evaluate_bop19's recalls equal the oracle's exactly once no (pair, threshold) decision lies inside those bands,
which the test asserts of its fixture."""
import json
import math
import os
import shutil

import numpy as np
import pytest
import torch

from oracle import bop_eval_oracle as bo
from oracle import render_oracle as ro
from sam6d_b200 import bop, bop_eval, meshio, render
from sam6d_b200.cli import eval_bop

pytestmark = pytest.mark.gpu

FLIP_Z = [-1, 0, 0, 0, 0, -1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1]
DEPTH_SCALE = 0.1
# (scene_id, im_id, height, width, focal, [(obj_id, visib_fract), ...])
IMAGES = [(1, 0, 480, 640, 600.0, [(1, 0.9), (1, 0.8), (2, 0.95)]),
          (1, 4, 480, 640, 600.0, [(2, 0.7), (3, 0.9), (1, 0.6)]),
          (2, 1, 240, 320, 300.0, [(3, 0.9), (3, 0.05), (1, 0.5)])]


def cylinder(r, h, n):
    a = 2 * np.pi * np.arange(n) / n
    ring = np.stack([r * np.cos(a), r * np.sin(a)], 1)
    v = np.concatenate([np.c_[ring, np.full(n, -h / 2)], np.c_[ring, np.full(n, h / 2)], [[0, 0, -h / 2], [0, 0, h / 2]]])
    f = []
    for i in range(n):
        j = (i + 1) % n
        f += [[i, j, n + j], [i, n + j, n + i], [2 * n, j, i], [2 * n + 1, n + i, n + j]]
    return v.astype(np.float32), np.asarray(f, np.int32)


def box(a, b, c, n):
    """a box subdivided into n x n quads per face (vertices on the surface for MSSD)"""
    vs, fs = [], []
    g = np.linspace(-1, 1, n + 1)
    for axis in range(3):
        for sign in (-1.0, 1.0):
            base = len(vs and np.concatenate(vs))
            uu, ww = np.meshgrid(g, g, indexing="ij")
            p = np.zeros(((n + 1) ** 2, 3))
            p[:, axis] = sign
            p[:, (axis + 1) % 3], p[:, (axis + 2) % 3] = uu.reshape(-1), ww.reshape(-1)
            vs.append(p)
            for i in range(n):
                for k in range(n):
                    q = base + i * (n + 1) + k
                    fs += [[q, q + n + 1, q + n + 2], [q, q + n + 2, q + 1]]
    v = np.concatenate(vs) * np.array([a, b, c])
    return v.astype(np.float32), np.asarray(fs, np.int32)


def make_meshes(detail=1):
    """{obj_id: (vertices (V,3) f32 mm, faces (F,3) i32)}: detail scales the vertex counts"""
    v1, f1 = ro.icosphere(1 + detail, 1.0)
    return {1: (v1 * np.array([40.0, 25.0, 15.0], np.float32), f1), 2: cylinder(20.0, 50.0, 24 * detail),
            3: box(25.0, 15.0, 10.0, 2 * detail)}


def models_info(meshes):
    info = {}
    for o, (v, _) in meshes.items():
        d = np.linalg.norm(v[:, None].astype(np.float64) - v[None], axis=2).max() if len(v) < 6000 else 2 * np.linalg.norm(v, axis=1).max()
        info[str(o)] = {"diameter": float(d)}
    info["2"]["symmetries_continuous"] = [{"axis": [0, 0, 1], "offset": [0, 0, 0]}]
    info["3"]["symmetries_discrete"] = [FLIP_Z]
    return info


def write_ply(path, v, f):
    with open(path, "w") as fh:
        fh.write(f"ply\nformat ascii 1.0\nelement vertex {len(v)}\nproperty float x\nproperty float y\nproperty float z\n"
                 f"element face {len(f)}\nproperty list uchar int vertex_indices\nend_header\n")
        fh.writelines(f"{x!r} {y!r} {z!r}\n" for x, y, z in v.tolist())
        fh.writelines(f"3 {a} {b} {c}\n" for a, b, c in f.tolist())


def _rot(rng):
    from scipy.spatial.transform import Rotation
    return Rotation.random(random_state=rng).as_matrix()


def write_split(root, dataset="toy", images=IMAGES, meshes=None, seed=0):
    """a BOP split at root/dataset: models_eval, test/<scene>/{rgb,depth,scene_*.json}, test_targets_bop19.json.  Each image's
    instances sit on a grid across the image at 600-900 mm; the test depth is the nearest rendered GT surface in units of
    DEPTH_SCALE mm.  -> list of GT records (scene_id, im_id, obj_id, R, t, visib_fract, W)"""
    from PIL import Image
    meshes = meshes or make_meshes()
    rng = np.random.RandomState(seed)
    ds = os.path.join(root, dataset)
    os.makedirs(os.path.join(ds, "models_eval"), exist_ok=True)
    for o, (v, f) in meshes.items():
        write_ply(os.path.join(ds, "models_eval", f"obj_{o:06d}.ply"), v, f)
    with open(os.path.join(ds, "models_eval", "models_info.json"), "w") as fh:
        json.dump(models_info(meshes), fh)
    dev = {o: render.upload(meshio.Mesh(v, f)) for o, (v, f) in meshes.items()}
    scenes, gts, targets = {}, [], []
    for s, im, H, W, foc, insts in images:
        K = np.array([[foc, 0, W / 2 - 0.5], [0, foc, H / 2 + 0.25], [0, 0, 1]])
        depth = np.zeros((H, W), np.float32)
        scene = scenes.setdefault(s, ({}, {}, {}))
        scene[0][str(im)], scene[1][str(im)] = [], []
        scene[2][str(im)] = {"cam_K": K.reshape(-1).tolist(), "depth_scale": DEPTH_SCALE}
        counts = {}
        for k, (o, vis) in enumerate(insts):
            z = 600.0 + 300.0 * rng.rand()
            cx = (k + 0.5) / len(insts) * W - W / 2 + rng.uniform(-10, 10)
            t = np.array([cx * z / foc, rng.uniform(-0.15, 0.15) * H * z / foc, z])
            R = _rot(rng)
            pose = np.eye(4, dtype=np.float32)
            pose[:3, :3], pose[:3, 3] = R, t
            d = render.render([dev[o]], torch.from_numpy(pose[None, None]).cuda(), K, H, W)["depth"][0, 0].cpu().numpy()
            depth = np.where((d > 0) & ((depth == 0) | (d < depth)), d, depth)
            R32, t32 = pose[:3, :3].astype(np.float64), pose[:3, 3].astype(np.float64)
            scene[0][str(im)].append({"cam_R_m2c": R32.reshape(-1).tolist(), "cam_t_m2c": t32.tolist(), "obj_id": o})
            scene[1][str(im)].append({"visib_fract": vis})
            gts.append(dict(scene_id=s, im_id=im, obj_id=o, R=R32, t=t32, visib=vis, W=W))
            counts[o] = counts.get(o, 0) + (vis >= 0.1)
        targets += [{"scene_id": s, "im_id": im, "obj_id": o, "inst_count": n} for o, n in counts.items() if n]
        sdir = os.path.join(ds, "test", f"{s:06d}")
        os.makedirs(os.path.join(sdir, "rgb"), exist_ok=True)
        os.makedirs(os.path.join(sdir, "depth"), exist_ok=True)
        Image.fromarray(np.zeros((H, W, 3), np.uint8)).save(os.path.join(sdir, "rgb", f"{im:06d}.png"))
        Image.fromarray(np.round(depth / DEPTH_SCALE).astype(np.uint16)).save(os.path.join(sdir, "depth", f"{im:06d}.png"))
    for s, (g, gi, cam) in scenes.items():
        sdir = os.path.join(ds, "test", f"{s:06d}")
        for name, obj in (("scene_gt", g), ("scene_gt_info", gi), ("scene_camera", cam)):
            with open(os.path.join(sdir, f"{name}.json"), "w") as fh:
                json.dump(obj, fh)
    with open(os.path.join(ds, "test_targets_bop19.json"), "w") as fh:
        json.dump(targets, fh)
    return gts


def write_results(path, gts, mode, seed=1):
    """mode "gt": every GT pose, valid instances scored above invalid ones; "far": every GT pose moved 2 m sideways;
    "perturbed": per GT a translation of 0.005-0.6 x the diameter and a rotation of up to 25 degrees (every other GT's
    best estimate within 0.05 x the diameter and 2 degrees), a second lower-scored
    estimate per object of an image (beyond inst_count where there is one instance), and estimates of objects and images
    that are not targets"""
    from scipy.spatial.transform import Rotation
    rng = np.random.RandomState(seed)
    diam = {1: 2 * 40.0, 2: 2 * math.hypot(20, 25), 3: 2 * math.sqrt(25 ** 2 + 15 ** 2 + 10 ** 2)}
    lines = []
    for k, g in enumerate(gts):
        R, t = g["R"], g["t"].copy()
        if mode == "gt":
            lines += bop.csv_rows(g["scene_id"], g["im_id"], [g["obj_id"]], [0.9 if g["visib"] >= 0.1 else 0.2], [R], [t], 0.5)
        elif mode == "far":
            lines += bop.csv_rows(g["scene_id"], g["im_id"], [g["obj_id"]], [0.9], [R], [t + [2000.0, 0, 0]], 0.5)
        else:
            for j, score in enumerate((rng.uniform(0.5, 1.0), rng.uniform(0.0, 0.5))):
                # every other GT's best estimate is close (up to 0.05 x diameter, 2 degrees), the rest spread wide
                near = j == 0 and k % 2 == 0
                d = rng.randn(3)
                d *= rng.uniform(0.005, 0.05 if near else 0.6) * diam[g["obj_id"]] / np.linalg.norm(d)
                deg = rng.uniform(0, 2 if near else 25)
                Rp = Rotation.from_rotvec(rng.randn(3) * np.radians(deg) / math.sqrt(3)).as_matrix() @ R
                lines += bop.csv_rows(g["scene_id"], g["im_id"], [g["obj_id"]], [score], [Rp], [t + d], 0.5)
            if k == 0:
                lines += bop.csv_rows(g["scene_id"], g["im_id"], [7], [0.99], [R], [t], 0.5)        # not a target object
                lines += bop.csv_rows(g["scene_id"], 99, [g["obj_id"]], [0.99], [R], [t], 0.5)      # not a target image
    with open(path, "w") as fh:
        fh.writelines(lines)
    return path


@pytest.fixture(scope="module")
def split(tmp_path_factory):
    root = str(tmp_path_factory.mktemp("bop_eval"))
    gts = write_split(root)
    shutil.copytree(os.path.join(root, "toy"), os.path.join(root, "itodd"))
    return root, gts


def _meshes_of(root, dataset="toy"):
    out = {}
    for o in (1, 2, 3):
        v, f, _ = meshio.load_ply(os.path.join(root, dataset, "models_eval", f"obj_{o:06d}.ply"))
        out[o] = (v, f.astype(np.int32))
    return out


def _render_fn(meshes):
    dev = {o: render.upload(meshio.Mesh(v, f)) for o, (v, f) in meshes.items()}

    def fn(o, R, t, K, H, W):
        pose = np.eye(4, dtype=np.float32)
        pose[:3, :3], pose[:3, 3] = R, t
        return render.render([dev[o]], torch.from_numpy(pose[None, None]).cuda(), K, H, W)["depth"][0, 0].cpu().numpy()
    return fn


def test_kernels_match_oracle(split, tmp_path):
    root, gts = split
    meshes = _meshes_of(root)
    info = json.load(open(os.path.join(root, "toy", "models_eval", "models_info.json")))
    res = bop_eval.load_results(write_results(str(tmp_path / "r.csv"), gts, "perturbed"))
    pairs = [(r, g) for r in range(len(res["score"])) for g in gts
             if (res["scene_id"][r], res["im_id"][r], res["obj_id"][r]) == (g["scene_id"], g["im_id"], g["obj_id"])]
    assert len(pairs) > 20
    objs = [1, 2, 3]
    syms64 = {o: bo.symmetries(info[str(o)]) for o in objs}
    est = np.array([np.r_[res["R"][r].reshape(-1), res["t"][r]] for r, _ in pairs]).astype(np.float32)
    gt = np.array([np.r_[g["R"].reshape(-1), g["t"]] for _, g in pairs]).astype(np.float32)
    Ks = {im[:2]: (im[4], im[4], im[3] / 2 - 0.5, im[2] / 2 + 0.25) for im in IMAGES}
    Kp = np.array([Ks[(g["scene_id"], g["im_id"])] for _, g in pairs], np.float32)
    syms = [np.array([np.r_[R.reshape(-1), t] for R, t in syms64[o]], np.float32) for o in objs]
    out = bop_eval.mssd_mspd(est, gt, np.array([objs.index(g["obj_id"]) for _, g in pairs], np.int32), Kp,
                             [meshes[o][0] for o in objs], syms).cpu().numpy()
    worst = [0.0, 0.0]
    for i, (r, g) in enumerate(pairs):
        o = g["obj_id"]
        X = meshes[o][0].astype(np.float64)
        # the oracle on the kernel's own fp32 inputs (poses and symmetry transforms rounded as uploaded)
        s32 = [(s[:9].astype(np.float64).reshape(3, 3), s[9:].astype(np.float64)) for s in syms[objs.index(o)]]
        Re, te = est[i, :9].astype(np.float64).reshape(3, 3), est[i, 9:].astype(np.float64)
        Rg, tg = gt[i, :9].astype(np.float64).reshape(3, 3), gt[i, 9:].astype(np.float64)
        K = np.array([[Kp[i, 0], 0, Kp[i, 2]], [0, Kp[i, 1], Kp[i, 3]], [0, 0, 1]], np.float64)
        m3, m2 = bo.mssd(Re, te, Rg, tg, X, s32), bo.mspd(Re, te, Rg, tg, X, s32, K)
        b3, b2 = bo.mssd_band(te, tg, X, s32), bo.mspd_band(Re, te, tg, X, s32, K)
        assert abs(out[i, 0] - m3) <= b3, (i, out[i, 0], m3, b3)
        assert abs(out[i, 1] - m2) <= b2, (i, out[i, 1], m2, b2)
        worst = [max(worst[0], abs(out[i, 0] - m3) / b3), max(worst[1], abs(out[i, 1] - m2) / b2)]
    print(f"[bop_eval] {len(pairs)} pairs: worst |gpu - oracle| / bound: MSSD {worst[0]:.3f}, MSPD {worst[1]:.3f}")

    # VSD counts of every pair of the 640 x 480 scene whose spheres overlap, on the renders the evaluator would make
    fn = _render_fn(meshes)
    sel = [i for i, (r, g) in enumerate(pairs) if g["scene_id"] == 1 and g["obj_id"] == 2]
    assert len(sel) >= 4
    from PIL import Image
    ims = sorted({pairs[i][1]["im_id"] for i in sel})
    K = np.array([[600.0, 0, 319.5], [0, 600.0, 240.25], [0, 0, 1]])
    dt = [(np.array(Image.open(os.path.join(root, "toy", "test", "000001", "depth", f"{im:06d}.png"))).astype(np.float64)
           * DEPTH_SCALE).astype(np.float32) for im in ims]
    de = [fn(2, est[i, :9].reshape(3, 3), est[i, 9:], K, 480, 640) for i in sel]
    dg = [fn(2, gt[i, :9].reshape(3, 3), gt[i, 9:], K, 480, 640) for i in sel]
    diam = info["2"]["diameter"]
    cnt = bop_eval.vsd_counts(torch.from_numpy(np.stack(de)).cuda(), torch.from_numpy(np.stack(dg)).cuda(),
                              torch.from_numpy(np.stack(dt)).cuda(), [ims.index(pairs[i][1]["im_id"]) for i in sel], K, 15.0,
                              diam).cpu().numpy()
    for k, i in enumerate(sel):
        d_t = dt[ims.index(pairs[i][1]["im_id"])]
        want = bo.vsd_counts(de[k], dg[k], d_t, K, 15.0, diam)
        m = bo.vsd_margin_pixels(de[k], dg[k], d_t, K, 15.0, diam)
        assert want[0] > 0
        assert np.abs(cnt[k] - np.array(want)).max() <= m, (k, cnt[k], want, m)


def _oracle(root, dataset, csv):
    meshes = _meshes_of(root, dataset)
    return bo.evaluate(root, dataset, csv, _render_fn(meshes), load_vertices=lambda p: meshio.load_ply(p)[0].astype(np.float64))


@pytest.mark.parametrize("dataset", ["toy", "itodd"])
def test_evaluate_matches_oracle(split, tmp_path, dataset):
    root, gts = split
    csv = write_results(str(tmp_path / "r.csv"), gts, "perturbed")
    got = bop_eval.evaluate_bop19(root, dataset, csv)
    want = _oracle(root, dataset, csv)
    assert want["ambiguous"] == 0, "the fixture puts an error inside a threshold's rounding band"
    assert got["n_gt"] == want["n_gt"] == sum(g["visib"] >= 0.1 for g in gts)
    assert got["n_targets"] == 7 and got["n_estimates"] == 8
    for e in ("mssd", "mspd"):
        np.testing.assert_array_equal(np.array(got[f"recall_{e}"]), want[f"recall_{e}"])
    np.testing.assert_array_equal(np.array(got["recall_vsd"]).reshape(-1), want["recall_vsd"])
    # a spread of outcomes, not all 0 or 1
    for e in ("vsd", "mssd", "mspd"):
        assert 0.0 < got[f"ar_{e}"] < 1.0
    assert got["ar"] == pytest.approx((got["ar_vsd"] + got["ar_mssd"] + got["ar_mspd"]) / 3)
    print(f"[bop_eval] {dataset}: AR {got['ar']:.4f} (VSD {got['ar_vsd']:.4f} MSSD {got['ar_mssd']:.4f} MSPD {got['ar_mspd']:.4f})")


def test_itodd_delta(split, tmp_path):
    """a copy of the split whose test depth lies 10 mm in front of every object surface, scored as "toy" (delta = 15 mm) and as
    "itodd" (delta = 5 mm) with the GT poses: the surfaces are visible at 15 mm (e_VSD = 0) and hidden at 5 mm (no visible
    pixel, e_VSD = 1)"""
    from PIL import Image
    root, gts = split
    new = str(tmp_path / "shifted")
    for ds in ("toy", "itodd"):
        shutil.copytree(os.path.join(root, "toy"), os.path.join(new, ds))
        for scene in ("000001", "000002"):
            ddir = os.path.join(new, ds, "test", scene, "depth")
            for name in os.listdir(ddir):
                raw = np.array(Image.open(os.path.join(ddir, name))).astype(np.int64)
                raw = np.where(raw > 0, raw - round(10.0 / DEPTH_SCALE), 0)
                Image.fromarray(raw.astype(np.uint16)).save(os.path.join(ddir, name))
    csv = write_results(str(tmp_path / "gt.csv"), gts, "gt")
    a = bop_eval.evaluate_bop19(new, "toy", csv, error_types=("vsd",))
    b = bop_eval.evaluate_bop19(new, "itodd", csv, error_types=("vsd",))
    assert a["ar_vsd"] == 1.0 and b["ar_vsd"] == 0.0
    assert a["ar"] == a["ar_vsd"] and "ar_mssd" not in a
    for ds, got in (("toy", a), ("itodd", b)):
        want = _oracle(new, ds, csv)
        assert want["ambiguous"] == 0
        np.testing.assert_array_equal(np.array(got["recall_vsd"]).reshape(-1), want["recall_vsd"])


def test_gt_and_far_results_and_cli(split, tmp_path):
    root, gts = split
    gt_csv = write_results(str(tmp_path / "gt.csv"), gts, "gt")
    got = bop_eval.evaluate_bop19(root, "toy", gt_csv)
    assert got["ar"] == 1.0 and got["ar_vsd"] == got["ar_mssd"] == got["ar_mspd"] == 1.0
    far = bop_eval.evaluate_bop19(root, "toy", write_results(str(tmp_path / "far.csv"), gts, "far"))
    assert far["ar"] == 0.0 and far["n_estimates"] == 7 + 1
    out = tmp_path / "out"
    assert eval_bop.main(["--bop_root", root, "--dataset_name", "toy", "--result_csv", gt_csv, "--output_dir", str(out)]) == 0
    saved = json.load(open(out / "scores_bop19_toy.json"))
    assert saved["ar"] == 1.0 and saved["n_gt"] == got["n_gt"] and saved["recall_mssd"] == [1.0] * 10
