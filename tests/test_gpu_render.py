"""GPU: the template rasteriser (csrc/render.cu through sam6d_b200.render) against oracle/render_oracle.py -- triangle id, mask,
depth and f16 object coordinates bit for bit, colours within 1 -- and the two template CLIs feeding the ISM and PEM CLIs."""
import json
import os

import numpy as np
import pytest
import torch

from oracle import render_oracle as ro
from sam6d_b200 import meshio, render

pytestmark = pytest.mark.gpu


def _soup(seed=0, n=160, dup=40):
    """overlapping random triangles, the last `dup` exact copies of earlier ones (exact depth ties the copies must lose)"""
    rng = np.random.RandomState(seed)
    v = rng.uniform(-30, 30, (3 * n, 3)).astype(np.float32)
    f = np.arange(3 * n, dtype=np.int32).reshape(n, 3)
    f = np.concatenate([f, f[rng.choice(n, dup, replace=False)]])
    return dict(vertices=v, faces=f, colors=rng.randint(0, 256, (3 * n, 3)).astype(np.uint8))


def _textured(seed=1):
    v, f = ro.icosphere(2, 35.0)
    rng = np.random.RandomState(seed)
    uv = np.stack([np.arctan2(v[:, 1], v[:, 0]) / (2 * np.pi) + 0.5, v[:, 2] / 70.0 + 0.5], 1).astype(np.float32)
    return dict(vertices=v, faces=f, uv=uv, texture=rng.randint(0, 256, (37, 53, 3)).astype(np.uint8))


def _hull_mesh(golden_dir):
    from scipy.spatial import ConvexHull
    gold = torch.load(os.path.join(golden_dir, "pem_input.pt"), weights_only=False)
    pts_mm = gold["model_points"].numpy().astype(np.float64) * 1000.0
    hull = ConvexHull(pts_mm)
    remap = {v: i for i, v in enumerate(hull.vertices)}
    faces = np.array([[remap[a] for a in s] for s in hull.simplices], np.int32)
    colors = np.random.RandomState(0).randint(40, 255, (len(hull.vertices), 3)).astype(np.uint8)
    return dict(vertices=pts_mm[hull.vertices].astype(np.float32), faces=faces, colors=colors)


def _to_mesh(d):
    return render.upload(meshio.Mesh(d["vertices"], d["faces"], d.get("colors"), d.get("uv"), d.get("texture")))


def _radius(d):
    return float(np.linalg.norm(d["vertices"], axis=1).max())


def _poses(meshes):
    return np.stack([render.level0_template_poses(4.0 * _radius(m)) for m in meshes]).astype(np.float32)


def _compare(meshes, size, base=0.8):
    poses = _poses(meshes)
    K = render.template_K(size)
    out = render.render([_to_mesh(m) for m in meshes], torch.from_numpy(poses).cuda(), K, size, size, base_color=base)
    torch.cuda.synchronize()
    gpu = {k: v.cpu().numpy() for k, v in out.items()}
    ref = ro.render(meshes, poses, K, size, size, base_color=base)
    np.testing.assert_array_equal(gpu["tri"], ref["tri"])
    np.testing.assert_array_equal(gpu["mask"], ref["mask"])
    np.testing.assert_array_equal(gpu["depth"].view(np.int32), ref["depth"].view(np.int32))
    np.testing.assert_array_equal(gpu["xyz"].view(np.int16), ref["xyz"].view(np.int16))
    d = np.abs(gpu["rgb"].astype(np.int32) - ref["rgb"].astype(np.int32))
    print(f"{size}^2, {len(meshes)} x 42 views: {int((ref['mask'] > 0).sum())} object pixels, rgb max |gpu - oracle| {d.max()}, "
          f"{int((d > 0).sum())} channels differ; dropped {gpu['dropped'].tolist()}")
    assert d.max() <= 1
    np.testing.assert_array_equal(gpu["dropped"], ref["dropped"])
    for o in range(len(meshes)):
        assert (ref["mask"][o] > 0).sum(axis=(1, 2)).min() > 0, "every view sees its object"
    return out


def test_gpu_matches_oracle_512():
    """a 12-triangle cube whose faces cover ~10^4 px each (the one-CTA-per-triangle path), a vertex-coloured icosphere and a
    triangle soup with exact depth ties, 3 objects x 42 views in one call"""
    cv, cf = ro.cube(50.0)
    iv, ifc = ro.icosphere(2, 40.0)
    ico = dict(vertices=iv, faces=ifc, colors=np.random.RandomState(2).randint(0, 256, (len(iv), 3)).astype(np.uint8))
    _compare([dict(vertices=cv, faces=cf), ico, _soup()], 512, base=[[0.8] * 3, [0.8] * 3, [0.8] * 3])


def test_gpu_matches_oracle_textured_and_hull(golden_dir):
    _compare([_textured(), _hull_mesh(golden_dir), _soup(seed=5, n=60, dup=20)], 192, base=0.4)


def test_dropped_and_deterministic():
    v, f = ro.icosphere(2, 1.0)
    mesh = dict(vertices=v, faces=f)
    poses = np.tile(np.eye(4, dtype=np.float32), (1, 2, 1, 1))
    poses[0, 0, 2, 3] = 0.5                                                          # camera inside the sphere: vertices behind it
    poses[0, 1, 2, 3] = 4.0
    K = render.template_K(128)
    runs = [render.render([_to_mesh(mesh)], torch.from_numpy(poses).cuda(), K, 128, 128) for _ in range(2)]
    torch.cuda.synchronize()
    ref = ro.render([mesh], poses, K, 128, 128)
    assert int(runs[0]["dropped"][0]) > 0 and int(runs[0]["dropped"][0]) == int(ref["dropped"][0])
    np.testing.assert_array_equal(runs[0]["tri"].cpu().numpy(), ref["tri"])
    for k in ("rgb", "mask", "xyz", "tri", "depth", "dropped"):
        assert torch.equal(runs[0][k], runs[1][k]), k


def test_rejects_bad_meshes():
    v, f = ro.icosphere(0)
    m = _to_mesh(dict(vertices=v, faces=f))
    with pytest.raises(ValueError):
        render.render([meshio.Mesh(m.vertices, m.faces + 100)], torch.eye(4).reshape(1, 1, 4, 4).cuda(), render.template_K(32), 32, 32)
    with pytest.raises(RuntimeError):
        render.render([m], torch.eye(4).reshape(1, 1, 4, 4).double().cuda(), render.template_K(32), 32, 32)


def _write_ply(path, m):
    V, F = m["vertices"], m["faces"]
    with open(path, "w") as fh:
        fh.write("ply\nformat ascii 1.0\nelement vertex %d\nproperty float x\nproperty float y\nproperty float z\n" % len(V))
        if m.get("colors") is not None:
            fh.write("property uchar red\nproperty uchar green\nproperty uchar blue\n")
        if m.get("uv") is not None:
            fh.write("property float texture_u\nproperty float texture_v\n")
        fh.write("element face %d\nproperty list uchar int vertex_indices\nend_header\n" % len(F))
        for i in range(len(V)):
            row = ["%.6f" % x for x in V[i]]
            row += ["%d" % c for c in m["colors"][i]] if m.get("colors") is not None else []
            row += ["%.7f" % x for x in m["uv"][i]] if m.get("uv") is not None else []
            fh.write(" ".join(row) + "\n")
        for f in F:
            fh.write("3 %d %d %d\n" % tuple(f))


@pytest.fixture(scope="module")
def custom_templates(tmp_path_factory, golden_dir):
    from sam6d_b200.cli import render_custom_templates as cli
    out = str(tmp_path_factory.mktemp("custom"))
    cad = os.path.join(out, "obj.ply")
    _write_ply(cad, _hull_mesh(golden_dir))
    assert cli.main(["--cad_path", cad, "--output_dir", out]) == 0
    return out, cad


def test_custom_cli_files_agree_with_poses(custom_templates):
    import cv2
    out, cad = custom_templates
    tdir = os.path.join(out, "templates")
    poses = np.load(os.path.join(tdir, "template_poses.npy"))
    assert poses.shape == (42, 4, 4)
    K = render.template_K(512)
    worst = 0.0
    for i in range(42):
        mask = cv2.imread(os.path.join(tdir, f"mask_{i}.png"), 0)
        xyz = np.load(os.path.join(tdir, f"xyz_{i}.npy"))
        assert xyz.dtype == np.float16 and xyz.shape == (512, 512, 3) and mask.shape == (512, 512)
        yy, xx = np.nonzero(mask == 255)
        assert len(yy) > 1000
        assert (xyz[mask == 0] == 0).all()
        p = xyz[yy, xx].astype(np.float64) @ poses[i, :3, :3].T + poses[i, :3, 3] * 1000.0   # template_poses.npy holds metres
        u = K[0, 0] * p[:, 0] / p[:, 2] + K[0, 2]
        v = K[1, 1] * p[:, 1] / p[:, 2] + K[1, 2]
        err = np.hypot(u - (xx + 0.5), v - (yy + 0.5))
        worst = max(worst, float(err.max()))
    print(f"max |K (R xyz + t) - pixel centre| over 42 views: {worst:.3f} px")
    assert worst < 0.75


def test_rendered_arrays_give_the_template_bank_of_the_files(custom_templates, golden_dir):
    from sam6d_b200 import inputs
    from sam6d_b200.cli import pem_run_inference_custom as pem_cli, render_custom_templates as cli
    out, cad = custom_templates
    files = pem_cli.read_templates(os.path.join(out, "templates"))
    mesh = meshio.load_ply_mesh(cad)
    r = max(np.linalg.norm(mesh.vertices.max(axis=0)), np.linalg.norm(mesh.vertices.min(axis=0)))
    res = cli.render_views([render.upload(mesh)], cli.view_poses(4.0 * float(r))[None], 512, [[0.8] * 3])
    arrays = ([x.cpu().numpy() for x in res["rgb"][0]], [x.cpu().numpy() for x in res["mask"][0]],
              [x.cpu().numpy().astype(np.float32) for x in res["xyz"][0]])
    a = inputs.get_templates_from_arrays(*files, rng=np.random.RandomState(0))
    b = inputs.get_templates_from_arrays(*arrays, rng=np.random.RandomState(0))
    for la, lb in zip(a, b):
        assert len(la) == len(lb) == 42
        for x, y in zip(la, lb):
            assert torch.equal(x, y)


def test_custom_templates_then_ism_cli_then_pem_cli(custom_templates, golden_dir):
    import cv2
    from sam6d_b200.cli import ism_run_inference_custom as ism_cli, pem_run_inference_custom as pem_cli
    out, cad = custom_templates
    gold = torch.load(os.path.join(golden_dir, "pem_input.pt"), weights_only=False)
    cv2.imwrite(os.path.join(out, "rgb.png"), gold["rgb"].numpy()[:, :, ::-1])
    cv2.imwrite(os.path.join(out, "depth.png"), gold["depth"].numpy().astype(np.uint16))
    json.dump(dict(cam_K=gold["cam_K"], depth_scale=gold["depth_scale"]), open(os.path.join(out, "camera.json"), "w"))
    common = ["--output_dir", out, "--cad_path", cad, "--rgb_path", os.path.join(out, "rgb.png"), "--depth_path", os.path.join(out, "depth.png"),
              "--cam_path", os.path.join(out, "camera.json")]
    assert ism_cli.main(common + ["--random_weights", "--stability_score_thresh", "0.0", "--pred_iou_thresh", "-10", "--confidence_thresh", "-1",
                                  "--points_per_side", "8"]) == 0
    dets = json.load(open(os.path.join(out, "sam6d_results", "detection_ism.json")))
    print(f"ISM CLI on rendered templates: {len(dets)} detections")
    assert len(dets) >= 1
    for d in dets:
        assert d["segmentation"]["size"] == [480, 640] and np.isfinite(d["score"])
    np.random.seed(0)
    assert pem_cli.main(common + ["--seg_path", os.path.join(out, "sam6d_results", "detection_ism.json"), "--random_weights",
                                  "--det_score_thresh", "-1"]) == 0
    res = json.load(open(os.path.join(out, "sam6d_results", "detection_pem.json")))
    assert 1 <= len(res) <= len(dets)
    for r in res:
        R = np.array(r["R"])
        assert np.allclose(R @ R.T, np.eye(3), atol=1e-4) and np.isfinite(np.array(r["t"])).all()


def test_bop_cli_two_objects(tmp_path, golden_dir):
    from sam6d_b200.cli import render_bop_templates as cli
    import cv2
    models = tmp_path / "BOP" / "ycbv" / "models"
    models.mkdir(parents=True)
    tex = _textured()
    cv2.imwrite(str(models / "obj_000002.png"), tex["texture"][:, :, ::-1])
    _write_ply(str(models / "obj_000001.ply"), _hull_mesh(golden_dir))
    _write_ply(str(models / "obj_000002.ply"), tex)
    with open(models / "obj_000002.ply") as fh:
        body = fh.read()
    (models / "obj_000002.ply").write_text(body.replace("format ascii 1.0\n", "format ascii 1.0\ncomment TextureFile obj_000002.png\n"))
    info = {"1": {"diameter": 2.0 * _radius(_hull_mesh(golden_dir))}, "2": {"diameter": 70.0}}
    (models / "models_info.json").write_text(json.dumps(info))
    out = tmp_path / "BOP-Templates"
    assert cli.main(["--dataset_name", "ycbv", "--bop_root", str(tmp_path / "BOP"), "--output_dir", str(out), "--size", "128"]) == 0
    for oid in ("obj_000001", "obj_000002"):
        d = out / "ycbv" / oid
        for i in range(42):
            assert (d / f"rgb_{i}.png").exists() and (d / f"mask_{i}.png").exists() and (d / f"xyz_{i}.npy").exists()
        poses = np.load(d / "template_poses.npy")
        assert poses.shape == (42, 4, 4)
        np.testing.assert_allclose(poses[:, 2, 3], 2.0 * info[oid[-1]]["diameter"] / 1000.0, rtol=1e-9)
        m = cv2.imread(str(d / "mask_0.png"), 0)
        assert (m == 255).sum() > 100
    rgb2 = cv2.imread(str(out / "ycbv" / "obj_000002" / "rgb_20.png"))
    assert len(np.unique(rgb2.reshape(-1, 3), axis=0)) > 50                          # the texture was read and sampled
