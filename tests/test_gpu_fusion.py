"""GPU: TSDF fusion and marching-tetrahedra extraction on sm_90a (csrc/fusion.cu, sam6d_b200/fusion.py) against
oracle/fusion_oracle.py and against the meshes the views were rendered from (render.render of tests/_symmetry_meshes).

- integration equals the float32 oracle bit for bit (tsdf, weight, colour sums and counts) on a 48^3 volume, with and without
  masks, with voxels outside the images and behind a camera, zeroed depth and the carving branch; chunked integration equals
  one launch and two runs are identical;
- extraction on the GPU's volume equals the oracle's vertex, colour and face arrays element for element;
- end to end from 162 rendered views at 480 x 640: the fused mesh is closed, within a derived Chamfer bound of the original
  surface, coloured like it away from face edges, and renders to the original's masks within a derived IoU bound;
- the fused PLY feeds SAM6D.onboard and fuse_object_model -> run_sam6d --cad_path;
- the ops wrappers reject bad arguments before launching."""
import json
import math
import os

import numpy as np
import pytest
import torch

import _symmetry_meshes as sm
from oracle import fusion_oracle as fo

pytestmark = pytest.mark.gpu


def _render(mesh, poses, K, H, W, ambient=1.0):
    """rendered rgb, depth (mm), mask of T views; the rasteriser samples pixel c at u = c + 1/2, so its principal point is
    shifted by +1/2 to put fusion's pixel c (the ray through u = c) on the same ray"""
    from sam6d_b200 import render
    Kr = np.array(K, np.float64).copy()
    Kr[0, 2] += 0.5
    Kr[1, 2] += 0.5
    out = render.render([render.upload(mesh)], torch.from_numpy(np.asarray(poses, np.float32))[None].cuda(), Kr, H, W, ambient=ambient)
    return out["rgb"][0], out["depth"][0], out["mask"][0]


def _small_case(seed=0):
    """12 views at 120 x 160 of the colour-faced cube, 300 mm away, plus one camera 40 mm from the centre (inside the volume's
    box, so voxels lie behind it) and one turned away (every voxel outside its image)"""
    from sam6d_b200 import render
    mesh = sm.build("cube_colours")
    poses = render.template_poses(0, distance=300.0)[::4][:10]
    near = render.template_poses(0, distance=40.0)[5:6]
    away = poses[:1].copy()
    away[0, :3, :3] = np.diag([1.0, -1.0, -1.0]) @ away[0, :3, :3]
    poses = np.concatenate([poses, near, away])
    K = np.array([[140.0, 0, 80.0], [0, 140.0, 60.0], [0, 0, 1]])
    rgb, depth, mask = _render(mesh, poses, K, 120, 160)
    depth = depth.clone()
    g = torch.Generator(device="cuda").manual_seed(seed)
    depth[torch.rand(depth.shape, device="cuda", generator=g) < 0.05] = 0          # missing depth
    return mesh, poses, K, rgb.contiguous(), depth.contiguous(), mask.contiguous()


def _oracle_state(vol, rgb, depth, mask, K, poses):
    from sam6d_b200 import fusion
    K4, P12 = fusion.pack_views(K, poses, len(poses))
    return fo.integrate(rgb.cpu().numpy(), depth.cpu().numpy(), None if mask is None else mask.cpu().numpy(), K4, P12,
                        vol.dims, vol.bbox_min, np.float32(vol.voxel), np.float32(vol.trunc), np.float32(fusion.ZNEAR_MM))


def _equal(a, b):
    for k in ("tsdf", "weight", "csum", "ccount"):
        assert a[k].dtype == b[k].dtype and np.array_equal(a[k].view(np.uint32) if k == "tsdf" else a[k],
                                                           b[k].view(np.uint32) if k == "tsdf" else b[k]), k


@pytest.mark.parametrize("with_mask", [True, False])
def test_integration_matches_float32_oracle(with_mask):
    from sam6d_b200 import fusion
    mesh, poses, K, rgb, depth, mask = _small_case()
    vol = fusion.TsdfVolume((-72.0, -72.0, -72.0), (72.0, 72.0, 72.0), 3.0)
    assert vol.dims == (48, 48, 48)
    m = mask if with_mask else None
    vol.integrate(rgb, depth, m, K, poses, 1.0)
    got, want = vol.state(), _oracle_state(vol, rgb, depth, m, K, poses)
    _equal(got, want)
    w = got["weight"]
    print(f"mask={with_mask}: weight range {w.min()}..{w.max()}, {np.mean(w > 0):.3f} of voxels observed, "
          f"{int(got['ccount'].sum())} colour samples")
    assert w.max() <= len(poses) - 1 and w.min() < w.max() and got["ccount"].sum() > 0
    if with_mask:
        assert (got["tsdf"][w > 0] == 1).mean() > 0.3                 # carved free space


def test_chunked_integration_and_repeat_are_identical(monkeypatch):
    from sam6d_b200 import fusion
    _, poses, K, rgb, depth, mask = _small_case(1)
    args = (rgb.cpu().numpy(), depth.cpu().numpy(), mask.cpu().numpy(), K, poses, 1.0)
    box = ((-72.0, -72.0, -72.0), (72.0, 72.0, 72.0), 3.0)
    one = fusion.TsdfVolume(*box).integrate(*args).state()
    again = fusion.TsdfVolume(*box).integrate(*args).state()
    monkeypatch.setattr(fusion, "FUSION_BUDGET_BYTES", 120 * 160 * 12 * 3)          # 3 views per launch
    chunked = fusion.TsdfVolume(*box).integrate(*args).state()
    _equal(one, again)
    _equal(one, chunked)


def test_depth_scale_and_raw_dtypes_leave_inputs_unchanged():
    """raw depth in 0.1 mm units as a CUDA float32 tensor (the dtype integrate could alias), a CUDA uint16 tensor and a numpy
    uint16 array: each fuses like the float32 oracle fed raw * 0.1 scaled on the host, the caller's arrays are unchanged, and
    a second integration of the same inputs gives the same volume"""
    from sam6d_b200 import fusion
    _, poses, K, rgb, depth, mask = _small_case(2)
    box = ((-72.0, -72.0, -72.0), (72.0, 72.0, 72.0), 3.0)
    u16 = torch.round(depth / 0.1).to(torch.int32).cpu().numpy().astype(np.uint16)
    raws = [(depth / 0.1).contiguous(), torch.from_numpy(u16).cuda(), u16]
    bits = lambda t: t.view(torch.int16) if t.dtype == torch.uint16 else t       # noqa: E731  (compared through int16)
    for raw in raws:
        before = bits(raw).clone() if isinstance(raw, torch.Tensor) else raw.copy()
        host = (bits(raw).cpu().numpy().view(u16.dtype) if isinstance(raw, torch.Tensor) and raw.dtype == torch.uint16
                else raw.cpu().numpy() if isinstance(raw, torch.Tensor) else raw).astype(np.float32) * np.float32(0.1)
        first = fusion.TsdfVolume(*box).integrate(rgb, raw, mask, K, poses, 0.1)
        second = fusion.TsdfVolume(*box).integrate(rgb, raw, mask, K, poses, 0.1)
        same = torch.equal(bits(raw), before) if isinstance(raw, torch.Tensor) else np.array_equal(raw, before)
        assert same, f"integrate changed the caller's {type(raw).__name__} depth"
        want = fo.integrate(rgb.cpu().numpy(), host, mask.cpu().numpy(), *fusion.pack_views(K, poses, len(poses)), first.dims,
                            first.bbox_min, np.float32(first.voxel), np.float32(first.trunc), np.float32(fusion.ZNEAR_MM))
        _equal(first.state(), want)
        _equal(first.state(), second.state())
        assert first.state()["weight"].max() > 0


def test_extraction_matches_oracle():
    from sam6d_b200 import fusion
    mesh, poses, K, rgb, depth, mask = _small_case()
    vol = fusion.TsdfVolume((-72.0, -72.0, -72.0), (72.0, 72.0, 72.0), 3.0).integrate(rgb, depth, mask, K, poses, 1.0)
    st = vol.state()
    for mw in (1, 3):
        v, c, f = (x.cpu().numpy() for x in vol.mesh_tensors(mw))
        ov, oc, of = fo.mesh(st["tsdf"], st["weight"], st["csum"], st["ccount"], vol.bbox_min, np.float32(vol.voxel), mw)
        print(f"min_weight {mw}: {len(v)} vertices, {len(f)} faces")
        assert len(f) > 100
        assert np.array_equal(v.view(np.uint32), ov.view(np.uint32)) and np.array_equal(c, oc) and np.array_equal(f, of)
    m = vol.mesh()
    assert m.vertices.dtype == np.float32 and m.faces.dtype == np.int64 and m.colors.dtype == np.uint8


def _closed(faces):
    d = np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])
    key = d[:, 0] * (faces.max() + 1) + d[:, 1]
    rkey = d[:, 1] * (faces.max() + 1) + d[:, 0]
    return len(np.unique(key)) == len(key) and np.isin(key, rkey).all()


def _blob_point(d, r=50.0):
    """the smooth surface _symmetry_meshes.blob samples: r s(d) d for unit directions d (..., 3)"""
    x, y, z = d[..., 0], d[..., 1], d[..., 2]
    s = 1.0 + 0.3 * x + 0.2 * y * y + 0.25 * x * z + 0.3 * y * z * z + 0.15 * x * y + 0.1 * z
    return r * s[..., None] * d


def _inscribed_blob():
    """_symmetry_meshes.blob with its north-pole vertex moved from r onto the surface it samples, r s(+z) = 1.1 r: as built,
    that vertex sits 5 mm below the surface, a dimple no curvature bound covers.  Every vertex then lies on the smooth
    surface (within float32 rounding), so the mesh is a polyhedron inscribed in it."""
    mesh = sm.build("blob")
    v = np.asarray(mesh.vertices, np.float64).copy()
    v[0] = _blob_point(np.array([0.0, 0.0, 1.0]))
    return type(mesh)(vertices=v.astype(np.float32), faces=mesh.faces, colors=mesh.colors)


def _blob_kappa_max(n=600, e=1e-4):
    """the largest principal-curvature magnitude of the smooth blob surface, from its first and second fundamental forms
    (central differences of step e in float64) on two spherical charts, |z| <= cos(pi/4) and |x| <= cos(pi/4), which
    together cover the sphere of directions"""
    kmax = 0.0
    th = np.linspace(0.25 * np.pi, 0.75 * np.pi, n)[:, None]
    ph = np.linspace(0, 2 * np.pi, 2 * n, endpoint=False)[None, :]
    charts = (lambda t, p: np.stack(np.broadcast_arrays(np.sin(t) * np.cos(p), np.sin(t) * np.sin(p), np.cos(t)), -1),
              lambda t, p: np.stack(np.broadcast_arrays(np.cos(t), np.sin(t) * np.sin(p), np.sin(t) * np.cos(p)), -1))
    for ch in charts:
        P = lambda a, b: _blob_point(ch(a, b))        # noqa: E731
        p0 = P(th, ph)
        Pt, Pp = (P(th + e, ph) - P(th - e, ph)) / (2 * e), (P(th, ph + e) - P(th, ph - e)) / (2 * e)
        Ptt = (P(th + e, ph) - 2 * p0 + P(th - e, ph)) / e ** 2
        Ppp = (P(th, ph + e) - 2 * p0 + P(th, ph - e)) / e ** 2
        Ptp = (P(th + e, ph + e) - P(th + e, ph - e) - P(th - e, ph + e) + P(th - e, ph - e)) / (4 * e * e)
        N = np.cross(Pt, Pp)
        N /= np.linalg.norm(N, axis=-1, keepdims=True)
        E, F, G = (Pt * Pt).sum(-1), (Pt * Pp).sum(-1), (Pp * Pp).sum(-1)
        L, M, Nn = (Ptt * N).sum(-1), (Ptp * N).sum(-1), (Ppp * N).sum(-1)
        a, b, c = E * G - F * F, -(E * Nn + G * L - 2 * F * M), L * Nn - M * M     # det(II - k I) = 0
        disc = np.sqrt(np.maximum(b * b - 4 * a * c, 0.0))
        kmax = max(kmax, float((np.maximum(np.abs(-b + disc), np.abs(-b - disc)) / (2 * a)).max()))
    return kmax


def _facet_deviation(mesh, steps=32):
    """the largest radial distance between the facets and the smooth blob surface, on a barycentric grid of 1/steps per face
    (the radial segment meets the surface, so this bounds the distance)"""
    v, f = np.asarray(mesh.vertices, np.float64), np.asarray(mesh.faces)
    g = np.linspace(0, 1, steps + 1)
    uu, vv = np.meshgrid(g, g)
    keep = uu + vv <= 1
    uu, vv = uu[keep], vv[keep]
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    pts = (a[:, None] + uu[None, :, None] * (b - a)[:, None] + vv[None, :, None] * (c - a)[:, None]).reshape(-1, 3)
    r = np.linalg.norm(pts, axis=1)
    return float(np.abs(r - np.linalg.norm(_blob_point(pts / r[:, None]), axis=1)).max())


def _fuse_views(name, resolution=128, H=480, W=640, f=600.0, distance=400.0):
    from sam6d_b200 import fusion, render
    mesh = _inscribed_blob() if name == "blob" else sm.build(name)
    poses = render.template_poses(level=1, distance=distance)
    K = np.array([[f, 0, W / 2.0], [0, f, H / 2.0], [0, 0, 1]])
    rgb, depth, mask = _render(mesh, poses, K, H, W)
    lo, hi, voxel, trunc = fusion.view_bounds(depth, mask, K, poses, 1.0, resolution=resolution)
    vol = fusion.TsdfVolume(lo, hi, voxel, trunc).integrate(rgb, depth, mask, K, poses, 1.0)
    return mesh, vol, vol.mesh(), (poses, K, H, W)


def test_end_to_end_blob_geometry():
    from scipy.spatial import cKDTree
    from sam6d_b200 import meshio, render
    mesh, vol, fused, (poses, K, H, W) = _fuse_views("blob")
    h, f = vol.voxel, K[0, 0]
    assert _closed(fused.faces), "the fused mesh is open"
    # Max bound.  A corner is negative only if some view's pixel depth d lies in front of it (d < z), i.e. it lies behind a
    # surface point seen on a ray that passes within s = (sqrt(2) / 2) z_max / f mm of it (the pixel snap is <= 1/2 px per
    # axis), by less than trunc along that ray: inside the object, or outside by at most the sagitta trunc^2 / (2 r_min) of a
    # ray grazing the rim (r_min = the smallest radius of curvature).  The rendered surface is a polyhedron inscribed in
    # the smooth one, within delta of it (_facet_deviation), so the sagitta term is taken on the smooth surface, with r_min
    # = 1 / the largest principal curvature computed from its analytic form, plus delta on each side.  Likewise a non-negative corner is outside or within s
    # of the surface.  A vertex lies on a lattice edge (length <= sqrt(3) h) between corners of both kinds, so it is within
    # s + trunc^2 / (2 r_min) + 2 delta + sqrt(3) h of the surface; the surface is covered by the 162 views, and the same argument
    # bounds the surface's distance to the mesh.  Mean: the lattice term, a vertex's distance along its edge from the
    # crossing, averages at most half the edge, so the mean is bounded by half the max bound.
    # Distances are measured between dense surface samples, which over-estimate point-to-surface distances: stricter.
    z_max = 400.0 + float(np.linalg.norm(mesh.vertices, axis=1).max())
    s = math.sqrt(2) / 2 * z_max / f
    r_min = 1.0 / _blob_kappa_max()
    delta = _facet_deviation(mesh)
    assert np.abs(np.linalg.norm(_blob_point(mesh.vertices / np.linalg.norm(mesh.vertices, axis=1, keepdims=True)), axis=1)
                  - np.linalg.norm(mesh.vertices, axis=1)).max() < 1e-4                  # inscribed
    bound = s + vol.trunc ** 2 / (2 * r_min) + 2 * delta + math.sqrt(3) * h
    rng = np.random.RandomState(0)
    a = meshio.sample_surface(np.asarray(mesh.vertices), np.asarray(mesh.faces), 400000, rng)
    b = meshio.sample_surface(fused.vertices, fused.faces, 400000, rng)
    d_ab = cKDTree(b).query(a)[0]
    d_ba = cKDTree(a).query(b)[0]
    print(f"blob: voxel {h:.3f} mm, {len(fused.vertices)} vertices, {len(fused.faces)} faces; Chamfer mean {d_ab.mean():.3f} / "
          f"{d_ba.mean():.3f}, max {d_ab.max():.3f} / {d_ba.max():.3f} mm; r_min {r_min:.2f} mm, facet deviation {delta:.3f} mm, "
          f"bound max {bound:.3f}, mean {bound / 2:.3f}")
    assert max(d_ab.max(), d_ba.max()) <= bound
    assert max(d_ab.mean(), d_ba.mean()) <= bound / 2
    # silhouettes from the 42 template views: the fused surface lies within `bound` of the original, so its mask lies between
    # the original mask eroded and dilated by e = bound f / z_min px (+1 px of rasterisation): IoU >= (A - P (e + 1)) /
    # (A + P (e + 1)) with A the original mask's area and P its boundary pixel count
    tp = render.template_poses(0, distance=400.0)
    _, _, m0 = _render(mesh, tp, K, H, W)
    _, _, m1 = _render(fused, tp, K, H, W)
    m0, m1 = m0.cpu().numpy() > 0, m1.cpu().numpy() > 0
    z_min = 400.0 - float(np.linalg.norm(mesh.vertices, axis=1).max())
    e = bound * f / z_min
    for k in range(len(tp)):
        A = m0[k].sum()
        inner = m0[k][1:-1, 1:-1] & m0[k][:-2, 1:-1] & m0[k][2:, 1:-1] & m0[k][1:-1, :-2] & m0[k][1:-1, 2:]
        P = A - inner.sum()
        iou = (m0[k] & m1[k]).sum() / (m0[k] | m1[k]).sum()
        lim = (A - P * (e + 1)) / (A + P * (e + 1))
        assert iou >= lim, (k, iou, lim)
    print(f"blob masks: e = {e:.2f} px, smallest IoU over 42 views "
          f"{min(((m0[k] & m1[k]).sum() / (m0[k] | m1[k]).sum()) for k in range(len(tp))):.4f}")


def test_end_to_end_cube_colours():
    _, vol, fused, _ = _fuse_views("cube_colours")
    assert _closed(fused.faces)
    # A vertex's colour comes from the two corners of its lattice edge (within sqrt(3) h of it), each averaging pixels whose
    # depth lies within trunc of that corner along the pixel's ray.  So every pixel it averages sees a surface point within
    # trunc + sqrt(3) h + s of the vertex (s the pixel snap, as in the blob test); a vertex farther than that from every
    # cube edge therefore averages one face's pixels only, and ambient = 1 renders that face's colour (within 1 level of
    # the u8 albedo's round trip).  2 voxels is not enough: a grazing ray can reach the next face within trunc = 4 voxels.
    s = math.sqrt(2) / 2 * (400.0 + 70.0) / 600.0
    reach = vol.trunc + math.sqrt(3) * vol.voxel + s
    v = fused.vertices.astype(np.float64)
    half = 40.0
    # distance to the nearest cube edge: the second-largest of |half - |x_i||
    gap = np.sort(np.abs(half - np.abs(v)), axis=1)
    far = (gap[:, 1] > reach) & (gap[:, 0] < vol.voxel * 2)
    assert far.sum() > 100
    face = np.argmin(np.abs(half - np.abs(v)), axis=1) * 2 + (v[np.arange(len(v)), np.argmin(np.abs(half - np.abs(v)), axis=1)] > 0)
    want = sm.FACE_COLOURS[face[far]].astype(int)
    err = np.abs(fused.colors[far].astype(int) - want).max()
    print(f"cube: {far.sum()} vertices farther than {reach:.2f} mm from an edge, max colour error {err}")
    assert err <= 2


@pytest.fixture(scope="module")
def blob_scene(tmp_path_factory):
    """42 rendered views of the blob at 240 x 320 in BOP scene layout (depth_scale 0.1, mask/ and mask_visib/)"""
    from PIL import Image
    from sam6d_b200 import render
    root = tmp_path_factory.mktemp("fuse") / "scene"
    mesh = sm.build("blob")
    poses = render.template_poses(0, distance=400.0)
    K = np.array([[300.0, 0, 160.0], [0, 300.0, 120.0], [0, 0, 1]])
    rgb, depth, mask = _render(mesh, poses, K, 240, 320)
    rgb, depth, mask = rgb.cpu().numpy(), depth.cpu().numpy(), mask.cpu().numpy()
    for d in ("rgb", "depth", "mask", "mask_visib"):
        os.makedirs(root / d)
    cams, gts = {}, {}
    for i in range(len(poses)):
        Image.fromarray(rgb[i]).save(root / "rgb" / f"{i:06d}.png")
        Image.fromarray(np.round(depth[i] / 0.1).astype(np.uint16)).save(root / "depth" / f"{i:06d}.png")
        Image.fromarray(mask[i]).save(root / "mask" / f"{i:06d}_000000.png")
        Image.fromarray(mask[i]).save(root / "mask_visib" / f"{i:06d}_000000.png")
        cams[str(i)] = dict(cam_K=K.reshape(-1).tolist(), depth_scale=0.1)
        gts[str(i)] = [dict(obj_id=1, cam_R_m2c=poses[i, :3, :3].reshape(-1).tolist(), cam_t_m2c=poses[i, :3, 3].tolist())]
    json.dump(cams, open(root / "scene_camera.json", "w"))
    json.dump(gts, open(root / "scene_gt.json", "w"))
    return str(root)


def test_fused_model_feeds_onboard_and_run_sam6d(blob_scene, golden_dir, tmp_path):
    import cv2
    from sam6d_b200 import meshio
    from sam6d_b200.cli import fuse_object_model, run_sam6d
    from test_gpu_icp import _sam6d, _scene_meshes
    ply = str(tmp_path / "obj.ply")
    assert fuse_object_model.main(["--scene_dir", blob_scene, "--obj_id", "1", "--output_ply", ply, "--resolution", "96"]) == 0
    fused = meshio.load_ply_mesh(ply)
    assert len(fused.faces) > 1000 and fused.colors is not None and _closed(fused.faces)
    ob = _sam6d().onboard(fused, template_size=192, rng=np.random.RandomState(0))
    assert ob is not None
    _, (rgb, depth, K, scale) = _scene_meshes(golden_dir)
    cv2.imwrite(str(tmp_path / "rgb.png"), rgb[:, :, ::-1])
    cv2.imwrite(str(tmp_path / "depth.png"), depth)
    json.dump(dict(cam_K=np.asarray(K).reshape(-1).tolist(), depth_scale=float(scale)), open(tmp_path / "camera.json", "w"))
    out = tmp_path / "out"
    assert run_sam6d.main(["--output_dir", str(out), "--cad_path", ply, "--rgb_path", str(tmp_path / "rgb.png"),
                           "--depth_path", str(tmp_path / "depth.png"), "--cam_path", str(tmp_path / "camera.json"),
                           "--segmentor_model", "fastsam", "--random_weights", "--confidence_thresh", "-1", "--det_score_thresh", "-1",
                           "--template_size", "192"]) == 0
    pem = json.load(open(out / "sam6d_results" / "detection_pem.json"))
    print(f"run_sam6d on the fused model: {len(pem)} poses")
    assert pem and all(np.isfinite(np.asarray(p["R"], float)).all() for p in pem)


def test_ops_reject_bad_arguments():
    from sam6d_b200 import _lib, ops
    dev = "cuda"
    n = 8
    vol = (torch.ones(n, n, n, device=dev), torch.zeros(n, n, n, dtype=torch.int32, device=dev),
           torch.zeros(n, n, n, 3, dtype=torch.int32, device=dev), torch.zeros(n, n, n, dtype=torch.int32, device=dev))
    rgb = torch.zeros(1, 4, 4, 3, dtype=torch.uint8, device=dev)
    depth = torch.ones(1, 4, 4, device=dev)
    K = torch.tensor([[10.0, 10.0, 2.0, 2.0]], device=dev)
    P = torch.tensor([[1.0, 0, 0, 0, 1, 0, 0, 0, 1, 0, 0, 100]], device=dev)
    ok = dict(rgb=rgb, depth=depth, mask=None, K=K, pose=P)
    box = ((0.0, 0.0, 0.0), 1.0, 4.0, 1.0)
    before = _lib.launch_count()
    bad = [dict(rgb=rgb.cpu()), dict(depth=depth.double()), dict(depth=depth[:, :3]), dict(K=K[:, :3]),
           dict(pose=P * float("nan")), dict(mask=torch.zeros(1, 4, 4, device=dev)), dict(mask=torch.zeros(1, 3, 4, dtype=torch.uint8, device=dev))]
    for b in bad:
        a = dict(ok, **b)
        with pytest.raises(RuntimeError):
            ops.tsdf_integrate(a["rgb"], a["depth"], a["mask"], a["K"], a["pose"], *vol, *box)
    for bx in [((0.0, 0.0, 0.0), 0.0, 4.0, 1.0), ((0.0, 0.0, 0.0), 1.0, -1.0, 1.0), ((0.0, float("inf"), 0.0), 1.0, 4.0, 1.0)]:
        with pytest.raises(RuntimeError):
            ops.tsdf_integrate(rgb, depth, None, K, P, *vol, *bx)
    big = torch.ones(2, 2, 513, device=dev)
    with pytest.raises(RuntimeError, match="512"):
        ops.tsdf_mesh(big, big.int(), torch.zeros(2, 2, 513, 3, dtype=torch.int32, device=dev), big.int(), (0, 0, 0), 1.0)
    with pytest.raises(RuntimeError):
        ops.tsdf_mesh(vol[0].cpu(), *vol[1:], (0, 0, 0), 1.0)
    for mw in (0, -1):
        with pytest.raises(RuntimeError, match="min_weight"):
            ops.tsdf_mesh(*vol, (0, 0, 0), 1.0, min_weight=mw)
    assert _lib.launch_count() == before
    with pytest.raises(_lib.Sam6dError, match="invalid argument"):
        _lib.call("sam6d_tsdf_mesh_count", vol[0], vol[1], n, n, n, 0, vol[1], vol[1], vol[1])
    # the C ABI itself refuses an oversize volume and a NULL volume field with -22, launching nothing
    with pytest.raises(_lib.Sam6dError, match="invalid argument"):
        _lib.call("sam6d_tsdf_integrate", rgb, depth, None, K, P, 1, 4, 4, 0.0, 0.0, 0.0, 1.0, 4.0, 1.0, 513, n, n, *vol)
    with pytest.raises(_lib.Sam6dError, match="invalid argument"):
        _lib.call("sam6d_tsdf_mesh_count", None, vol[1], n, n, n, 1, vol[1], vol[1], vol[1])
    ops.tsdf_integrate(rgb, depth, None, K, P, *vol, *box)
    torch.cuda.synchronize()
