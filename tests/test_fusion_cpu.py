"""CPU: TSDF fusion's host side and its numpy oracle (oracle/fusion_oracle.py, sam6d_b200/fusion.py, meshio.save_ply,
cli/fuse_object_model.py).

- The extraction rule on analytic volumes: a sphere on a 32^3 lattice gives a closed, consistently wound 2-manifold with
  Euler characteristic 2 (a torus 0), an enclosed volume inside a bound derived from the voxel size, and face normals along
  +grad tsdf.  All 16 sign patterns of each Kuhn tetrahedron give the expected triangle count and winding.  A half-space of
  zero weights opens the mesh exactly along the lattice plane where observed voxels meet unobserved ones.
- save_ply -> load_ply_mesh round-trips exactly; the CLI's BOP-layout discovery, mask preference, skipped frames and errors;
  fusion.py's input checks raise before any device work."""
import json
import math
import os

import numpy as np
import pytest

from oracle import fusion_oracle as fo


def _volume(fn, n=32, h=1.0, trunc=4.0, lo=0.0):
    """tsdf = clip(f / trunc, -1, 1) of a signed distance f sampled at the voxel centres of an n^3 lattice"""
    c = lo + (np.arange(n) + 0.5) * h
    z, y, x = np.meshgrid(c, c, c, indexing="ij")
    f = fn(x, y, z)
    tsdf = np.clip(f / trunc, -1, 1).astype(np.float32)
    shape = tsdf.shape
    return tsdf, np.ones(shape, np.int32), np.zeros(shape + (3,), np.uint32), np.zeros(shape, np.int32)


def _sphere(R=10.0, ctr=(16.0, 16.0, 16.0)):
    return lambda x, y, z: np.sqrt((x - ctr[0]) ** 2 + (y - ctr[1]) ** 2 + (z - ctr[2]) ** 2) - R


def _torus(Rmaj=9.0, rmin=4.0, ctr=(16.0, 16.0, 16.0)):
    return lambda x, y, z: np.sqrt((np.sqrt((x - ctr[0]) ** 2 + (y - ctr[1]) ** 2) - Rmaj) ** 2 + (z - ctr[2]) ** 2) - rmin


def _edges(faces):
    """directed edges (F*3, 2)"""
    return np.concatenate([faces[:, [0, 1]], faces[:, [1, 2]], faces[:, [2, 0]]])


def _closed_manifold(faces):
    """every undirected edge in exactly two faces, once in each direction -> the number of undirected edges"""
    d = _edges(faces)
    assert len(np.unique(d, axis=0)) == len(d), "a directed edge appears twice: inconsistent winding or non-manifold"
    rev = set(map(tuple, d[:, ::-1]))
    assert all(tuple(e) in rev for e in d), "an edge with one face: the mesh is open"
    return len(d) // 2


def _enclosed_volume(v, f):
    a, b, c = v[f[:, 0]].astype(np.float64), v[f[:, 1]].astype(np.float64), v[f[:, 2]].astype(np.float64)
    return np.einsum("ij,ij->i", a, np.cross(b, c)).sum() / 6.0


def test_sphere_is_closed_manifold_with_bounded_volume_and_outward_normals():
    h, R = 1.0, 10.0
    vol = _volume(_sphere(R))
    v, col, f = fo.mesh(*vol, bbox_min=(0, 0, 0), voxel=h)
    assert len(f) > 1000 and len(v) == len(np.unique(f))               # only used vertices are kept
    E = _closed_manifold(f)
    assert len(v) - E + len(f) == 2
    # Marching tetrahedra returns the zero set of the piecewise-linear interpolant L of the corner values.  The corners of
    # every tetrahedron the surface crosses lie within its diameter sqrt(3) h < trunc of the surface, so no clipping
    # touches them and L interpolates f = |p - c| - R exactly at the corners.  On a simplex of diameter D, |f - L| <=
    # M D^2 / 2 with M the largest second directional derivative of f, 1 / |p - c| <= 1 / (R - sqrt(3) h) there.  So the
    # surface lies in the shell |f| <= eps = (3 h^2 / 2) / (R - sqrt(3) h), and it bounds a volume between the balls of
    # radius R -+ eps.
    eps = 1.5 * h * h / (R - math.sqrt(3) * h)
    r = np.linalg.norm(v - 16.0, axis=1)
    assert np.abs(r - R).max() <= eps
    V = _enclosed_volume(v, f)
    lo, hi = 4 / 3 * math.pi * (R - eps) ** 3, 4 / 3 * math.pi * (R + eps) ** 3
    print(f"sphere: V {len(v)} F {len(f)}, volume {V:.1f} in [{lo:.1f}, {hi:.1f}], max radial error {np.abs(r - R).max():.4f} "
          f"(bound {eps:.4f})")
    assert lo <= V <= hi
    # outward: each face normal along grad tsdf = (x - c) / |x - c| at its centroid
    a, b, c = v[f[:, 0]], v[f[:, 1]], v[f[:, 2]]
    n = np.cross(b - a, c - a)
    cen = (a + b + c) / 3.0 - 16.0
    nz = np.linalg.norm(n, axis=1) > 0
    assert (np.einsum("ij,ij->i", n, cen)[nz] > 0).all()
    assert (col == 128).all()                                           # no colour observed: grey


def test_torus_has_euler_characteristic_zero():
    vol = _volume(_torus())
    v, _, f = fo.mesh(*vol, bbox_min=(0, 0, 0), voxel=1.0)
    E = _closed_manifold(f)
    assert len(v) - E + len(f) == 0


@pytest.mark.parametrize("t", range(6))
def test_every_sign_pattern_of_a_tetrahedron(t):
    path = fo.tetrahedra()[t]
    corner = lambda c: np.array([c & 1, (c >> 1) & 1, (c >> 2) & 1], np.float64)    # noqa: E731
    for pat in range(16):
        tsdf = np.ones((2, 2, 2), np.float32)
        weight = np.zeros((2, 2, 2), np.int32)
        vals = {}
        for j, c in enumerate(path):
            x, y, z = corner(c).astype(int)
            vals[c] = -0.5 - 0.1 * j if (pat >> j) & 1 else 0.5 + 0.1 * j
            tsdf[z, y, x] = vals[c]
            weight[z, y, x] = 1                                         # only this tetrahedron has 4 observed corners
        v, _, f = fo.mesh(tsdf, weight, np.zeros((2, 2, 2, 3), np.uint32), np.zeros((2, 2, 2), np.int32), (0, 0, 0), 1.0)
        n_in = bin(pat).count("1")
        assert len(f) == {0: 0, 4: 0, 1: 1, 3: 1, 2: 2}[n_in], (t, pat)
        if not len(f):
            continue
        # the linear interpolant over the tetrahedron: its gradient g solves (c_j - c_0) . g = val_j - val_0
        A = np.stack([corner(c) - corner(path[0]) for c in path[1:]])
        g = np.linalg.solve(A, np.array([vals[c] - vals[path[0]] for c in path[1:]]))
        for tri in f:
            a, b, c = v[tri].astype(np.float64)
            assert np.dot(np.cross(b - a, c - a), g) > 0, (t, pat, tri)
        assert len(v) == {1: 3, 3: 3, 2: 4}[n_in]


def test_unobserved_half_space_opens_the_mesh_along_the_seam():
    tsdf, weight, csum, cnt = _volume(_sphere())
    m = 16
    weight[:, :, :m] = 0                                                # voxels with x index < 16 never observed
    v, _, f = fo.mesh(tsdf, weight, csum, cnt, (0, 0, 0), 1.0)
    d = _edges(f)
    rev = set(map(tuple, d[:, ::-1]))
    boundary = np.array([e for e in d if tuple(e) not in rev])
    assert len(boundary) > 0 and len(np.unique(d, axis=0)) == len(d)
    # a tetrahedron with a corner at x index < m emits nothing, so the open rim lies on lattice edges within the plane
    # x index = m: vertex x = (m + 0.5) h exactly; every other edge keeps its two faces
    assert np.array_equal(np.unique(v[boundary.reshape(-1), 0]), np.array([m + 0.5], np.float32))
    assert (v[:, 0] >= m + 0.5).all()
    weight[:] = 1
    _closed_manifold(fo.mesh(tsdf, weight, csum, cnt, (0, 0, 0), 1.0)[2])


def test_min_weight_and_colour_interpolation():
    tsdf, weight, csum, cnt = _volume(_sphere(R=6.0, ctr=(8, 8, 8)), n=16)
    cnt[:] = 2
    csum[...] = np.array([20, 100, 201], np.uint32)                     # mean colour 10, 50, 100.5
    v, col, f = fo.mesh(tsdf, weight, csum, cnt, (0, 0, 0), 1.0)
    assert (col == np.array([10, 50, 100], np.uint8)).all()             # 100.5 rounds half to even
    v2, _, f2 = fo.mesh(tsdf, weight, csum, cnt, (0, 0, 0), 1.0, min_weight=2)
    assert len(f2) == 0


def test_integration_oracle_f32_matches_f64_rule():
    """the float32 restatement and the float64 one fuse the same analytic views to within float32 rounding"""
    rng = np.random.RandomState(0)
    T, H, W = 3, 24, 32
    depth = (300.0 + rng.rand(T, H, W) * 20).astype(np.float32)
    depth[:, :2] = 0
    mask = (rng.rand(T, H, W) > 0.3).astype(np.uint8)
    rgb = rng.randint(0, 256, (T, H, W, 3)).astype(np.uint8)
    K4 = np.tile(np.array([[40.0, 40.0, 16.0, 12.0]], np.float32), (T, 1))
    P12 = np.zeros((T, 12), np.float32)
    P12[:, [0, 4, 8]] = 1
    P12[:, 11] = 300.0
    args = (rgb, depth, mask, K4, P12, (12, 10, 8), (-30.0, -25.0, -20.0), 5.0, 20.0, 1.0)
    s32 = fo.integrate(*args)
    s64 = fo.integrate(*args, dtype=np.float64)
    assert s32["weight"].max() == T and (s32["weight"] == s64["weight"]).mean() > 0.99
    same = s32["weight"] == s64["weight"]
    assert np.abs(s32["tsdf"][same] - s64["tsdf"][same]).max() < 1e-5
    assert s32["ccount"].sum() > 0


def test_save_ply_round_trip(tmp_path):
    from sam6d_b200 import meshio
    rng = np.random.RandomState(1)
    v = (rng.randn(50, 3) * 100).astype(np.float32)
    f = rng.randint(0, 50, (80, 3)).astype(np.int64)
    c = rng.randint(0, 256, (50, 3)).astype(np.uint8)
    p = str(tmp_path / "m.ply")
    meshio.save_ply(p, meshio.Mesh(v, f, c))
    m = meshio.load_ply_mesh(p)
    assert m.vertices.dtype == np.float32 and np.array_equal(m.vertices, v)
    assert np.array_equal(m.faces, f) and np.array_equal(m.colors, c) and m.uv is None
    meshio.save_ply(p, meshio.Mesh(v, f))
    m = meshio.load_ply_mesh(p)
    assert m.colors is None and np.array_equal(m.faces, f)
    with pytest.raises(ValueError):
        meshio.save_ply(p, meshio.Mesh(v, f + 50, c))


# ---- the CLI's file discovery ---------------------------------------------------------------------------------------------
def _png(path, a):
    from PIL import Image
    os.makedirs(os.path.dirname(path), exist_ok=True)
    Image.fromarray(a).save(path)


def _scene(root, ids_with_obj=(0, 2), n=4, masks=("mask", "mask_visib"), H=8, W=10):
    os.makedirs(root, exist_ok=True)
    cams, gts = {}, {}
    for i in range(n):
        cams[str(i)] = dict(cam_K=[50.0, 0, 5, 0, 50.0, 4, 0, 0, 1], depth_scale=0.1)
        gt = [dict(obj_id=9, cam_R_m2c=list(np.eye(3).reshape(-1)), cam_t_m2c=[0, 0, 500.0])]
        if i in ids_with_obj:
            gt.append(dict(obj_id=3, cam_R_m2c=list(np.eye(3).reshape(-1)), cam_t_m2c=[1.0, 2.0, 400.0 + i]))
        gts[str(i)] = gt
        _png(os.path.join(root, "rgb", f"{i:06d}.png"), np.full((H, W, 3), 40 * i, np.uint8))
        _png(os.path.join(root, "depth", f"{i:06d}.png"), np.full((H, W), 4000 + i, np.uint16))
        for k in range(len(gt)):
            for mdir in masks:
                _png(os.path.join(root, mdir, f"{i:06d}_{k:06d}.png"), np.full((H, W), 255 if mdir == "mask" else 7, np.uint8))
    json.dump(cams, open(os.path.join(root, "scene_camera.json"), "w"))
    json.dump(gts, open(os.path.join(root, "scene_gt.json"), "w"))


def test_cli_discovery(tmp_path):
    from sam6d_b200.cli import fuse_object_model as cli
    up, down = str(tmp_path / "up"), str(tmp_path / "down")
    _scene(up)
    _scene(down, ids_with_obj=(1,), masks=("mask_visib",))
    fr, skipped, mdir = cli.scene_frames(up, 3)
    assert [os.path.basename(f["rgb"]) for f in fr] == ["000000.png", "000002.png"] and skipped == 2
    assert os.path.basename(mdir) == "mask" and fr[0]["mask"].endswith(os.path.join("mask", "000000_000001.png"))
    assert fr[1]["pose"][2, 3] == 402.0 and fr[0]["depth_scale"] == 0.1
    fr2, skipped2, mdir2 = cli.scene_frames(down, 3)
    assert len(fr2) == 1 and skipped2 == 3 and os.path.basename(mdir2) == "mask_visib"
    assert len(cli.scene_frames(up, 3, frame_step=2)[0]) == 2 and len(cli.scene_frames(up, 3, frame_step=3)[0]) == 1
    rgb, depth, masks, K, poses = cli.load_views(fr + fr2)
    assert rgb.shape == (3, 8, 10, 3) and depth.dtype == np.float32 and masks.shape == (3, 8, 10)
    assert depth[0, 0, 0] == np.float32(4000) * np.float32(0.1) and masks[0].max() == 255 and masks[2].max() == 7
    assert K.shape == (3, 3, 3) and poses.shape == (3, 4, 4)


def test_cli_errors(tmp_path, capsys):
    from sam6d_b200.cli import fuse_object_model as cli
    s = str(tmp_path / "s")
    _scene(s)
    out = str(tmp_path / "o.ply")

    def fails(argv, msg):
        with pytest.raises(SystemExit):
            cli.main(argv)
        assert msg in capsys.readouterr().err

    fails(["--scene_dir", str(tmp_path / "nope"), "--obj_id", "3", "--output_ply", out], "no scene folder")
    fails(["--scene_dir", s, "--obj_id", "4", "--output_ply", out], "shows obj_id 4")
    fails(["--scene_dir", s, "--obj_id", "3", "--output_ply", out, "--frame_step", "0"], "--frame_step")
    fails(["--scene_dir", s, "--obj_id", "3", "--output_ply", out, "--trunc_voxels", "nan"], "--trunc_voxels")
    fails(["--scene_dir", s, "--obj_id", "3", "--output_ply", out, "--resolution", "64", "--voxel_size", "2"], "not allowed")
    os.remove(os.path.join(s, "mask", "000002_000001.png"))
    fails(["--scene_dir", s, "--obj_id", "3", "--output_ply", out], "no mask/000002_000001.png")
    os.remove(os.path.join(s, "depth", "000000.png"))
    fails(["--scene_dir", s, "--obj_id", "3", "--output_ply", out], "image 0 has no depth file")
    os.remove(os.path.join(s, "scene_gt.json"))
    fails(["--scene_dir", s, "--obj_id", "3", "--output_ply", out], "no scene_gt.json")
    assert not os.path.exists(out)


# ---- fusion.py's checks: ValueError / TypeError before the device is touched ---------------------------------------------------
def _views(T=2, H=6, W=8):
    return (np.zeros((T, H, W, 3), np.uint8), np.full((T, H, W), 1000, np.uint16), np.full((T, H, W), 255, np.uint8),
            np.array([[50.0, 0, 4], [0, 50.0, 3], [0, 0, 1]]), np.tile(np.eye(4), (T, 1, 1)))


def test_fusion_input_checks(monkeypatch):
    from sam6d_b200 import fusion, ops
    monkeypatch.setattr(ops, "tsdf_integrate", lambda *a, **k: pytest.fail("reached the device"))
    monkeypatch.setattr(ops, "tsdf_mesh", lambda *a, **k: pytest.fail("reached the device"))
    rgb, depth, masks, K, poses = _views()
    poses[:, 2, 3] = 500.0
    ok = dict(rgb_u8=rgb, depth_raw=depth, masks=masks, cam_K=K, poses_m2c=poses, depth_scale=0.1)
    assert fusion.check_views(**ok)[:3] == (2, 6, 8)
    bad = [dict(depth_scale=0.0), dict(depth_scale=float("nan")), dict(depth_scale=-1.0), dict(depth_scale=1e300),
           dict(rgb_u8=rgb[..., :2]), dict(rgb_u8=rgb.astype(np.float32)), dict(depth_raw=depth.astype(np.float64)),
           dict(depth_raw=depth[:1]), dict(masks=masks.astype(bool)), dict(masks=masks[:, :3]), dict(cam_K=np.stack([K] * 3)),
           dict(poses_m2c=poses[:1]), dict(poses_m2c=np.where(np.eye(4, dtype=bool), np.nan, poses)), dict(cam_K=K + np.inf),
           dict(depth_raw=np.zeros((0, 6, 8), np.uint16), rgb_u8=np.zeros((0, 6, 8, 3), np.uint8), masks=None)]
    for b in bad:
        with pytest.raises((ValueError, TypeError)):
            fusion.check_views(**dict(ok, **b))
        with pytest.raises((ValueError, TypeError)):
            fusion.fuse(*dict(ok, **b).values())
    lo, hi, voxel, trunc = fusion.view_bounds(depth, masks, K, poses, 0.1, resolution=16)
    # a 100 mm deep plane in front of the camera: x over columns 0..7 at (c - 4) 100 / 50
    assert np.allclose([lo[0] + 6 * voxel, hi[0] - 6 * voxel], [-8.0, 6.0]) and trunc == 4 * voxel
    assert voxel == pytest.approx(14.0 / 16)
    with pytest.raises(ValueError, match="no view"):
        fusion.view_bounds(depth, np.zeros_like(masks), K, poses, 0.1)
    for args in [((0, 0, 0), (10, 10, 10), 0.0), ((0, 0, 0), (10, 10, 10), float("inf")), ((0, 0, 0), (0, 10, 10), 1.0),
                 ((0, 0, 0), (10, 10, 10), 1.0, -1.0), ((0, 0, 0), (513, 10, 10), 1.0), ((0, 0, float("nan")), (1, 1, 1), 0.1)]:
        with pytest.raises(ValueError):
            fusion.TsdfVolume(*args, device="cpu")
