"""CPU: the template renderer's view set against the reference's level-0 poses, the rasteriser rules of oracle/render_oracle.py on
hand-built cases, PLY reading of textured and vertex-coloured models, and the argument surface of the two template CLIs."""
import os

import numpy as np
import pytest
import torch

from oracle import render_oracle as ro
from sam6d_b200 import meshio, render


# ---- view set ------------------------------------------------------------------------------------------------------------

def test_level0_poses_match_reference_as_a_set(golden_dir):
    ref = torch.load(os.path.join(golden_dir, "template_poses_level0.pt"))["obj_poses"].numpy()
    ours = render.level0_template_poses(1000.0)
    assert ours.shape == (42, 4, 4)
    d = np.abs(ours[:, None, :3, :3] - ref[None, :, :3, :3]).max(axis=(2, 3))
    match = d.argmin(axis=1)
    print("ours -> reference:", match.tolist(), f"max rotation difference {d.min(axis=1).max():.2e}")
    assert sorted(match.tolist()) == list(range(42))                                 # a bijection
    assert d.min(axis=1).max() < 1e-5
    assert np.abs(ours[:, :3, 3] - ref[match, :3, 3]).max() < 1e-3                  # (0, 0, 1000) up to rounding
    R = ours[:, :3, :3]
    assert np.allclose(R @ R.transpose(0, 2, 1), np.eye(3), atol=1e-12)
    assert np.allclose(np.linalg.det(R), 1.0, atol=1e-12)
    np.testing.assert_allclose(ours[:, 3], np.tile([0, 0, 0, 1.0], (42, 1)))


def test_level0_order_is_elevation_then_azimuth():
    P = render.level0_template_poses(2.0)
    cam = -np.einsum("tji,tj->ti", P[:, :3, :3], P[:, :3, 3])                        # camera centre = -R^T t
    np.testing.assert_allclose(np.linalg.norm(cam, axis=1), 2.0, atol=1e-12)
    el = np.round(np.degrees(np.arctan2(cam[:, 2], np.hypot(cam[:, 0], cam[:, 1]))), 6)
    az = np.round(np.degrees(np.arctan2(cam[:, 0], cam[:, 1])), 6)
    keys = list(zip(el, az))
    assert keys == sorted(keys)
    assert el[0] == -90 and el[-1] == 90


def test_template_K():
    np.testing.assert_allclose(render.template_K(512), [[560, 0, 256], [0, 560, 256], [0, 0, 1]])
    np.testing.assert_allclose(render.template_K(256), [[280, 0, 128], [0, 280, 128], [0, 0, 1]])


# ---- rasteriser rules ------------------------------------------------------------------------------------------------------

def _coverage(X, Y, faces, H, W):
    """per-triangle coverage counts of every pixel: (F, H, W) bool, from the oracle's integer rules"""
    X, Y = np.asarray(X, np.int64), np.asarray(Y, np.int64)
    s = ro.setup(faces, X, Y, np.ones(len(X), np.float32), np.ones(len(X), bool))
    yy, xx = np.mgrid[0:H, 0:W]
    out = []
    for f in range(len(faces)):
        cov, *_ = ro.cover(s, np.full(H * W, f), xx.ravel(), yy.ravel())
        out.append(cov.reshape(H, W) & (s["state"][f] == 1))
    return np.stack(out)


def _polygon_inside(px, py, H, W):
    """pixel centres inside a convex polygon (vertices in fixed point, either winding) under the top-left rule"""
    px, py = np.asarray(px, np.int64), np.asarray(py, np.int64)
    area2 = np.sum(px * np.roll(py, -1) - np.roll(px, -1) * py)
    if area2 < 0:                       # the rasteriser's positive orientation: edge(s, e, P) > 0 inside
        px, py = px[::-1], py[::-1]
    yy, xx = np.mgrid[0:H, 0:W]
    cx, cy = xx.astype(np.int64) * 256 + 128, yy.astype(np.int64) * 256 + 128
    inside = np.ones((H, W), bool)
    for i in range(len(px)):
        sx, sy, ex, ey = px[i], py[i], px[(i + 1) % len(px)], py[(i + 1) % len(px)]
        e = (ex - sx) * (cy - sy) - (ey - sy) * (cx - sx)
        inside &= ro._inside(e, ex - sx, ey - sy)
    return inside


@pytest.mark.parametrize("seed", range(6))
def test_quad_split_covers_each_pixel_once(seed):
    rng = np.random.RandomState(seed)
    H = W = 24
    if seed == 0:    # corners and diagonal exactly on pixel centres: every tie goes through the fill rule
        X, Y = np.array([3, 19, 19, 3]) * 256 + 128, np.array([4, 4, 20, 20]) * 256 + 128
    else:            # a random convex quad (corners on a circle, sorted by angle) in fixed point
        ang = np.sort(rng.uniform(0, 2 * np.pi, 4))
        X = np.rint((12 + 10 * np.cos(ang)) * 256).astype(np.int64)
        Y = np.rint((12 + 10 * np.sin(ang)) * 256).astype(np.int64)
        if seed % 2:
            X, Y = (X // 128) * 128, (Y // 128) * 128                               # half-pixel grid: many exact ties
    for faces in (np.array([[0, 1, 2], [0, 2, 3]]), np.array([[0, 2, 1], [3, 2, 0]]), np.array([[1, 2, 3], [1, 3, 0]])):
        cov = _coverage(X, Y, faces, H, W)
        count = cov.sum(axis=0)
        assert count.max() <= 1, "a pixel covered twice along the shared edge"
        np.testing.assert_array_equal(count == 1, _polygon_inside(X, Y, H, W))


def _hull(px, py):
    """integer convex hull (monotone chain), counter-clockwise in (x, y)"""
    pts = sorted(set(zip(px.tolist(), py.tolist())))

    def cross(o, a, b):
        return (a[0] - o[0]) * (b[1] - o[1]) - (a[1] - o[1]) * (b[0] - o[0])
    lower, upper = [], []
    for p in pts:
        while len(lower) >= 2 and cross(lower[-2], lower[-1], p) <= 0:
            lower.pop()
        lower.append(p)
    for p in reversed(pts):
        while len(upper) >= 2 and cross(upper[-2], upper[-1], p) <= 0:
            upper.pop()
        upper.append(p)
    h = lower[:-1] + upper[:-1]
    return np.array([p[0] for p in h]), np.array([p[1] for p in h])


@pytest.mark.parametrize("view", [0, 7, 20, 33, 41])
def test_convex_mesh_mask_is_the_projected_hull(view):
    v, f = ro.icosphere(2, 30.0)
    H = W = 96
    K = render.template_K(96)
    P = render.level0_template_poses(120.0)[view].astype(np.float32)
    P[:3, 3] += np.array([3.3, -2.1, 0.0], np.float32)                              # off-centre, no symmetry
    out = ro.render_view(dict(vertices=v, faces=f), P, K, H, W)
    X, Y, _, ok = ro.vertex_pass(v, P, K, 1e-3)
    assert ok.all()
    hx, hy = _hull(X, Y)
    np.testing.assert_array_equal(out["mask"] == 255, _polygon_inside(hx, hy, H, W))
    assert out["dropped"] == 0


def _quads_mesh(z_a, z_b):
    """two overlapping axis-aligned quads facing the camera, faces 0-1 at depth z_a, faces 2-3 at z_b"""
    v = np.array([[-2, -2, z_a], [1, -2, z_a], [1, 1, z_a], [-2, 1, z_a],
                  [-1, -1, z_b], [2, -1, z_b], [2, 2, z_b], [-1, 2, z_b]], np.float32)
    f = np.array([[0, 1, 2], [0, 2, 3], [4, 5, 6], [4, 6, 7]], np.int32)
    return dict(vertices=v, faces=f)


def test_nearest_wins_and_equal_depth_goes_to_lower_id():
    K = np.array([[32.0, 0, 16], [0, 32.0, 16], [0, 0, 1]])
    P = np.eye(4, dtype=np.float32)
    ov = np.zeros((32, 32), bool)
    ov[12:20, 12:20] = True                      # centres 12.5 .. 19.5 px: inside quad A (8 .. 20 px at z = 8) and quad B at z 6 or 8
    near_b = ro.render_view(_quads_mesh(8.0, 6.0), P, K, 32, 32)
    near_a = ro.render_view(_quads_mesh(6.0, 8.0), P, K, 32, 32)
    assert np.isin(near_b["tri"][ov], [2, 3]).all() and np.allclose(near_b["depth"][ov], 6.0, rtol=1e-6)
    assert np.isin(near_a["tri"][ov], [0, 1]).all() and np.allclose(near_a["depth"][ov], 6.0, rtol=1e-6)
    # the same quad twice: every pixel is an exact depth tie, and the lower face ids win all of them
    dup = dict(vertices=_quads_mesh(8.0, 8.0)["vertices"][[0, 1, 2, 3, 0, 1, 2, 3]], faces=_quads_mesh(8.0, 8.0)["faces"])
    tie = ro.render_view(dup, P, K, 32, 32)
    m = tie["mask"] == 255
    assert m.sum() == 12 * 12 and np.isin(tie["tri"][m], [0, 1]).all() and np.allclose(tie["depth"][m], 8.0, rtol=1e-6)
    # a tilted quad crossing a flat one: per pixel the nearer surface, whichever id it has
    v = np.array([[-2, -2, 6], [2, -2, 6], [2, 2, 10], [-2, 2, 10], [-2, -2, 8], [2, -2, 8], [2, 2, 8], [-2, 2, 8]], np.float32)
    f = np.array([[4, 5, 6], [4, 6, 7], [0, 1, 2], [0, 2, 3]], np.int32)
    out = ro.render_view(dict(vertices=v, faces=f), P, K, 32, 32)
    m = out["mask"] == 255
    flat = np.isin(out["tri"], [0, 1])
    assert flat.any() and (m & ~flat).any()
    assert np.allclose(out["depth"][m & flat], 8.0, rtol=1e-6) and (out["depth"][m & ~flat] <= 8.0 * (1 + 1e-6)).all()


def test_xyz_lies_on_the_triangle_and_reprojects_to_the_pixel_centre():
    # vertices whose projections fall on the 1/256 px grid (dyadic coordinates, power-of-two depths and focal length), so the
    # fixed-point snap is exact and what remains is the float32 perspective interpolation
    K = np.array([[64.0, 0, 32], [0, 64.0, 32], [0, 0, 1]])
    rng = np.random.RandomState(3)
    verts, faces = [], []
    for k in range(6):
        for z in rng.choice([2.0, 4.0, 8.0], 3):
            u, v = rng.randint(2 * 256, 62 * 256, 2) / 256.0
            verts.append([(u - 32) * z / 64.0, (v - 32) * z / 64.0, z])
        faces.append([3 * k, 3 * k + 1, 3 * k + 2])
    V, F = np.asarray(verts, np.float32), np.asarray(faces, np.int32)
    out = ro.render_view(dict(vertices=V, faces=F), np.eye(4, dtype=np.float32), K, 64, 64)
    yy, xx = np.nonzero(out["mask"] == 255)
    assert len(yy) > 200
    p = out["xyz32"][yy, xx].astype(np.float64)
    u = 64.0 * p[:, 0] / p[:, 2] + 32
    v = 64.0 * p[:, 1] / p[:, 2] + 32
    err = np.hypot(u - (xx + 0.5), v - (yy + 0.5))
    print(f"max reprojection error {err.max():.2e} px over {len(err)} pixels")
    assert err.max() < 1e-3
    tri = F[out["tri"][yy, xx]]
    a, b, c = (V[tri[:, k]].astype(np.float64) for k in range(3))
    n = np.cross(b - a, c - a)
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    assert np.abs(np.sum((p - a) * n, axis=1)).max() < 1e-5 * np.abs(p).max()        # on the plane
    np.testing.assert_array_equal(out["xyz"][yy, xx], out["xyz32"][yy, xx].astype(np.float16))


def test_vertex_behind_the_camera_is_dropped():
    v, f = ro.icosphere(1, 1.0)
    P = np.eye(4, dtype=np.float32)
    P[2, 3] = 0.5                                                                      # camera inside the sphere
    out = ro.render_view(dict(vertices=v, faces=f), P, render.template_K(64), 64, 64)
    assert out["dropped"] > 0 and out["dropped"] < len(f)


# ---- PLY -------------------------------------------------------------------------------------------------------------------

def _write_ply(path, V, F, colors=None, uv=None, tex=None, binary=False):
    props = ["property float x", "property float y", "property float z"]
    if colors is not None:
        props += ["property uchar red", "property uchar green", "property uchar blue"]
    if uv is not None:
        props += ["property float texture_u", "property float texture_v"]
    head = ["ply", "format " + ("binary_little_endian" if binary else "ascii") + " 1.0"]
    if tex is not None:
        head.append(f"comment TextureFile {tex}")
    head += [f"element vertex {len(V)}"] + props + [f"element face {len(F)}", "property list uchar int vertex_indices", "end_header"]
    with open(path, "wb") as fh:
        fh.write(("\n".join(head) + "\n").encode())
        if binary:
            dt = [("x", "<f4"), ("y", "<f4"), ("z", "<f4")] + ([("red", "u1"), ("green", "u1"), ("blue", "u1")] if colors is not None else []) \
                + ([("texture_u", "<f4"), ("texture_v", "<f4")] if uv is not None else [])
            rec = np.zeros(len(V), dtype=dt)
            rec["x"], rec["y"], rec["z"] = V[:, 0], V[:, 1], V[:, 2]
            if colors is not None:
                rec["red"], rec["green"], rec["blue"] = colors[:, 0], colors[:, 1], colors[:, 2]
            if uv is not None:
                rec["texture_u"], rec["texture_v"] = uv[:, 0], uv[:, 1]
            fh.write(rec.tobytes())
            for f in F:
                fh.write(np.uint8(3).tobytes() + np.asarray(f, "<i4").tobytes())
        else:
            for i in range(len(V)):
                row = ["%.6f" % x for x in V[i]]
                row += ["%d" % c for c in colors[i]] if colors is not None else []
                row += ["%.6f" % x for x in uv[i]] if uv is not None else []
                fh.write((" ".join(row) + "\n").encode())
            for f in F:
                fh.write(("3 %d %d %d\n" % tuple(f)).encode())


@pytest.mark.parametrize("binary", [False, True])
def test_load_ply_mesh_textured_and_coloured(tmp_path, binary):
    import cv2
    V, F = ro.icosphere(1, 25.0)
    rng = np.random.RandomState(0)
    uv = rng.uniform(0, 1, (len(V), 2)).astype(np.float32)
    tex = rng.randint(0, 256, (16, 24, 3)).astype(np.uint8)
    cv2.imwrite(str(tmp_path / "obj.png"), tex[:, :, ::-1])
    textured = str(tmp_path / "textured.ply")
    _write_ply(textured, V, F, uv=uv, tex="obj.png", binary=binary)
    m = meshio.load_ply_mesh(textured)
    np.testing.assert_allclose(m.vertices, V, atol=1e-5)
    np.testing.assert_array_equal(m.faces, F)
    np.testing.assert_allclose(m.uv, uv, atol=1e-5)
    np.testing.assert_array_equal(m.texture, tex)
    assert m.colors is None and m.texture_file == str(tmp_path / "obj.png")
    v3, f3, c3 = meshio.load_ply(textured)                                           # the 3-tuple reader is unchanged
    np.testing.assert_array_equal(v3, m.vertices)
    np.testing.assert_array_equal(f3, F.astype(np.int64))
    assert f3.dtype == np.int64 and v3.dtype == np.float32 and c3 is None

    col = rng.randint(0, 256, (len(V), 3)).astype(np.uint8)
    coloured = str(tmp_path / "coloured.ply")
    _write_ply(coloured, V, F, colors=col, binary=binary)
    m = meshio.load_ply_mesh(coloured)
    np.testing.assert_array_equal(m.colors, col)
    assert m.uv is None and m.texture is None and m.texture_file is None
    v3, f3, c3 = meshio.load_ply(coloured)
    np.testing.assert_array_equal(c3, col)
    assert c3.dtype == np.uint8 and f3.shape == F.shape


def test_load_ply_mesh_st_coordinates(tmp_path):
    p = tmp_path / "st.ply"
    p.write_text("ply\nformat ascii 1.0\nelement vertex 3\nproperty float x\nproperty float y\nproperty float z\nproperty float s\n"
                 "property float t\nelement face 1\nproperty list uchar int vertex_indices\nend_header\n"
                 "0 0 0 0.1 0.2\n1 0 0 0.3 0.4\n0 1 0 0.5 0.6\n3 0 1 2\n")
    m = meshio.load_ply_mesh(str(p))
    np.testing.assert_allclose(m.uv, [[0.1, 0.2], [0.3, 0.4], [0.5, 0.6]], atol=1e-6)
    assert m.texture is None


# ---- CLIs and host checks --------------------------------------------------------------------------------------------------

def _actions(ap):
    return {a.dest: a for a in ap._actions if a.dest != "help"}


def test_custom_cli_arguments_match_reference():
    from sam6d_b200.cli import render_custom_templates as cli
    acts = _actions(cli.get_parser())
    # SAM-6D/Render/render_custom_templates.py: untyped values, so any value given on the command line is truthy
    ref = dict(cad_path=None, output_dir=None, normalize=True, colorize=False, base_color=0.05)
    for k, default in ref.items():
        assert acts[k].default == default and acts[k].type is None and acts[k].option_strings == [f"--{k}"]
    assert set(acts) - set(ref) == {"size", "poses"}
    a = cli.get_parser().parse_args(["--cad_path", "x.ply", "--output_dir", "o", "--normalize", "False", "--colorize", "0"])
    assert a.normalize and a.colorize and a.size == 512 and a.poses is None


def test_bop_cli_arguments_match_reference():
    from sam6d_b200.cli import render_bop_templates as cli
    acts = _actions(cli.get_parser())
    assert acts["dataset_name"].default is None and acts["dataset_name"].type is None
    assert set(acts) - {"dataset_name"} == {"bop_root", "output_dir", "size", "poses"}


def test_poses_file_scales_to_the_framing_distance(tmp_path, golden_dir):
    from sam6d_b200.cli import render_custom_templates as cli
    ref = torch.load(os.path.join(golden_dir, "template_poses_level0.pt"))["obj_poses"].numpy()
    path = str(tmp_path / "obj_poses_level0.npy")
    np.save(path, ref)
    P = cli.view_poses(400.0, path)
    np.testing.assert_allclose(P[:, :3, :3], ref[:, :3, :3])
    np.testing.assert_allclose(P[:, :3, 3], np.tile([0, 0, 400.0], (42, 1)), atol=1e-6)
    np.testing.assert_allclose(cli.to_metres(P)[:, :3, 3], np.tile([0, 0, 0.4], (42, 1)), atol=1e-9)


def test_render_rejects_cpu_tensors():
    v, f = ro.icosphere(0)
    mesh = meshio.Mesh(torch.from_numpy(v), torch.from_numpy(f))
    with pytest.raises(RuntimeError, match="CUDA"):
        render.render([mesh], torch.eye(4).reshape(1, 1, 4, 4), render.template_K(32), 32, 32)
