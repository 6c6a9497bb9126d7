"""CPU: the float64 restatement of the point-to-plane ICP refinement (oracle/icp_oracle.py) on cases whose answer is known,
the surface normals of meshio.sample_surface, and the --icp_iters option of the three CLIs."""
import numpy as np
import pytest

from oracle import icp_oracle as io
from sam6d_b200 import meshio


def box_mesh(hx, hy, hz):
    """a closed box centred at the origin, outward faces"""
    v = np.array([[x, y, z] for x in (-hx, hx) for y in (-hy, hy) for z in (-hz, hz)], dtype=np.float32)
    quads = [(0, 1, 3, 2), (4, 6, 7, 5), (0, 4, 5, 1), (2, 3, 7, 6), (0, 2, 6, 4), (1, 5, 7, 3)]
    faces = np.array([t for a, b, c, d in quads for t in ((a, b, c), (a, c, d))], dtype=np.int64)
    return v, faces


def random_rotation(rng):
    q = rng.normal(size=4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def perturb(R, t, rng, deg, shift):
    """(R, t) composed with a rotation of `deg` degrees about a random axis and moved by `shift` in a random direction"""
    axis = rng.normal(size=3)
    axis /= np.linalg.norm(axis)
    d = rng.normal(size=3)
    return R @ io.so3_exp(np.radians(deg) * axis), t + shift * d / np.linalg.norm(d)


def box_scene(seed, n_obs=400, m=1024):
    rng = np.random.RandomState(seed)
    v, f = box_mesh(0.05, 0.03, 0.02)
    Q, Nn = meshio.sample_surface(v, f, m, rng, return_normals=True)
    Q, Nn = Q.astype(np.float64), Nn.astype(np.float64)
    r = float(np.linalg.norm(Q, axis=1).max())
    R, t = random_rotation(rng), np.array([0.02, -0.01, 0.6])
    P = Q[rng.choice(m, n_obs, replace=False)] @ R.T + t
    return rng, Q, Nn, r, R, t, P


def test_oracle_recovers_a_known_pose():
    rng, Q, Nn, r, R, t, P = box_scene(0)
    R0, t0 = perturb(R, t, rng, 5.0, 0.05 * r)
    res = io.refine(R0, t0, P, Q, Nn, r, 30)
    assert res["history"][-1]["stop"] and res["iters_run"] < 30
    assert np.abs(res["R"] - R).max() < 1e-9 and np.abs(res["t"] - t).max() < 1e-9, (res["R"] - R, res["t"] - t)
    assert res["inliers"] == len(P) and res["rms"] < 1e-9


def test_oracle_trims_planted_outliers():
    rng, Q, Nn, r, R, t, P = box_scene(1)
    # 10 % outliers on a plane 2 r behind the object: at least r from every sample, beyond tau_0 = 0.3 r
    uv = rng.uniform(-2 * r, 2 * r, size=(len(P) // 10, 2))
    out_obj = np.concatenate([uv, np.full((len(uv), 1), 2 * r)], axis=1)
    P_all = np.concatenate([P, out_obj @ R.T + t])
    R0, t0 = perturb(R, t, rng, 5.0, 0.05 * r)
    res = io.refine(R0, t0, P_all, Q, Nn, r, 30)
    for s in res["history"]:
        assert not s["inlier"][len(P):].any()
    assert np.abs(res["R"] - R).max() < 1e-9 and np.abs(res["t"] - t).max() < 1e-9
    assert res["inliers"] == len(P)


def test_damping_holds_the_unobservable_directions_of_a_plane():
    rng = np.random.RandomState(2)
    m = 1024
    Q = np.concatenate([rng.uniform(-0.05, 0.05, size=(m, 2)), np.zeros((m, 1))], axis=1)
    Nn = np.tile([0.0, 0.0, 1.0], (m, 1))
    r = float(np.linalg.norm(Q, axis=1).max())
    R, t = random_rotation(rng), np.array([0.01, 0.02, 0.5])
    P = Q[rng.choice(m, 500, replace=False)] @ R.T + t
    # start: rotated 4 degrees about the plane normal, moved 0.03 r in the plane and 0.02 r along the normal (object frame)
    R0 = R @ io.so3_exp([0.0, 0.0, np.radians(4.0)])
    t0 = t + R @ np.array([0.02 * r, -0.02 * r, 0.02 * r])
    res = io.refine(R0, t0, P, Q, Nn, r, 20)
    for s in res["history"]:
        if s["applied"]:
            assert np.all(s["delta"][[2, 3, 4]] == 0.0)           # w_z, v_x, v_y: no row of J reaches them
    dR, dt = R0.T @ res["R"], R0.T @ (res["t"] - t0)
    assert abs(np.arctan2(dR[1, 0], dR[0, 0])) < 1e-6                # rotation about the normal stays at its start
    assert np.abs(dt[:2]).max() < 1e-6 * r                            # so does the in-plane translation
    assert abs((R.T @ (res["t"] - t))[2]) < 1e-9                      # the normal offset is removed
    assert res["inliers"] == len(P)


def test_fewer_than_32_inliers_returns_the_start_pose():
    rng, Q, Nn, r, R, t, P = box_scene(3)
    res = io.refine(R, t, P[:31], Q, Nn, r, 10)
    assert res["iters_run"] == 0 and res["inliers"] == 31
    assert np.array_equal(res["R"], R) and np.array_equal(res["t"], t)


def test_nearest_ties_go_to_the_lowest_index():
    Q = np.array([[1.0, 0, 0], [-1.0, 0, 0], [0, 1.0, 0], [1.0, 0, 0]])
    j, d1, d2 = io.nearest(np.array([[0.0, 0, 0], [2.0, 0, 0]]), Q)
    assert j.tolist() == [0, 0] and d1.tolist() == [1.0, 1.0] and d2.tolist() == [1.0, 1.0]


def test_tau_schedule():
    assert [io.tau_fraction(k) for k in range(6)] == [0.3, 0.15, 0.075, 0.05, 0.05, 0.05]


def test_sample_surface_normals_keep_the_draws():
    v, f = box_mesh(0.05, 0.03, 0.02)
    v = v * 1000
    p0 = meshio.sample_surface(v, f, 2000, np.random.RandomState(7))
    p1, n1 = meshio.sample_surface(v, f, 2000, np.random.RandomState(7), return_normals=True)
    assert np.array_equal(p0, p1) and n1.dtype == np.float32 and n1.shape == p1.shape
    assert np.abs(np.linalg.norm(n1, axis=1) - 1).max() < 1e-6
    # each point lies on a box face: its normal is that face's axis, perpendicular to both of the face's edge directions
    half = np.array([50.0, 30.0, 20.0])
    axis = np.argmax(np.abs(n1), axis=1)
    assert np.abs(np.abs(n1[np.arange(len(n1)), axis]) - 1).max() < 1e-6
    assert np.allclose(np.abs(p1[np.arange(len(p1)), axis]), half[axis], atol=1e-3)
    # the same on an irregular mesh: every normal is perpendicular to the edges of the face the point was drawn on
    rng = np.random.RandomState(8)
    verts = rng.normal(size=(30, 3)).astype(np.float32)
    faces = rng.randint(0, 30, size=(40, 3))
    faces = faces[(faces[:, 0] != faces[:, 1]) & (faces[:, 1] != faces[:, 2]) & (faces[:, 0] != faces[:, 2])]
    g = np.random.RandomState(9)
    pts, nrm = meshio.sample_surface(verts, faces, 500, g, return_normals=True)
    a, b, c = (verts[faces[:, k]].astype(np.float64) for k in range(3))
    area = 0.5 * np.linalg.norm(np.cross(b - a, c - a), axis=1)
    fi = np.minimum(np.searchsorted(np.cumsum(area), np.random.RandomState(9).random_sample(500) * area.sum()), len(faces) - 1)
    for e in (b - a, c - a):
        en = e[fi] / np.linalg.norm(e[fi], axis=1, keepdims=True)
        assert np.abs((en * nrm).sum(1)).max() < 1e-5
    assert np.array_equal(pts, meshio.sample_surface(verts, faces, 500, np.random.RandomState(9)))


def test_sample_surface_accepts_a_generator():
    v, f = box_mesh(1.0, 2.0, 3.0)
    p, n = meshio.sample_surface(v, f, 100, np.random.default_rng(3), return_normals=True)
    q, m = meshio.sample_surface(v, f, 100, np.random.default_rng(3), return_normals=True)
    assert np.array_equal(p, q) and np.array_equal(n, m)
    with pytest.raises(ValueError):
        meshio.sample_surface(v, np.zeros((0, 3), np.int64), 10, np.random.default_rng(3), return_normals=True)


def test_icp_model_draws_from_its_own_seed():
    from sam6d_b200 import pipeline
    v, f = box_mesh(50.0, 30.0, 20.0)
    np.random.seed(11)
    before = np.random.get_state()[1].copy()
    p, n = pipeline.icp_model(v, f)
    assert np.array_equal(np.random.get_state()[1], before)
    assert p.shape == (pipeline.ICP_SAMPLES, 3) and p.dtype == np.float32 and np.abs(p).max() <= 0.05 + 1e-6
    p2, n2 = pipeline.icp_model(v, f)
    assert np.array_equal(p, p2) and np.array_equal(n, n2)


def test_cli_parsers_accept_icp_iters():
    from sam6d_b200.cli import pem_run_inference_custom as pem_cli, run_bop, run_sam6d
    req = ["--cad_path", "o.ply", "--rgb_path", "r.png", "--depth_path", "d.png", "--cam_path", "c.json", "--output_dir", "out"]
    bop = ["--bop_root", "b", "--dataset_name", "ycbv", "--output_dir", "out"]
    for parser, base in ((pem_cli.get_parser(), []), (run_sam6d.get_parser(), req), (run_bop.get_parser(), bop)):
        assert parser.parse_args(base).icp_iters == 0
        assert parser.parse_args(base + ["--icp_iters", "10"]).icp_iters == 10
