"""GPU: the point-to-plane ICP refinement (csrc/icp.cu through ops.icp_refine) against the float64 restatement of
oracle/icp_oracle.py, and the pipeline's opt-in refinement (SAM6D(..., icp_iters)).

Bounds.  u = 2^-24.  The kernel rounds the pose to fp32 (the oracle is fed that fp32 pose) and forms y = R^T (p - t) in fp32:
one rounding of p - t and a three-term dot product, so each component is within 5u (|R|^T |p - t|) of the exact value;
E_y is the norm of that vector.  A squared distance D = |y - q|^2 evaluated in fp32 from the perturbed y is within
dD(D) = 2 sqrt(D) E_y + E_y^2 + 6u D of the exact one (three differences, three products, two sums of non-negative terms).
The nearest sample is decided where the float64 margin to the second-nearest exceeds dD of both; the inlier test where
|D - tau^2| exceeds dD(D) + 2u tau^2 (tau^2 rounded to fp32).  Elsewhere the kernel's choice must be one the bound allows,
and the number of undecided points is printed.  The normal equations are rebuilt in float64 from the kernel's own
correspondences and inliers: each entry of the rotation columns of J moves by at most E_y / r (|n| = 1) and e by at most
E_y / r, so an entry of A = sum J^T J moves by at most sum |J_a| d_c + |J_c| d_a + d_a d_c, plus 1e-12 relative for the
fp64 sums.  The update is a linear solve of that system: its error is bounded through the oracle's condition number,
kappa (|dA| / |A| + |db| / |b|) / (1 - kappa |dA| / |A|) |delta|, plus the fp32 rounding of the returned pose."""
import math
import os

import numpy as np
import pytest
import torch

from oracle import icp_oracle as io

pytestmark = pytest.mark.gpu

U = 2.0 ** -24


@pytest.fixture(scope="module")
def ops():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from sam6d_b200 import ops as _ops
    return _ops


def _rot(rng):
    q = rng.normal(size=4)
    w, x, y, z = q / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def _perturb(R, t, rng, deg, shift):
    axis = rng.normal(size=3)
    d = rng.normal(size=3)
    return R @ io.so3_exp(np.radians(deg) * axis / np.linalg.norm(axis)), t + shift * d / np.linalg.norm(d)


def hull_mesh_mm(golden_dir):
    """the 1.6 k-face test mesh: the convex hull of the example object's model points, in mm"""
    from scipy.spatial import ConvexHull
    g = torch.load(os.path.join(golden_dir, "pem_input.pt"), weights_only=False)
    pts = g["model_points"].numpy().astype(np.float64) * 1000.0
    hull = ConvexHull(pts)
    remap = {v: i for i, v in enumerate(hull.vertices)}
    return pts[hull.vertices].astype(np.float32), np.array([[remap[a] for a in s] for s in hull.simplices], dtype=np.int64)


def bumpy_sphere_mm(level=5):
    """the 10 k-vertex test mesh (level 5): an icosphere stretched to 60 x 40 x 30 mm with bumps, so no rotation is a symmetry"""
    from oracle import render_oracle as ro
    v, f = ro.icosphere(level, 1.0)
    v = v.astype(np.float64)
    v = v * (1.0 + 0.15 * np.sin(3 * v[:, :1]) * np.cos(2 * v[:, 1:2]))
    return (v * np.array([60.0, 40.0, 30.0])).astype(np.float32), f.astype(np.int64)


def _objects(golden_dir, m=4096):
    from sam6d_b200 import meshio
    meshes = [hull_mesh_mm(golden_dir), bumpy_sphere_mm(3)]
    Q, Nn = zip(*[meshio.sample_surface(v, f, m, np.random.RandomState(10 + i), return_normals=True) for i, (v, f) in enumerate(meshes)])
    return meshes, np.stack(Q) / np.float32(1000.0), np.stack(Nn)


def _observations(meshes, obj, n, rng, deg=5.0, shift=0.02):
    """per instance: a posed noisy subset of its object's surface with 10 % background points, the true pose and a perturbed
    start pose, fp32"""
    from sam6d_b200 import meshio
    B = len(obj)
    P = np.empty((B, n, 3), np.float32)
    R0, t0 = np.empty((B, 3, 3), np.float32), np.empty((B, 3), np.float32)
    radius = np.empty(B, np.float32)
    for b, o in enumerate(obj):
        v, f = meshes[o]
        pts = meshio.sample_surface(v, f, n, rng).astype(np.float64) / 1000.0
        r = float(np.linalg.norm(v, axis=1).max()) / 1000.0
        R, t = _rot(rng), np.array([rng.uniform(-0.1, 0.1), rng.uniform(-0.1, 0.1), rng.uniform(0.4, 0.9)])
        pts += rng.normal(scale=0.001, size=pts.shape)
        k = n // 10
        pts[:k] = np.concatenate([rng.uniform(-2 * r, 2 * r, size=(k, 2)), np.full((k, 1), 1.6 * r)], axis=1)
        P[b] = pts @ R.T + t
        Rp, tp = _perturb(R, t, rng, rng.uniform(0, deg), shift * r)
        R0[b], t0[b], radius[b] = Rp, tp, r
    return P, R0, t0, radius


def _run(ops, R0, t0, P, Q, Nn, obj, radius, iters, system=True):
    c = lambda a, dt=torch.float32: torch.from_numpy(np.ascontiguousarray(a)).to(dt).cuda()      # noqa: E731
    out = ops.icp_refine(c(R0), c(t0), c(P), c(Q), c(Nn), c(obj, torch.int32), c(radius), iters, system=system)
    torch.cuda.synchronize()
    return [x.cpu().numpy() for x in out]


def _sym(s):
    A = np.zeros((6, 6))
    A[np.triu_indices(6)] = s[:21]
    return A + np.triu(A, 1).T


def _system_bounds(y, q, n, r, E):
    """A, b, sse of the inliers in float64 and their entrywise bounds for a perturbation of at most E (per point) in y"""
    A, b, sse = io.normal_equations(y, q, n, r)
    ys, qs = y / r, q / r
    e = (n * (ys - qs)).sum(1)
    J = np.concatenate([np.cross(ys, n), n], axis=1)
    d = np.zeros_like(J)
    d[:, :3] = (E / r)[:, None]
    de = E / r
    aJ = np.abs(J)
    bA = aJ.T @ d + d.T @ aJ + d.T @ d + 1e-12 * (aJ.T @ aJ)
    bb = aJ.T @ de + d.T @ np.abs(e) + d.T @ de + 1e-12 * (aJ.T @ np.abs(e))
    bs = float((2 * np.abs(e) * de + de * de).sum() + 1e-12 * (e @ e))
    return A, b, sse, bA, bb, bs


def check_one_iteration(R0, t0, P, Q, Nn, obj, radius, res, label, k=0):
    """one kernel iteration (res = icp_refine(..., 1, system=True) on numpy) against io.step from the same fp32 pose"""
    Rg, tg, inl_g, rms_g, it_g, corr, sums = res
    und_j = und_i = 0
    worst = 0.0
    for b in range(len(obj)):
        Qo, No, r = Q[obj[b]].astype(np.float64), Nn[obj[b]].astype(np.float64), float(radius[b])
        s = io.step(R0[b], t0[b], P[b], Qo, No, r, k)
        dpt = P[b].astype(np.float64) - t0[b].astype(np.float64)
        E = 5 * U * np.linalg.norm(np.abs(dpt) @ np.abs(R0[b].astype(np.float64)), axis=1)
        dD = lambda D: 2 * np.sqrt(D) * E + E * E + 6 * U * D        # noqa: E731
        jg = np.where(corr[b] >= 0, corr[b], -1 - corr[b])
        ing = corr[b] >= 0
        # correspondences: equal where decided, within the bound elsewhere
        dec = np.isinf(s["dsecond"]) | ((s["dsecond"] - s["dmin"]) > dD(s["dmin"]) + dD(s["dsecond"]))
        assert np.array_equal(jg[dec], s["j"][dec]), (label, b)
        Dg = ((s["y"] - Qo[jg]) ** 2).sum(1)
        assert np.all(Dg - s["dmin"] <= dD(Dg) + dD(s["dmin"])), (label, b)
        und_j += int((~dec).sum())
        # inlier sets: equal where decided
        tau2 = (r * io.tau_fraction(k)) ** 2
        dec_i = dec & (np.abs(s["dmin"] - tau2) > dD(s["dmin"]) + 2 * U * tau2)
        assert np.array_equal(ing[dec_i], s["inlier"][dec_i]), (label, b)
        und_i += int((~dec_i).sum())
        # the system, rebuilt in float64 on the kernel's correspondences and inliers
        A, bv, sse, bA, bb, bs = _system_bounds(s["y"][ing], Qo[jg[ing]], No[jg[ing]], r, E[ing])
        Ag = _sym(sums[b])
        assert sums[b, 27] == ing.sum() == inl_g[b], (label, b)
        ratio = max(float((np.abs(Ag - A) / np.maximum(bA, 1e-300)).max()), float((np.abs(sums[b, 21:27] - bv) / np.maximum(bb, 1e-300)).max()),
                    abs(sums[b, 28] - sse) / max(bs, 1e-300))
        assert ratio <= 1.0, (label, b, ratio)
        worst = max(worst, ratio)
        assert abs(rms_g[b] - r * math.sqrt(sums[b, 28] / sums[b, 27])) <= 4 * U * rms_g[b] + 1e-12
        # the update: the oracle's solve of the rebuilt system, within its condition-number bound
        if ing.sum() < io.MIN_INLIERS:
            assert it_g[b] == 0 and np.array_equal(Rg[b], R0[b]) and np.array_equal(tg[b], t0[b]), (label, b)
            continue
        delta, Ad = io.solve(A, bv)
        kappa = np.linalg.cond(Ad)
        rel = np.linalg.norm(bA) / np.linalg.norm(Ad)
        assert kappa * rel < 0.5
        dd = kappa * (rel + np.linalg.norm(bb) / np.linalg.norm(bv)) / (1 - kappa * rel) * np.linalg.norm(delta) + 1e-12
        R64, t64 = R0[b].astype(np.float64), t0[b].astype(np.float64)
        Ro, to = R64 @ io.so3_exp(delta[:3]), t64 + R64 @ (r * delta[3:])
        assert np.abs(Rg[b] - Ro).max() <= 2 * dd + U, (label, b)
        assert np.abs(tg[b] - to).max() <= r * dd + U * np.abs(to).max(), (label, b)
        assert it_g[b] == 1
    print(f"{label}: {und_j} undecided correspondences, {und_i} undecided inlier tests of {P.shape[0] * P.shape[1]} points; "
          f"largest system error / bound {worst:.3f}")
    return worst


def test_one_iteration_bench_shape(ops, golden_dir):
    """B = 32, N = 2048, M = 4096, two objects"""
    meshes, Q, Nn = _objects(golden_dir)
    rng = np.random.RandomState(0)
    obj = np.arange(32) % 2
    P, R0, t0, radius = _observations(meshes, obj, 2048, rng)
    res = _run(ops, R0, t0, P, Q, Nn, obj, radius, 1)
    check_one_iteration(R0, t0, P, Q, Nn, obj, radius, res, "B=32")
    # plausible wrong answers fail the bounds: point-to-point normal equations, and point-to-plane without the 1/r scaling
    Rg, tg, inl_g, rms_g, it_g, corr, sums = res
    b = 0
    Qo, No, r = Q[obj[b]].astype(np.float64), Nn[obj[b]].astype(np.float64), float(radius[b])
    s = io.step(R0[b], t0[b], P[b], Qo, No, r, 0)
    ing = corr[b] >= 0
    jg = np.where(ing, corr[b], -1 - corr[b])
    E = 5 * U * np.linalg.norm(np.abs(P[b].astype(np.float64) - t0[b]) @ np.abs(R0[b].astype(np.float64)), axis=1)
    A, _, _, bA, _, _ = _system_bounds(s["y"][ing], Qo[jg[ing]], No[jg[ing]], r, E[ing])
    ys = s["y"][ing] / r
    A_pp = np.zeros((6, 6))
    for y in ys:                                                          # rows [-[y]x, I] of the point-to-point residual
        Jp = np.concatenate([-np.array([[0, -y[2], y[1]], [y[2], 0, -y[0]], [-y[1], y[0], 0]]), np.eye(3)], axis=1)
        A_pp += Jp.T @ Jp
    A_m, _, _ = io.normal_equations(s["y"][ing], Qo[jg[ing]], No[jg[ing]], 1.0)
    Ag = _sym(sums[b])
    assert (np.abs(Ag - A) <= bA).all()
    assert not (np.abs(Ag - A_pp) <= bA).all()
    assert not (np.abs(Ag - A_m) <= bA).all()


def test_edges(ops, golden_dir, capsys):
    meshes, Q, Nn = _objects(golden_dir)
    rng = np.random.RandomState(1)
    for B, N in ((1, 2048), (3, 1001), (2, 3)):                            # B = 1; N not a multiple of the CTA width; tiny N
        obj = np.arange(B) % 2
        P, R0, t0, radius = _observations(meshes, obj, N, rng)
        check_one_iteration(R0, t0, P, Q, Nn, obj, radius, _run(ops, R0, t0, P, Q, Nn, obj, radius, 1), f"B={B} N={N}")
    # M = 1
    obj = np.zeros(2, np.int64)
    P, R0, t0, radius = _observations(meshes, obj, 512, rng)
    res = _run(ops, R0, t0, P, Q[:, :1], Nn[:, :1], obj, radius, 1)
    assert (np.where(res[5] >= 0, res[5], -1 - res[5]) == 0).all()
    check_one_iteration(R0, t0, P, Q[:, :1], Nn[:, :1], obj, radius, res, "M=1")
    # duplicate observed points: 512 distinct points, four copies each
    P4 = np.repeat(P[:, :512], 4, axis=1)
    res = _run(ops, R0, t0, P4, Q, Nn, obj, radius, 1)
    assert (res[5].reshape(2, 512, 4) == res[5].reshape(2, 512, 4)[..., :1]).all()
    check_one_iteration(R0, t0, P4, Q, Nn, obj, radius, res, "duplicates")


def test_samples_at_the_shared_memory_limit(ops, golden_dir):
    from sam6d_b200 import meshio
    from sam6d_b200._lib import Sam6dError
    m = ops.icp_max_samples()
    assert m >= 4096
    meshes, _, _ = _objects(golden_dir)
    q, n = meshio.sample_surface(*meshes[0], m + 1, np.random.RandomState(3), return_normals=True)
    Q, Nn = (q / np.float32(1000.0))[None], n[None]
    obj = np.zeros(2, np.int64)
    P, R0, t0, radius = _observations(meshes[:1], obj, 2048, np.random.RandomState(4))
    check_one_iteration(R0, t0, P, Q[:, :m], Nn[:, :m], obj, radius, _run(ops, R0, t0, P, Q[:, :m], Nn[:, :m], obj, radius, 1), f"M={m}")
    with pytest.raises(Sam6dError, match="invalid argument"):
        _run(ops, R0, t0, P, Q, Nn, obj, radius, 1)


def test_exact_ties_go_to_the_lowest_index(ops):
    """pairs of samples m +- h on a dyadic grid and observed points at their midpoints, identity pose: every distance is exact
    in fp32, so each point is tied between its pair; repeated samples tie at distance 0"""
    rng = np.random.RandomState(5)
    K = 300
    cells = rng.choice(16 ** 3, K, replace=False)
    mids = np.stack([cells // 256, (cells // 16) % 16, cells % 16], axis=1) / 16.0 - 0.5
    h = rng.choice([-1.0, 1.0], size=(K, 3)) / 128.0
    h[:, 2] = 0.0
    Q = np.empty((2 * K + 20, 3))
    Q[0:2 * K:2], Q[1:2 * K:2] = mids + h, mids - h
    Q[2 * K:] = Q[:20]                                                     # repeats of the first 20 samples
    Nn = rng.normal(size=Q.shape)
    Nn /= np.linalg.norm(Nn, axis=1, keepdims=True)
    P = np.concatenate([mids, Q[:20]])[None]
    obj, radius = np.zeros(1, np.int64), np.array([np.linalg.norm(Q, axis=1).max()], np.float32)
    res = _run(ops, np.eye(3)[None], np.zeros((1, 3)), P, Q[None], Nn[None], obj, radius, 1)
    j = np.where(res[5][0] >= 0, res[5][0], -1 - res[5][0])
    assert np.array_equal(j, np.concatenate([2 * np.arange(K), np.arange(20)]))


def test_too_few_inliers_and_invalid_instances(ops, golden_dir):
    """an instance with fewer than 32 inliers comes back bit for bit; so does one with an out-of-range object (inliers -1)"""
    meshes, Q, Nn = _objects(golden_dir)
    P, R0, t0, radius = _observations(meshes, [0, 1, 0, 0], 2048, np.random.RandomState(6))
    obj = np.array([0, 1, 0, 5])                                          # object 5 does not exist
    P[1] += np.float32(10 * radius[1])                                    # every point 10 r away: no inlier
    P[2, :-31] += np.float32(10 * radius[2])                              # only the last 31 surface points can be inliers
    Rg, tg, inl, rms, it = _run(ops, R0, t0, P, Q, Nn, obj, radius, 10, system=False)
    for b in (1, 2, 3):
        assert np.array_equal(Rg[b], R0[b]) and np.array_equal(tg[b], t0[b]) and it[b] == 0, b
    assert inl[1] == 0 and 0 < inl[2] < 32 and inl[3] == -1 and inl[0] > 1000 and it[0] >= 1
    # iters = 0: every pose unchanged
    Rg, tg, inl, rms, it = _run(ops, R0, t0, P, Q, Nn, obj, radius, 0, system=False)
    assert np.array_equal(Rg, R0) and np.array_equal(tg, t0) and (it == 0).all()


def test_deterministic(ops, golden_dir):
    meshes, Q, Nn = _objects(golden_dir)
    obj = np.arange(32) % 2
    P, R0, t0, radius = _observations(meshes, obj, 2048, np.random.RandomState(7))
    a = _run(ops, R0, t0, P, Q, Nn, obj, radius, 10)
    b = _run(ops, R0, t0, P, Q, Nn, obj, radius, 10)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def rendered_scene(v_mm, f, seed):
    """render the mesh at a known pose, back-project its mask pixels, add 1 mm noise and 10 % background-plane outliers, sample
    2048 points; start from the pose perturbed by 5 degrees and 1 cm"""
    from sam6d_b200 import meshio, render
    rng = np.random.RandomState(seed)
    H, W, fx, cx, cy = 480, 640, 600.0, 320.0, 240.0
    R, t = _rot(rng), np.array([0.02, -0.01, 0.6])
    pose = np.eye(4, dtype=np.float32)
    pose[:3, :3], pose[:3, 3] = R, t
    mesh = render.upload(meshio.Mesh(vertices=(v_mm / 1000.0).astype(np.float32), faces=f.astype(np.int32)))
    depth = render.render([mesh], torch.from_numpy(pose)[None, None].cuda(), np.array([[fx, 0, cx], [0, fx, cy], [0, 0, 1]]), H, W)["depth"]
    depth = depth[0, 0].cpu().numpy().astype(np.float64)
    ys, xs = np.nonzero(depth > 0)
    z = depth[ys, xs]
    obs = np.stack([(xs + 0.5 - cx) * z / fx, (ys + 0.5 - cy) * z / fx, z], axis=1)
    obs += rng.normal(scale=0.001, size=obs.shape)
    n_bg = 2048 // 10
    sel = obs[rng.choice(len(obs), 2048 - n_bg, replace=len(obs) < 2048 - n_bg)]
    lo, hi = obs.min(0), obs.max(0)
    bg = np.stack([rng.uniform(lo[0], hi[0], n_bg), rng.uniform(lo[1], hi[1], n_bg), np.full(n_bg, t[2] + 0.15)], axis=1)
    P = np.concatenate([sel, bg])[rng.permutation(2048)]
    R0, t0 = _perturb(R, t, rng, 5.0, 0.01)
    return P.astype(np.float32), R, t, R0.astype(np.float32), t0.astype(np.float32)


@pytest.mark.parametrize("mesh", ["hull_1.6k_faces", "bumpy_sphere_10k_vertices"])
def test_converges_on_rendered_depth(ops, golden_dir, mesh):
    from sam6d_b200 import pipeline
    v, f = hull_mesh_mm(golden_dir) if mesh.startswith("hull") else bumpy_sphere_mm(5)
    Q, Nn = pipeline.icp_model(v, f)
    r = np.float32(np.linalg.norm(v, axis=1).max() / 1000.0)
    P, R, t, R0, t0 = rendered_scene(v, f, 11)
    Rg, tg, inl, rms, it = _run(ops, R0[None], t0[None], P[None], Q[None], Nn[None], np.zeros(1), np.array([r]), 20, system=False)
    o = io.refine(R0, t0, P, Q, Nn, float(r), 20)
    e_start = (io.rotation_error_deg(R0, R), 1000 * np.linalg.norm(t0 - t))
    e_gpu = (io.rotation_error_deg(Rg[0], R), 1000 * np.linalg.norm(tg[0] - t))
    e_ora = (io.rotation_error_deg(o["R"], R), 1000 * np.linalg.norm(o["t"] - t))
    print(f"{mesh}: r = {1000 * r:.1f} mm; start {e_start[0]:.3f} deg {e_start[1]:.3f} mm; after {it[0]} iterations: GPU "
          f"{e_gpu[0]:.4f} deg {e_gpu[1]:.4f} mm ({inl[0]} inliers, rms {1000 * rms[0]:.3f} mm), oracle {e_ora[0]:.4f} deg "
          f"{e_ora[1]:.4f} mm ({o['inliers']} inliers, {o['iters_run']} iterations)")
    # a correspondence or inlier decision that fp32 flips moves one of ~2000 equally weighted points, about 1 mm / 2000 in
    # translation and (1 mm / r) / 2000 in rotation per flip: the GPU's final errors stay within 0.02 deg / 0.05 mm of the oracle's
    assert abs(e_gpu[0] - e_ora[0]) <= 0.02 and abs(e_gpu[1] - e_ora[1]) <= 0.05
    assert e_gpu[0] < e_start[0] / 5 and e_gpu[1] < e_start[1] / 5


# ---- the pipeline's opt-in refinement -------------------------------------------------------------------------------------------
_MODEL = {}


def _sam6d():
    from sam6d_b200.pipeline import SAM6D
    if "m" not in _MODEL:
        _MODEL["m"] = SAM6D(segmentor="fastsam", random_weights=True, confidence_thresh=-1, det_score_thresh=-1)
    return _MODEL["m"]


def _scene_meshes(golden_dir):
    from sam6d_b200 import meshio
    v, f = hull_mesh_mm(golden_dir)
    cols = np.random.RandomState(0).randint(40, 255, (len(v), 3)).astype(np.uint8)
    g = torch.load(os.path.join(golden_dir, "pem_input.pt"), weights_only=False)
    frame = (g["rgb"].numpy().astype(np.uint8), g["depth"].numpy().astype(np.uint16), g["cam_K"], g["depth_scale"])
    return [meshio.Mesh(vertices=(v * s).astype(np.float32), faces=f, colors=cols) for s in (1.0, 0.7)], frame


def test_pipeline_frame_with_icp(golden_dir):
    model = _sam6d()
    meshes, frame = _scene_meshes(golden_dir)
    try:
        model.icp_iters = 0
        objs0 = model.onboard_objects(meshes, obj_ids=[3, 7], template_size=192, rng=np.random.RandomState(0))
        res0 = model.detect_objects(*frame, objs0, rng=np.random.RandomState(5))
        model.icp_iters = 10
        objs1 = model.onboard_objects(meshes, obj_ids=[3, 7], template_size=192, rng=np.random.RandomState(0))
        res1 = model.detect_objects(*frame, objs1, rng=np.random.RandomState(5))
    finally:
        model.icp_iters = 0
    # onboarding with ICP: every other field equal, so the caller's draws are untouched
    for k in ("ref_cls", "ref_patch", "poses_m", "cloud_m", "bank", "model_points_m", "radii", "obj_ids"):
        a, b = getattr(objs0, k), getattr(objs1, k)
        for x, y in (zip(a, b) if k == "bank" else [(a, b)]):
            assert (torch.equal(x, y) if isinstance(x, torch.Tensor) else np.array_equal(x, y)), k
    icp = objs1.pose_inputs.icp
    assert objs0.pose_inputs.icp is None and icp[0].shape == (2, 4096, 3) and icp[1].shape == (2, 4096, 3)
    # the frame: the same records and scores, only R and t refined (time is the host clock)
    drop = lambda recs, keys: [{k: v for k, v in r.items() if k not in keys} for r in recs]          # noqa: E731
    assert drop(res0.ism, ("time",)) == drop(res1.ism, ("time",)) and len(res1.pem) == len(res0.pem) > 0
    assert drop(res0.pem, ("time", "R", "t")) == drop(res1.pem, ("time", "R", "t"))
    assert any(a["R"] != b["R"] or a["t"] != b["t"] for a, b in zip(res0.pem, res1.pem))
    out0, out1 = res0.frame.out, res1.frame.out
    assert torch.equal(out1["pem_R"], out0["pred_R"]) and torch.equal(out1["pem_t"], out0["pred_t"])
    assert torch.equal(out1["pred_R"], res1.R) and "pem_R" not in out0
    print(f"frame: {len(res1.pem)} poses, ICP inliers {out1['icp_inliers'].tolist()}, rms (mm) "
          f"{[round(1000 * x, 3) for x in out1['icp_rms'].tolist()]}")


def test_run_bop_pem_with_icp(golden_dir, tmp_path):
    import json
    import sys
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import _bop_golden as bg
    gold = bg.load(golden_dir)
    split = str(tmp_path / "bop")
    os.makedirs(split)
    split = bg.write_split(gold, split)
    det_path = tmp_path / "dets.json"
    json.dump(gold["detections"], open(det_path, "w"))
    tdir = os.path.join(split, "BOP-Templates")
    model = _sam6d()
    try:
        model.icp_iters = 0
        l0 = model.run_bop_pem(str(det_path), split, "lmo", tdir, None, rng=np.random.RandomState(3))
        model.icp_iters = 10
        l1 = model.run_bop_pem(str(det_path), split, "lmo", tdir, None, rng=np.random.RandomState(3))
    finally:
        model.icp_iters = 0
    assert len(l0) == len(l1) == 12
    cols = lambda line: line.rstrip("\n").split(",")                      # noqa: E731
    # scene_id, im_id, obj_id, score equal; R and t may differ; time is the host clock
    assert [cols(x)[:4] for x in l0] == [cols(x)[:4] for x in l1]
    assert sum(cols(a)[4:6] != cols(b)[4:6] for a, b in zip(l0, l1)) >= 1
