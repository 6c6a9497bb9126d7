"""GPU: template-scoring aggregations (csrc/ism.cu with mean / median / max / avg_5) and the ISM's denser view sets.

- The kernel against oracle/ism_agg_oracle.py at P in {0, 1, 200}, T in {42, 162, 642} (the level-0 / 1 / 2 view sets),
  O in {1, 8, 21, 33}: similarities and scores within test_template_score's tolerance (atol 2e-6, rtol 1e-5; mean adds its
  fp32 summation bound T x 2^-24, the sum of T values in [0, 1] taken in another order); median and max are, bit for bit,
  one of the kernel's own similarities of that (proposal, object) -- exactly torch.median / torch.max of them; object and
  template indices equal the oracle's except at near-ties, where the oracle's two best values lie within that tolerance.
- avg_5 bit-identical to the one-CTA-per-proposal kernel it replaced (tests/golden/template_score_avg5.pt, recorded on an
  H100 by tools/make_golden_template_score_avg5.py): indices, scores, per-object scores and the similarity tensor.
- The reference's own compute_semantic_score with every aggregation (tests/golden/ism_aggregation.pt).
- Shapes past the shared-memory limit are rejected; O x T far past the one-CTA-per-proposal kernel's cap is not a limit.
- dist.sharded_semantic_score with each aggregation equals the unsharded call.
- SAM6D.onboard at level_templates 1 / 2 (and 2 "upper"): 162 / 642 / 341 ISM references, PEM bank and model points
  bit-identical to a level-0 onboard; a detect_objects frame with the median at level 2."""
import hashlib
import os

import numpy as np
import pytest
import torch

from oracle import ism_agg_oracle as ia
from oracle import ism_oracle as io

pytestmark = pytest.mark.gpu

ATOL, RTOL = 2e-6, 1e-5                     # test_template_score's tolerance (tests/test_gpu_kernels.py)


def _score(q, r, agg, want_sim=True):
    from sam6d_b200 import ism, ops
    qn = ism._normalized(q.cuda())
    rn = ops.l2norm_rows(r.cuda().float().contiguous())
    return [x.cpu() if x is not None else None for x in ops.template_score(qn, rn, want_sim=want_sim, aggregation=agg)]


def _oracle_sim(q, r, chunk=8):
    """oracle similarities in proposal chunks (the reference's P-fold replication of the references, chunk by chunk)"""
    if q.shape[0] == 0:
        return torch.zeros(0, r.shape[0], r.shape[1])
    return torch.cat([io.pairwise_similarity(q[i:i + chunk], r) for i in range(0, q.shape[0], chunk)])


def _near_tie(v, idx, tol):
    """rows of v (n, k) whose best value is within tol of another entry (so the oracle's argmax idx may differ)"""
    best = v.gather(1, idx[:, None])
    others = v.clone()
    others.scatter_(1, idx[:, None], -float("inf"))
    return (best[:, 0] - others.max(dim=1).values) <= tol


def _check_against_oracle(q, r, agg, sim_oracle=None):
    P, O, T = q.shape[0], r.shape[0], r.shape[1]
    sim, obj, bo, bs, bt = _score(q, r, agg)
    scores = _oracle_sim(q, r) if sim_oracle is None else sim_oracle
    torch.testing.assert_close(sim, scores, atol=ATOL, rtol=RTOL)
    per = ia.aggregate(scores, agg) if P else torch.zeros(0, O)
    tol = ATOL + RTOL + (T * 2.0 ** -24 if agg == "mean" else 0.0)
    torch.testing.assert_close(obj, per, atol=tol, rtol=RTOL)
    if P == 0:
        assert bo.numel() == bs.numel() == bt.numel() == 0
        return
    # median and max: one of the kernel's own similarities, the one torch picks
    if agg in ("median", "max"):
        assert torch.equal(obj, ia.aggregate(sim, agg))
        assert (sim == obj[..., None]).any(dim=-1).all()
    if agg == "avg_5":
        # the same 5 values <= 1 summed in another order: within 2 x 4 u x 5 / 5 = 4.8e-7
        torch.testing.assert_close(obj, ia.aggregate(sim, agg), atol=4.8e-7, rtol=0)
    # first-max object and template, except at near-ties of the oracle
    o_best, o_obj = per.max(dim=-1)
    free = ~_near_tie(per, o_obj, 2 * tol)
    assert torch.equal(bo.long()[free], o_obj[free]), agg
    assert torch.equal(bs, obj.gather(1, bo.long()[:, None])[:, 0])
    assert torch.equal(bo.long(), obj.max(dim=-1).indices)                     # first max over the kernel's own scores
    rows = scores[torch.arange(P), bo.long()]
    o_t = rows.max(dim=-1).indices
    free_t = ~_near_tie(rows, o_t, 2 * (ATOL + RTOL))
    assert torch.equal(bt.long()[free_t], o_t[free_t]), agg
    assert torch.equal(bt.long(), sim[torch.arange(P), bo.long()].max(dim=-1).indices)


@pytest.mark.parametrize("agg", ia.AGGREGATIONS)
@pytest.mark.parametrize("T", [42, 162, 642])
@pytest.mark.parametrize("O", [1, 8, 21, 33])
def test_kernel_matches_oracle(agg, T, O):
    for P in (0, 1, 200):
        q, r = ia.make_tied_descriptors(P, O, T, 256, seed=11 * O + T + P)
        _check_against_oracle(q, r, agg)


@pytest.mark.parametrize("agg", ia.AGGREGATIONS)
def test_kernel_matches_reference_golden(golden_dir, agg):
    """the reference's own compute_semantic_score (tools/make_golden_ism_aggregation.py), ties and T < 5 included"""
    from sam6d_b200 import ism
    g = torch.load(os.path.join(golden_dir, "ism_aggregation.pt"), weights_only=False)
    thresh = g["meta"]["confidence_thresh"]
    for (O, T), c in g["cases"].items():
        q, r = ia.make_tied_descriptors(c["P"], O, T, c["C"], c["seed"])
        w = c[agg]
        _, obj, bo, _, _ = _score(q, r, agg, want_sim=False)
        tol = ATOL + RTOL + (T * 2.0 ** -24 if agg == "mean" else 0.0)
        torch.testing.assert_close(obj, w["per_obj"], atol=tol, rtol=RTOL)
        sel, pobj, sem, bt = ism.compute_semantic_score(q.cuda(), r.cuda(), agg, thresh)
        near = _near_tie(w["per_obj"], w["per_obj"].max(dim=-1).indices, 2 * tol)
        assert torch.equal(sel.cpu(), w["idx_selected"]), (O, T)
        free = ~near[w["idx_selected"]]
        assert torch.equal(pobj.cpu()[free], w["pred_idx_objects"][free]), (O, T)
        assert torch.equal(bt.cpu()[free], w["best_template"][free]), (O, T)
        torch.testing.assert_close(sem.cpu(), w["semantic_score"], atol=tol, rtol=RTOL)
        if O > 1:
            assert not (bo == 1).any()                                      # object 1 repeats object 0: first max wins


def test_avg5_bit_identical_to_previous_kernel(golden_dir):
    from sam6d_b200.synth import make_descriptors
    g = torch.load(os.path.join(golden_dir, "template_score_avg5.pt"), weights_only=False)
    C = g["meta"]["C"]
    assert len(g["cases"]) == 24
    for (P, O, T), c in g["cases"].items():
        q, r = make_descriptors(P=P, O=O, T=T, C=C, seed=c["seed"])
        assert q.double().sum().item() == c["input_checksum"]["q"] and r.double().sum().item() == c["input_checksum"]["ref"]
        sim, obj, bo, bs, bt = _score(q, r, "avg_5")
        assert torch.equal(bo, c["best_obj"]) and torch.equal(bt, c["best_tmpl"]), (P, O, T)
        assert torch.equal(bs, c["best_score"]) and torch.equal(obj, c["obj_score"]), (P, O, T)
        assert hashlib.sha256(sim.contiguous().numpy().tobytes()).hexdigest() == c["sim_sha256"], (P, O, T)


def test_over_limit_shapes_are_rejected():
    from sam6d_b200 import _lib, ops
    q = ops.l2norm_rows(torch.randn(4, 64, device="cuda"))
    for O, T, agg in ((1, 4097, "median"), (1, 8000, "avg_5"), (65536, 1, "max")):
        r = ops.l2norm_rows(torch.randn(O * T, 64, device="cuda")).reshape(O, T, 64)
        with pytest.raises(_lib.Sam6dError, match="invalid argument"):
            ops.template_score(q, r, want_sim=False, aggregation=agg)


def test_large_object_template_products_run():
    """O x T = 65536 similarities per proposal: past the 51 k of the one-CTA-per-proposal kernel's shared memory"""
    P, O, T, C = 9, 16, 4096, 64
    q, r = ia.make_tied_descriptors(P, O, T, C, seed=3)
    for agg in ("median", "avg_5"):
        _check_against_oracle(q, r, agg)


@pytest.mark.parametrize("agg", ia.AGGREGATIONS)
def test_sharded_semantic_score_equals_unsharded(agg):
    from sam6d_b200 import dist as sdist, ism
    q, r = ia.make_tied_descriptors(200, 21, 162, 256, seed=5)
    q, r = q.cuda(), r.cuda()
    want = ism.compute_semantic_score(q, r, agg)
    got = sdist.sharded_semantic_score(q, r, 0, aggregation_function=agg)
    for a, b in zip(got, want):
        assert torch.equal(a, b)
    # two shards combined by the first-max rule of the all-gather: the unsharded result
    recs = []
    for lo, hi in (sdist.shard_range(21, 0, 2), sdist.shard_range(21, 1, 2)):
        obj, score, tmpl = sdist._local_best(q, r[lo:hi].contiguous(), agg)
        recs.append(torch.stack([score, (obj + lo).float(), tmpl.float()], dim=1))
    allrec = torch.stack(recs)
    win = torch.argmax(allrec[:, :, 0], dim=0)
    rec = allrec[win, torch.arange(200, device=q.device)]
    keep = rec[:, 0] > 0.2
    assert torch.equal(rec[keep, 1].long(), want[1]) and torch.equal(rec[keep, 0], want[2]) and torch.equal(rec[keep, 2].long(), want[3])


# ---- SAM6D with denser view sets -------------------------------------------------------------------------------------------
def _meshes(golden_dir):
    """two CADs: the convex hull of the example frame's object samples at two scales"""
    from scipy.spatial import ConvexHull
    from sam6d_b200 import meshio
    g = torch.load(os.path.join(golden_dir, "pem_input.pt"), weights_only=False)
    pts = g["model_points"].numpy().astype(np.float64) * 1000.0
    hull = ConvexHull(pts)
    remap = {v: i for i, v in enumerate(hull.vertices)}
    faces = np.array([[remap[a] for a in s] for s in hull.simplices], dtype=np.int64)
    cols = np.random.RandomState(0).randint(40, 255, (len(hull.vertices), 3)).astype(np.uint8)
    meshes = [meshio.Mesh(vertices=(pts[hull.vertices] * s).astype(np.float32), faces=faces, colors=cols) for s in (1.0, 0.7)]
    frame = (g["rgb"].numpy().astype(np.uint8), g["depth"].numpy().astype(np.uint16), g["cam_K"], g["depth_scale"])
    return meshes, frame


@pytest.fixture(scope="module")
def sam6d():
    from sam6d_b200.pipeline import SAM6D
    return SAM6D(segmentor="fastsam", random_weights=True, confidence_thresh=-1, det_score_thresh=-1)


def _onboard(model, mesh, level, dist):
    model.level_templates, model.pose_distribution = level, dist
    try:
        return model.onboard(mesh, template_size=192, rng=np.random.RandomState(0))
    finally:
        model.level_templates, model.pose_distribution = 0, "all"


def test_onboard_view_sets(sam6d, golden_dir):
    from sam6d_b200 import render
    meshes, _ = _meshes(golden_dir)
    base = _onboard(sam6d, meshes[0], 0, "all")
    assert base.ref_cls.shape[0] == 42 and base.poses_m.shape == (42, 4, 4)
    for level, dist, T in ((1, "all", 162), (2, "all", 642), (2, "upper", 341)):
        ob = _onboard(sam6d, meshes[0], level, dist)
        assert ob.ref_cls.shape == (T, base.ref_cls.shape[1]) and ob.ref_patch.shape == (T,) + tuple(base.ref_patch.shape[1:])
        assert ob.poses_m.shape == (T, 4, 4)
        # the geometric score's poses are the set's own views, at the framing distance of the level-0 ones
        R = render.template_poses(level, dist)[:, :3, :3]
        np.testing.assert_allclose(ob.poses_m[:, :3, :3], R, atol=1e-12)
        np.testing.assert_allclose(np.linalg.norm(ob.poses_m[:, :3, 3], axis=1), np.linalg.norm(base.poses_m[0, :3, 3]), rtol=1e-12)
        # the PEM's template bank and model points come from the 42 level-0 views and the same draws
        assert torch.equal(ob.bank[0], base.bank[0]) and torch.equal(ob.bank[1], base.bank[1])
        assert np.array_equal(ob.model_points_m, base.model_points_m) and np.array_equal(ob.cloud_m, base.cloud_m)
        del ob


def test_detect_objects_median_at_level2(sam6d, golden_dir):
    meshes, frame = _meshes(golden_dir)
    sam6d.level_templates, sam6d.aggregation_function = 2, "median"
    try:
        objs = sam6d.onboard_objects(meshes, obj_ids=[4, 9], template_size=192, rng=np.random.RandomState(0))
        assert objs.ref_cls.shape[:2] == (2, 642) and objs.poses_m.shape == (2, 642, 4, 4)
        res = sam6d.detect_objects(*frame, objs, rng=np.random.RandomState(5))
    finally:
        sam6d.level_templates, sam6d.aggregation_function = 0, "avg_5"
    assert res.reason is None and len(res.ism) >= 1 and len(res.pem) >= 1
    assert {r["category_id"] for r in res.ism} <= {4, 9}
    assert all(np.isfinite(r["score"]) for r in res.ism + res.pem)
