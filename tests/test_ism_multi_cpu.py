"""CPU: the multi-object ISM post-processing oracle (oracle/ism_multi_oracle.py) against tests/golden/ism_multi.pt, pinned to
the reference's own Detections / Instance_Segmentation_Model methods by tools/make_golden_ism_multi.py; and the host side of
SAM6D.onboard_objects / detect_objects: ObjectSet stacking, the random-draw order and the category ids of the records."""
import os
from types import SimpleNamespace

import numpy as np
import pytest
import torch


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "ism_multi.pt"), weights_only=False)


def _oracle_frame(inp, per_object_poses):
    from oracle import ism_multi_oracle as imo
    after_small = torch.nonzero(imo.remove_very_small_detections(inp["masks"], inp["boxes"])).flatten()
    O = inp["ref_desc"].shape[0]
    poses = inp["poses"].unsqueeze(0).repeat(O, 1, 1, 1) if per_object_poses else inp["poses"]
    s = imo.score_objects(inp["desc"][after_small], inp["ref_desc"], inp["q_patch"][after_small], inp["ref_patch"], inp["masks"][after_small],
                          inp["depth"], inp["K"], inp["depth_scale"], inp["boxes"][after_small], poses, inp["pointcloud"])
    idx_sel = after_small[s["idx_sel"]]
    k = imo.nms_per_object(inp["boxes"][idx_sel], s["score"], s["pred_obj"])
    return dict(after_small=after_small, idx_sel=idx_sel, pred_obj=s["pred_obj"], best_t=s["best_t"], score=s["score"],
                final_index=idx_sel[k], final_object=s["pred_obj"][k], final_score=s["score"][k])


@pytest.mark.parametrize("tag", ["o3_spread", "o3_one", "o8_spread", "o8_empty"])
@pytest.mark.parametrize("per_object_poses", [False, True])
def test_oracle_frame_matches_reference(gold, tag, per_object_poses):
    from oracle import ism_multi_oracle as imo
    case = gold["frames"][tag]
    inp = imo.make_multi_inputs(**case["kw"])
    chk = float(sum(inp[k].double().sum() for k in ("masks", "depth", "desc", "ref_desc", "q_patch", "ref_patch", "poses", "pointcloud")))
    assert chk == case["input_checksum"], "the seeded inputs are not the ones the fixture was made from"
    got = _oracle_frame(inp, per_object_poses)
    for k, v in got.items():
        assert torch.equal(v, case[k]), k
    # the cases cover what they are named for: a size filter that removes, a tie of final scores, empty and single objects
    assert len(case["after_small"]) < case["kw"]["N"] and 1 not in case["final_index"].tolist()
    objs = set(case["pred_obj"].tolist())
    O = case["kw"]["O"]
    assert {"o3_one": objs == {0}, "o8_empty": objs == set(range(O - 1))}.get(tag, objs == set(range(O)))
    fo = case["final_object"]
    assert torch.equal(fo, fo.sort(stable=True).values)


def test_oracle_per_object_poses_are_used():
    """different poses per object change the geometric score of exactly the proposals on the objects whose poses changed"""
    from oracle import ism_multi_oracle as imo
    inp = imo.make_multi_inputs(N=40, O=3, seed=0)
    keep = torch.nonzero(imo.remove_very_small_detections(inp["masks"], inp["boxes"])).flatten()
    args = (inp["desc"][keep], inp["ref_desc"], inp["q_patch"][keep], inp["ref_patch"], inp["masks"][keep], inp["depth"], inp["K"],
            inp["depth_scale"], inp["boxes"][keep])
    poses = inp["poses"].unsqueeze(0).repeat(3, 1, 1, 1)
    a = imo.score_objects(*args, poses, inp["pointcloud"])
    poses = poses.clone()
    poses[2, :, :3, :3] = poses[2, :, :3, :3].flip(0)
    b = imo.score_objects(*args, poses, inp["pointcloud"])
    changed = a["geometric"] != b["geometric"]
    assert changed.any() and torch.equal(changed & (a["pred_obj"] != 2), torch.zeros_like(changed))


@pytest.mark.parametrize("tag", ["o3", "o8", "o8_two_used", "one"])
def test_oracle_nms_per_object(gold, tag):
    from oracle import ism_multi_oracle as imo
    from oracle.sam_dec_oracle import nms
    case = gold["nms"][tag]
    boxes, scores, obj = imo.make_nms_case(**case["kw"])
    assert torch.equal(boxes, case["boxes"]) and torch.equal(scores, case["scores"]) and torch.equal(obj, case["object_ids"])
    keep = imo.nms_per_object(boxes, scores, obj)
    assert torch.equal(keep, case["keep"])
    assert len(scores.unique()) < len(scores)                                   # exact score ties
    if tag == "one":
        assert torch.equal(keep, nms(boxes, scores, 0.25))


# ---- host side of onboard_objects / detect_objects ----------------------------------------------------------------------------
def _fake_sam6d(T=4, C=8, Nm=16):
    """a SAM6D without models, ICP or verification whose onboarding of one mesh draws from rng in onboard's order (cloud, PEM
    samples, model points) and builds arrays from the draws"""
    from sam6d_b200.pipeline import SAM6D, Onboarded

    def onboard(mesh, template_size=512, rng=None, refs=None):
        rng = rng if rng is not None else np.random
        cloud = rng.rand(2048, 3)
        tem = rng.rand(3)
        mp = rng.rand(Nm, 3) * mesh
        return Onboarded(ref_cls=torch.full((T, C), float(mesh)), ref_patch=torch.full((T, 256, C), float(tem[0])),
                         poses_m=np.tile(np.eye(4), (T, 1, 1)) * mesh, cloud_m=cloud, bank=(torch.full((1, 2048, 3), tem[1]),
                                                                                             torch.full((1, 2048, 256), tem[2])),
                         model_points_m=mp)
    m = SAM6D.__new__(SAM6D)
    m._onboard_mesh = onboard
    m.icp_iters, m.verify, m.device = 0, False, torch.device("cpu")
    return m


def test_onboard_objects_stacks_in_draw_order():
    m = _fake_sam6d()
    objs = m.onboard_objects([1.0, 2.0, 3.0], rng=np.random.RandomState(7))
    assert objs.obj_ids == [1, 2, 3]
    assert objs.ref_cls.shape == (3, 4, 8) and objs.ref_patch.shape == (3, 4, 256, 8)
    assert objs.poses_m.shape == (3, 4, 4, 4) and objs.cloud_m.shape == (3, 2048, 3)
    assert objs.bank[0].shape == (3, 2048, 3) and objs.bank[1].shape == (3, 2048, 256)
    assert objs.model_points_m.shape == (3, 16, 3) and objs.model_points_m.dtype == np.float32 and objs.radii.shape == (3,)
    # object after object from one generator: the same draws as onboarding the three meshes in a row
    rng = np.random.RandomState(7)
    for o, mesh in enumerate([1.0, 2.0, 3.0]):
        one = m._onboard_mesh(mesh, rng=rng)
        assert torch.equal(objs.ref_cls[o], one.ref_cls) and torch.equal(objs.ref_patch[o], one.ref_patch)
        assert np.array_equal(objs.cloud_m[o], one.cloud_m) and np.array_equal(objs.poses_m[o], one.poses_m)
        assert torch.equal(objs.bank[0][o], one.bank[0][0]) and torch.equal(objs.bank[1][o], one.bank[1][0])
        mp = one.model_points_m.astype(np.float32)
        assert np.array_equal(objs.model_points_m[o], mp)
        assert objs.radii[o] == np.max(np.linalg.norm(mp, axis=1))


def test_onboard_objects_ids():
    m = _fake_sam6d()
    assert m.onboard_objects([1.0, 2.0], obj_ids=[5, 9]).obj_ids == [5, 9]
    for bad in ([5, 5], [1], [1, 2, 3]):
        with pytest.raises(ValueError):
            m.onboard_objects([1.0, 2.0], obj_ids=bad)
    with pytest.raises(ValueError):
        m.onboard_objects([])


def test_records_category_ids():
    from sam6d_b200.pipeline import ism_records
    boxes = np.array([[0, 0, 4, 4], [1, 2, 5, 7], [3, 3, 9, 9]])
    counts = [[0, 5], [2, 3], [1, 1]]
    one = ism_records(boxes, np.array([0.5, 0.4, 0.3]), counts, (10, 12), 0.1)
    assert [r["category_id"] for r in one] == [1, 1, 1]
    obj_ids, det_obj = np.array([4, 11, 21]), np.array([2, 0, 2])
    multi = ism_records(boxes, np.array([0.5, 0.4, 0.3]), counts, (10, 12), 0.1, category_ids=obj_ids[det_obj])
    assert [r["category_id"] for r in multi] == [21, 4, 21]
    assert [{k: v for k, v in r.items() if k != "category_id"} for r in multi] == [{k: v for k, v in r.items() if k != "category_id"} for r in one]
    assert all(type(r["category_id"]) is int for r in multi)
