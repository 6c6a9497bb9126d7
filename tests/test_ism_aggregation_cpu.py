"""CPU: oracle/ism_agg_oracle.py against the outputs of the reference's own compute_semantic_score with every template
aggregation (tests/golden/ism_aggregation.pt, tools/make_golden_ism_aggregation.py), and the host-side checks of the
aggregation argument."""
import os

import pytest
import torch

from oracle import ism_agg_oracle as ia

GOLDEN = "ism_aggregation.pt"


def _cases(golden_dir):
    return torch.load(os.path.join(golden_dir, GOLDEN), weights_only=False)


@pytest.mark.parametrize("agg", ia.AGGREGATIONS)
def test_oracle_matches_reference_golden(golden_dir, agg):
    g = _cases(golden_dir)
    thresh = g["meta"]["confidence_thresh"]
    for (O, T), c in g["cases"].items():
        q, r = ia.make_tied_descriptors(c["P"], O, T, c["C"], c["seed"])
        assert q.double().sum().item() == c["input_checksum"]["q"] and r.double().sum().item() == c["input_checksum"]["ref"]
        idx, obj, sem, bt, _, per = ia.compute_semantic_score(q, r, agg, thresh)
        w = c[agg]
        assert torch.equal(idx, w["idx_selected"]) and torch.equal(obj, w["pred_idx_objects"]) and torch.equal(bt, w["best_template"])
        assert torch.equal(sem, w["semantic_score"]) and torch.equal(per, w["per_obj"])
        assert w["reference"] == (agg != "avg_5" or T >= 5)


def test_golden_covers_the_view_sets_ties_and_short_template_lists(golden_dir):
    g = _cases(golden_dir)["cases"]
    assert {(O, T) for O in (1, 8, 21) for T in (42, 162, 642)} <= set(g)
    assert any(T < 5 for _, T in g)
    c = g[(8, 42)]
    q, r = ia.make_tied_descriptors(c["P"], 8, 42, c["C"], c["seed"])
    assert torch.equal(r[:, 0], r[:, 1]) and torch.equal(r[0], r[1]) and torch.equal(q[0], q[1])
    # object 1 repeats object 0: the first maximum wins, so no proposal is assigned to object 1
    for agg in ia.AGGREGATIONS:
        assert not (c[agg]["pred_idx_objects"] == 1).any()


def test_median_is_the_lower_median():
    s = torch.tensor([[[0.4, 0.1, 0.3, 0.2]]])
    assert ia.aggregate(s, "median").item() == pytest.approx(0.2)
    assert ia.aggregate(s[..., :3], "median").item() == pytest.approx(0.3)


def test_unknown_aggregation_is_rejected():
    from sam6d_b200 import ism, ops
    with pytest.raises(NotImplementedError):
        ism.compute_semantic_score(torch.zeros(2, 8), torch.zeros(1, 3, 8), "avg_3")
    with pytest.raises(NotImplementedError):
        ia.aggregate(torch.zeros(1, 1, 3), "avg_3")
    assert set(ops.TEMPLATE_AGGREGATIONS) == set(ia.AGGREGATIONS)


def test_sharded_semantic_score_passes_the_aggregation(monkeypatch):
    """the default per-shard scorer receives the aggregation (the kernel call itself is a GPU test)"""
    from sam6d_b200 import dist as sdist
    seen = []

    def fake(desc, refs, aggregation_function="avg_5"):
        seen.append(aggregation_function)
        P = desc.shape[0]
        return torch.zeros(P, dtype=torch.long), torch.ones(P), torch.zeros(P, dtype=torch.long)
    monkeypatch.setattr(sdist, "_local_best", fake)
    sdist.sharded_semantic_score(torch.zeros(3, 8), torch.zeros(2, 4, 8), 0, aggregation_function="median")
    sdist.sharded_semantic_score(torch.zeros(3, 8), torch.zeros(2, 4, 8), 0)
    assert seen == ["median", "avg_5"]
