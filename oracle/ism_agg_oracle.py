"""oracle/ism_agg_oracle.py -- TEST INFRASTRUCTURE ONLY.

oracle/ism_oracle.py's compute_semantic_score with every template aggregation the reference's matching_config selects
(Instance_Segmentation_Model.compute_semantic_score, ISM/model/detector.py:260-296):
    mean     torch.sum(scores, dim=-1) / T
    median   torch.median(scores, dim=-1)[0]             the lower median, sorted[(T - 1) // 2]
    max      torch.max(scores, dim=-1)[0]
    avg_5    torch.mean(torch.topk(scores, k=5)[0])      k = min(5, T): the reference's topk raises when T < 5
Parity status: PINNED.  tools/make_golden_ism_aggregation.py runs the reference's own compute_semantic_score with each
aggregation and finds this restatement bit-identical; the outputs are tests/golden/ism_aggregation.pt, checked by
tests/test_ism_aggregation_cpu.py (this oracle) and tests/test_gpu_ism_aggregation.py (csrc/ism.cu).
"""
import torch

from oracle import ism_oracle as io

AGGREGATIONS = ("mean", "median", "max", "avg_5")


def aggregate(scores: torch.Tensor, aggregation: str) -> torch.Tensor:
    """(P,O,T) similarities -> (P,O) per-object scores"""
    if aggregation == "mean":
        return torch.sum(scores, dim=-1) / scores.shape[-1]
    if aggregation == "median":
        return torch.median(scores, dim=-1)[0]
    if aggregation == "max":
        return torch.max(scores, dim=-1)[0]
    if aggregation == "avg_5":
        return torch.mean(torch.topk(scores, k=min(5, scores.shape[-1]), dim=-1)[0], dim=-1)
    raise NotImplementedError(aggregation)


def compute_semantic_score(desc: torch.Tensor, ref_desc: torch.Tensor, aggregation: str = "avg_5", confidence_thresh: float = 0.2,
                           scores: torch.Tensor = None):
    """-> (idx_selected, pred_obj, semantic_score, best_template, scores (P,O,T), per_obj (P,O)); `scores` may be passed in
    when the similarities are already known"""
    if scores is None:
        scores = io.pairwise_similarity(desc, ref_desc)
    per_obj = aggregate(scores, aggregation)
    score_per_proposal, assigned = torch.max(per_obj, dim=-1)
    idx_sel = torch.arange(len(score_per_proposal))[score_per_proposal > confidence_thresh]
    pred_obj = assigned[idx_sel]
    sem = score_per_proposal[idx_sel]
    _, best_t = torch.max(scores[idx_sel, ...], dim=-1)
    best_template = torch.gather(best_t, 1, pred_obj[:, None].repeat(1, best_t.shape[1]))[:, 0]
    return idx_sel, pred_obj, sem, best_template, scores, per_obj


def make_tied_descriptors(P: int, O: int, T: int, C: int, seed: int):
    """synth.make_descriptors with exact ties planted: template 1 of every object repeats template 0, object 1 repeats object 0
    (O > 1), and proposal 1 repeats proposal 0 (P > 1)"""
    q, ref = io.make_descriptors(P=P, O=O, T=T, C=C, seed=seed)
    if T > 1:
        ref[:, 1] = ref[:, 0]
    if O > 1:
        ref[1] = ref[0]
    if P > 1:
        q[1] = q[0]
    return q, ref
