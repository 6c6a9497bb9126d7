"""Multi-GPU plumbing: proposals are independent (SURVEY.md 8e), so the path shards by contiguous proposal chunks with no
data-path collective; the only exchange is one all-gather of the final poses (16 fp32 per pose: R 9, t 3, score 1, pad 3)
over NCCL / NVLink.  ISM template scoring shards the O x T reference descriptors by object instead (every rank scores all
proposals against its objects; one all-gather of 12 bytes per proposal and rank picks the winner).  One process per GPU,
torch.distributed for the rendezvous."""
import functools
from typing import Dict, Tuple

import torch
import torch.distributed as dist

POSE_FLOATS = 16


def shard_range(total: int, rank: int, world: int) -> Tuple[int, int]:
    """contiguous chunk [lo, hi) of `total` proposals owned by `rank` (sizes differ by at most one)"""
    base, rem = divmod(total, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def pack_poses(end_points: Dict[str, torch.Tensor]) -> torch.Tensor:
    R, t, s = end_points["pred_R"], end_points["pred_t"], end_points["pred_pose_score"]
    B = R.shape[0]
    out = torch.zeros(B, POSE_FLOATS, dtype=torch.float32, device=R.device)
    out[:, :9] = R.reshape(B, 9)
    out[:, 9:12] = t
    out[:, 12] = s
    return out


def unpack_poses(p: torch.Tensor) -> Dict[str, torch.Tensor]:
    return dict(pred_R=p[:, :9].reshape(-1, 3, 3), pred_t=p[:, 9:12], pred_pose_score=p[:, 12])


def all_gather_poses(local: torch.Tensor, counts=None) -> torch.Tensor:
    """local (B_local,16) -> (sum B,16) on every rank.  Equal chunk sizes use one all_gather_into_tensor; ragged chunks
    (counts = per-rank sizes) pad to the maximum and trim."""
    if not dist.is_initialized() or dist.get_world_size() == 1:
        return local
    world = dist.get_world_size()
    if counts is None or len(set(counts)) == 1:
        out = torch.empty(world * local.shape[0], POSE_FLOATS, dtype=local.dtype, device=local.device)
        dist.all_gather_into_tensor(out, local.contiguous())
        return out
    mx = max(counts)
    padded = torch.zeros(mx, POSE_FLOATS, dtype=local.dtype, device=local.device)
    padded[: local.shape[0]] = local
    out = torch.empty(world * mx, POSE_FLOATS, dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(out, padded)
    return torch.cat([out[r * mx: r * mx + counts[r]] for r in range(world)], dim=0)


def _local_best(proposal_descriptors: torch.Tensor, ref_descriptors: torch.Tensor, aggregation_function: str = "avg_5"):
    """fused kernel on this rank's object shard: per proposal (best local object, its aggregated score, its best template)"""
    from . import ism, ops
    qn = ism._normalized(proposal_descriptors)
    rn = ops.l2norm_rows(ref_descriptors.float().contiguous())
    _, _, best_obj, best_score, best_tmpl = ops.template_score(qn, rn, want_sim=False, aggregation=aggregation_function)
    return best_obj.long(), best_score, best_tmpl.long()


def sharded_semantic_score(proposal_descriptors: torch.Tensor, local_ref_descriptors: torch.Tensor, obj_lo: int,
                           confidence_thresh: float = 0.2, local_best=None, aggregation_function: str = "avg_5"):
    """compute_semantic_score (ISM/model/detector.py:260-296) with the reference descriptors sharded by object:
    this rank holds objects [obj_lo, obj_lo + O_local) (shard_range over the O objects, ascending with the rank).
    Every rank returns the same (idx_selected_proposals, pred_idx_objects, semantic_score, best_template) the unsharded call
    gives: per-object scores do not depend on the sharding, and ties go to the lowest object index (first maximum) because
    lower ranks own lower indices.  aggregation_function: as ism.compute_semantic_score.  `local_best(desc, refs)` defaults
    to the CUDA kernel with that aggregation; tests inject the CPU oracle (which then applies its own aggregation)."""
    fn = local_best or functools.partial(_local_best, aggregation_function=aggregation_function)
    P = proposal_descriptors.shape[0]
    if local_ref_descriptors.shape[0] == 0:                       # a rank may own no object (O < world)
        score = torch.full((P,), -1.0, dtype=torch.float32, device=proposal_descriptors.device)
        obj = torch.zeros(P, dtype=torch.long, device=score.device)
        tmpl = torch.zeros(P, dtype=torch.long, device=score.device)
    else:
        obj, score, tmpl = fn(proposal_descriptors, local_ref_descriptors)
    rec = torch.stack([score.float(), (obj + obj_lo).float(), tmpl.float()], dim=1).contiguous()   # exact: indices << 2^24
    if dist.is_initialized() and dist.get_world_size() > 1:
        world = dist.get_world_size()
        allrec = torch.empty(world * P, 3, dtype=torch.float32, device=rec.device)
        dist.all_gather_into_tensor(allrec, rec)
        allrec = allrec.view(world, P, 3)
        win = torch.argmax(allrec[:, :, 0], dim=0)                # first maximum over ranks = lowest object index on ties
        rec = allrec[win, torch.arange(P, device=rec.device)]
    keep = rec[:, 0] > confidence_thresh
    idx_selected = torch.arange(P, device=rec.device)[keep]
    return idx_selected, rec[keep, 1].long(), rec[keep, 0], rec[keep, 2].long()
