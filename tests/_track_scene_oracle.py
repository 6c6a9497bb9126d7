"""Numpy restatement of the multi-instance tracker (sam6d_b200/csrc/track.cu at sam6d_track_points_scene,
sam6d_b200/track.py with max_instances > 1), on top of oracle/track_oracle.py's dilation, back-projection and selection.

track_points_scene() gives every pixel to at most one of L tracks with the kernel's float32 operations in the kernel's order
and the kernel's walk over the tracks (strict <, so exact ties stay with the lower j), so it reproduces the candidate sets,
counts, selected pixels and points bit for bit.  merge_drops() and starts() restate the tracker's merge and start rules."""
import numpy as np

from oracle import track_oracle as to

F32 = np.float32


def eligible(rdepth, depth_raw, depth_scale, K, centre, radius, margin):
    """-> (elig (L,H,W) bool: conditions 1-3 of sam6d_track_points per track, d2 (L,H,W) float32 squared gate distances)"""
    rdepth = np.asarray(rdepth, F32)
    p = to.back_project(np.asarray(depth_raw), depth_scale, K)
    c = np.asarray(centre, F32)[:, None, None, :]
    r = np.asarray(radius, F32)[:, None, None]
    d = p[None] - c
    d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    return to.dilate(rdepth > 0, int(margin)) & (p[None, ..., 2] > 0) & (r > 0) & (d2 <= r * r), d2


def owners(rdepth, depth_raw, depth_scale, K, centre, radius, margin) -> np.ndarray:
    """-> (H,W) int64: the track each pixel goes to, -1 for none.  Walking j = 0 .. L-1: the eligible track with the least
    rendered depth among those rendered there (> 0), else the eligible track with the least d2 / r^2 (float32)"""
    rdepth = np.asarray(rdepth, F32)
    elig, d2 = eligible(rdepth, depth_raw, depth_scale, K, centre, radius, margin)
    r = np.asarray(radius, F32)
    L, H, W = elig.shape
    front, band = np.full((H, W), -1, np.int64), np.full((H, W), -1, np.int64)
    front_z, band_q = np.zeros((H, W), F32), np.zeros((H, W), F32)
    with np.errstate(divide="ignore", invalid="ignore"):
        for j in range(L):
            rz = rdepth[j]
            f = elig[j] & (rz > 0) & ((front < 0) | (rz < front_z))
            front[f], front_z[f] = j, rz[f]
            q = d2[j] / (r[j] * r[j])
            b = elig[j] & ~(rz > 0) & ((band < 0) | (q < band_q))
            band[b], band_q[b] = j, q[b]
    return np.where(front >= 0, front, band)


def track_points_scene(rdepth, depth_raw, depth_scale, K, centre, radius, margin, n):
    """-> (pts (L,n,3) float32, count (L,) int64, index (L,n) int64 pixel y W + x or -1, cand (L,H,W) bool)"""
    own = owners(rdepth, depth_raw, depth_scale, K, centre, radius, margin)
    L = np.asarray(rdepth).shape[0]
    cand = own[None] == np.arange(L)[:, None, None]
    p = to.back_project(np.asarray(depth_raw), depth_scale, K).reshape(-1, 3)
    pts = np.zeros((L, n, 3), F32)
    index = np.full((L, n), -1, np.int64)
    count = np.zeros(L, np.int64)
    for j in range(L):
        flat = np.flatnonzero(cand[j])                   # raster order
        count[j] = len(flat)
        if len(flat):
            index[j] = flat[to.select(len(flat), n)]
            pts[j] = p[index[j]]
    return pts, count, index, cand


def merge_drops(track_ids, centroids, rho, assoc_scale) -> set:
    """one object's live tracks (ids, centroids (k,3) metres) after the ICP -> the ids the merge rule drops: walking the tracks
    by ascending id, a track within assoc_scale x rho of a kept (older) track's centroid is dropped"""
    kept, drop = [], set()
    for i in np.argsort(np.asarray(track_ids), kind="stable"):
        c = np.asarray(centroids[i], np.float64)
        if any(np.linalg.norm(c - k) <= assoc_scale * rho for k in kept):
            drop.add(int(track_ids[i]))
        else:
            kept.append(c)
    return drop


def starts(scores, centroids, live_centroids, free, rho, start_score, assoc_scale) -> list:
    """one object's PEM instances (scores, centroids (k,3) metres) -> the instances that start tracks, in start order: by
    descending score (stable), the best one whatever its score when the object has no live track; every other needs
    score >= start_score and a centroid farther than assoc_scale x rho from every live track's, those started here included;
    at most `free` of them"""
    live = [np.asarray(c, np.float64) for c in live_centroids]
    out = []
    for i in np.argsort(-np.asarray(scores, np.float64), kind="stable"):
        if len(out) == free:
            break
        c = np.asarray(centroids[i], np.float64)
        if live and (scores[i] < start_score or any(np.linalg.norm(c - k) <= assoc_scale * rho for k in live)):
            continue
        out.append(int(i))
        live.append(c)
    return out
