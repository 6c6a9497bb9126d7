"""Numpy restatement of the tracker (sam6d_b200/csrc/track.cu at sam6d_track_points, sam6d_b200/track.py).

track_points() is the observed-point selection with every float32 operation that decides membership (depth, back-projection,
squared distance to the gate centre, the comparison) in float32 in the kernel's order, so it reproduces the candidate set,
the counts, the selected pixels and the points bit for bit; the dilation is boolean and the rank arithmetic is in Python
integers.  lost() and detection_due() restate the tracker's loss rule and detection schedule."""
import numpy as np

F32 = np.float32


def dilate(sil: np.ndarray, m: int) -> np.ndarray:
    """(O,H,W) bool silhouettes -> dilated by a (2m+1)^2 square window, as two separable max passes (rows, then columns)"""
    O, H, W = sil.shape
    h = np.zeros_like(sil)
    for d in range(-min(m, W), min(m, W) + 1):
        lo, hi = max(0, -d), min(W, W - d)
        h[:, :, lo:hi] |= sil[:, :, lo + d:hi + d]
    v = np.zeros_like(sil)
    for d in range(-min(m, H), min(m, H) + 1):
        lo, hi = max(0, -d), min(H, H - d)
        v[:, lo:hi, :] |= h[:, lo + d:hi + d, :]
    return v


def back_project(depth_raw: np.ndarray, depth_scale: float, K) -> np.ndarray:
    """(H,W) raw depth -> (H,W,3) float32 camera points: z = (float32(raw) * depth_scale) / 1000, x = ((u - cx) * z) / fx,
    y = ((v - cy) * z) / fy, each operation in float32"""
    K = np.asarray(K, np.float64).reshape(3, 3).astype(F32)
    H, W = depth_raw.shape
    z = (depth_raw.astype(F32) * F32(depth_scale)) / F32(1000.0)
    xs = np.arange(W, dtype=F32)[None, :]
    ys = np.arange(H, dtype=F32)[:, None]
    x = ((xs - K[0, 2]) * z) / K[0, 0]
    y = ((ys - K[1, 2]) * z) / K[1, 1]
    return np.stack([x, y, z], axis=-1).astype(F32)


def candidates(rdepth, depth_raw, depth_scale, K, centre, radius, margin) -> np.ndarray:
    """-> (O,H,W) bool: dilated silhouette, positive observed depth, inside the gate ((dx^2 + dy^2) + dz^2 <= r^2 in float32)"""
    rdepth = np.asarray(rdepth, F32)
    p = back_project(np.asarray(depth_raw), depth_scale, K)
    c = np.asarray(centre, F32)[:, None, None, :]
    r = np.asarray(radius, F32)[:, None, None]
    d = p[None] - c
    d2 = (d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1]) + d[..., 2] * d[..., 2]
    return dilate(rdepth > 0, int(margin)) & (p[None, ..., 2] > 0) & (r > 0) & (d2 <= r * r)


def select(count: int, n: int) -> np.ndarray:
    """ranks of the n outputs among count candidates: floor(i count / n) when count >= n, i mod count when 0 < count < n"""
    i = np.arange(n, dtype=np.int64)
    if count >= n:
        return i * count // n
    return i % count if count else np.full(n, -1, np.int64)


def track_points(rdepth, depth_raw, depth_scale, K, centre, radius, margin, n):
    """-> (pts (O,n,3) float32, count (O,) int64, index (O,n) int64 pixel y W + x or -1, cand (O,H,W) bool)"""
    cand = candidates(rdepth, depth_raw, depth_scale, K, centre, radius, margin)
    O, H, W = cand.shape
    p = back_project(np.asarray(depth_raw), depth_scale, K).reshape(-1, 3)
    pts = np.zeros((O, n, 3), F32)
    index = np.full((O, n), -1, np.int64)
    count = np.zeros(O, np.int64)
    for o in range(O):
        flat = np.flatnonzero(cand[o])                   # raster order
        count[o] = len(flat)
        if len(flat):
            index[o] = flat[select(len(flat), n)]
            pts[o] = p[index[o]]
    return pts, count, index, cand


def lost(inliers: int, rms: float, n: int, min_inlier_fraction: float, max_rms_m: float) -> bool:
    """a track is lost when its ICP ends with fewer than min_inlier_fraction of the n points as inliers, or above max_rms_m"""
    return inliers < min_inlier_fraction * n or rms > max_rms_m


def detection_due(first: bool, lost_last_frame: bool, frames_since_detection: int, redetect_interval: int) -> bool:
    """detection runs on the first frame, on the frame after a track was lost, and once redetect_interval frames have passed
    without one"""
    return first or lost_last_frame or frames_since_detection >= redetect_interval
