"""Float64 restatement of the distinct coarse hypotheses (csrc/coarse.cu, sam6d_coarse_pick_distinct in include/sam6d_b200.h).
Not in the reference: SAM-6D keeps only the best coarse hypothesis.

Per proposal, K greedy rounds over the n2 retained hypotheses (R_j, t_j, score_j) = Rt[top[j]], scores[j], all live at the start:
  1. pick i = the first argmax of the live scores; a NaN score is never picked; in round 0 an all-NaN row picks hypothesis 0, a
     later round with nothing to pick ends the selection;
  2. slot r = i, valid; i is no longer live;
  3. every live j that is not distinct from i is no longer live: j is distinct when trace(R_i^T R_j) < cos_thr or
     |t_i - t_j|^2 >= d2_min, with cos_thr = 1 + 2 cos(min_angle) and d2_min = min_dist^2 rounded to fp32 (thresholds()).
Slots from count on are copies of slot 0 with valid 0.

The kernel evaluates the trace and the squared distance in fp32, rounded to nearest without fused multiply-adds, in the order
the header states.  With u = 2^-24 and gamma_n = n u / (1 - n u), the fp32 trace of nine products summed left to right is
within gamma_9 sum_e |R_i[e] R_j[e]| of the exact one, and the fp32 squared distance (three rounded differences, three rounded
squares, two additions, all terms >= 0) within gamma_5 d2.  A comparison whose outcome can change inside those bounds is
"undecided": only rows without one must equal the kernel.  fp32=True evaluates both quantities in the kernel's fp32 order
instead (numpy float32 rounds every operation to nearest), which the kernel must match on every row."""
import numpy as np

U = 2.0 ** -24


def _gamma(n):
    return n * U / (1.0 - n * U)


def thresholds(min_angle, min_dist):
    """-> (cos_thr, d2_min), the fp32 values the kernel compares against, as float64"""
    return (float(np.float32(1.0 + 2.0 * np.cos(np.radians(float(min_angle))))), float(np.float32(float(min_dist) ** 2)))


def _trace_d2(hi, hj, fp32):
    """hi (12,), hj (m,12) [R row-major, t] -> trace(R_i^T R_j) (m,), |t_i - t_j|^2 (m,), and their rounding bounds"""
    if fp32:
        a, b = hi.astype(np.float32), hj.astype(np.float32)
        tr = a[0] * b[:, 0]
        for e in range(1, 9):
            tr = tr + a[e] * b[:, e]
        d = a[9:12] - b[:, 9:12]
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        z = np.zeros(len(hj))
        return tr.astype(np.float64), d2.astype(np.float64), z, z
    a, b = hi.astype(np.float64), hj.astype(np.float64)
    p = a[None, :9] * b[:, :9]
    d = a[None, 9:12] - b[:, 9:12]
    d2 = (d * d).sum(axis=1)
    return p.sum(axis=1), d2, _gamma(9) * np.abs(p).sum(axis=1) * (1 + 1e-12), _gamma(5) * d2 * (1 + 1e-12)


def _argmax_first(score, live):
    best, bi = -np.inf, None
    for j in np.flatnonzero(live):
        v = score[j]
        if v > best or (v == best and (bi is None or j < bi)):     # NaN compares false: never picked
            best, bi = v, j
    return bi


def pick_one(hyp, score, K, cos_thr, d2_min, fp32=False):
    """hyp (n2,12) float, score (n2,) -> (picks: indices into hyp of the valid slots, number of undecided comparisons made)"""
    n2 = len(hyp)
    live = np.ones(n2, bool)
    picks, n_und = [], 0
    for r in range(K):
        i = _argmax_first(score, live)
        if i is None:
            if r > 0:
                break
            i = 0
        picks.append(int(i))
        live[i] = False
        js = np.flatnonzero(live)
        if len(js) == 0:
            continue
        tr, d2, btr, bd2 = _trace_d2(hyp[i], hyp[js], fp32)
        sure = (tr + btr < cos_thr) | (d2 - bd2 >= d2_min)           # distinct whatever the rounding
        maybe = (tr - btr < cos_thr) | (d2 + bd2 >= d2_min)          # distinct for some rounding
        n_und += int((maybe & ~sure).sum())
        live[js[~((tr < cos_thr) | (d2 >= d2_min))]] = False
    return picks, n_und


def pick_distinct(Rt, top, scores, K, cos_thr, d2_min, fp32=False):
    """Rt (B,n1,12), top (B,n2), scores (B,n2) -> R (B,K,3,3), t (B,K,3), score (B,K) float64 (of the fp32 inputs), valid (B,K)
    u8, count (B) i32, pick (B,K) i64 (index into top, slot 0's repeated past count), undecided (B) comparisons per row"""
    Rt, top, scores = np.asarray(Rt), np.asarray(top), np.asarray(scores)
    B = Rt.shape[0]
    R, t = np.zeros((B, K, 3, 3)), np.zeros((B, K, 3))
    sc, valid = np.zeros((B, K)), np.zeros((B, K), np.uint8)
    count, pick, und = np.zeros(B, np.int32), np.zeros((B, K), np.int64), np.zeros(B, np.int64)
    for b in range(B):
        hyp = Rt[b, top[b]]
        picks, und[b] = pick_one(hyp, scores[b].astype(np.float64), K, cos_thr, d2_min, fp32)
        count[b] = len(picks)
        full = picks + [picks[0]] * (K - len(picks))
        pick[b] = full
        valid[b, :len(picks)] = 1
        R[b] = hyp[full, :9].reshape(K, 3, 3)
        t[b] = hyp[full, 9:12]
        sc[b] = scores[b][full]
    return R, t, sc, valid, count, pick, und
