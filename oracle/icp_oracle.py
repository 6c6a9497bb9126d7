"""Float64 restatement of the point-to-plane ICP refinement (sam6d_b200/csrc/icp.cu, include/sam6d_b200.h at sam6d_icp_refine).

Every step runs in float64: the transform y = R^T (p - t), the nearest sample (an exact tie to the lowest index), the
inlier test |y - q|^2 < tau_k^2, the normal equations in coordinates divided by the object radius r, the damped Cholesky
solve and the right update R <- R Exp(w), t <- t + R (r v).  The GPU kernel evaluates the transform and the search in fp32;
the tests hold it to this restatement within bounds derived from that rounding.  step() runs one iteration from a given
pose, so a test can start it from the GPU's fp32 inputs; refine() runs K iterations with the kernel's stopping rules."""
import numpy as np

MIN_INLIERS = 32
STEP_TOL = 1e-7
DAMPING = 1e-4


def tau_fraction(k: int) -> float:
    """inlier radius of iteration k as a fraction of the object radius (csrc/icp.cu: icp_tau_fraction)"""
    return max(0.3 * 2.0 ** -k, 0.05)


def so3_exp(w) -> np.ndarray:
    w = np.asarray(w, dtype=np.float64)
    th2 = float(w @ w)
    th = np.sqrt(th2)
    if th < 1e-4:
        a, b = 1.0 - th2 / 6.0 + th2 * th2 / 120.0, 0.5 - th2 / 24.0 + th2 * th2 / 720.0
    else:
        a, b = np.sin(th) / th, (1.0 - np.cos(th)) / th2
    K = np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])
    return np.eye(3) + a * K + b * (K @ K)


def nearest(y: np.ndarray, Q: np.ndarray, chunk: int = 256):
    """-> (j (N,) the lowest index of the nearest sample, its squared distance (N,), the second-smallest squared distance over
    the other samples (N,), inf when M = 1)"""
    j = np.empty(len(y), np.int64)
    d1, d2 = np.empty(len(y)), np.empty(len(y))
    for s in range(0, len(y), chunk):
        d = ((y[s:s + chunk, None, :] - Q[None, :, :]) ** 2).sum(-1)
        rows = np.arange(d.shape[0])
        j[s:s + chunk] = np.argmin(d, axis=1)              # argmin returns the first of equal minima
        d1[s:s + chunk] = d[rows, j[s:s + chunk]]
        d[rows, j[s:s + chunk]] = np.inf
        d2[s:s + chunk] = d.min(axis=1)
    return j, d1, d2


def normal_equations(y: np.ndarray, q: np.ndarray, n: np.ndarray, r: float):
    """inlier points y, their samples q and normals n (object frame, metres) -> (A (6,6), b (6,), sum e^2) in units of r"""
    ys, qs = y / r, q / r
    e = (n * (ys - qs)).sum(1)
    J = np.concatenate([np.cross(ys, n), n], axis=1)
    return J.T @ J, J.T @ e, float(e @ e)


def solve(A: np.ndarray, b: np.ndarray):
    """(A + lambda I) delta = b with lambda = 1e-4 trace(A) / 6, by Cholesky -> delta (6,), the damped matrix"""
    Ad = A + DAMPING * np.trace(A) / 6.0 * np.eye(6)
    L = np.linalg.cholesky(Ad)
    return np.linalg.solve(L.T, np.linalg.solve(L, b)), Ad


def step(R, t, P, Q, Nn, r: float, k: int) -> dict:
    """one iteration k from pose (R, t) -> dict: y, j, dmin, dsecond (nearest()'s distances), inlier mask, count, A, b, sse,
    rms (metres), delta, R, t (the updated pose, or the input pose when fewer than MIN_INLIERS are inliers), stop (the instance
    stops after this iteration), applied"""
    R, t = np.asarray(R, np.float64), np.asarray(t, np.float64)
    P, Q, Nn = np.asarray(P, np.float64), np.asarray(Q, np.float64), np.asarray(Nn, np.float64)
    y = (P - t) @ R                                        # rows R^T (p - t)
    j, dmin, dsecond = nearest(y, Q)
    tau = r * tau_fraction(k)
    inl = dmin < tau * tau
    cnt = int(inl.sum())
    A, b, sse = normal_equations(y[inl], Q[j[inl]], Nn[j[inl]], r)
    out = dict(y=y, j=j, dmin=dmin, dsecond=dsecond, inlier=inl, count=cnt, A=A, b=b, sse=sse, rms=r * np.sqrt(sse / cnt) if cnt else 0.0,
               delta=None, R=R, t=t, stop=True, applied=False)
    if cnt < MIN_INLIERS:
        return out
    delta, _ = solve(A, b)
    w, v = delta[:3], delta[3:]
    out.update(delta=delta, R=R @ so3_exp(w), t=t + R @ (r * v), applied=True,
               stop=bool(np.linalg.norm(w) < STEP_TOL and np.linalg.norm(v) < STEP_TOL))
    return out


def refine(R0, t0, P, Q, Nn, r: float, iters: int) -> dict:
    """K iterations with the kernel's stopping rules -> dict: R, t, inliers and rms of the last iteration evaluated, iters_run
    (updates applied), history (every step's dict)"""
    R, t = np.asarray(R0, np.float64), np.asarray(t0, np.float64)
    hist, n_run = [], 0
    for k in range(iters):
        s = step(R, t, P, Q, Nn, r, k)
        hist.append(s)
        R, t = s["R"], s["t"]
        n_run += s["applied"]
        if s["stop"]:
            break
    last = hist[-1] if hist else dict(count=0, rms=0.0)
    return dict(R=R, t=t, inliers=last["count"], rms=last["rms"], iters_run=n_run, history=hist)


def rotation_error_deg(Ra, Rb) -> float:
    c = (np.trace(np.asarray(Ra, np.float64).T @ np.asarray(Rb, np.float64)) - 1.0) / 2.0
    return float(np.degrees(np.arccos(np.clip(c, -1.0, 1.0))))
