"""Float64 restatement of the depth agreement of pose hypotheses (sam6d_b200/csrc/verify.cu, include/sam6d_b200.h at
sam6d_pose_verify) and of its score (sam6d_b200/ops.py: verify_score).

Per pixel of hypothesis p: dr = rdepth * rscale, do = depth, e = do - dr, all in float64 (the kernel rounds dr and e to fp32).
Classes: silhouette dr > 0; occluded, fit and violation need the silhouette and do > 0 and are e < -tau, |e| <= tau and
e > tau; mask is the hypothesis's mask row != 0 and mask_fit mask and fit.  The score is fit_frac x cover with
fit_frac = n_fit / (n_fit + n_viol) and cover = n_mask_fit / n_mask, each 0 when its denominator is 0.  undecided() marks the
pixels whose class the kernel's fp32 rounding can change, so a test can hold the kernel to this restatement exactly elsewhere."""
import numpy as np

U = 2.0 ** -24
NAMES = ("n_sil", "n_occ", "n_fit", "n_viol", "n_mask", "n_mask_fit")


def classes(rdepth, depth, mask, mrow, tau, rscale):
    """rdepth (P,H,W), depth (H,W), mask (M,H,W), mrow (P), tau (P), rscale -> dict of (P,H,W) bool arrays, one per class
    (sil, occ, fit, viol, mask, mask_fit), and e (P,H,W) float64"""
    rd = np.asarray(rdepth, np.float64)
    dr = rd * float(rscale)
    do = np.asarray(depth, np.float64)[None]
    tau = np.asarray(tau, np.float64).reshape(-1, 1, 1)
    e = do - dr
    sil = dr > 0
    seen = sil & (do > 0)
    fit = seen & (np.abs(e) <= tau)
    m = np.asarray(mask)[np.asarray(mrow, np.int64)] != 0
    return dict(sil=sil, occ=seen & (e < -tau), fit=fit, viol=seen & (e > tau), mask=m, mask_fit=m & fit, e=e)


def counts(rdepth, depth, mask, mrow, tau, rscale) -> np.ndarray:
    """-> (P,6) int64 in the order of NAMES"""
    c = classes(rdepth, depth, mask, mrow, tau, rscale)
    return np.stack([c[k].reshape(len(c[k]), -1).sum(axis=1) for k in ("sil", "occ", "fit", "viol", "mask", "mask_fit")], axis=1)


def score(c):
    """counts (P,6) -> (fit_frac, cover, verify) float64 (P,) each"""
    c = np.asarray(c, np.float64)
    seen, n_mask = c[:, 2] + c[:, 3], c[:, 4]
    fit_frac = np.divide(c[:, 2], seen, out=np.zeros_like(seen), where=seen > 0)
    cover = np.divide(c[:, 5], n_mask, out=np.zeros_like(n_mask), where=n_mask > 0)
    return fit_frac, cover, fit_frac * cover


def undecided(rdepth, depth, tau, rscale):
    """(P,H,W) bool: silhouette pixels with do > 0 whose e lies within the fp32 rounding bound of +-tau.  With rscale and tau
    the fp32 values the kernel uses, dr32 = dr (1 + d1) and e32 = (do - dr32)(1 + d2) with |d1|, |d2| <= u, so
    |e32 - e| <= u |dr| + u (|e| + u |dr|) <= u (|e| + 2 |dr|).  Elsewhere the kernel's class is the oracle's (the silhouette
    and do > 0 tests are exact: the product of two positive normal floats does not round to 0 at render depths)."""
    c = classes(rdepth, depth, np.zeros((1,) + np.shape(depth), np.uint8), np.zeros(len(rdepth), np.int64), tau, rscale)
    dr = np.asarray(rdepth, np.float64) * float(rscale)
    tau = np.asarray(tau, np.float64).reshape(-1, 1, 1)
    bound = U * (np.abs(c["e"]) + 2 * np.abs(dr))
    seen = c["sil"] & (np.asarray(depth, np.float64)[None] > 0)
    return seen & (np.abs(np.abs(c["e"]) - tau) <= bound)
