"""Float64 oracle of the VOC07 linear-SVM evaluation (scripts/clf_voc07.py:56-105 of the reference).

- `synthetic_voc07`: seeded VOC07-shaped features (numpy PCG64): non-negative, L2-normalised, multi-label, with
  difficult (-1) labels in both splits and classes of different difficulty, so that different costs win.
- `objective` / `newton_cg`: liblinear's L2R_L2LOSS_SVC objective, the optimum every LinearSVC fit converges to, and
  a batched float64 truncated Newton solve of it to |grad f| <= 1e-10 |grad f(0)|.
- `stratified_folds` (sklearn's StratifiedKFold without shuffling, restated in virtex_b200.svm) and
  `average_precision` (sklearn's average_precision_score), restated so that no test needs sklearn.
"""
import hashlib

import numpy as np

from virtex_b200.svm import SVM_COSTS, stratified_folds  # noqa: F401  (re-exported: the fold restatement)

GOLDEN = "voc07_svm.pt"
SEED = 2007
N_TRAIN, N_TEST, DIM, CLASSES = 5011, 4952, 2048, 20
FOLDS = 3


def synthetic_voc07(n_train=N_TRAIN, n_test=N_TEST, dim=DIM, classes=CLASSES, seed=SEED):
    """(features_train, targets_train, features_test, targets_test): float32 [n, dim], int32 [n, classes]."""
    rng = np.random.Generator(np.random.PCG64(seed))
    freq = rng.uniform(0.03, 0.25, classes)                 # class frequencies
    strength = np.geomspace(0.08, 1.2, classes)             # signal strength: hard .. easy classes
    rng.shuffle(strength)
    protos = np.maximum(rng.standard_normal((classes, dim)), 0.0) * (rng.random((classes, dim)) < 0.15)
    protos /= np.maximum(np.linalg.norm(protos, axis=1, keepdims=True), 1e-30)  # an empty prototype stays 0
    shared = np.maximum(rng.standard_normal(dim), 0.0)
    shared /= np.linalg.norm(shared)

    def split(n):
        present = rng.random((n, classes)) < freq
        difficult = present & (rng.random((n, classes)) < 0.12)
        weight = present * strength * np.where(difficult, 0.3, 1.0) * rng.uniform(0.5, 1.5, (n, classes))
        x = (np.maximum(rng.standard_normal((n, dim)), 0.0) * 0.03 + 0.5 * shared
             + weight @ protos)
        x /= np.linalg.norm(x, axis=1, keepdims=True)
        t = np.where(difficult, -1, present.astype(np.int32)).astype(np.int32)
        return x.astype(np.float32), t

    xtr, ttr = split(n_train)
    xte, tte = split(n_test)
    return xtr, ttr, xte, tte


def feature_digest(xtr, xte):
    h = hashlib.sha256()
    h.update(np.ascontiguousarray(xtr, np.float32).tobytes())
    h.update(np.ascontiguousarray(xte, np.float32).tobytes())
    return h.hexdigest()


def problems(ttr, costs=SVM_COSTS, folds=FOLDS, positive_weight=2.0):
    """(y [n, K] +-1, fold ids [n, K], cw [n, P]): the signed per-sample cost y_i * c_ip of every problem
    p = (k * len(costs) + ci) * (folds + 1) + f, f = folds being the full fit (the layout of virtex_b200.svm)."""
    y = np.where(ttr == 1, 1.0, -1.0)
    fold = np.stack([stratified_folds(y[:, k], folds) for k in range(y.shape[1])], 1)
    n, K = y.shape
    keep = np.ones((n, K, folds + 1))
    keep[:, :, :folds] = fold[:, :, None] != np.arange(folds)
    cy = (np.where(y > 0, positive_weight, 1.0) * y)[:, :, None, None] * np.asarray(costs)[None, None, :, None] \
        * keep[:, :, None, :]
    return y, fold, cy.reshape(n, -1)


def augment(x):
    """x~ = [x, 1] in float64."""
    return np.concatenate([np.asarray(x, np.float64), np.ones((len(x), 1))], 1)


def objective(xa, cy, W):
    """f_p(W[:, p]) for every column: 1/2 |w|^2 + sum_i c_ip max(0, 1 - y_i x~_i . w)^2, float64."""
    m = np.maximum(0.0, 1.0 - np.sign(cy) * (xa @ W))
    return 0.5 * (W * W).sum(0) + (np.abs(cy) * m * m).sum(0)


def newton_cg(xa, cy, tol=1e-10, forcing=0.1, max_newton=100, max_cg=1000):
    """Batched truncated Newton (CG to the forcing term, exact line search) on every column of cy; returns W and the
    Newton steps taken per problem."""
    n, D = xa.shape
    P = cy.shape[1]
    c, y = np.abs(cy), np.sign(cy)
    W = np.zeros((D, P))
    running = np.ones(P, bool)
    steps = np.zeros(P, int)
    g0 = None
    for _ in range(max_newton):
        z = xa @ W
        act = (c > 0) & (y * z < 1)
        dact = np.where(act, c, 0.0)
        g = W + xa.T @ (2.0 * dact * (z - y))
        gn = np.linalg.norm(g, axis=0)
        if g0 is None:
            g0 = gn.copy()
        running &= gn > tol * g0
        if not running.any():
            break
        r = np.where(running, -g, 0.0)
        d = r.copy()
        s = np.zeros_like(W)
        rr = (r * r).sum(0)
        cg = running.copy()
        for _ in range(max_cg):
            hd = d + xa.T @ (2.0 * dact * (xa @ d))
            alpha = np.where(cg, rr / np.where(cg, (d * hd).sum(0), 1.0), 0.0)
            s += alpha * d
            r -= alpha * hd
            rr_new = (r * r).sum(0)
            cg &= rr_new > (forcing * gn) ** 2
            if not cg.any():
                break
            d = r + np.where(cg, rr_new / np.where(rr > 0, rr, 1.0), 0.0) * d
            rr = rr_new
        W += line_search(z, xa @ s, c, y, (W * s).sum(0), (s * s).sum(0)) * s * running
        steps += running
    return W, steps


def line_search(z, t, c, y, ws, ss, iters=200):
    """Minimiser of the convex piecewise quadratic phi(a) = f(w + a s) for every column (bracketed Newton)."""
    lo, hi = np.zeros(z.shape[1]), np.full(z.shape[1], np.inf)
    a = np.ones(z.shape[1])
    for _ in range(iters):
        act = (c > 0) & (y * (z + a * t) < 1)
        d1 = ws + a * ss + (2.0 * c * act * (z + a * t - y) * t).sum(0)
        d2 = ss + (2.0 * c * act * t * t).sum(0)
        lo = np.where(d1 < 0, a, lo)
        hi = np.where(d1 > 0, a, hi)
        an = a - d1 / np.where(d2 > 0, d2, 1.0)
        bad = ~((an > lo) & (an < hi))
        an = np.where(bad, np.where(np.isinf(hi), 2 * a, 0.5 * (lo + hi)), an)
        an = np.where(d1 == 0, a, an)
        if np.array_equal(an, a):
            break
        a = an
    return a


def average_precision(positive, scores):
    """sklearn's average_precision_score: sum over distinct thresholds (descending) of (R_k - R_{k-1}) P_k, tied
    scores forming one threshold; 0 without a positive."""
    positive = np.asarray(positive, bool)
    scores = np.asarray(scores, np.float64)
    if not positive.any():
        return 0.0
    order = np.argsort(-scores, kind="mergesort")
    s, yp = scores[order], positive[order]
    ends = np.r_[np.nonzero(np.diff(s))[0], len(s) - 1]
    tps = np.cumsum(yp)[ends].astype(np.float64)
    precision = tps / (ends + 1)
    recall = tps / tps[-1]
    return float(np.sum(np.diff(np.r_[0.0, recall]) * precision))


def evaluate(W, xtr, ttr, xte, tte, costs=SVM_COSTS, folds=FOLDS):
    """CV APs [K, costs, folds], test APs of the full fits [K, costs], best cost index [K] (the reference's rule:
    first cost whose mean CV AP is strictly above the running best, which starts at 0.0) and test AP [K]."""
    y, fold, _ = problems(ttr, costs, folds)
    K, nc, F = ttr.shape[1], len(costs), folds + 1
    ztr, zte = augment(xtr) @ W, augment(xte) @ W
    cv = np.zeros((K, nc, folds))
    te = np.zeros((K, nc))
    for k in range(K):
        keep = tte[:, k] != -1
        for ci in range(nc):
            for f in range(folds):
                p = (k * nc + ci) * F + f
                held = fold[:, k] == f
                cv[k, ci, f] = average_precision(y[held, k] > 0, ztr[held, p])
            p = (k * nc + ci) * F + folds
            te[k, ci] = average_precision(tte[keep, k] == 1, zte[keep, p])
    best = np.zeros(K, int)
    for k in range(K):
        b = 0.0
        for ci in range(nc):
            if cv[k, ci].mean() > b:
                b, best[k] = cv[k, ci].mean(), ci
    return cv, te, best, te[np.arange(K), best]
