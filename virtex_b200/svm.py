"""VOC07 linear-SVM evaluation on the sm_90a kernels: the second stage of scripts/clf_voc07.py.

The reference trains, per class, `LinearSVC(C, class_weight={1: 2, -1: 1}, penalty="l2", loss="squared_hinge",
max_iter=2000)` for every cost in (0.01, 0.1, 1.0, 10.0), scores each cost by 3-fold `cross_val_score(...,
scoring="average_precision")`, keeps the first cost with the best mean CV AP (strict `>` against a running best that
starts at 0.0), and reports that fit's `average_precision_score` on the test set, difficult (-1) test entries excluded
(clf_voc07.py:56-105).  `pool.map` runs that function once per class (:216-229).

`train_test_svms` solves every one of those fits -- K classes x costs x (folds + 1), the last one on all of trainval
-- as one column of a single batched truncated-Newton solve of liblinear's L2R_L2LOSS_SVC objective (the optimum
LinearSVC converges to, with the intercept a regularised coordinate of x~ = [x, 1]), and scores every held-out fold
and every full fit on the device.  See include/virtex_b200.h (VOC07 linear SVMs) for the kernels.
"""
import dataclasses
import warnings

import numpy as np
import torch

from . import ops

SVM_COSTS = (0.01, 0.1, 1.0, 10.0)
# Per-problem stopping rule: |grad f| <= GRAD_TOL |grad f(0)|, or the exact line search decreased f by at most
# DECREASE_TOL * f.  The fp32 products put a floor under |grad f| for the larger costs, so the second rule is the one
# that stops most C = 10 problems.  On the VOC07-shaped synthetic features (tests/voc07_oracle.py) every problem stops
# within 15 Newton steps, at most 4.5e-8 * f* above the float64 optimum; DECREASE_TOL = 1e-10 left 36 of 320
# problems stuck at the Newton-step cap on the fp32 noise floor.
GRAD_TOL = 1e-7
DECREASE_TOL = 1e-8
MAX_NEWTON = 60
MAX_CG = 256
_ALIGN = 64          # rows / features / problems padded to the GEMM's 64-wide tiles


class SvmConvergenceWarning(UserWarning):
    """A problem stopped at the Newton-step or CG-iteration cap (sklearn's ConvergenceWarning)."""


@dataclasses.dataclass
class SvmResults:
    test_ap: torch.Tensor        # float64 [K]: test AP of each class's selected fit (the reference's pool_output)
    mean_ap: float               # mean of test_ap
    best_cost: torch.Tensor      # float64 [K]
    cv_ap: torch.Tensor          # float64 [K, costs, folds]: AP of each held-out fold
    coef: torch.Tensor           # float32 [K, d]: weights of the selected fit
    intercept: torch.Tensor      # float32 [K]
    test_ap_all: torch.Tensor    # float64 [K, costs]: test AP of the full fit at every cost
    weights: torch.Tensor        # float32 [K, costs, folds + 1, d + 1]: (w, b) of every problem, full fit last
    newton_steps: torch.Tensor   # int32 [K, costs, folds + 1]
    cg_iterations: torch.Tensor  # int32 [K, costs, folds + 1], over all Newton steps


def _up(x, m):
    return (x + m - 1) // m * m


def stratified_folds(y, n_splits):
    """Test-fold id of every sample: sklearn's StratifiedKFold(n_splits) without shuffling, restated
    (sklearn/model_selection/_split.py, StratifiedKFold._make_test_folds)."""
    y = np.asarray(y)
    _, y_idx, y_inv = np.unique(y, return_index=True, return_inverse=True)
    _, class_perm = np.unique(y_idx, return_inverse=True)   # classes in order of first appearance
    y_encoded = class_perm[y_inv.reshape(-1)]
    n_classes = len(y_idx)
    if np.all(n_splits > np.bincount(y_encoded)):
        raise ValueError(f"n_splits={n_splits} cannot be greater than the number of members in each class.")
    y_order = np.sort(y_encoded)
    allocation = np.asarray([np.bincount(y_order[i::n_splits], minlength=n_classes) for i in range(n_splits)])
    folds = np.empty(len(y), dtype=np.int64)
    for k in range(n_classes):
        folds[y_encoded == k] = np.arange(n_splits).repeat(allocation[:, k])
    return folds


def _features(x, name):
    x = torch.as_tensor(x)
    if x.dim() != 2:
        raise ValueError(f"{name} must be 2-D [samples, features], got shape {tuple(x.shape)}")
    return x


def _targets(t, n, name):
    t = np.asarray(t.cpu() if torch.is_tensor(t) else t)
    if t.ndim != 2 or t.shape[0] != n:
        raise ValueError(f"{name} must be [samples, classes] with {n} samples, got shape {t.shape}")
    if not np.isin(t, (-1, 0, 1)).all():
        raise ValueError(f"{name} must hold 1 (present), 0 (absent) or -1 (difficult)")
    return t.astype(np.int64)


def train_test_svms(features_train, targets_train, features_test, targets_test, costs=SVM_COSTS, folds=3,
                    positive_weight=2.0):
    """The reference's `pool.map(train_test_single_svm, ...)` over all classes, on the GPU.

    features_*: [n, d] (CUDA tensors, or CPU tensors / numpy arrays, which are moved to the current CUDA device);
    targets_*: [n, K] with 1 = present, 0 = absent, -1 = difficult.  Training targets map 0 -> -1 (difficult images
    train as negatives); difficult test entries are left out of the test AP.  Runs on torch's current stream."""
    xtr, xte = _features(features_train, "features_train"), _features(features_test, "features_test")
    n, d = xtr.shape
    nt = xte.shape[0]
    if xte.shape[1] != d:
        raise ValueError(f"features_test has {xte.shape[1]} features, features_train {d}")
    ttr = _targets(targets_train, n, "targets_train")
    tte = _targets(targets_test, nt, "targets_test")
    K = ttr.shape[1]
    if tte.shape[1] != K:
        raise ValueError(f"targets_test has {tte.shape[1]} classes, targets_train {K}")
    costs = tuple(float(c) for c in costs)
    if not costs or min(costs) <= 0 or folds < 2 or positive_weight <= 0:
        raise ValueError("needs positive costs, folds >= 2 and a positive positive_weight")
    n_pad, dp = _up(n, _ALIGN), _up(d + 1, _ALIGN)
    if n_pad > 16384 or nt > 16384:
        raise ValueError("at most 16384 training (rounded up to 64) and 16384 test samples")
    device = xtr.device if xtr.is_cuda else torch.device("cuda", torch.cuda.current_device())
    xtr = xtr.to(device=device, dtype=torch.float32).contiguous()
    xte = xte.to(device=device, dtype=torch.float32).contiguous()

    ytr = np.where(ttr == 1, 1, -1)
    for k in range(K):
        if len(np.unique(ytr[:, k])) < 2:
            raise ValueError(f"class {k}: the training targets hold one label value only; "
                             "the number of classes has to be greater than one")
    fold_id = np.stack([stratified_folds(ytr[:, k], folds) for k in range(K)], 1)        # [n, K]

    nc, F = len(costs), folds + 1
    P_real = K * nc * F
    P = _up(P_real, _ALIGN)
    # cy[i, p] = y_i * c_ip, problem p = (k * nc + ci) * F + f; f < folds holds fold f out, f = folds is the full fit
    cw = np.where(ytr == 1, positive_weight, 1.0) * ytr                                 # [n, K]
    keep = np.ones((n, K, F))
    keep[:, :, :folds] = fold_id[:, :, None] != np.arange(folds)
    cy_np = np.zeros((n_pad, P), np.float32)
    cy_np[:n, :P_real] = (cw[:, :, None, None] * np.asarray(costs)[None, None, :, None] * keep[:, :, None, :]
                          ).reshape(n, P_real)
    cy = torch.from_numpy(cy_np).to(device)

    sol = _solve(xtr, xte, cy, dp, P)
    Z, Zt, flags = sol["z"], sol["z_test"], sol["flags"]

    # average precision: held-out folds over the training scores, full fits over the test scores
    lab_tr = torch.from_numpy((ttr == 1).astype(np.int8)).to(device)
    lab_te = torch.from_numpy(tte.astype(np.int8)).to(device)                 # -1: left out
    fold_dev = torch.from_numpy(fold_id.astype(np.int8)).to(device)
    kk, cc, ff = np.meshgrid(np.arange(K), np.arange(nc), np.arange(F), indexing="ij")
    pidx = (kk * nc + cc) * F + ff
    cv = np.stack([pidx[:, :, :folds].ravel(), kk[:, :, :folds].ravel(), ff[:, :, :folds].ravel()], 1)
    te = np.stack([pidx[:, :, folds].ravel(), kk[:, :, folds].ravel(), np.full(K * nc, -1)], 1)
    cv_ap = _average_precision(Z, n, lab_tr, fold_dev, cv, device).reshape(K, nc, folds)
    test_all = _average_precision(Zt, nt, lab_te, None, te, device).reshape(K, nc)

    best = np.full(K, -1)
    for k in range(K):
        best_ap = 0.0
        for ci in range(nc):
            m = float(cv_ap[k, ci].mean())
            if m > best_ap:
                best_ap, best[k] = m, ci
        if best[k] < 0:
            raise RuntimeError(f"class {k}: no cost reached a mean cross-validation AP above 0")

    w_all = sol["w"][:d + 1, :P_real].t().reshape(K, nc, F, d + 1).cpu()
    fl = flags[:, :P_real].cpu()
    status = fl[0].reshape(K, nc, F)
    capped = (status == 2) | (fl[5].reshape(K, nc, F) != 0)
    if bool(capped.any()):
        warnings.warn(f"{int(capped.sum())} of {P_real} SVM problems stopped at the Newton-step ({MAX_NEWTON}) or "
                      f"CG-iteration ({MAX_CG}) cap before converging", SvmConvergenceWarning, stacklevel=2)
    sel = torch.from_numpy(best)
    w_best = w_all[torch.arange(K), sel, folds]
    test_ap = torch.from_numpy(test_all[np.arange(K), best])
    return SvmResults(test_ap=test_ap, mean_ap=float(test_ap.mean()),
                      best_cost=torch.tensor([costs[c] for c in best], dtype=torch.float64),
                      cv_ap=torch.from_numpy(cv_ap), coef=w_best[:, :d].clone(), intercept=w_best[:, d].clone(),
                      test_ap_all=torch.from_numpy(test_all), weights=w_all,
                      newton_steps=fl[1].reshape(K, nc, F).clone(), cg_iterations=fl[4].reshape(K, nc, F).clone())


def _average_precision(scores, n, labels, folds, cols, device):
    cols_dev = torch.from_numpy(np.ascontiguousarray(cols, dtype=np.int32)).to(device)
    ap = torch.empty(len(cols), dtype=torch.float64, device=device)
    ops.call("vtx_svm_average_precision", scores.data_ptr(), scores.stride(0), n, labels.data_ptr(), labels.stride(0),
             ops._p(folds), folds.stride(0) if folds is not None else 0, cols_dev.data_ptr(), len(cols),
             ap.data_ptr(), ops._stream())
    return ap.cpu().numpy()


def _pinned_counts(n):
    return torch.zeros(n, dtype=torch.int32, pin_memory=True)


def _gemm(A, B, D, M, K, a_mn, tile_n=0):
    # fp32 D[M, P] = A . B over the concatenated split operands: no split-K, no atomics (deterministic)
    ops.gemm(A, B, D, M, D.shape[1], K, a_mn=a_mn, b_mn=1, tile_n=tile_n)


def _solve(xtr, xte, cy, dp, P):
    """Batched truncated Newton over the P columns of cy; returns the weights W [dp, P] (row d = the intercept), the
    training scores z = X~ W [n_pad, P], the test scores [nt_pad, P] and the per-problem flags."""
    dev = xtr.device
    n, d = xtr.shape
    n_pad = cy.shape[0]
    nt = xte.shape[0]
    nt_pad = _up(nt, _ALIGN)
    st = ops._stream()
    bf, f32, f64, i32 = torch.bfloat16, torch.float32, torch.float64, torch.int32
    xcat = torch.empty(n_pad, 3 * dp, dtype=bf, device=dev)
    xstk = torch.empty(3 * n_pad, dp, dtype=bf, device=dev)
    ops.call("vtx_svm_split_x", xtr.data_ptr(), xtr.stride(0), n, d, n_pad, dp, xcat.data_ptr(), xstk.data_ptr(), st)
    vec = lambda rows: torch.zeros(rows, P, dtype=f32, device=dev)  # noqa: E731
    W, G, R, Dv, S, HD = (vec(dp) for _ in range(6))
    Z, T, dact = vec(n_pad), vec(n_pad), vec(n_pad)
    wop, dop = (torch.zeros(3 * dp, P, dtype=bf, device=dev) for _ in range(2))
    uop = torch.zeros(3 * n_pad, P, dtype=bf, device=dev)
    sl = 32  # VTX_SVM_SLICES
    part_loss, part_rr = (torch.zeros(sl, P, dtype=f64, device=dev) for _ in range(2))
    part_g, part_dhd = (torch.zeros(3, sl, P, dtype=f64, device=dev) for _ in range(2))
    scal = torch.zeros(7, P, dtype=f64, device=dev)   # VTX_SVM_NSCAL
    flags = torch.zeros(6, P, dtype=i32, device=dev)  # VTX_SVM_NFLAGS
    running = torch.zeros(MAX_CG + 1, dtype=i32, device=dev)
    running_host = _pinned_counts(MAX_CG + 1)
    p_ = lambda t: t.data_ptr()  # noqa: E731

    for _ in range(MAX_NEWTON + 1):
        _gemm(xcat, wop, Z, n_pad, 3 * dp, 0)
        ops.call("vtx_svm_margin", p_(Z), p_(cy), n_pad, P, p_(uop), p_(dact), p_(part_loss), st)
        _gemm(xstk, uop, G, dp, 3 * n_pad, 1, tile_n=64)
        ops.call("vtx_svm_axpy_dot", p_(G), p_(W), dp, P, 1, p_(part_g), st)
        ops.call("vtx_svm_newton_begin", p_(part_loss), p_(part_g), P, p_(scal), p_(flags), GRAD_TOL, MAX_NEWTON,
                 p_(running[MAX_CG:]), st)
        if int(running[MAX_CG].item()) == 0:  # the one host synchronisation of a Newton step
            break
        ops.call("vtx_svm_cg_start", p_(G), p_(R), p_(Dv), p_(S), p_(flags), dp, P, p_(dop), st)
        _cg(xcat, xstk, dop, uop, T, HD, Dv, R, S, dact, part_dhd, part_rr, scal, flags, running, running_host,
            n_pad, dp, P, st)
        # exact line search along s: t = X~ s
        ops.call("vtx_svm_split_cols", p_(S), dp, P, p_(dop), st)
        _gemm(xcat, dop, T, n_pad, 3 * dp, 0)
        ops.call("vtx_svm_axpy_dot", p_(S), p_(W), dp, P, 0, p_(part_dhd), st)
        ops.call("vtx_svm_line_search", p_(Z), p_(T), p_(cy), n_pad, P, p_(part_dhd), p_(scal), p_(flags),
                 DECREASE_TOL, st)
        ops.call("vtx_svm_newton_step", p_(W), p_(S), p_(scal), dp, P, p_(wop), st)

    # Z holds X~ W of the final W (the loop ends right after computing it); the test scores use the same operand
    xcat_t = torch.empty(nt_pad, 3 * dp, dtype=bf, device=dev)
    ops.call("vtx_svm_split_x", xte.data_ptr(), xte.stride(0), nt, d, nt_pad, dp, xcat_t.data_ptr(), 0, st)
    Zt = vec(nt_pad)
    _gemm(xcat_t, wop, Zt, nt_pad, 3 * dp, 0)
    return {"w": W, "z": Z, "z_test": Zt, "flags": flags}


def _cg(xcat, xstk, dop, vop, T, HD, Dv, R, S, dact, part_dhd, part_rr, scal, flags, running, running_host, n_pad, dp,
        P, st):
    """CG on H s = -g for every problem still running, in lockstep.  The host never waits for the device here: each
    iteration queues a copy of the count of problems still in CG to pinned memory, and the loop stops issuing once
    a copy that has already landed reads 0 (iterations issued meanwhile are no-ops for finished problems)."""
    p_ = lambda t: t.data_ptr()  # noqa: E731
    pending = []
    for j in range(MAX_CG):
        _gemm(xcat, dop, T, n_pad, 3 * dp, 0)
        ops.call("vtx_svm_hess_mid", p_(T), p_(dact), n_pad, P, p_(vop), st)
        _gemm(xstk, vop, HD, dp, 3 * n_pad, 1, tile_n=64)
        ops.call("vtx_svm_axpy_dot", p_(HD), p_(Dv), dp, P, 1, p_(part_dhd), st)
        ops.call("vtx_svm_cg_update", p_(S), p_(R), p_(Dv), p_(HD), p_(part_dhd[1]), p_(scal), p_(flags), dp, P,
                 p_(part_rr), st)
        ops.call("vtx_svm_cg_scalars", p_(part_rr), P, p_(scal), p_(flags), MAX_CG, p_(running[j:]), st)
        running_host[j:j + 1].copy_(running[j:j + 1], non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        pending.append((ev, j))
        ops.call("vtx_svm_cg_direction", p_(R), p_(Dv), p_(scal), p_(flags), dp, P, p_(dop), st)
        finished = False
        while pending and pending[0][0].query():
            finished |= int(running_host[pending.pop(0)[1]]) == 0
        if finished:
            return
