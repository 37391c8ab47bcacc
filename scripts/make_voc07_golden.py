"""Write tests/golden/voc07_svm.pt: the reference's VOC07 SVM stage on the seeded synthetic features of
tests/voc07_oracle.py, and the float64 optimum of every one of its 320 LinearSVC problems.

The reference function `train_test_single_svm` (scripts/clf_voc07.py:56-105) is taken from the unmodified reference
file (its definition only: the script's module-level imports need the dataset and TensorBoard stack) and run once per
class, as the reference's pool.map does.  Needs sklearn and a reference checkout ($VIRTEX_REFERENCE_ROOT).  The fixture
holds no feature arrays: the tests regenerate them from the seed and check their SHA-256.

    VIRTEX_REFERENCE_ROOT=/path/to/virtex python scripts/make_voc07_golden.py
"""
import ast
import logging
import multiprocessing as mp
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402
from tests import voc07_oracle as V  # noqa: E402


def reference_function():
    import sklearn
    from sklearn.metrics import average_precision_score
    from sklearn.model_selection import cross_val_score
    from sklearn.svm import LinearSVC
    path = os.path.join(ref_shim.REFERENCE_ROOT, "scripts", "clf_voc07.py")
    tree = ast.parse(open(path).read(), path)
    fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "train_test_single_svm")
    ns = {"np": np, "LinearSVC": LinearSVC, "cross_val_score": cross_val_score,
          "average_precision_score": average_precision_score, "logger": logging.getLogger("clf_voc07")}
    exec(compile(ast.Module([fn], []), path, "exec"), ns)
    return ns["train_test_single_svm"], sklearn.__version__


def _sklearn_detail(args):
    """The CV APs and best cost that train_test_single_svm computes internally (it returns the test AP only)."""
    from sklearn.model_selection import cross_val_score
    from sklearn.svm import LinearSVC
    xtr, ytr = args
    y = np.where(ytr == 0, -1, ytr)
    cv = []
    for cost in V.SVM_COSTS:
        clf = LinearSVC(C=cost, class_weight={1: 2, -1: 1}, penalty="l2", loss="squared_hinge", max_iter=2000)
        cv.append(cross_val_score(clf, xtr, y, cv=3, scoring="average_precision"))
    return np.asarray(cv)


def _run_ref(args):
    fn, _ = reference_function()
    return fn(args)


def main():
    if not ref_shim.available():
        raise SystemExit("reference tree not found: set VIRTEX_REFERENCE_ROOT to a checkout of the reference")
    xtr, ttr, xte, tte = V.synthetic_voc07()
    K = ttr.shape[1]
    _, version = reference_function()
    t0 = time.time()
    with mp.Pool() as pool:
        ref_test_ap = pool.map(_run_ref, [(xtr, ttr[:, k], xte, tte[:, k], str(k)) for k in range(K)])
        ref_cv = pool.map(_sklearn_detail, [(xtr, ttr[:, k]) for k in range(K)])
    print(f"reference (sklearn {version}): mAP {np.mean(ref_test_ap):.6f} in {time.time() - t0:.1f} s", flush=True)
    ref_cv = np.stack(ref_cv)                                           # [K, costs, folds]
    ref_best = np.zeros(K, int)
    for k in range(K):
        b = 0.0
        for ci in range(len(V.SVM_COSTS)):
            if ref_cv[k, ci].mean() > b:
                b, ref_best[k] = ref_cv[k, ci].mean(), ci

    y, fold, cy = V.problems(ttr)
    xa = V.augment(xtr)
    t0 = time.time()
    W, steps = V.newton_cg(xa, cy)
    f_opt = V.objective(xa, cy, W)
    cv, te, best, test_ap = V.evaluate(W, xtr, ttr, xte, tte)
    print(f"oracle: mAP {test_ap.mean():.6f}, Newton steps {steps.min()}..{steps.max()}, {time.time() - t0:.1f} s; "
          f"best costs {sorted(set(np.asarray(V.SVM_COSTS)[best].tolist()))}; reference best costs "
          f"{sorted(set(np.asarray(V.SVM_COSTS)[ref_best].tolist()))}", flush=True)
    assert len(set(best.tolist())) >= 2, "the synthetic classes must not all select the same cost"
    out = {
        "sklearn_version": version,
        "features_sha256": V.feature_digest(xtr, xte),
        "fold_ids": torch.from_numpy(fold.astype(np.int8)),
        "ref_cv_ap": torch.from_numpy(ref_cv),
        "ref_test_ap": torch.tensor(ref_test_ap, dtype=torch.float64),
        "ref_best_cost": torch.tensor(np.asarray(V.SVM_COSTS)[ref_best]),
        "ref_mean_ap": float(np.mean(ref_test_ap)),
        "oracle_objective": torch.from_numpy(f_opt),
        "oracle_cv_ap": torch.from_numpy(cv),
        "oracle_test_ap_all": torch.from_numpy(te),
        "oracle_best_cost": torch.tensor(np.asarray(V.SVM_COSTS)[best]),
        "oracle_test_ap": torch.from_numpy(test_ap),
        "oracle_mean_ap": float(test_ap.mean()),
        "oracle_newton_steps": torch.from_numpy(steps),
    }
    torch.save(out, os.path.join(ROOT, "tests", "golden", V.GOLDEN))


if __name__ == "__main__":
    main()
