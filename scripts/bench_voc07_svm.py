"""Time the VOC07 SVM stage (virtex_b200.svm.train_test_svms) at the VOC07 shape: 5011 trainval / 4952 test images,
2048 features, 20 classes, 4 costs x (3 folds + full fit) = 320 LinearSVC problems, on the seeded synthetic features
of tests/voc07_oracle.py.

- GPU: CUDA events around whole calls, each ending in a device synchronise, after a warm-up call; median of --runs.
- GEMMs: one separate profiled call counts every product's FLOPs from its shape and times it with CUDA events.
- CPU: the same 320 fits through sklearn's LinearSVC / cross_val_score / average_precision_score with one process per
  class over all cores (the reference's mp.Pool), when sklearn is importable; otherwise "not measured".
Prints one JSON line.

    python scripts/bench_voc07_svm.py [--runs 5] [--no-cpu]
"""
import argparse
import json
import multiprocessing as mp
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import voc07_oracle as V  # noqa: E402
from virtex_b200 import ops, svm  # noqa: E402


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def _sklearn_class(args):
    """One class of the reference's SVM stage through sklearn: per cost a 3-fold CV AP and a full fit; the first cost
    with the best mean CV AP scores the test set (difficult entries excluded)."""
    from sklearn.metrics import average_precision_score
    from sklearn.model_selection import cross_val_score
    from sklearn.svm import LinearSVC
    xtr, ttr, xte, tte = args
    y = np.where(ttr == 1, 1, -1)
    best, best_clf = 0.0, None
    for cost in svm.SVM_COSTS:
        clf = LinearSVC(C=cost, class_weight={1: 2, -1: 1}, penalty="l2", loss="squared_hinge", max_iter=2000)
        m = cross_val_score(clf, xtr, y, cv=3, scoring="average_precision").mean()
        clf.fit(xtr, y)
        if m > best:
            best, best_clf = m, clf
    keep = tte != -1
    return average_precision_score(tte[keep] == 1, best_clf.decision_function(xte[keep]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    torch.cuda.set_device(0)
    xtr, ttr, xte, tte = V.synthetic_voc07()
    gx, gxt = torch.from_numpy(xtr).cuda(), torch.from_numpy(xte).cuda()

    res = svm.train_test_svms(gx, ttr, gxt, tte)               # warm-up
    times = []
    for _ in range(a.runs):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        res = svm.train_test_svms(gx, ttr, gxt, tte)
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))

    ops.start_gemm_profile()
    svm.train_test_svms(gx, ttr, gxt, tte)
    prof = ops.stop_gemm_profile()
    gemm_ms = sum(p[0] for p in prof)
    gemm_flops = sum(p[1] for p in prof)

    out = {
        "workload": "voc07_svm", "card": _card(), "problems": int(res.weights.shape[0] * res.weights.shape[1]
                                                                  * res.weights.shape[2]),
        "gpu_ms_median": round(statistics.median(times), 2), "gpu_ms_runs": [round(t, 2) for t in times],
        "mean_ap": res.mean_ap, "newton_steps_max": int(res.newton_steps.max()),
        "cg_iterations_max": int(res.cg_iterations.max()),
        "gemms": len(prof), "gemm_tflop": round(gemm_flops / 1e12, 3), "gemm_ms": round(gemm_ms, 2),
        "gemm_tflops_per_s": round(gemm_flops / gemm_ms / 1e9, 1),
        "gemm_share_of_call": round(gemm_ms / statistics.median(times), 3),
    }
    try:
        import sklearn  # noqa: F401
        have_sklearn = True
    except ImportError:
        have_sklearn = False
    if have_sklearn and not a.no_cpu:
        t0 = time.perf_counter()
        with mp.Pool(os.cpu_count()) as pool:
            cpu_ap = pool.map(_sklearn_class, [(xtr, ttr[:, k], xte, tte[:, k]) for k in range(ttr.shape[1])])
        out["cpu_sklearn_s"] = round(time.perf_counter() - t0, 2)
        out["cpu_cores"] = os.cpu_count()
        out["cpu_mean_ap"] = float(np.mean(cpu_ap))
    else:
        out["cpu_sklearn_s"] = "not measured"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
