"""Time the CIDEr metric (virtex_b200.metrics) on the COCO-val2017-shaped seeded corpus of tests/cider_oracle.py:
5000 images, about 27 000 references of about 10.5 words, a Zipf vocabulary of 10 000 words.

- cider: `cider(predictions, ground_truth)` end to end (splitting, interning, copies, kernels, the one read back).
- device: the device part alone from the packed int32 arrays -- copies in, the ground-truth tables, the predictions'
  pass -- between CUDA events.
- evaluate: `CocoCaptionsEvaluator.evaluate` with the ground truth's tables cached (identity tokenizer).
- cpu: the float64 restatement (tests/cider_oracle.py, the reference's dict-of-tuples algorithm) on this host.
Medians of --runs after one warm-up call.  Prints one JSON line with the card's name and power limit.

    python scripts/bench_cider.py [--runs 7]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import cider_oracle as C  # noqa: E402
from virtex_b200 import metrics as M  # noqa: E402


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def _wall(fn, runs):
    fn()
    times = []
    for _ in range(runs):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(times), min(times), max(times)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=7)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    pred, gt = C.synthetic_corpus(2017, 5000)
    refs = sum(len(v) for v in gt.values())

    score = M.cider(pred, gt)
    cider_ms = _wall(lambda: M.cider(pred, gt), args.runs)

    pg = M.PackedGroundTruth(gt)
    pp = M.PackedPredictions(pred, pg)

    def device():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        mean, _, _ = M.CiderTables(pg).score(pp, 6.0)
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1)

    device()
    dev_ms = sorted(device() for _ in range(args.runs))

    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "captions.json")
        with open(path, "w") as f:
            json.dump({"annotations": [{"image_id": k, "caption": c} for k, v in gt.items() for c in v]}, f)
        t0 = time.perf_counter()
        ev = M.CocoCaptionsEvaluator(path, lambda d: {k: list(v) for k, v in d.items()})
        build_ms = (time.perf_counter() - t0) * 1e3
    preds = [{"image_id": k, "caption": v[0]} for k, v in pred.items()]
    eval_ms = _wall(lambda: ev.evaluate(preds), args.runs)
    assert ev.evaluate(preds)["CIDEr"] == 100 * score

    t0 = time.perf_counter()
    cpu_score = C.cider(pred, gt)
    cpu_ms = (time.perf_counter() - t0) * 1e3

    out = {
        "card": _card(), "images": len(gt), "references": refs,
        "cider_ms": round(cider_ms[0], 2), "cider_ms_range": [round(cider_ms[1], 2), round(cider_ms[2], 2)],
        "device_ms": round(statistics.median(dev_ms), 3), "device_ms_range": [round(dev_ms[0], 3), round(dev_ms[-1], 3)],
        "evaluate_ms": round(eval_ms[0], 2), "evaluate_ms_range": [round(eval_ms[1], 2), round(eval_ms[2], 2)],
        "evaluator_init_ms": round(build_ms, 1),
        "cpu_oracle_ms": round(cpu_ms, 1), "score": score, "cpu_score": cpu_score,
        "abs_diff": abs(score - cpu_score), "runs": args.runs,
    }
    print(json.dumps(out))


if __name__ == "__main__":
    main()
