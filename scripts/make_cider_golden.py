"""Write tests/golden/cider.pt: the reference's `cider` on the seeded corpora of tests/cider_oracle.py and on its
literal edge cases.

`virtex/utils/metrics.py` of the unmodified reference ($VIRTEX_REFERENCE_ROOT) is loaded as a module of its own; at
load time it imports only numpy, torch and the standard library, so no Java is needed for `cider`.  Its `np` is then
replaced by a proxy whose `mean` records the list of per-image scores the function averages.  The fixture holds no
seeded corpus: the tests regenerate them from the seed and check their SHA-256.

    VIRTEX_REFERENCE_ROOT=/path/to/virtex python scripts/make_cider_golden.py
"""
import importlib.util
import os
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import ref_shim  # noqa: E402
from tests import cider_oracle as C  # noqa: E402


def reference_module():
    path = os.path.join(ref_shim.REFERENCE_ROOT, "virtex", "utils", "metrics.py")
    spec = importlib.util.spec_from_file_location("reference_metrics", path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    recorded = []

    def mean(a, *args, **kwargs):
        if isinstance(a, list):     # the corpus mean over images; per-image means take a 4-element ndarray
            recorded.append(np.asarray(a, np.float64).copy())
        return np.mean(a, *args, **kwargs)

    proxy = types.SimpleNamespace(**{k: getattr(np, k) for k in ("log", "sqrt", "array", "e")})
    proxy.mean = mean
    mod.np = proxy
    return mod, recorded


def run(mod, recorded, pred, gt, sigma):
    recorded.clear()
    t0 = time.perf_counter()
    score = float(mod.cider(pred, gt, sigma=sigma))
    dt = time.perf_counter() - t0
    assert len(recorded) == 1 and float(np.mean(recorded[0])) == score
    ours = C.cider_details(pred, gt, sigma=sigma)
    err = float(np.abs(ours["img_scores"] - recorded[0]).max())
    print(f"  sigma {sigma:6.2f}: reference {score:.15f} ({dt:.2f} s), oracle {ours['score']:.15f}, "
          f"max per-image |diff| {err:.1e}", flush=True)
    assert err <= 1e-12 and abs(ours["score"] - score) <= 1e-12
    return {"sigma": sigma, "ref_score": score, "ref_img_scores": torch.from_numpy(recorded[0])}


def main():
    if not ref_shim.available():
        raise SystemExit("reference tree not found: set VIRTEX_REFERENCE_ROOT to a checkout of the reference")
    mod, recorded = reference_module()
    seeded = {}
    for name, seed, images in C.CORPORA:
        pred, gt = C.synthetic_corpus(seed, images)
        refs = sum(len(v) for v in gt.values())
        print(f"{name}: {images} images, {refs} references", flush=True)
        sigmas = C.SIGMAS if images <= 1000 else C.SIGMAS[:1]
        seeded[name] = {"seed": seed, "images": images, "sha256": C.corpus_digest(pred, gt),
                        "runs": [run(mod, recorded, pred, gt, s) for s in sigmas]}
    edge = []
    for name, pred, gt, sigma in C.edge_cases():
        print(f"edge case {name}", flush=True)
        edge.append(dict(name=name, predictions=pred, ground_truth=gt, **run(mod, recorded, pred, gt, sigma)))
    torch.save({"seeded": seeded, "edge": edge}, os.path.join(ROOT, "tests", "golden", C.GOLDEN))


if __name__ == "__main__":
    main()
