#!/usr/bin/env python
"""Times the reference's five task ablations (virtex_b200/configs/task_ablations/) on pipeline-built batches.

    python scripts/bench_task_ablations.py [--batch 256] [--steps 20] [--warmup 5]

Prints one JSON line each for:
  * the GPU's name and power limit, read in the same run;
  * `Trainer.step` of every config at `--batch`, on a batch built by GpuInputPipeline.from_config (256 x 256 uint8
    images with random-resized-crop parameters, ragged captions or category lists), timed with CUDA events over
    `--steps` steps after `--warmup` steps; two rounds, the configs alternating within each, and the peak memory;
  * the masked-LM collate kernel (vtx_collate_masked_lm) for 256 captions, CUDA events over 1000 launches, beside the
    host restatement of the reference's per-sample Python masking (MaskedLmDataset.__getitem__'s masking lines) for
    the same 256 captions.
Measurement infrastructure only -- nothing in `virtex_b200/` imports this.
"""
import argparse
import json
import os
import random
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import gpu_identity  # noqa: E402
from tests import masked_lm_oracle as MO  # noqa: E402

CONFIGS = ("bicaptioning_R_50_L1_H2048", "captioning_R_50_L1_H2048", "masked_lm_R_50_L1_H2048",
           "token_classification_R_50", "multilabel_classification_R_50")


def captions(B, g):
    return [[MO.SOS] + [int(x) for x in g.integers(4, 10000, int(g.integers(6, 40)))] + [MO.EOS] for _ in range(B)]


def make_batch(pipe, B, seed=0):
    g = np.random.default_rng(seed)
    images = [g.integers(0, 256, (256, 256, 3), dtype=np.uint8) for _ in range(B)]
    params = [pipe.sample_train_params(g, 256, 256) for _ in range(B)]
    if pipe.task == "multilabel_classification":
        lists = [[int(x) for x in g.choice(np.arange(1, 81), int(g.integers(1, 12)), replace=False)] for _ in range(B)]
    else:
        lists = captions(B, g)
    return pipe(images, params, lists)


def time_steps(step, steps, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def run_config(name, B, steps, warmup, dev):
    from virtex_b200.config import Config
    from virtex_b200.data_gpu import GpuInputPipeline
    from virtex_b200.factories import PretrainingModelFactory
    from virtex_b200.trainer import Trainer
    cfg = Config(f"task_ablations/{name}.yaml")
    torch.manual_seed(0)
    model = PretrainingModelFactory.from_config(cfg).to(dev).train()
    trainer = Trainer(model, cfg)
    batch = make_batch(GpuInputPipeline.from_config(cfg, dev), B)
    torch.cuda.reset_peak_memory_stats()
    ms = time_steps(lambda: trainer.step(batch), steps, warmup)
    loss = float(trainer.step(batch)[0])
    out = {"config": name, "batch": B, "ms_per_step": round(ms, 2), "images_s": round(B / ms * 1e3, 1),
           "loss": round(loss, 4), "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 1),
           "steps": steps, "warmup": warmup}
    del model, trainer, batch
    torch.cuda.empty_cache()
    return out


def run_masking(dev, B=256, launches=1000):
    from virtex_b200 import ops
    g = np.random.default_rng(5)
    lists = captions(B, g)
    offs = np.zeros(B + 1, np.int64)
    offs[1:] = np.cumsum([len(t) for t in lists])
    flat = torch.tensor([x for t in lists for x in t], dtype=torch.int64, device=dev)
    offs_d = torch.from_numpy(offs).to(dev)
    T = MO.MAX_LEN
    cap = torch.empty(B, T, dtype=torch.int64, device=dev)
    lab, lens = torch.empty_like(cap), torch.empty(B, dtype=torch.int64, device=dev)
    seed = torch.tensor([7], dtype=torch.int64, device=dev)

    def launch():
        ops.call("vtx_collate_masked_lm", flat.data_ptr(), offs_d.data_ptr(), cap.data_ptr(), lab.data_ptr(),
                 lens.data_ptr(), B, T, MO.MAX_LEN, MO.UNK, MO.MASK, MO.VOCAB, 0.15, 0.85, 0.10, seed.data_ptr(),
                 ops._stream())

    us = time_steps(launch, launches, 50) * 1e3
    rng = random.Random(0)
    reps = 20
    t0 = time.perf_counter()
    for _ in range(reps):
        for t in lists:
            MO.reference_item(t[1:-1], rng)
    host_us = (time.perf_counter() - t0) / reps * 1e6
    return {"captions": B, "kernel_us_per_launch": round(us, 2), "launches": launches,
            "host_python_masking_us": round(host_us, 1), "host_reps": reps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print(json.dumps({"gpu": gpu_identity(0)}), flush=True)
    for rnd in range(2):
        for name in CONFIGS:
            print(json.dumps({"round": rnd, "step": run_config(name, a.batch, a.steps, a.warmup, dev)}), flush=True)
    print(json.dumps({"masking": run_masking(dev)}), flush=True)


if __name__ == "__main__":
    main()
