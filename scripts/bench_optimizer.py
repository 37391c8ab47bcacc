#!/usr/bin/env python
"""Times the fused optimiser tail with SGD against AdamW on the R50-L1-H1024 bicaptioning model (69.5 M parameters).

    python scripts/bench_optimizer.py [--batch 256] [--windows 8] [--steps 20]

Prints one JSON line each for:
  * the GPU's name and power limit, read in the same run;
  * `Trainer.optimizer_step` alone (global-norm clip + step kernel + conv weight re-pack) with SGD and with AdamW;
  * `Trainer.step` at `--batch` with each optimiser;
  * the eager alternative over the same 202 parameter groups: clip_grad_norm_ + Lookahead(torch.optim.AdamW) with
    foreach=True and with fused=True.
Each case runs in `--windows` windows of `--steps` steps (a multiple of the Lookahead k = 5), timed with CUDA events;
the cases of one comparison alternate window by window in this one process, and the median window is reported.
`bytes_est` is what the step kernel must move at least (SGD: p, g, momentum read; p, momentum, bf16 mirror written;
AdamW: p, g, m, v read; p, m, v, bf16 mirror written), `gb_s_est` that divided by the measured time.
Measurement infrastructure only -- nothing in `virtex_b200/` imports this.
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import gpu_identity  # noqa: E402
from oracle import virtex_oracle as O  # noqa: E402

BYTES_PER_ELEMENT = {"sgd": 4 * 3 + 4 * 2 + 2, "adamw": 4 * 4 + 4 * 3 + 2}


def window_ms(fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def alternate(cases, windows, steps):
    """{name: median ms per step} over `windows` alternating windows of every case (one warm-up window each)."""
    for fn in cases.values():
        window_ms(fn, steps)
    times = {name: [] for name in cases}
    for _ in range(windows):
        for name, fn in cases.items():
            times[name].append(window_ms(fn, steps))
    return {name: statistics.median(t) for name, t in times.items()}, times


def build(optimizer, dev):
    from virtex_b200.config import Config
    from virtex_b200.factories import PretrainingModelFactory
    from virtex_b200.trainer import Trainer
    cfg = Config("_base_bicaptioning_R_50_L1_H1024.yaml", ["MODEL.TEXTUAL.DROPOUT", 0.0,
                                                           "OPTIM.OPTIMIZER_NAME", optimizer])
    torch.manual_seed(0)
    model = PretrainingModelFactory.from_config(cfg).to(dev).train()
    return cfg, model, Trainer(model, cfg)


def eager_adamw(cfg, model, dev, **kind):
    """clip_grad_norm_ + Lookahead(AdamW) over copies of the model's 202 parameters, one group each (the reference's
    OptimizerFactory), with gradients set once."""
    from virtex_b200.factories import param_group_hparams
    from virtex_b200.optim import Lookahead
    groups, params = [], []
    g = torch.Generator(device=dev).manual_seed(1)
    for name, p in model.named_parameters():
        q = torch.nn.Parameter(p.detach().clone())
        q.grad = torch.randn(q.shape, device=dev, generator=g) * 1e-3
        params.append(q)
        lr, wd = param_group_hparams(cfg, name)
        groups.append({"params": [q], "lr": lr * 1e-3, "weight_decay": wd})
    opt = Lookahead(torch.optim.AdamW(groups, **kind), k=cfg.OPTIM.LOOKAHEAD.STEPS, alpha=cfg.OPTIM.LOOKAHEAD.ALPHA)

    def step():
        torch.nn.utils.clip_grad_norm_(params, cfg.OPTIM.CLIP_GRAD_NORM)
        opt.step()
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--windows", type=int, default=8)
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    assert a.steps % 5 == 0, "windows must hold whole Lookahead cycles"
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print(json.dumps({"gpu": gpu_identity(0)}), flush=True)
    built = {name: build(name, dev) for name in ("sgd", "adamw")}
    numel = sum(p.numel() for p in built["sgd"][1].parameters())
    for _, _, tr in built.values():
        tr.arena.grads.normal_(0.0, 1e-3)
        tr.iteration = 1000  # past the warm-up: a non-zero learning rate

    cases = {name: tr.optimizer_step for name, (_, _, tr) in built.items()}
    cfg, model, _ = built["adamw"]
    cases["eager_adamw_foreach"] = eager_adamw(cfg, model, dev, foreach=True)
    cases["eager_adamw_fused"] = eager_adamw(cfg, model, dev, fused=True)
    med, times = alternate(cases, a.windows, a.steps)
    for name, ms in med.items():
        line = {"case": "optimizer_step", "impl": name, "ms": round(ms, 4), "params": numel,
                "windows_ms": [round(t, 4) for t in times[name]]}
        kind = "adamw" if "adamw" in name else "sgd"
        line["bytes_est"] = BYTES_PER_ELEMENT[kind] * numel
        line["gb_s_est"] = round(line["bytes_est"] / (ms * 1e-3) / 1e9, 1)
        print(json.dumps(line), flush=True)
    del cases
    torch.cuda.empty_cache()

    batch = {k: v.to(dev) for k, v in O.synth_batch(a.batch, seed=3, ragged=True).items()}
    steps = {name: (lambda tr=tr: tr.step(batch)) for name, (_, _, tr) in built.items()}
    med, times = alternate(steps, max(2, a.windows // 2), 5)
    for name, ms in med.items():
        loss = float(built[name][2].step(batch).sum())
        print(json.dumps({"case": "Trainer.step", "impl": name, "batch": a.batch, "ms": round(ms, 3),
                          "images_s": round(a.batch / ms * 1e3, 1), "loss": round(loss, 4),
                          "windows_ms": [round(t, 3) for t in times[name]],
                          "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2**30, 1)}), flush=True)


if __name__ == "__main__":
    main()
