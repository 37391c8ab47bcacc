#!/usr/bin/env python
"""Times the token-classification pretext step (ResNet-50 + LinearTextualHead, V = 10000, batch 256, bf16).

    python scripts/bench_classification.py [--batch 256] [--steps 50] [--warmup 10]

Prints one JSON line each for:
  * the GPU's name and power limit, read in the same run;
  * `Trainer.step` of TokenClassificationModel, timed with CUDA events over `--steps` steps after `--warmup` steps;
  * the eager PyTorch incumbent of the same step: torchvision resnet50(zero_init_residual=True) run up to layer4 as
    scripts/gpu_incumbent.py runs it, mean pool + nn.Linear, the reference's per-image K-hot loss loop
    (virtex/models/classification.py:74-96), backward, clip_grad_norm_(10) and SGD, under bf16 autocast;
  * a separate torch.profiler run of a few training steps and one eval forward: GPU time of each new kernel.
Measurement infrastructure only -- nothing in `virtex_b200/` imports this.
"""
import argparse
import json
import os
import sys

import torch
import torchvision
from torch import nn
from torch.nn import functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import gpu_identity  # noqa: E402

IGNORE = [0, 1, 2, 3]


def make_batch(B, dev, seed=0):
    g = torch.Generator().manual_seed(seed)
    labels = torch.randint(4, 10000, (B, 30), generator=g)
    lengths = torch.randint(8, 31, (B,), generator=g)
    labels[:, 0] = 1
    labels[torch.arange(B), lengths - 1] = 2
    labels[torch.arange(30)[None, :] >= lengths[:, None]] = 0
    return {"image": torch.randn(B, 3, 224, 224, generator=g).to(dev), "labels": labels.to(dev),
            "caption_tokens": labels.to(dev)}


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


def build_trainer(dev):
    from virtex_b200.config import Config
    from virtex_b200.factories import PretrainingModelFactory
    from virtex_b200.trainer import Trainer
    cfg = Config("_base_bicaptioning_R_50_L1_H1024.yaml",
                 ["MODEL.NAME", "token_classification", "MODEL.TEXTUAL.NAME", "none", "OPTIM.NO_DECAY", "none"])
    torch.manual_seed(0)
    model = PretrainingModelFactory.from_config(cfg).to(dev).train()
    return model, Trainer(model, cfg)


def run_ours(batch, steps, warmup, dev):
    model, trainer = build_trainer(dev)
    ms = time_steps(lambda: trainer.step(batch), steps, warmup)
    loss = float(trainer.step(batch)[0])
    return {"impl": "virtex_b200 Trainer.step", "ms_per_step": round(ms, 3),
            "images_s": round(batch["image"].shape[0] / ms * 1e3, 1), "steps": steps, "warmup": warmup,
            "loss": round(loss, 4), "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2**30, 1)}


class EagerTokenClassification(nn.Module):
    def __init__(self, vocab=10000):
        super().__init__()
        self.cnn = torchvision.models.resnet50(weights=None, zero_init_residual=True)
        self.cnn.fc = nn.Identity()
        self.output = nn.Linear(2048, vocab)

    def forward(self, batch):
        x = batch["image"]
        for name, layer in self.cnn.named_children():
            x = layer(x)
            if name == "layer4":
                break
        logprobs = F.log_softmax(self.output(x.flatten(2).mean(-1)), dim=1)
        loss = 0.0
        for b in range(logprobs.shape[0]):  # the reference's per-image loop over unique, non-ignored labels
            unique = [int(u) for u in batch["labels"][b].unique() if int(u) not in IGNORE]
            loss = loss - logprobs[b, unique].mean()
        return loss / logprobs.shape[0]


def run_incumbent(batch, steps, warmup, dev):
    torch.backends.cudnn.benchmark = True
    torch.manual_seed(0)
    model = EagerTokenClassification().to(dev).to(memory_format=torch.channels_last).train()
    cnn = [p for n, p in model.named_parameters() if n.startswith("cnn.")]
    rest = [p for n, p in model.named_parameters() if not n.startswith("cnn.")]
    opt = torch.optim.SGD([{"params": cnn, "lr": 0.2}, {"params": rest, "lr": 0.001}], momentum=0.9, weight_decay=1e-4)
    b = dict(batch, image=batch["image"].contiguous(memory_format=torch.channels_last))
    out = {}

    def step():
        opt.zero_grad()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = model(b)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(model.parameters(), 10.0)
        opt.step()
        out["loss"] = loss

    ms = time_steps(step, steps, warmup)
    return {"impl": f"eager torch {torch.__version__} + torchvision {torchvision.__version__}, bf16 autocast, "
                    "cudnn.benchmark, channels_last", "ms_per_step": round(ms, 3),
            "images_s": round(batch["image"].shape[0] / ms * 1e3, 1), "steps": steps, "warmup": warmup,
            "loss": round(float(out["loss"]), 4)}


def run_profile(batch, dev, steps=5):
    """GPU time per step of the new kernels (the top-k: per eval forward), from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    model, trainer = build_trainer(dev)
    for _ in range(3):
        trainer.step(batch)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            trainer.step(batch)
        model.eval()
        with torch.no_grad():
            model(batch)
        torch.cuda.synchronize()
    per = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        t = ev.cuda_time_total if t is None else t
        for key in ("group_mean_fwd", "group_mean_bwd", "khot_xent", "topk_rows"):
            if key in ev.key:
                per[key] = per.get(key, 0.0) + t
    runs = {"group_mean_fwd": steps + 1, "group_mean_bwd": steps, "khot_xent": steps + 1, "topk_rows": 1}
    return {"profiler_us_per_launch": {k: round(v / runs[k], 2) for k, v in per.items()}, "profiled_steps": steps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print(json.dumps({"gpu": gpu_identity(0)}), flush=True)
    batch = make_batch(a.batch, dev)
    print(json.dumps({"ours": run_ours(batch, a.steps, a.warmup, dev)}), flush=True)
    torch.cuda.empty_cache()
    print(json.dumps({"incumbent": run_incumbent(batch, a.steps, a.warmup, dev)}), flush=True)
    torch.cuda.empty_cache()
    print(json.dumps({"kernels": run_profile(batch, dev)}), flush=True)


if __name__ == "__main__":
    main()
