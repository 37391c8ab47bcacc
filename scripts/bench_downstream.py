"""Time the downstream classification path on one GPU (scripts/clf_linear.py, scripts/clf_voc07.py):

    python scripts/bench_downstream.py [--arch resnet50] [--batch 256] [--iters 20] [--warmup 5] [--rounds 3]

Eval-mode forward of a torchvision ResNet (`--arch`: resnet18, resnet34, resnet50, resnet101, resnet152,
wide_resnet50_2 or wide_resnet101_2) at 224 x 224, three ways, alternated within one process so that clock and power
drift hit all three alike:
  * infer     -- Engine.backbone_infer (eval BN folded into the GEMM epilogues);
  * forward   -- Engine.backbone_forward(training=False) (raw conv outputs, then a BN + ReLU (+ residual) pass each);
  * eager     -- the same torchvision model, channels_last, bf16 autocast, cuDNN.
Then a full linear-probe iteration (frozen eval-mode backbone, CE, SGD on fc) and a fine-tuning iteration (train mode,
SGD on every parameter) through ResNetParams.forward.  HBM bytes of the two engine schedules are computed from the
layer shapes (activation reads and writes of every GEMM and every elementwise pass; weights excluded), so that the
passes the fold removes show up as bandwidth.  Prints the card's name and power limit, then one JSON line."""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm",
                            "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable ({e})"
    return q


def activation_bytes(cnn, B, H=224):
    """(infer, forward) bytes of activations read + written by the eval forward of `cnn` (a ResNetParams), from the
    shapes of its weights."""
    e = 2  # bf16
    Ho = (H - 1) // 2 + 1
    Hp = (Ho - 1) // 2 + 1
    stem = B * Ho * Ho * 64 * e
    infer = fwd = stem + 2 * stem + B * Hp * Hp * 64 * e  # GEMM write, BN+ReLU+maxpool read, pool write (both)
    Hc, Cin = Hp, 64
    for li in range(1, 5):
        for blk in getattr(cnn, f"layer{li}"):
            stride = blk.stride
            Hn = (Hc - 1) // stride + 1
            ds = blk.downsample is not None
            if not hasattr(blk, "conv3"):  # basic block: conv1 (stride) x -> a1, conv2 a1 (+ shortcut) -> out
                C = blk.conv1.weight.shape[0]
                x, a1, out = B * Hc * Hc * Cin * e, B * Hn * Hn * C * e, B * Hn * Hn * C * e
                infer += (x + a1) + (x + out if ds else 0) + (a1 + out + out)
                fwd += (x + a1) + 2 * a1 + (a1 + out) + (x + out if ds else 0)
                fwd += out + (out if ds else x) + out  # bn2 (+ downsample BN) + residual + ReLU pass
                Hc, Cin = Hn, C
                continue
            width, C4 = blk.conv1.weight.shape[0], blk.conv3.weight.shape[0]
            x, a1, a2, out = B * Hc * Hc * Cin * e, B * Hc * Hc * width * e, B * Hn * Hn * width * e, \
                B * Hn * Hn * C4 * e
            # folded: conv1 x -> a1, conv2 a1 -> a2, [downsample x -> shortcut], conv3 a2 + shortcut -> out
            infer += (x + a1) + (a1 + a2) + (x + out if ds else 0) + (a2 + out + out)
            # unfused: every conv writes y and a BN pass reads it back and writes the activation (+ reads the shortcut)
            fwd += (x + a1) + 2 * a1 + (a1 + a2) + 2 * a2 + (a2 + out) + (x + out if ds else 0)
            fwd += out + (out if ds else x) + out  # bn3 (+ downsample BN) + residual + ReLU pass
            Hc, Cin = Hn, C4
    return infer, fwd


def timed(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arch", default="resnet50", help="torchvision ResNet name")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--classes", type=int, default=1000)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_downstream.py measures the GPU path: no CUDA device")
    import torchvision
    from virtex_b200.modules import ResNetParams
    from oracle import virtex_oracle as O
    from tests import downstream_oracle as DO

    print(f"card: {card()}", flush=True)
    torch.manual_seed(0)
    dev = torch.device("cuda")
    width = ResNetParams(a.arch).out_channels
    if a.arch == "resnet50":
        state = DO.synth_state(0, a.classes)
    else:  # the same recipe on the other architecture's parameter tree
        spec = O.Spec(backbone=a.arch, hidden=128, layers=1, heads=2, ffn=256, caption_backward=False)
        full = O.synth_state(spec, 0, bn3_gain=0.25)
        state = {k[len(DO.PREFIX):]: v for k, v in full.items() if k.startswith(DO.PREFIX)}
        g = torch.Generator().manual_seed(7000)
        state["fc.weight"] = torch.randn(a.classes, width, generator=g) * 0.01
        state["fc.bias"] = torch.randn(a.classes, generator=g) * 0.1
    cnn = ResNetParams(a.arch)
    cnn.fc = nn.Linear(width, a.classes)
    cnn.load_state_dict(state, strict=True)
    cnn = cnn.to(dev).eval()
    image = torch.randn(a.batch, 3, 224, 224, device=dev)
    label = torch.randint(0, a.classes, (a.batch,), device=dev)
    with torch.no_grad():
        cnn(image[:2])  # builds the engine
    eng = cnn._vtx_engine
    tv = getattr(torchvision.models, a.arch)(num_classes=a.classes)
    tv.load_state_dict(state, strict=True)
    tv = tv.to(dev).to(memory_format=torch.channels_last).eval()
    image_cl = image.contiguous(memory_format=torch.channels_last)

    def eager():
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
            tv(image_cl)

    ways = {"infer": lambda: eng.backbone_infer(image),
            "forward": lambda: eng.backbone_forward(image, training=False),
            "eager": eager}
    for fn in ways.values():
        for _ in range(a.warmup):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in ways}
    for _ in range(a.rounds):
        for k, fn in ways.items():
            times[k].append(timed(fn, a.iters))
    # same outputs: pooled features of the folded and the unfused engine forward
    f1 = eng.backbone_infer(image)[0].float().view(a.batch, -1, width).mean(1)
    f2 = eng.backbone_forward(image, training=False)[0].float().view(a.batch, -1, width).mean(1)
    pooled_rel = ((f1 - f2).norm() / f2.norm()).item()

    # linear probe: frozen eval-mode backbone, only fc trains
    for n, p in cnn.named_parameters():
        p.requires_grad = n.startswith("fc.")
    opt = torch.optim.SGD([p for p in cnn.parameters() if p.requires_grad], lr=0.3, momentum=0.9)

    def probe():
        opt.zero_grad()
        F.cross_entropy(cnn(image), label).backward()
        opt.step()

    # fine-tuning: train mode, every parameter
    ft = ResNetParams(a.arch)
    ft.fc = nn.Linear(width, a.classes)
    ft.load_state_dict(state, strict=True)
    ft = ft.to(dev).train()
    opt_ft = torch.optim.SGD(ft.parameters(), lr=0.025, momentum=0.9, weight_decay=1e-4)

    def finetune():
        opt_ft.zero_grad()
        F.cross_entropy(ft(image), label).backward()
        opt_ft.step()

    iters = {"probe": probe, "finetune": finetune}
    for fn in iters.values():
        for _ in range(a.warmup):
            fn()
    torch.cuda.synchronize()
    for k, fn in iters.items():
        times[k] = [timed(fn, a.iters) for _ in range(a.rounds)]

    b_inf, b_fwd = activation_bytes(cnn, a.batch)
    best = {k: min(v) for k, v in times.items()}
    res = {"arch": a.arch, "batch": a.batch, "image": 224, "card": card(),
           "ms": {k: [round(x, 3) for x in v] for k, v in times.items()},
           "best_ms": {k: round(v, 3) for k, v in best.items()},
           "activation_bytes": {"infer": b_inf, "forward": b_fwd},
           "activation_GBps": {"infer": round(b_inf / best["infer"] / 1e6, 1),
                               "forward": round(b_fwd / best["forward"] / 1e6, 1)},
           "images_per_s": {k: round(a.batch / best[k] * 1e3, 1) for k in best},
           "pooled_rel_infer_vs_forward": pooled_rel}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
