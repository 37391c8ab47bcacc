#!/usr/bin/env python
"""Times the identity bottlenecks' masked-residual 1x1 dgrads, dx = dy1 . W1 + m3 (.) dOut (with and without the
previous block's fused BN-backward sums), on the streaming kernel (csrc/gemm_resid.cu, tile_n = 0) against the
persistent GEMM (tile_n = 256 forces it).

    python scripts/bench_residual_dgrad.py [--seconds 0.5] [--gap 1.0] [--rounds 2]

The shapes are the four ResNet-50 stages at batch 256.  Layer4 (K = 512) takes the persistent kernel either way; it
is listed so that both sides of the selection are on record.  The two routes alternate, every case after
`--gap` seconds of idle GPU (a power-capped card otherwise starts a case at the clocks the previous one left), warmed
up and launched back to back for at least `--seconds`, timed with CUDA events.  Bytes are bench.py's `min_bytes` of
the launch (operands read once, D written once, plus the residual, y and mask reads); the fraction is of the H100 SXM
data-sheet 3.35 TB/s.  One JSON line per case, preceded by one naming the GPU and its power limit.
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import gpu_identity  # noqa: E402
from scripts.bench_gemm_epilogues import time_launches  # noqa: E402
from virtex_b200 import ops  # noqa: E402

# (M, N, K, layer): M = 256 images x the stage's positions, N = the block's output channels, K = its width
SHAPES = [
    (802816, 256, 64, "layer1"),
    (200704, 512, 128, "layer2"),
    (50176, 1024, 256, "layer3"),
    (12544, 2048, 512, "layer4"),
]
HBM_TBS = 3.35


def min_bytes(M, N, K, bnr):
    extra = 2 * M * N + M * N // 8 + ((2 * M * N + M * N // 8) if bnr else 0)
    return 2 * (M * K + N * K) + 2 * M * N + extra


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=0.5, help="least timed window per case")
    ap.add_argument("--gap", type=float, default=1.0, help="idle seconds before each case")
    ap.add_argument("--rounds", type=int, default=2, help="alternations of the two routes per case")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_residual_dgrad.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    print(json.dumps({"gpu": gpu_identity(0)}), flush=True)
    g = torch.Generator().manual_seed(0)
    for M, N, K, layer in SHAPES:
        dy1 = (torch.randn(M, K, generator=g) * 0.5).bfloat16().to(dev)
        w1 = (torch.randn(K, N, generator=g) * 0.1).bfloat16().to(dev)
        dout = torch.randn(M, N, generator=g).bfloat16().to(dev)
        m3 = torch.randint(0, 256, (M, N // 8), generator=g, dtype=torch.uint8).to(dev)
        y = torch.randn(M, N, generator=g).bfloat16().to(dev)
        bnp = torch.stack([torch.zeros(N), torch.ones(N), torch.ones(N), torch.zeros(N)]).contiguous().to(dev)
        mb = torch.randint(0, 256, (M, N // 8), generator=g, dtype=torch.uint8).to(dev)
        sums = torch.zeros(2, N, device=dev)
        D = torch.empty(M, N, dtype=torch.bfloat16, device=dev)
        for bnr in (False, True):
            by = min_bytes(M, N, K, bnr)
            res = {0: [], 256: []}
            for _ in range(args.rounds):
                for tile_n in (0, 256):
                    def fn():
                        ops.gemm(dy1, w1, D, M, N, K, b_mn=1, residual=dout, residual_mask=m3,
                                 bnr=(y, bnp, sums, mb) if bnr else None, tile_n=tile_n)
                    torch.cuda.synchronize()
                    time.sleep(args.gap)
                    ms, _ = time_launches(fn, args.seconds)
                    res[tile_n].append(ms)
            for tile_n, route in ((0, "auto"), (256, "persistent")):
                us = min(res[tile_n]) * 1e3
                print(json.dumps({"layer": layer, "M": M, "N": N, "K": K, "bnr": bnr, "route": route,
                                  "tile_n": tile_n, "us": round(us, 1), "us_all": [round(v * 1e3, 1) for v in res[tile_n]],
                                  "GBps": round(by / (us * 1e-6) / 1e9, 1),
                                  "frac_hbm": round(by / (us * 1e-6) / (HBM_TBS * 1e12), 3)}), flush=True)
        del dy1, w1, dout, m3, y, bnp, mb, sums, D
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
