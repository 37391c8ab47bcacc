#!/usr/bin/env python
"""Times single `ops.gemm` launches of the step's biased linear layers against the same GEMM with other epilogues.

    python scripts/bench_gemm_epilogues.py [--seconds 0.5] [--tile-n 0]

Every shape runs in three variants on the same operands (A [M, K] and B [N, K], both K-major) and with the same tile
width: with `bias=` (bf16 output), without it (plain bf16 output) and with an fp32 output.  Each case starts after
`--gap` seconds of idle GPU, is warmed up and then launched back to back for at least `--seconds`, timed with CUDA
events.  The idle gap matters on a power-capped card: a case that follows a power-hungry one starts at lower clocks, so
without it a faster kernel in one case makes the next case look slower.  One JSON line per case, preceded by one line
naming the GPU and its power limit.
"""
import argparse
import json
import math
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import gpu_identity  # noqa: E402
from virtex_b200 import ops  # noqa: E402

# (M, N, K, layer) at batch 256, caption length 30, hidden 1024: M = 7680 caption tokens, 12544 = 256 x 7 x 7 image
# positions
SHAPES = [
    (7680, 10000, 1024, "vocabulary projection"),
    (7680, 4096, 1024, "linear1"),
    (7680, 1024, 1024, "q, self/cross out-proj"),
    (7680, 3072, 1024, "self-attn qkv"),
    (7680, 1024, 4096, "linear2"),
    (12544, 2048, 1024, "cross-attn k/v of the memory"),
    (12544, 1024, 2048, "visual projection"),
]


def time_launches(fn, seconds):
    """Milliseconds per launch of fn over a window of at least `seconds` (after a warm-up)."""
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        fn()
    e1.record()
    e1.synchronize()
    n = max(20, math.ceil(seconds * 1e3 / (e0.elapsed_time(e1) / 5)))
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=0.5, help="least timed window per case")
    ap.add_argument("--gap", type=float, default=1.0, help="idle seconds before each case")
    ap.add_argument("--tile-n", type=int, default=0, help="tile width of every launch (0: the host's heuristic)")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gemm_epilogues.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    print(json.dumps({"gpu": gpu_identity(0)}), flush=True)
    g = torch.Generator().manual_seed(0)
    for M, N, K, layer in SHAPES:
        A = (torch.randn(M, K, generator=g) * 0.5).bfloat16().to(dev)
        B = (torch.randn(N, K, generator=g) * 0.05).bfloat16().to(dev)
        bias = torch.randn(N, generator=g).to(dev)
        D = torch.empty(M, N, dtype=torch.bfloat16, device=dev)
        D32 = torch.empty(M, N, dtype=torch.float32, device=dev)
        variants = {
            "bias": lambda: ops.gemm(A, B, D, M, N, K, bias=bias, tile_n=args.tile_n),
            "plain": lambda: ops.gemm(A, B, D, M, N, K, tile_n=args.tile_n),
            "f32": lambda: ops.gemm(A, B, D32, M, N, K, out_f32=True, tile_n=args.tile_n),
        }
        for name, fn in variants.items():
            torch.cuda.synchronize()
            time.sleep(args.gap)
            ms, n = time_launches(fn, args.seconds)
            print(json.dumps({"M": M, "N": N, "K": K, "layer": layer, "epilogue": name, "tile_n": args.tile_n,
                              "launches": n, "us": round(ms * 1e3, 2),
                              "tflops": round(2.0 * M * N * K / (ms * 1e-3) / 1e12, 1)}), flush=True)
        del A, B, bias, D, D32
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
