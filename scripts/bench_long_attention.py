#!/usr/bin/env python
"""Times attention past 32 queries and 64 keys: the long kernels behind vtx_attn_fwd / _bwd, and training steps at the
crops and caption lengths that reach them.

    python scripts/bench_long_attention.py [--steps 20] [--warmup 5] [--launches 50]

Prints one JSON line each for:
  * the GPU's name and power limit, read in the same run;
  * every kernel shape at B = 256 images and A = 16 heads (R50-L1-H1024): vtx_attn_fwd and vtx_attn_fwd + _bwd beside
    torch's F.scaled_dot_product_attention (bf16, the same boolean mask, forward and forward + autograd backward), CUDA
    events over `--launches` launches after a warm-up, and the bytes each kernel must move at least (q, k, v, o and the
    fp32 LSE forward; q, k, v, dO, LSE, dq, dk, dv backward), computed from the shapes;
  * `Trainer.step` of R50-L1-H1024 (the base config) at batch 256, crops 224 / 320 / 384 and MAX_CAPTION_LENGTH 30 / 64,
    on batches built by GpuInputPipeline.from_config, timed with CUDA events over `--steps` steps after `--warmup`,
    with the peak memory.
Measurement infrastructure only -- nothing in `virtex_b200/` imports this.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import gpu_identity  # noqa: E402

B, A = 256, 16
# (Tq, Tk, mask mode): cross-attention over 9x9 / 12x12 / 20x20 grids (crops 288 / 384 / 640) from 30 tokens, causal
# self-attention of 64- and 128-token captions, masked-LM (key padding only) self-attention of 64 tokens
SHAPES = ((30, 81, 0), (30, 144, 0), (30, 400, 0), (64, 64, 1), (128, 128, 1), (64, 64, 2))


def time_ms(fn, n, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def run_kernel(Tq, Tk, mode, launches, dev):
    from virtex_b200 import ops
    H = A * 64
    g = torch.Generator(device=dev).manual_seed(Tq + Tk + mode)
    q = torch.randn(B * Tq, H, device=dev, generator=g).to(torch.bfloat16)
    k = torch.randn(B * Tk, H, device=dev, generator=g).to(torch.bfloat16)
    v = torch.randn(B * Tk, H, device=dev, generator=g).to(torch.bfloat16)
    do = torch.randn(B * Tq, H, device=dev, generator=g).to(torch.bfloat16)
    lengths = torch.randint(max(1, Tq // 2), Tq + 1, (B,), device=dev, generator=g)
    o, dq = torch.empty_like(q), torch.empty_like(q)
    dk, dv = torch.empty_like(k), torch.empty_like(v)
    lse = torch.empty(B * A * (-(-Tq // 32) * 32), device=dev)
    seed = torch.tensor([3], dtype=torch.int64, device=dev)
    lp = lengths.data_ptr() if mode else 0
    s = ops._stream()

    def fwd():
        ops.call("vtx_attn_fwd", q.data_ptr(), H, k.data_ptr(), H, v.data_ptr(), H, o.data_ptr(), H, lse.data_ptr(), B,
                 A, Tq, Tk, lp, mode, 0.1, seed.data_ptr(), 11, s)

    def bwd():
        ops.call("vtx_attn_bwd", q.data_ptr(), H, k.data_ptr(), H, v.data_ptr(), H, do.data_ptr(), H, lse.data_ptr(),
                 dq.data_ptr(), H, dk.data_ptr(), H, dv.data_ptr(), H, B, A, Tq, Tk, lp, mode, 0.1, seed.data_ptr(), 11,
                 s)

    # SDPA on [B, A, T, 64] views of the same tensors, mask True = attend
    i = torch.arange(Tq, device=dev)[:, None]
    j = torch.arange(Tk, device=dev)[None, :]
    if mode == 0:
        mask = torch.ones(B, 1, Tq, Tk, dtype=torch.bool, device=dev)
    else:
        mask = (j[None] < lengths.view(B, 1, 1))
        if mode == 1:
            mask = mask & (j <= i)[None]
        mask = mask[:, None]
    qh, kh, vh, doh = (t.view(B, -1, A, 64).transpose(1, 2) for t in (q, k, v, do))
    qg, kg, vg = (t.detach().clone().requires_grad_(True) for t in (qh, kh, vh))

    def sdpa_fwd():
        return F.scaled_dot_product_attention(qh, kh, vh, attn_mask=mask, dropout_p=0.1)

    def sdpa_fwd_bwd():
        out = F.scaled_dot_product_attention(qg, kg, vg, attn_mask=mask, dropout_p=0.1)
        torch.autograd.grad(out, (qg, kg, vg), doh)

    fwd_bytes = 2 * (2 * B * Tq * H + 2 * B * Tk * H) + 4 * B * A * Tq
    bwd_bytes = 2 * (2 * B * Tq * H + 2 * B * Tk * H) + 4 * B * A * Tq + 2 * (B * Tq * H + 2 * B * Tk * H)
    t_fwd = time_ms(fwd, launches)
    t_fb = time_ms(lambda: (fwd(), bwd()), launches)
    t_sf = time_ms(sdpa_fwd, launches)
    t_sfb = time_ms(sdpa_fwd_bwd, launches)
    out = {"Tq": Tq, "Tk": Tk, "mask": mode, "B": B, "heads": A, "p": 0.1,
           "vtx_fwd_us": round(t_fwd * 1e3, 1), "vtx_fwd_bwd_us": round(t_fb * 1e3, 1),
           "sdpa_fwd_us": round(t_sf * 1e3, 1), "sdpa_fwd_bwd_us": round(t_sfb * 1e3, 1),
           "fwd_min_bytes": fwd_bytes, "fwd_bwd_min_bytes": fwd_bytes + bwd_bytes,
           "vtx_fwd_GBps": round(fwd_bytes / t_fwd / 1e6, 1),
           "vtx_fwd_bwd_GBps": round((fwd_bytes + bwd_bytes) / t_fb / 1e6, 1), "launches": launches}
    return out


def run_step(crop, max_len, steps, warmup, dev):
    from virtex_b200.config import Config
    from virtex_b200.data_gpu import GpuInputPipeline
    from virtex_b200.factories import PretrainingModelFactory
    from virtex_b200.trainer import Trainer
    cfg = Config(None, ["DATA.IMAGE_CROP_SIZE", crop, "DATA.MAX_CAPTION_LENGTH", max_len])
    torch.manual_seed(0)
    model = PretrainingModelFactory.from_config(cfg).to(dev).train()
    trainer = Trainer(model, cfg)
    pipe = GpuInputPipeline.from_config(cfg, dev)
    g = np.random.default_rng(0)
    side = crop + crop // 8
    images = [g.integers(0, 256, (side, side, 3), dtype=np.uint8) for _ in range(B)]
    params = [pipe.sample_train_params(g, side, side) for _ in range(B)]
    # caption lengths spread up to the maximum, so that T (the batch's longest) is max_len
    lists = [[1] + [int(x) for x in g.integers(4, 10000, int(g.integers(4, max_len - 1)))] + [2] for _ in range(B)]
    lists[0] = [1] + [5] * (max_len - 2) + [2]
    batch = pipe(images, params, lists)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    ms = time_ms(lambda: trainer.step(batch), steps, warmup)
    loss = trainer.step(batch).sum().item()
    out = {"crop": crop, "max_caption_length": max_len, "T": int(batch["caption_tokens"].shape[1]),
           "keys": (crop // 32) ** 2, "batch": B, "ms_per_step": round(ms, 2), "images_s": round(B / ms * 1e3, 1),
           "loss": round(loss, 4), "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 1),
           "steps": steps, "warmup": warmup}
    del model, trainer, batch
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--launches", type=int, default=50)
    a = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print(json.dumps({"gpu": gpu_identity(0)}), flush=True)
    for Tq, Tk, mode in SHAPES:
        print(json.dumps({"kernel": run_kernel(Tq, Tk, mode, a.launches, dev)}), flush=True)
    for crop in (224, 320, 384):
        for max_len in (30, 64):
            print(json.dumps({"step": run_step(crop, max_len, a.steps, a.warmup, dev)}), flush=True)


if __name__ == "__main__":
    main()
