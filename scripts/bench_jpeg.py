"""JPEG decoding on the GPU: batch 256 of 640x480 quality-90 4:2:0 synthetic JPEGs without restart markers.

Prints the card and its power limit (read in this run), then
  - the device decode time per batch (CUDA events, warmed up, >= 1 s of timed work) and per stage,
  - the histogram of synchronisation rounds,
  - the host header-parse time per image,
  - the bytes per image crossing PCIe, compressed against decoded,
  - end to end: pipe(jpeg_bytes, ...) against cv2.imdecode on the host (1 core and all cores) + pipe(arrays, ...).

    python scripts/bench_jpeg.py [--batch 256] [--seconds 1.0]
"""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.make_jpeg_golden import cv2_jpeg, synth  # noqa: E402
from virtex_b200 import jpeg  # noqa: E402
from virtex_b200.data_gpu import GpuInputPipeline  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unknown"


def timed(fn, seconds):
    fn()
    torch.cuda.synchronize()
    n, t0 = 0, time.perf_counter()
    while time.perf_counter() - t0 < 0.2:  # warm-up
        fn()
        n += 1
    torch.cuda.synchronize()
    per = (time.perf_counter() - t0) / n
    iters = max(3, int(seconds / per))
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    w0 = time.perf_counter()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters, (time.perf_counter() - w0) / iters * 1e3, iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--seconds", type=float, default=1.0)
    ap.add_argument("--distinct", type=int, default=32, help="distinct images, repeated over the batch")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_jpeg.py measures on a CUDA device"
    import cv2
    print("card:", card())
    B = args.batch
    files = [cv2_jpeg(synth(480, 640, 100 + k, noise=12.0), 90, "420") for k in range(args.distinct)]
    bufs = [files[k % len(files)] for k in range(B)]
    res = {"batch": B, "bytes_per_image": float(np.mean([len(b) for b in bufs])),
           "decoded_bytes_per_image": 480 * 640 * 3}
    # host parse
    t0 = time.perf_counter()
    for _ in range(3):
        heads = [jpeg.parse(b) for b in bufs]
    res["host_parse_us_per_image"] = (time.perf_counter() - t0) / (3 * B) * 1e6
    assert all(h.supported for h in heads)
    # device decode
    dec = jpeg.decoder_for("cuda")
    out = jpeg.decode(bufs, "cuda")
    assert out.fallbacks == 0
    ref = cv2.cvtColor(cv2.imdecode(np.frombuffer(bufs[0], np.uint8), cv2.IMREAD_COLOR), cv2.COLOR_BGR2RGB)
    assert np.array_equal(out[0].cpu().numpy(), ref)
    res["rounds_histogram"] = np.bincount(dec.last_rounds).tolist()
    ev_ms, wall_ms, iters = timed(lambda: jpeg.decode(bufs, "cuda"), args.seconds)
    res["decode_batch_ms_events"], res["decode_batch_ms_wall"], res["decode_iters"] = ev_ms, wall_ms, iters
    # per stage (device time between stage boundaries of one call)
    stages = {}
    for _ in range(5):
        dec.stage_events = []
        jpeg.decode(bufs, "cuda")
        torch.cuda.synchronize()
        ev = dec.stage_events
        for (_, a), (name, b) in zip(ev[:-1], ev[1:]):
            stages.setdefault(name, []).append(a.elapsed_time(b))
    dec.stage_events = None
    res["stage_ms"] = {k: float(np.median(v)) for k, v in stages.items()}
    # status read: one D2H of 2B int32 per batch
    st = torch.zeros(2 * B, dtype=torch.int32, device="cuda")
    t0 = time.perf_counter()
    for _ in range(200):
        st.cpu()
    res["status_d2h_us"] = (time.perf_counter() - t0) / 200 * 1e6
    # end to end through the input pipeline
    pipe = GpuInputPipeline("cuda")
    rng = np.random.default_rng(0)
    params = [pipe.sample_train_params(rng, 480, 640) for _ in range(B)]
    toks = [[1, 5, 6, 7, 2]] * B

    def host_decode(b):
        return cv2.cvtColor(cv2.imdecode(np.frombuffer(b, np.uint8), cv2.IMREAD_COLOR), cv2.COLOR_BGR2RGB)

    arrays = [host_decode(b) for b in bufs]
    g1 = pipe(bufs, params, toks)["_image_u8"].clone()
    assert torch.equal(g1, pipe(arrays, params, toks)["_image_u8"])
    res["pipe_jpeg_ms"] = timed(lambda: pipe(bufs, params, toks), args.seconds)[1]
    res["pipe_arrays_only_ms"] = timed(lambda: pipe(arrays, params, toks), args.seconds)[1]
    cv2.setNumThreads(1)
    t0 = time.perf_counter()
    for b in bufs:
        host_decode(b)
    res["cv2_decode_1core_ms"] = (time.perf_counter() - t0) * 1e3
    cores = os.cpu_count() or 1
    with ThreadPoolExecutor(cores) as ex:
        list(ex.map(host_decode, bufs))
        t0 = time.perf_counter()
        list(ex.map(host_decode, bufs))
        res["cv2_decode_allcores_ms"] = (time.perf_counter() - t0) * 1e3
    res["cores"] = cores
    res["cv2_1core_plus_pipe_arrays_ms"] = res["cv2_decode_1core_ms"] + res["pipe_arrays_only_ms"]
    res["cv2_allcores_plus_pipe_arrays_ms"] = res["cv2_decode_allcores_ms"] + res["pipe_arrays_only_ms"]
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
