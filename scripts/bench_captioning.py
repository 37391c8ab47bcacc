#!/usr/bin/env python
"""Captioning throughput: the engine's incremental decoder against the eager-PyTorch incumbent, by beam search or by
nucleus sampling.

    python scripts/bench_captioning.py --batch 256 --beam 5 --max-steps 30 --heads L1_H1024 L4_H1024 L1_H2048
    python scripts/bench_captioning.py --decoder nucleus_sampling --nucleus-size 0.9

Setting of scripts/eval_captioning.py: batch 256, 224 x 224 images, beam 5 (per-node 2), 30 decoding steps; random-init
weights with the EOS column of `textual.output.bias` at -30 so that both paths run all 30 steps.  Engine: image ->
tokens through `model({"image": x})` (backbone with folded BN, one decoder position per step over the cache).
Incumbent, alternating with the engine in the same process: torchvision resnet50 + scripts/gpu_incumbent.py's `Head`
under bf16 autocast, eval mode, recomputing the whole prefix every step, with the search's rules vectorised (the
repetition penalty as one scatter); for nucleus sampling, the reference's rules (SOS-prefixed prefix, sort + cumsum
nucleus, last-token ban, multinomial draw) on whole batches.  Prints one JSON line per head with the card's name and power limit; decode FLOPs
are counted from the shapes (GEMMs and attention; the backbone separately).  `--profile` adds one torch.profiler run of
the engine per head, reporting the share of the decode span in which no kernel of the run was executing.
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F
import torchvision

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
from gpu_incumbent import Head  # noqa: E402

SOS, EOS, V = 1, 2, 10000
R50_GFLOP = 4.09  # multiply-adds x 2 of a torchvision ResNet-50 to layer4 at 224 x 224, per image


def card():
    q = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name(0)


def decode_flops(B, beam, steps, L, H, Sk=49, Cv=2048, sampler=False):
    """FLOPs of the incremental decode (everything after the backbone), from the shapes."""
    f = 2 * B * Sk * Cv * H + L * 2 * B * Sk * H * 2 * H  # visual projection, cross-attention K|V
    for t in range(steps):
        rows, keys = (B, t + 1) if sampler else (B, 1) if t == 0 else (B * beam, t)
        per_layer = 2 * rows * H * (3 * H + H + H + H + 8 * H) + 4 * rows * H * (keys + Sk)
        f += L * per_layer + 2 * rows * H * V
    return f


def build(L, H, B):
    from virtex_b200.modules import TorchvisionVisualBackbone, TransformerDecoderTextualHead
    torch.manual_seed(0)
    visual = TorchvisionVisualBackbone("resnet50", visual_feature_size=2048)
    textual = TransformerDecoderTextualHead(2048, V, H, L, H // 64, 4 * H, dropout=0.1)
    return visual, textual


class Incumbent:
    def __init__(self, L, H, beam, steps, nucleus_size=None):
        self.cnn = torchvision.models.resnet50(weights=None).cuda().eval()
        self.cnn.fc = torch.nn.Identity()
        self.head = Head(2048, V, H, L, H // 64, 4 * H, 0.1).cuda().eval()
        with torch.no_grad():
            self.head.output.bias[EOS] = -30.0
        self.beam, self.steps, self.nucleus_size = beam, steps, nucleus_size

    @torch.no_grad()
    def __call__(self, image):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            x = image
            for name, layer in self.cnn.named_children():
                x = layer(x)
                if name == "layer4":
                    break
            B, beam, steps = image.shape[0], self.beam, self.steps

            def step(tokens):
                feats = x.repeat_interleave(tokens.shape[0] // B, 0)
                lengths = torch.full((tokens.shape[0],), tokens.shape[1], device=tokens.device)
                return self.head(feats, tokens, lengths)[:, -1].float()

            if self.nucleus_size is not None:
                return self._sample(step, B, image.device)
            lp = F.log_softmax(step(torch.full((B, 1), SOS, device=image.device)), 1)
            scores, tok = lp.topk(beam)
            pred = tok.reshape(B * beam, 1)
            scores = scores.reshape(B * beam)
            rows = torch.arange(B * beam, device=image.device)
            for _ in range(steps - 1):
                last = pred[:, -1]
                if bool((last == EOS).all()):
                    break
                lp = F.log_softmax(step(pred), 1)
                lp[rows, last] = -10000
                ended = last == EOS
                lp[ended] = float("-inf")
                lp[ended, EOS] = 0.0
                v, i = lp.topk(2)
                cand = (v + scores[:, None]).view(B, beam * 2)
                best, sel = cand.topk(beam)
                parent = (torch.arange(B, device=image.device)[:, None] * beam + sel // 2).reshape(-1)
                pred = torch.cat([pred[parent], i.view(B, beam * 2).gather(1, sel).reshape(-1, 1)], 1)
                scores = best.reshape(-1)
            return pred[::beam]

    def _sample(self, step, B, device):
        pred = torch.full((B, 1), SOS, device=device)
        rows = torch.arange(B, device=device)
        for _ in range(self.steps):
            last = pred[:, -1]
            if bool((last == EOS).all()):
                break
            logits = step(pred)
            sorted_logits, sorted_idx = torch.sort(logits, descending=True)
            remove = torch.cumsum(F.softmax(sorted_logits, -1), -1) > self.nucleus_size
            remove[:, 1:] = remove[:, :-1].clone()
            remove[:, 0] = False
            logits[remove.scatter(1, sorted_idx, remove)] = -1e12
            logits[rows, last] = -1e12
            tok = torch.multinomial(F.softmax(logits, -1), 1).view(B)
            tok[last == EOS] = EOS
            pred = torch.cat([pred, tok[:, None]], 1)
        return pred[:, 1:]


def timed(fn, reps):
    out = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1))
    return out


def gap_share(model, image, eng):
    """Share of the decode span (first to last kernel after the backbone) with no kernel executing."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        model({"image": image})
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if e.device_type.name == "CUDA" and e.device_resource_id is not None),
                key=lambda e: e.time_range.start)
    k = [e for e in ev if "attn_decode" in e.name]
    start = k[0].time_range.start if k else ev[0].time_range.start
    span_ev = [e for e in ev if e.time_range.start >= start]
    busy, cur_s, cur_e = 0.0, None, None
    for e in span_ev:
        s, t = e.time_range.start, e.time_range.end
        if cur_e is None or s > cur_e:
            if cur_e is not None:
                busy += cur_e - cur_s
            cur_s, cur_e = s, t
        else:
            cur_e = max(cur_e, t)
    busy += cur_e - cur_s
    span = span_ev[-1].time_range.end - start
    return 1.0 - busy / span, len(span_ev)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--beam", type=int, default=5)
    ap.add_argument("--max-steps", type=int, default=30)
    ap.add_argument("--heads", nargs="+", default=["L1_H1024", "L4_H1024", "L1_H2048"])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--decoder", choices=["beam_search", "nucleus_sampling"], default="beam_search")
    ap.add_argument("--nucleus-size", type=float, default=0.9)
    a = ap.parse_args()
    from virtex_b200.factories import CaptionDecoderFactory
    from virtex_b200.models import ForwardCaptioningModel
    gpu = card()
    B, beam, steps = a.batch, a.beam, a.max_steps
    sampler = a.decoder == "nucleus_sampling"
    if sampler:
        beam = 1
    image = torch.randn(B, 3, 224, 224, generator=torch.Generator().manual_seed(0)).cuda()
    for spec in a.heads:
        L, H = (int(p[1:]) for p in spec.split("_"))
        visual, textual = build(L, H, B)
        if sampler:
            dec = CaptionDecoderFactory.create("nucleus_sampling", eos_index=EOS, max_steps=steps,
                                               nucleus_size=a.nucleus_size)
        else:
            dec = CaptionDecoderFactory.create("beam_search", eos_index=EOS, max_steps=steps, beam_size=beam)
        model = ForwardCaptioningModel(visual, textual, decoder=dec).cuda().eval()
        with torch.no_grad():
            model.textual.output.bias[EOS] = -30.0
        eng = model.engine
        inc = Incumbent(L, H, beam, steps, a.nucleus_size if sampler else None)
        with torch.no_grad():
            out = model({"image": image})["predictions"]
            ref = inc(image)
            assert out.shape == (B, steps) and ref.shape == (B, steps), (out.shape, ref.shape)
            t_eng, t_inc, t_bb = [], [], []
            for _ in range(a.reps):  # alternate the two paths
                t_eng += timed(lambda: model({"image": image}), 1)
                t_inc += timed(lambda: inc(image), 1)
                t_bb += timed(lambda: eng.backbone_infer(image), 1)
        ms, ms_inc, ms_bb = min(t_eng), min(t_inc), min(t_bb)
        dec_ms = ms - ms_bb
        fl = decode_flops(B, beam, steps, L, H, sampler=sampler)
        row = {"head": spec, "card": gpu, "decoder": a.decoder, "batch": B, "beam": beam, "steps": steps,
               **({"nucleus_size": a.nucleus_size} if sampler else {}),
               "engine_images_s": round(B / ms * 1e3, 1), "engine_ms": [round(t, 2) for t in t_eng],
               "incumbent_images_s": round(B / ms_inc * 1e3, 1), "incumbent_ms": [round(t, 2) for t in t_inc],
               "speedup": round(ms_inc / ms, 2), "backbone_ms": round(ms_bb, 2), "decode_ms": round(dec_ms, 2),
               "decode_ms_per_step": round(dec_ms / steps, 3), "decode_gflop": round(fl / 1e9, 1),
               "decode_tflop_s": round(fl / dec_ms / 1e9, 1),
               "image_to_tokens_tflop_s": round((fl + B * R50_GFLOP * 1e9) / ms / 1e9, 1)}
        if a.profile:
            with torch.no_grad():
                share, n = gap_share(model, image, eng)
            row.update(decode_gap_share=round(share, 3), decode_kernels=n)
        print(json.dumps(row), flush=True)
        del model, eng, inc
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
