#!/usr/bin/env python
"""The incumbent on the same GPU: the reference's bicaptioning step as eager PyTorch (cuDNN convs, cuBLASLt linears,
SDPA attention) under bf16 autocast.  Measurement infrastructure only -- nothing in `virtex_b200/` imports this.

The reference itself is not needed, so the model is re-wired here from the library modules the reference
itself instantiates, exactly as it wires them:
  * torchvision `resnet50(zero_init_residual=True)` with `fc = Identity`, children run up to `layer4`
    (virtex/modules/visual_backbones.py:43-74);
  * `nn.Linear` visual projection, word+position embedding -> LayerNorm(eps 1e-8) -> dropout -> pad mask
    (virtex/modules/embedding.py:25-74), `nn.TransformerDecoder(nn.TransformerDecoderLayer(H, A, F, dropout, "gelu",
    batch_first=True, norm_first))`, tied output `nn.Linear` (virtex/modules/textual_heads.py:146-278);
  * two directions sharing visual projection / embedding / output (virtex/models/captioning.py:57-63), CE with
    ignore_index 0 on logits[:, :-1] vs tokens[:, 1:], summed (captioning.py:99-143);
  * loop body of scripts/pretrain_virtex.py:145-163: zero_grad -> autocast forward -> backward -> clip_grad_norm_(10)
    -> SGD(momentum 0.9, wd 1e-4, two lr groups) step.  bf16 autocast needs no GradScaler; Lookahead (a parameter
    interpolation every 5th step) and the LR scheduler are omitted, which only favours the incumbent.

Prints ONE JSON line: {"incumbent": {"variant", "pairs_s", "ms_per_step", ...}}.
"""
import argparse
import copy
import json

import torch
import torchvision
from torch import nn


class Embedding(nn.Module):
    def __init__(self, vocab, hidden, dropout, max_len=30):
        super().__init__()
        self.words = nn.Embedding(vocab, hidden, padding_idx=0)
        self.positions = nn.Embedding(max_len, hidden)
        self.layer_norm = nn.LayerNorm(hidden, eps=1e-8)
        self.dropout = nn.Dropout(dropout)

    def forward(self, tokens):
        pos = torch.arange(tokens.size(1), device=tokens.device).unsqueeze(0).expand_as(tokens)
        x = self.dropout(self.layer_norm(self.words(tokens) + self.positions(pos)))
        return x * (tokens != 0).unsqueeze(-1).type(x.dtype)


class Head(nn.Module):
    def __init__(self, vis, vocab, hidden, layers, heads, ffn, dropout, norm_first=False):
        super().__init__()
        self.visual_projection = nn.Linear(vis, hidden)
        self.embedding = Embedding(vocab, hidden, dropout)
        self.transformer = nn.TransformerDecoder(
            nn.TransformerDecoderLayer(hidden, heads, dim_feedforward=ffn, dropout=dropout, activation="gelu",
                                       batch_first=True, norm_first=norm_first),
            num_layers=layers, norm=nn.LayerNorm(hidden) if norm_first else None)
        self.apply(self._init_weights)  # textual_heads.py:205-216 (BERT-style N(0, 0.02))
        self.output = nn.Linear(hidden, vocab)
        self.output.weight = self.embedding.words.weight

    @staticmethod
    def _init_weights(m):
        if isinstance(m, nn.Linear):
            m.weight.data.normal_(0.0, 0.02)
        elif isinstance(m, nn.MultiheadAttention):
            m.in_proj_weight.data.normal_(0.0, 0.02)
            m.out_proj.weight.data.normal_(0.0, 0.02)
        elif isinstance(m, nn.Embedding):
            m.weight.data.normal_(0.0, 0.02)
            if m.padding_idx is not None:
                m.weight.data[m.padding_idx].zero_()

    def forward(self, feats, tokens, lengths):
        b, c = feats.shape[:2]
        mem = self.visual_projection(feats.reshape(b, c, -1).permute(0, 2, 1))
        t = tokens.size(1)
        pad = lengths.unsqueeze(1) < torch.ones_like(tokens).cumsum(dim=1)
        x = self.embedding(tokens)
        future = torch.triu(torch.full((t, t), float("-inf"), dtype=x.dtype, device=x.device), diagonal=1)
        return self.output(self.transformer(x, mem, tgt_mask=future, tgt_key_padding_mask=pad))


class Bicaptioning(nn.Module):
    def __init__(self, arch="resnet50", vocab=10000, hidden=1024, layers=1, heads=16, ffn=4096, dropout=0.1):
        super().__init__()
        self.cnn = getattr(torchvision.models, arch)(weights=None, zero_init_residual=True)
        width = self.cnn.fc.in_features  # layer4's channels: 512 for resnet18/34, 2048 for the bottleneck ResNets
        self.cnn.fc = nn.Identity()
        self.textual = Head(width, vocab, hidden, layers, heads, ffn, dropout)
        self.backward_textual = copy.deepcopy(self.textual)
        self.backward_textual.visual_projection = self.textual.visual_projection
        self.backward_textual.embedding = self.textual.embedding
        self.backward_textual.output = self.textual.output
        self.loss = nn.CrossEntropyLoss(ignore_index=0)
        self.vocab = vocab

    def forward(self, batch):
        x = batch["image"]
        for name, layer in self.cnn.named_children():
            x = layer(x)
            if name == "layer4":
                break
        lf = self.textual(x, batch["caption_tokens"], batch["caption_lengths"])
        lb = self.backward_textual(x, batch["noitpac_tokens"], batch["caption_lengths"])
        loss = self.loss(lf[:, :-1].contiguous().view(-1, self.vocab), batch["caption_tokens"][:, 1:].contiguous().view(-1))
        return loss + self.loss(lb[:, :-1].contiguous().view(-1, self.vocab),
                                batch["noitpac_tokens"][:, 1:].contiguous().view(-1))


def run(variant, arch, hidden, layers, heads, ffn, B, steps, warmup):
    dev = torch.device("cuda", 0)
    torch.backends.cudnn.benchmark = True
    torch.manual_seed(0)
    model = Bicaptioning(arch, hidden=hidden, layers=layers, heads=heads, ffn=ffn).to(dev).train()
    if variant == "channels_last":
        model = model.to(memory_format=torch.channels_last)
    cnn = [p for n, p in model.named_parameters() if n.startswith("cnn.")]
    rest = [p for n, p in model.named_parameters() if not n.startswith("cnn.")]
    opt = torch.optim.SGD([{"params": cnn, "lr": 0.2}, {"params": rest, "lr": 0.001}], momentum=0.9,
                          weight_decay=1e-4)
    g = torch.Generator().manual_seed(0)
    image = torch.randn(B, 3, 224, 224, generator=g).to(dev)
    if variant == "channels_last":
        image = image.contiguous(memory_format=torch.channels_last)
    tokens = torch.randint(4, 10000, (B, 30), generator=g)
    tokens[:, 0], tokens[:, -1] = 1, 2
    batch = {"image": image, "caption_tokens": tokens.to(dev), "noitpac_tokens": tokens.flip(1).contiguous().to(dev),
             "caption_lengths": torch.full((B,), 30, dtype=torch.int64, device=dev)}

    def step():
        opt.zero_grad()
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = model(batch)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(model.parameters(), 10.0)
        opt.step()
        return loss

    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        loss = step()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    return {"variant": f"eager torch {torch.__version__} + torchvision {torchvision.__version__}, bf16 autocast, "
                       f"cudnn.benchmark, {variant}", "pairs_s": round(B / ms * 1e3, 1), "ms_per_step": round(ms, 3),
            "batch": B, "steps": steps, "warmup": warmup, "loss": round(float(loss), 4),
            "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2**30, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--variant", default="channels_last", choices=["channels_last", "nchw"])
    ap.add_argument("--arch", default="resnet50")
    ap.add_argument("--hidden", type=int, default=1024)
    ap.add_argument("--layers", type=int, default=1)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=4)
    a = ap.parse_args()
    out = run(a.variant, a.arch, a.hidden, a.layers, a.hidden // 64, 4 * a.hidden, a.batch, a.steps, a.warmup)
    print(json.dumps({"incumbent": out}), flush=True)


if __name__ == "__main__":
    main()
