"""CPU oracle of the VirTex bicaptioning pretraining step -- TEST INFRASTRUCTURE, NOT PRODUCT.

A plain fp32 restatement (explicit formulas over basic torch CPU ops, gradients by CPU autograd) of the algorithm
the reference executes for `VirTexModel.forward` + backward + optimiser step.  Only `tests/`,
`__graft_entry__.smoke()` and `bench.py`'s CPU-baseline / `--impl reference` legs may import this module; the
product (`virtex_b200/`) never does.

Pinning: the reference ships no tests or golden vectors of its own (SURVEY.md section 8c) and its arithmetic lives
in torch / torchvision.  This restatement is therefore pinned against the *live* reference modules imported from
a reference checkout (`oracle/make_golden.py`), and the resulting fixtures are committed under
`tests/golden/`; `tests/test_oracle_golden.py` re-checks the oracle against them everywhere.

Reference call sites restated (file:line, relative to the reference root unless prefixed SP/ = site-packages):
  * ResNet-v1.5 to layer4          virtex/modules/visual_backbones.py:43-74 -> SP/torchvision/models/resnet.py:108-163,
                                   166-285 (Bottleneck, stride on the 3x3, zero_init_residual; wide: width_per_group
                                   128, :922-985)
  * basic-block ResNet-18 / 34     SP/torchvision/models/resnet.py:59-105 (BasicBlock: conv1 3x3 carries the stride,
                                   conv2 3x3, expansion 1, 512 output channels)
  * BatchNorm2d (train / eval)     SP/torchvision/models/resnet.py:147-155 (SURVEY Appendix C.2)
  * visual projection + embedding  virtex/modules/textual_heads.py:240-259, virtex/modules/embedding.py:46-74
  * post-/pre-norm decoder layer   SP/torch/nn/modules/transformer.py:1131-1199; MHA SP/torch/nn/functional.py:6244-6690
  * masks                          virtex/modules/textual_heads.py:255-256,280-292
  * tied output projection + CE    virtex/modules/textual_heads.py:199-200,277; virtex/models/captioning.py:69,99-143
  * optimiser step                 scripts/pretrain_virtex.py:145-163; virtex/factories.py:509-545;
                                   virtex/optim/lookahead.py:82-102; virtex/optim/lr_scheduler.py:174-183
"""
from __future__ import annotations

import math
import re
from collections import OrderedDict
from dataclasses import dataclass, field, replace
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

_RESNET_LAYERS = {"resnet18": [2, 2, 2, 2], "resnet34": [3, 4, 6, 3], "resnet50": [3, 4, 6, 3],
                  "resnet101": [3, 4, 23, 3], "resnet152": [3, 8, 36, 3], "wide_resnet50_2": [3, 4, 6, 3],
                  "wide_resnet101_2": [3, 4, 23, 3]}
# (block kind, width per group), as torchvision's constructors set them: a basic block is two 3x3 convs of `planes`
# channels; a bottleneck is planes * width_per_group / 64 channels wide inside and 4 * planes at its output.
_RESNET_BLOCK = {"resnet18": ("basic", 64), "resnet34": ("basic", 64), "resnet50": ("bottleneck", 64),
                 "resnet101": ("bottleneck", 64), "resnet152": ("bottleneck", 64),
                 "wide_resnet50_2": ("bottleneck", 128), "wide_resnet101_2": ("bottleneck", 128)}


def _is_basic(spec: "Spec") -> bool:
    return _RESNET_BLOCK[spec.backbone][0] == "basic"


@dataclass
class Spec:
    """Architecture of one bicaptioning model (what the reference's Config + factories resolve to)."""
    backbone: str = "resnet50"
    hidden: int = 1024
    layers: int = 1
    heads: int = 16
    ffn: int = 4096
    norm_first: bool = False
    vocab: int = 10000
    max_len: int = 30
    pad: int = 0
    visual_feature_size: Optional[int] = None  # default: the backbone's output width, 512 (basic blocks) or 2048
    caption_backward: bool = True
    mask_future: bool = True  # False: masked language modelling (virtex/factories.py:395 -> textual_heads.py:255-262)
    blocks: List[int] = field(default_factory=list)

    def __post_init__(self):
        if not self.blocks:
            self.blocks = list(_RESNET_LAYERS[self.backbone])
        if self.visual_feature_size is None:
            self.visual_feature_size = 512 if _is_basic(self) else 2048


# ----------------------------------------------------------------------------------------------- parameter inventory
def backbone_param_shapes(spec: Spec) -> "OrderedDict[str, Tuple[int, ...]]":
    """Names/shapes of `visual.cnn.*` parameters and buffers, in torchvision registration order."""
    kind, width_per_group = _RESNET_BLOCK[spec.backbone]
    basic = kind == "basic"
    k1, expansion = (3, 1) if basic else (1, 4)  # basic: conv1 3x3, conv2 3x3; bottleneck: 1x1, 3x3, 1x1 (conv3)
    out: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()

    def bn(prefix, c):
        out[prefix + ".weight"] = (c,)
        out[prefix + ".bias"] = (c,)
        out[prefix + ".running_mean"] = (c,)
        out[prefix + ".running_var"] = (c,)
        out[prefix + ".num_batches_tracked"] = ()

    p = "visual.cnn."
    out[p + "conv1.weight"] = (64, 3, 7, 7)
    bn(p + "bn1", 64)
    inplanes = 64
    for li, (planes, nblocks) in enumerate(zip([64, 128, 256, 512], spec.blocks), start=1):
        width = planes * width_per_group // 64
        for bi in range(nblocks):
            stride = 2 if (bi == 0 and li > 1) else 1
            q = f"{p}layer{li}.{bi}."
            out[q + "conv1.weight"] = (width, inplanes, k1, k1)
            bn(q + "bn1", width)
            out[q + "conv2.weight"] = (width, width, 3, 3)
            bn(q + "bn2", width)
            if not basic:
                out[q + "conv3.weight"] = (planes * expansion, width, 1, 1)
                bn(q + "bn3", planes * expansion)
            if stride != 1 or inplanes != planes * expansion:
                out[q + "downsample.0.weight"] = (planes * expansion, inplanes, 1, 1)
                bn(q + "downsample.1", planes * expansion)
            inplanes = planes * expansion
    return out


def head_param_shapes(spec: Spec) -> "OrderedDict[str, Tuple[int, ...]]":
    """Unique textual parameters: shared ones under `textual.*`, per-direction transformer under both prefixes."""
    H, Fd, V = spec.hidden, spec.ffn, spec.vocab
    out: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()
    out["textual.visual_projection.weight"] = (H, spec.visual_feature_size)
    out["textual.visual_projection.bias"] = (H,)
    out["textual.embedding.words.weight"] = (V, H)
    out["textual.embedding.positions.weight"] = (spec.max_len, H)
    out["textual.embedding.layer_norm.weight"] = (H,)
    out["textual.embedding.layer_norm.bias"] = (H,)
    dirs = ["textual"] + (["backward_textual"] if spec.caption_backward else [])
    for d in dirs:
        for l in range(spec.layers):
            q = f"{d}.transformer.layers.{l}."
            out[q + "self_attn.in_proj_weight"] = (3 * H, H)
            out[q + "self_attn.in_proj_bias"] = (3 * H,)
            out[q + "self_attn.out_proj.weight"] = (H, H)
            out[q + "self_attn.out_proj.bias"] = (H,)
            out[q + "multihead_attn.in_proj_weight"] = (3 * H, H)
            out[q + "multihead_attn.in_proj_bias"] = (3 * H,)
            out[q + "multihead_attn.out_proj.weight"] = (H, H)
            out[q + "multihead_attn.out_proj.bias"] = (H,)
            out[q + "linear1.weight"] = (Fd, H)
            out[q + "linear1.bias"] = (Fd,)
            out[q + "linear2.weight"] = (H, Fd)
            out[q + "linear2.bias"] = (H,)
            for n in ("norm1", "norm2", "norm3"):
                out[q + n + ".weight"] = (H,)
                out[q + n + ".bias"] = (H,)
        if spec.norm_first:
            out[f"{d}.transformer.norm.weight"] = (H,)
            out[f"{d}.transformer.norm.bias"] = (H,)
        if d == "textual":
            out["textual.output.bias"] = (V,)
    return out


_BUFFER_SUFFIXES = (".running_mean", ".running_var", ".num_batches_tracked")


def is_buffer(name: str) -> bool:
    return name.endswith(_BUFFER_SUFFIXES)


def unique_shapes(spec: Spec) -> "OrderedDict[str, Tuple[int, ...]]":
    out = backbone_param_shapes(spec)
    out.update(head_param_shapes(spec))
    return out


_SHARED_PREFIXES = ("visual_projection.", "embedding.", "output.")


def to_reference_state_dict(state: Dict[str, torch.Tensor], spec: Spec) -> Dict[str, torch.Tensor]:
    """Expand the unique-tensor dict into the reference's `state_dict()` key set (shared modules serialised under
    both `textual.*` and `backward_textual.*`, tied `output.weight`; virtex/models/captioning.py:57-63)."""
    sd = dict(state)
    sd["textual.output.weight"] = state["textual.embedding.words.weight"]
    if spec.caption_backward:
        for k, v in list(sd.items()):
            if k.startswith("textual.") and k[len("textual."):].startswith(_SHARED_PREFIXES):
                sd["backward_" + k] = v
    return sd


def from_reference_state_dict(sd: Dict[str, torch.Tensor], spec: Spec) -> Dict[str, torch.Tensor]:
    return OrderedDict((k, sd[k]) for k in unique_shapes(spec))


def synth_state(spec: Spec, seed: int = 0, randomize_bn: bool = True,
                bn3_gain: float = 1.0) -> "OrderedDict[str, torch.Tensor]":
    """Deterministic synthetic weights, reproducible anywhere from (spec, seed) alone.

    Scales follow the reference initialisers (Kaiming fan_out convs, N(0, 0.02) head weights) but BN affine
    parameters and running statistics are randomised when `randomize_bn` so that every gradient is exercised
    (fresh `zero_init_residual` makes 112 of 202 gradients identically zero; SURVEY section 8c gotcha (i)).
    `bn3_gain` scales the last BN gamma of every residual block (bn3 of a bottleneck, bn2 of a basic block; zero
    without `randomize_bn`, as zero_init_residual): with gain 1 a random 16-block residual stack amplifies any
    perturbation ~1.25x per block (bf16 rounding -> 50% feature error at layer4), which is a property of that random
    network, not of an implementation; bf16-vs-fp32 parity tests therefore use a residual branch gain of ~0.25.

    ResNet-50/101/152 draw every tensor in `unique_shapes` order from one generator seeded `seed`.  The wide and
    basic-block backbones draw theirs in registration order from a generator of their own, seeded 10_000 + seed and
    20_000 + seed, and take the textual tensors that the same head draws on a resnet50 backbone."""
    kind, width_per_group = _RESNET_BLOCK[spec.backbone]
    own_generator = kind == "basic" or width_per_group != 64
    if own_generator:
        g = torch.Generator().manual_seed((20_000 if kind == "basic" else 10_000) + seed)
        shapes = backbone_param_shapes(spec)
    else:
        g = torch.Generator().manual_seed(seed)
        shapes = unique_shapes(spec)
    last_bn = ".bn2." if kind == "basic" else ".bn3."
    out: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    for name, shape in shapes.items():
        if name.endswith("num_batches_tracked"):
            t = torch.zeros((), dtype=torch.int64)
        elif name.endswith("running_mean"):
            t = torch.randn(shape, generator=g) * 0.1 if randomize_bn else torch.zeros(shape)
        elif name.endswith("running_var"):
            t = torch.rand(shape, generator=g) + 0.5 if randomize_bn else torch.ones(shape)
        elif "visual.cnn" in name and name.endswith(".weight") and len(shape) == 4:
            fan_out = shape[0] * shape[2] * shape[3]
            t = torch.randn(shape, generator=g) * math.sqrt(2.0 / fan_out)
        elif "visual.cnn" in name and name.endswith(".weight"):  # BN gamma
            t = torch.rand(shape, generator=g) + 0.5 if randomize_bn else torch.ones(shape)
            if not randomize_bn and last_bn in name:
                t = torch.zeros(shape)
            elif last_bn in name:
                t = t * bn3_gain
        elif "visual.cnn" in name:  # BN beta
            t = torch.randn(shape, generator=g) * 0.1 if randomize_bn else torch.zeros(shape)
        elif re.search(r"(norm\d?|layer_norm)\.weight$", name):
            t = torch.rand(shape, generator=g) * 0.5 + 0.75 if randomize_bn else torch.ones(shape)
        elif re.search(r"(norm\d?|layer_norm)\.bias$", name):
            t = torch.randn(shape, generator=g) * 0.05 if randomize_bn else torch.zeros(shape)
        elif name.endswith("bias"):
            t = torch.randn(shape, generator=g) * 0.02
        else:
            t = torch.randn(shape, generator=g) * 0.02
            if name == "textual.embedding.words.weight":
                t[spec.pad].zero_()
        out[name] = t
    if own_generator:
        head = synth_state(replace(spec, backbone="resnet50", blocks=list(_RESNET_LAYERS["resnet50"])), seed,
                           randomize_bn, bn3_gain)
        out.update((k, v) for k, v in head.items() if not k.startswith("visual."))
    return out


def synth_batch(batch_size: int, seed: int = 0, max_len: int = 30, vocab: int = 10000, ragged: bool = False,
                image_size: int = 224) -> Dict[str, torch.Tensor]:
    """Synthetic batch with the reference's schema (virtex/data/datasets/captioning.py:69-100): `[SOS] ... [EOS]`
    right-padded with 0, `noitpac_tokens` = per-row reversal *before* padding, shared lengths."""
    g = torch.Generator().manual_seed(1000 + seed)
    image = torch.randn(batch_size, 3, image_size, image_size, generator=g)
    if ragged:
        lengths = torch.randint(5, max_len + 1, (batch_size,), generator=g)
        lengths[0] = max_len
    else:
        lengths = torch.full((batch_size,), max_len, dtype=torch.int64)
    tokens = torch.zeros(batch_size, max_len, dtype=torch.int64)
    noitpac = torch.zeros(batch_size, max_len, dtype=torch.int64)
    for b in range(batch_size):
        n = int(lengths[b])
        row = torch.randint(4, vocab, (n,), generator=g)
        row[0], row[-1] = 1, 2
        if ragged and n > 6:  # a few <unk> (= pad id 0) inside the caption: SURVEY section 8c gotcha (iv)
            row[3] = 0
        tokens[b, :n] = row
        noitpac[b, :n] = row.flip(0)
    return {"image_id": torch.arange(batch_size), "image": image, "caption_tokens": tokens,
            "noitpac_tokens": noitpac, "caption_lengths": lengths}


# ------------------------------------------------------------------------------------------------------- forward math
class _RoundBF16(torch.autograd.Function):
    """Round-to-bf16 in forward AND on the gradient in backward: marks where the bf16-autocast reference (and the
    CUDA path) materialise a bf16 tensor.  Used only by the `emulate_bf16` variants below."""

    @staticmethod
    def forward(ctx, x):
        return x.bfloat16().to(x.dtype)

    @staticmethod
    def backward(ctx, g):
        return g.bfloat16().to(g.dtype)


def _rb(x):
    return _RoundBF16.apply(x)


def _batch_norm(x, P, prefix, training, new_buffers, eps=1e-5, momentum=0.1, emulate_bf16=False):
    w, b = P[prefix + ".weight"], P[prefix + ".bias"]
    x_stat = x  # statistics come from the fp32 conv accumulators; the normalised tensor is the bf16-rounded one
    if emulate_bf16:
        x = _rb(x)
    if training:
        n = x.numel() // x.shape[1]
        mean = x_stat.mean(dim=(0, 2, 3))
        var_b = ((x_stat - mean[None, :, None, None]) ** 2).mean(dim=(0, 2, 3))  # biased
        if new_buffers is not None:
            with torch.no_grad():
                new_buffers[prefix + ".running_mean"] = (1 - momentum) * P[prefix + ".running_mean"] + momentum * mean
                new_buffers[prefix + ".running_var"] = ((1 - momentum) * P[prefix + ".running_var"]
                                                        + momentum * var_b * n / max(n - 1, 1))
                new_buffers[prefix + ".num_batches_tracked"] = P[prefix + ".num_batches_tracked"] + 1
    else:
        mean, var_b = P[prefix + ".running_mean"], P[prefix + ".running_var"]
    xhat = (x - mean[None, :, None, None]) * torch.rsqrt(var_b + eps)[None, :, None, None]
    return xhat * w[None, :, None, None] + b[None, :, None, None]


def backbone_forward(P, image, spec: Spec, training=True, new_buffers=None, record=None, emulate_bf16=False):
    """(B,3,H,W) -> (B,C,H/32,W/32), C = 512 for basic blocks and 2048 otherwise.  torchvision ResNet children
    conv1..layer4.  `record` (dict) optionally receives the stem's and every block's intermediates (y1, a1, y2, out)."""
    basic = _is_basic(spec)
    p = "visual.cnn."
    rb = _rb if emulate_bf16 else (lambda t: t)
    bn = lambda t, name: _batch_norm(t, P, name, training, new_buffers, emulate_bf16=emulate_bf16)
    x = F.conv2d(rb(image), rb(P[p + "conv1.weight"]), stride=2, padding=3)
    if record is not None:
        record["stem.y"] = x
    x = rb(torch.relu(bn(x, p + "bn1")))
    x = F.max_pool2d(x, kernel_size=3, stride=2, padding=1)
    if record is not None:
        record["stem.pool"] = x
    for li, nblocks in enumerate(spec.blocks, start=1):
        for bi in range(nblocks):
            stride = 2 if (bi == 0 and li > 1) else 1
            q = f"{p}layer{li}.{bi}."
            identity = x
            # the first 3x3 conv carries the stride: conv1 of a basic block, conv2 of a bottleneck
            out = F.conv2d(x, rb(P[q + "conv1.weight"]), stride=stride if basic else 1, padding=1 if basic else 0)
            if record is not None:
                record[q + "y1"] = out
            out = rb(torch.relu(bn(out, q + "bn1")))
            if record is not None:
                record[q + "a1"] = out
            out = F.conv2d(out, rb(P[q + "conv2.weight"]), stride=1 if basic else stride, padding=1)
            if record is not None:
                record[q + "y2"] = out
            if basic:
                out = bn(out, q + "bn2")
            else:
                out = rb(torch.relu(bn(out, q + "bn2")))
                out = F.conv2d(out, rb(P[q + "conv3.weight"]))
                out = bn(out, q + "bn3")
            if q + "downsample.0.weight" in P:
                identity = F.conv2d(x, rb(P[q + "downsample.0.weight"]), stride=stride)
                identity = bn(identity, q + "downsample.1")
            x = rb(torch.relu(out + identity))
            if record is not None:
                record[q + "out"] = x
    return x


def _layer_norm(x, w, b, eps):
    mu = x.mean(-1, keepdim=True)
    var = ((x - mu) ** 2).mean(-1, keepdim=True)
    return (x - mu) * torch.rsqrt(var + eps) * w + b


def _gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x * (1.0 / math.sqrt(2.0))))


def _mha(P, prefix, x_q, x_kv, heads, bias_mask, self_attn, drop=None, site=0):
    """Packed in-projection multi-head attention; bias_mask broadcastable to (B, heads, Tq, Tk) or None.
    `drop(probs, site)` (optional) is the dropout of the (B, heads, Tq, Tk) attention probabilities."""
    H = x_q.shape[-1]
    W, bvec = P[prefix + ".in_proj_weight"], P[prefix + ".in_proj_bias"]
    if self_attn:
        qkv = x_q @ W.t() + bvec
        q, k, v = qkv.split(H, dim=-1)
    else:
        q = x_q @ W[:H].t() + bvec[:H]
        kv = x_kv @ W[H:].t() + bvec[H:]
        k, v = kv.split(H, dim=-1)
    B, Tq, _ = q.shape
    Tk = k.shape[1]
    d = H // heads
    q = q.view(B, Tq, heads, d).transpose(1, 2)
    k = k.view(B, Tk, heads, d).transpose(1, 2)
    v = v.view(B, Tk, heads, d).transpose(1, 2)
    s = (q @ k.transpose(-1, -2)) * (1.0 / math.sqrt(d))
    if bias_mask is not None:
        s = s + bias_mask
    pr = torch.softmax(s, dim=-1)
    if drop is not None:
        pr = drop(pr, site)
    o = (pr @ v).transpose(1, 2).reshape(B, Tq, H)
    return o @ P[prefix + ".out_proj.weight"].t() + P[prefix + ".out_proj.bias"]


def head_forward(P, visual_features, tokens, lengths, spec: Spec, direction: str = "textual", drop=None):
    """(B,C,h,w), (B,T) int64, (B,) int64 -> logits (B,T,V).  Dropout is the identity (p = 0 / eval) unless `drop` is
    given: `drop(x, site)` is then applied at the reference's 7 dropout points, numbered as the CUDA engine numbers its
    dropout sites (di = 0 for "textual", 1 for "backward_textual"; sb = di * 1000 + 10 * (layer + 1)):
      embedding output after its LayerNorm, before the pad mask     di * 1000    x (B, T, H)
      self- / cross-attention probabilities                         sb + 0 / 2   x (B, heads, Tq, Tk)
      dropout1 / 2 / 3 of the residual branches                     sb + 1 / 3 / 5  x (B, T, H)
      the feed-forward hidden after GELU                            sb + 4       x (B, T, F)"""
    drop_ = drop if drop is not None else (lambda x, site: x)
    di = 0 if direction == "textual" else 1
    B, C, h, w = visual_features.shape
    vf = visual_features.reshape(B, C, h * w).permute(0, 2, 1)
    mem = vf @ P["textual.visual_projection.weight"].t() + P["textual.visual_projection.bias"]
    T = tokens.shape[1]
    # embedding (virtex/modules/embedding.py:58-73)
    emb = P["textual.embedding.words.weight"][tokens] + P["textual.embedding.positions.weight"][:T][None]
    emb = _layer_norm(emb, P["textual.embedding.layer_norm.weight"], P["textual.embedding.layer_norm.bias"], 1e-8)
    emb = drop_(emb, di * 1000)
    emb = emb * (tokens != spec.pad).unsqueeze(-1).to(emb.dtype)
    # masks
    pos = torch.arange(1, T + 1)[None, :]
    kpm = lengths[:, None] < pos  # True = padded key
    bias = torch.zeros(B, 1, T, T, dtype=emb.dtype)
    if spec.mask_future:
        bias = bias.masked_fill(torch.triu(torch.ones(T, T, dtype=torch.bool), diagonal=1)[None, None], float("-inf"))
    bias = bias.masked_fill(kpm[:, None, None, :], float("-inf"))
    x = emb
    for l in range(spec.layers):
        q = f"{direction}.transformer.layers.{l}."
        sb = di * 1000 + 10 * (l + 1)
        n1 = lambda t: _layer_norm(t, P[q + "norm1.weight"], P[q + "norm1.bias"], 1e-5)
        n2 = lambda t: _layer_norm(t, P[q + "norm2.weight"], P[q + "norm2.bias"], 1e-5)
        n3 = lambda t: _layer_norm(t, P[q + "norm3.weight"], P[q + "norm3.bias"], 1e-5)
        ff = lambda t: drop_(_gelu(t @ P[q + "linear1.weight"].t() + P[q + "linear1.bias"]), sb + 4) \
            @ P[q + "linear2.weight"].t() + P[q + "linear2.bias"]
        sa = lambda t: drop_(_mha(P, q + "self_attn", t, t, spec.heads, bias, True, drop, sb + 0), sb + 1)
        ca = lambda t: drop_(_mha(P, q + "multihead_attn", t, mem, spec.heads, None, False, drop, sb + 2), sb + 3)
        if spec.norm_first:
            x = x + sa(n1(x))
            x = x + ca(n2(x))
            x = x + drop_(ff(n3(x)), sb + 5)
        else:
            x = n1(x + sa(x))
            x = n2(x + ca(x))
            x = n3(x + drop_(ff(x), sb + 5))
    if spec.norm_first:
        x = _layer_norm(x, P[f"{direction}.transformer.norm.weight"], P[f"{direction}.transformer.norm.bias"], 1e-5)
    return x @ P["textual.embedding.words.weight"].t() + P["textual.output.bias"]


def caption_loss(logits, tokens, pad=0):
    """CrossEntropyLoss(ignore_index=pad) on logits[:, :-1] vs tokens[:, 1:] (virtex/models/captioning.py:111-114)."""
    V = logits.shape[-1]
    z = logits[:, :-1].reshape(-1, V)
    y = tokens[:, 1:].reshape(-1)
    lse = torch.logsumexp(z, dim=-1)
    picked = z.gather(1, y[:, None]).squeeze(1)
    valid = (y != pad).to(z.dtype)
    return ((lse - picked) * valid).sum() / valid.sum()


def masked_lm_loss(logits, labels, pad=0):
    """CrossEntropyLoss(ignore_index=pad) between every position's logits and its label (virtex/models/masked_lm.py:68-72)."""
    V = logits.shape[-1]
    z, y = logits.reshape(-1, V), labels.reshape(-1)
    lse = torch.logsumexp(z, dim=-1)
    picked = z.gather(1, y[:, None]).squeeze(1)
    valid = (y != pad).to(z.dtype)
    return ((lse - picked) * valid).sum() / valid.sum()


def masked_lm_forward(P, batch, spec: Spec, training=True, new_buffers=None, return_logits=False):
    """virtex/models/masked_lm.py:35-86 (spec.mask_future must be False)."""
    vf = backbone_forward(P, batch["image"], spec, training, new_buffers)
    logits = head_forward(P, vf, batch["caption_tokens"], batch["caption_lengths"], spec, "textual")
    loss = masked_lm_loss(logits, batch["masked_labels"], spec.pad)
    out = {"loss": loss, "loss_components": {"masked_lm": loss.detach().clone()}}
    if not training:
        pred = torch.argmax(logits, dim=-1)
        pred[batch["masked_labels"] == spec.pad] = spec.pad
        out["predictions"] = pred
    if return_logits:
        out["logits"] = logits
    return out


def synth_masked_batch(batch_size: int, seed: int = 0, max_len: int = 30, vocab: int = 10000, mask_index: int = 3,
                       mask_prob: float = 0.3, ragged: bool = True):
    """A captioning batch turned into a masked-LM batch the way virtex/data/datasets/masked_lm.py does in spirit:
    ~mask_prob of the real tokens (never [SOS]/[EOS]) are replaced by [MASK]; `masked_labels` holds the original id
    there and the padding id everywhere else (at least one label per caption)."""
    batch = synth_batch(batch_size, seed=seed, max_len=max_len, vocab=vocab, ragged=ragged)
    g = torch.Generator().manual_seed(seed + 777)
    tokens = batch["caption_tokens"].clone()
    labels = torch.zeros_like(tokens)
    for b in range(batch_size):
        n = int(batch["caption_lengths"][b])
        cand = [t for t in range(1, n - 1) if tokens[b, t] != 0]
        pick = [t for t in cand if torch.rand(1, generator=g).item() < mask_prob] or cand[:1]
        for t in pick:
            labels[b, t] = tokens[b, t]
            tokens[b, t] = mask_index
    batch["caption_tokens"], batch["masked_labels"] = tokens, labels
    return batch


def model_forward(P, batch, spec: Spec, training=True, new_buffers=None, return_logits=False):
    vf = backbone_forward(P, batch["image"], spec, training, new_buffers)
    logits_f = head_forward(P, vf, batch["caption_tokens"], batch["caption_lengths"], spec, "textual")
    loss_f = caption_loss(logits_f, batch["caption_tokens"], spec.pad)
    out = {"loss": loss_f, "loss_components": {"captioning_forward": loss_f.detach().clone()}}
    if spec.caption_backward:
        logits_b = head_forward(P, vf, batch["noitpac_tokens"], batch["caption_lengths"], spec, "backward_textual")
        loss_b = caption_loss(logits_b, batch["noitpac_tokens"], spec.pad)
        out["loss"] = loss_f + loss_b
        out["loss_components"]["captioning_backward"] = loss_b.detach().clone()
        if return_logits:
            out["backward_logits"] = logits_b
    if not training:
        out["predictions"] = torch.argmax(logits_f, dim=-1)
    if return_logits:
        out["logits"] = logits_f
        out["visual_features"] = vf
    return out


def _cast_batch(batch, dtype):
    b = dict(batch)
    b["image"] = batch["image"].to(dtype)
    return b


def cast_state(state, dtype):
    return OrderedDict((k, v.to(dtype) if v.is_floating_point() else v) for k, v in state.items())


def loss_and_grads(state, batch, spec: Spec, dtype=torch.float32):
    """One training-mode forward + backward.  Returns (output dict, grads by unique name, new BN buffers).
    `dtype=torch.float64` gives the well-conditioned ground truth used to pin the oracle against the reference."""
    P = {k: (v.clone().to(dtype).requires_grad_(True) if not is_buffer(k)
             else (v.clone().to(dtype) if v.is_floating_point() else v.clone())) for k, v in state.items()}
    batch = _cast_batch(batch, dtype)
    new_buffers: Dict[str, torch.Tensor] = {}
    fwd = masked_lm_forward if "masked_labels" in batch else model_forward
    out = fwd(P, batch, spec, training=True, new_buffers=new_buffers, return_logits=True)
    out["loss"].backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in P.items() if not is_buffer(k)}
    # NB: row `pad` of the tied word matrix still receives the vocabulary-projection gradient (class-0 logit);
    # only the *lookup* gradient is suppressed by nn.Embedding(padding_idx), and that one is already zero here
    # because padded positions are multiplied by the token mask after the embedding LayerNorm.
    out = {k: (v.detach() if torch.is_tensor(v) else v) for k, v in out.items()}
    return out, grads, new_buffers


# ------------------------------------------------------------------------------------------------------ optimiser step
@dataclass
class OptimCfg:
    """OPTIM.* defaults of configs/_base_bicaptioning_R_50_L1_H1024.yaml:44-69."""
    lr: float = 0.001
    cnn_lr: float = 0.2
    momentum: float = 0.9
    weight_decay: float = 1e-4
    no_decay: str = r".*textual.(embedding|transformer).*(norm.*|bias)"
    clip_grad_norm: float = 10.0
    lookahead: bool = True
    lookahead_alpha: float = 0.5
    lookahead_steps: int = 5
    warmup_steps: int = 10000
    num_iterations: int = 500000


def lr_multiplier(step: int, cfg: OptimCfg) -> float:
    """LinearWarmupCosineAnnealingLR (virtex/optim/lr_scheduler.py:174-183)."""
    if step < cfg.warmup_steps:
        return float(step) / float(max(1, cfg.warmup_steps))
    cos_factor = (step - cfg.warmup_steps) / (cfg.num_iterations - cfg.warmup_steps)
    return max(0.0, math.cos(cos_factor * (math.pi / 2)) ** 2)


def param_hparams(name: str, cfg: OptimCfg) -> Tuple[float, float]:
    """(lr, weight_decay) of one parameter: virtex/factories.py:529-533."""
    wd = 0.0 if re.match(cfg.no_decay, name) else cfg.weight_decay
    lr = cfg.cnn_lr if "cnn" in name else cfg.lr
    return lr, wd


class OracleTrainer:
    """Reference step sequence (scripts/pretrain_virtex.py:145-163) on the oracle model, fp32 CPU."""

    def __init__(self, state, spec: Spec, cfg: Optional[OptimCfg] = None):
        self.spec, self.cfg = spec, cfg or OptimCfg()
        self.state = OrderedDict((k, v.clone()) for k, v in state.items())
        self.momentum_buf: Dict[str, torch.Tensor] = {}
        self.slow = {k: v.clone() for k, v in self.state.items() if not is_buffer(k)}
        self.iteration = 0  # completed optimiser steps
        self.k_counter = 0

    def step(self, batch) -> Dict[str, torch.Tensor]:
        cfg = self.cfg
        out, grads, new_buffers = loss_and_grads(self.state, batch, self.spec)
        self.state.update(new_buffers)
        total = torch.sqrt(sum((g.double() ** 2).sum() for g in grads.values())).float()
        clip = min(1.0, cfg.clip_grad_norm / (float(total) + 1e-6))
        mult = lr_multiplier(self.iteration, cfg)  # step i uses lambda(i-1)
        for name, g in grads.items():
            lr, wd = param_hparams(name, cfg)
            p = self.state[name]
            g = g * clip + wd * p
            if name not in self.momentum_buf:
                self.momentum_buf[name] = g.clone()
            else:
                self.momentum_buf[name].mul_(cfg.momentum).add_(g)
            p.add_(self.momentum_buf[name], alpha=-lr * mult)
        if cfg.lookahead:
            self.k_counter += 1
            if self.k_counter >= cfg.lookahead_steps:
                self.k_counter = 0
                for name, slow in self.slow.items():
                    slow.add_(self.state[name] - slow, alpha=cfg.lookahead_alpha)
                    self.state[name].copy_(slow)
        self.iteration += 1
        out["grad_norm"] = total
        return out
