"""Basic-block ResNets (ResNet-18 / ResNet-34) for the CPU oracle -- TEST INFRASTRUCTURE, NOT PRODUCT.

`oracle.virtex_oracle` states the bicaptioning model for the bottleneck ResNets.  Its head, BatchNorm, losses and
trainer apply to any backbone; its parameter inventory, synthetic weights and `backbone_forward` assume bottlenecks.
This module supplies those three for torchvision's resnet18 / resnet34 (torchvision/models/resnet.py:59-105: conv1 3x3
(stride) -> bn1 -> ReLU -> conv2 3x3 -> bn2, + shortcut, ReLU; 512 output channels), and runs the oracle's
`model_forward`, `loss_and_grads` and `OracleTrainer` on them.  For any other backbone everything here is the oracle's
own.  Pinned against the reference's VirTexModel with TorchvisionVisualBackbone("resnet18", visual_feature_size=512)
by tests/golden/r18_l1_h128_post_b2.pt (scripts/make_basic_golden.py, tests/test_basic_resnet_cpu.py)."""
import contextlib
import math
from collections import OrderedDict
from typing import Tuple

import torch
import torch.nn.functional as F

from oracle import virtex_oracle as O

BLOCKS = {"resnet18": [2, 2, 2, 2], "resnet34": [3, 4, 6, 3]}
_BOTTLENECK_FORWARD = O.backbone_forward


def spec(backbone: str = "resnet18", **kwargs) -> O.Spec:
    """O.Spec of a model with this basic-block backbone: its blocks per layer and a 512-wide visual feature."""
    return O.Spec(backbone=backbone, blocks=list(BLOCKS[backbone]), visual_feature_size=512, **kwargs)


def backbone_param_shapes(s: O.Spec) -> "OrderedDict[str, Tuple[int, ...]]":
    """Names/shapes of `visual.cnn.*` parameters and buffers of a basic-block ResNet, in torchvision registration
    order."""
    out: "OrderedDict[str, Tuple[int, ...]]" = OrderedDict()

    def bn(prefix, c):
        for leaf, shape in (("weight", (c,)), ("bias", (c,)), ("running_mean", (c,)), ("running_var", (c,)),
                            ("num_batches_tracked", ())):
            out[f"{prefix}.{leaf}"] = shape

    p = "visual.cnn."
    out[p + "conv1.weight"] = (64, 3, 7, 7)
    bn(p + "bn1", 64)
    inplanes = 64
    for li, (planes, nblocks) in enumerate(zip([64, 128, 256, 512], s.blocks), start=1):
        for bi in range(nblocks):
            stride = 2 if (bi == 0 and li > 1) else 1
            q = f"{p}layer{li}.{bi}."
            out[q + "conv1.weight"] = (planes, inplanes, 3, 3)
            bn(q + "bn1", planes)
            out[q + "conv2.weight"] = (planes, planes, 3, 3)
            bn(q + "bn2", planes)
            if stride != 1 or inplanes != planes:
                out[q + "downsample.0.weight"] = (planes, inplanes, 1, 1)
                bn(q + "downsample.1", planes)
            inplanes = planes
    return out


def synth_state(s: O.Spec, seed: int = 0, randomize_bn: bool = True,
                residual_gain: float = 1.0) -> "OrderedDict[str, torch.Tensor]":
    """Deterministic synthetic weights from (spec, seed), by the rules of O.synth_state: Kaiming fan_out convs,
    randomised BN parameters and running statistics, and `residual_gain` on bn2's gamma, the last BN of every basic
    block (zero without `randomize_bn`, as zero_init_residual).  The textual tensors are O.synth_state's for the same
    head; the backbone tensors are drawn in registration order from a generator of their own."""
    if s.backbone not in BLOCKS:
        return O.synth_state(s, seed, randomize_bn, residual_gain)
    head = O.synth_state(O.Spec(**{**s.__dict__, "backbone": "resnet50", "blocks": [3, 4, 6, 3]}), seed,
                         randomize_bn, residual_gain)
    g = torch.Generator().manual_seed(20_000 + seed)
    out: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    for name, shape in backbone_param_shapes(s).items():
        last = ".bn2." in name and ".layer" in name
        if name.endswith("num_batches_tracked"):
            t = torch.zeros((), dtype=torch.int64)
        elif name.endswith("running_mean"):
            t = torch.randn(shape, generator=g) * 0.1 if randomize_bn else torch.zeros(shape)
        elif name.endswith("running_var"):
            t = torch.rand(shape, generator=g) + 0.5 if randomize_bn else torch.ones(shape)
        elif name.endswith(".weight") and len(shape) == 4:
            t = torch.randn(shape, generator=g) * math.sqrt(2.0 / (shape[0] * shape[2] * shape[3]))
        elif name.endswith(".weight"):  # BN gamma
            if not randomize_bn:
                t = torch.zeros(shape) if last else torch.ones(shape)
            else:
                t = (torch.rand(shape, generator=g) + 0.5) * (residual_gain if last else 1.0)
        else:  # BN beta
            t = torch.randn(shape, generator=g) * 0.1 if randomize_bn else torch.zeros(shape)
        out[name] = t
    out.update((k, v) for k, v in head.items() if not k.startswith("visual."))
    return out


def backbone_forward(P, image, spec: O.Spec, training=True, new_buffers=None, record=None, emulate_bf16=False):
    """(B,3,H,W) -> (B,512,H/32,W/32) for a basic-block backbone (O.backbone_forward for any other), in the dtype of
    P; autograd runs through it.  `record` receives the stem's and every block's intermediates (y1, a1, y2, out)."""
    if spec.backbone not in BLOCKS:
        return _BOTTLENECK_FORWARD(P, image, spec, training, new_buffers, record, emulate_bf16)
    p = "visual.cnn."
    rb = O._rb if emulate_bf16 else (lambda t: t)
    bn = lambda t, name: O._batch_norm(t, P, name, training, new_buffers, emulate_bf16=emulate_bf16)
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
            out = F.conv2d(x, rb(P[q + "conv1.weight"]), stride=stride, padding=1)
            if record is not None:
                record[q + "y1"] = out
            out = rb(torch.relu(bn(out, q + "bn1")))
            if record is not None:
                record[q + "a1"] = out
            out = F.conv2d(out, rb(P[q + "conv2.weight"]), padding=1)
            if record is not None:
                record[q + "y2"] = out
            out = bn(out, q + "bn2")
            if q + "downsample.0.weight" in P:
                identity = F.conv2d(x, rb(P[q + "downsample.0.weight"]), stride=stride)
                identity = bn(identity, q + "downsample.1")
            x = rb(torch.relu(out + identity))
            if record is not None:
                record[q + "out"] = x
    return x


@contextlib.contextmanager
def _basic_backbone():
    """The oracle's model functions look `backbone_forward` up in their module: run them on this one meanwhile."""
    O.backbone_forward = backbone_forward
    try:
        yield
    finally:
        O.backbone_forward = _BOTTLENECK_FORWARD


def model_forward(*args, **kwargs):
    with _basic_backbone():
        return O.model_forward(*args, **kwargs)


def loss_and_grads(*args, **kwargs):
    with _basic_backbone():
        return O.loss_and_grads(*args, **kwargs)


class OracleTrainer(O.OracleTrainer):
    def step(self, batch):
        with _basic_backbone():
            return super().step(batch)
