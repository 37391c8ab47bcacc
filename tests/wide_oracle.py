"""Wide ResNet backbones for the CPU oracle -- TEST INFRASTRUCTURE, NOT PRODUCT.

`oracle.virtex_oracle` states the bicaptioning model for torchvision's resnet50/101/152.  Its forward and backward
(`backbone_forward`, `model_forward`, `loss_and_grads`, `OracleTrainer`) read every conv's width from the weights they
are given, so they run the wide models unchanged; only the parameter inventory and the synthetic weights assume a
bottleneck as wide inside as its `planes`.  This module supplies those two for any torchvision ResNet name: a
bottleneck of `planes` has inner width planes * width_per_group / 64 (128 for wide_resnet50_2 / wide_resnet101_2,
torchvision/models/resnet.py:108-163) and output width 4 * planes.  For resnet50/101/152 everything here is the oracle's
own.  Pinned against the reference's VirTexModel with TorchvisionVisualBackbone("wide_resnet50_2") by
tests/golden/r50w2x_l1_h128_post_b2.pt (scripts/make_wide_golden.py, tests/test_wide_resnet_cpu.py)."""
import math
from collections import OrderedDict
from typing import Tuple

import torch

from oracle import virtex_oracle as O

BLOCKS = {"resnet50": [3, 4, 6, 3], "resnet101": [3, 4, 23, 3], "resnet152": [3, 8, 36, 3],
          "wide_resnet50_2": [3, 4, 6, 3], "wide_resnet101_2": [3, 4, 23, 3]}
WIDTH_PER_GROUP = {"wide_resnet50_2": 128, "wide_resnet101_2": 128}


def spec(backbone: str = "wide_resnet50_2", **kwargs) -> O.Spec:
    """O.Spec of a model with this backbone (its blocks per layer given explicitly, which O.Spec accepts for any name)."""
    return O.Spec(backbone=backbone, blocks=list(BLOCKS[backbone]), **kwargs)


def backbone_param_shapes(s: O.Spec) -> "OrderedDict[str, Tuple[int, ...]]":
    """Names/shapes of `visual.cnn.*` parameters and buffers in torchvision registration order, as
    O.backbone_param_shapes, with each bottleneck's inner width."""
    wpg = WIDTH_PER_GROUP.get(s.backbone, 64)
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
        width = planes * wpg // 64
        for bi in range(nblocks):
            stride = 2 if (bi == 0 and li > 1) else 1
            q = f"{p}layer{li}.{bi}."
            out[q + "conv1.weight"] = (width, inplanes, 1, 1)
            bn(q + "bn1", width)
            out[q + "conv2.weight"] = (width, width, 3, 3)
            bn(q + "bn2", width)
            out[q + "conv3.weight"] = (planes * 4, width, 1, 1)
            bn(q + "bn3", planes * 4)
            if stride != 1 or inplanes != planes * 4:
                out[q + "downsample.0.weight"] = (planes * 4, inplanes, 1, 1)
                bn(q + "downsample.1", planes * 4)
            inplanes = planes * 4
    return out


def synth_state(s: O.Spec, seed: int = 0, randomize_bn: bool = True,
                bn3_gain: float = 1.0) -> "OrderedDict[str, torch.Tensor]":
    """Deterministic synthetic weights from (spec, seed), by the rules of O.synth_state (Kaiming fan_out convs,
    randomised BN parameters and running statistics, `bn3_gain` on the last BN gamma of every bottleneck).  For
    resnet50/101/152 it is O.synth_state itself.  For a wide backbone the textual tensors are O.synth_state's and the
    backbone tensors are drawn in registration order from a generator of their own."""
    if s.backbone not in WIDTH_PER_GROUP:
        return O.synth_state(s, seed, randomize_bn, bn3_gain)
    head = O.synth_state(O.Spec(**{**s.__dict__, "backbone": "resnet50", "blocks": [3, 4, 6, 3]}), seed,
                         randomize_bn, bn3_gain)
    g = torch.Generator().manual_seed(10_000 + seed)
    out: "OrderedDict[str, torch.Tensor]" = OrderedDict()
    for name, shape in backbone_param_shapes(s).items():
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
                t = torch.zeros(shape) if ".bn3." in name else torch.ones(shape)
            else:
                t = (torch.rand(shape, generator=g) + 0.5) * (bn3_gain if ".bn3." in name else 1.0)
        else:  # BN beta
            t = torch.randn(shape, generator=g) * 0.1 if randomize_bn else torch.zeros(shape)
        out[name] = t
    out.update((k, v) for k, v in head.items() if not k.startswith("visual."))
    return out
