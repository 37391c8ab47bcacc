"""CPU oracle of the downstream classification evaluations -- TEST INFRASTRUCTURE, NOT PRODUCT.

`pretrained_model.visual.cnn` called as a torchvision ResNet (scripts/clf_linear.py:147-160,227-229,
scripts/clf_voc07.py:165): `oracle.virtex_oracle.backbone_forward` up to layer4, then the global average pool and an
`fc` linear layer, with nn.CrossEntropyLoss on the logits.  Pinned against the reference's own torchvision ResNet-50 by
the fixture scripts/make_downstream_golden.py writes (tests/test_downstream_cpu.py)."""
from collections import OrderedDict
from typing import Dict, Optional

import torch
import torch.nn.functional as F

from oracle import virtex_oracle as O

SPEC = O.Spec(hidden=128, layers=1, heads=2, ffn=256, caption_backward=False)  # only its backbone is used
NUM_CLASSES = 10
PREFIX = "visual.cnn."
# (state seed, batch seed, batch size, image size): a 224 x 224 batch (space-to-depth stem) and one whose size the
# stem's TMA boxes do not tile (im2col stem)
CASES = {"b2_224": (61, 71, 2, 224), "b3_200": (62, 72, 3, 200)}
GOLDEN = "downstream_r50_fc10.pt"
# sampled gradients and running statistics of the train-mode fixture
CONV_PROBES = ("conv1.weight", "layer1.0.conv2.weight", "layer2.0.downsample.0.weight", "layer4.2.conv3.weight")
BN_PROBES = ("bn1", "layer1.0.bn1", "layer3.0.downsample.1", "layer4.2.bn3")


def synth_state(seed: int, num_classes: int = NUM_CLASSES) -> "OrderedDict[str, torch.Tensor]":
    """ResNetParams state_dict keys (no prefix): the backbone of `O.synth_state` with randomised BN affine parameters
    and running statistics, plus `fc.*` drawn from the seed (clf_linear.py re-initialises fc with N(0, 0.01); the
    bias is random here so that its gradient path is exercised)."""
    full = O.synth_state(SPEC, seed, bn3_gain=0.25)
    state = OrderedDict((k[len(PREFIX):], v) for k, v in full.items() if k.startswith(PREFIX))
    g = torch.Generator().manual_seed(7000 + seed)
    state["fc.weight"] = torch.randn(num_classes, SPEC.visual_feature_size, generator=g) * 0.01
    state["fc.bias"] = torch.randn(num_classes, generator=g) * 0.1
    return state


def synth_batch(batch_size: int, seed: int, image_size: int, num_classes: int = NUM_CLASSES) -> Dict[str, torch.Tensor]:
    g = torch.Generator().manual_seed(3000 + seed)
    return {"image": torch.randn(batch_size, 3, image_size, image_size, generator=g),
            "label": torch.randint(0, num_classes, (batch_size,), generator=g)}


def case_inputs(case: str):
    seed, batch_seed, B, S = CASES[case]
    return synth_state(seed), synth_batch(B, batch_seed, S)


def cnn_forward(P, image, training: bool, new_buffers: Optional[dict] = None):
    """P keyed like ResNetParams' state_dict -> (pooled (B, 2048), logits (B, num_classes))."""
    Q = {PREFIX + k: v for k, v in P.items()}
    nb = {} if new_buffers is not None else None
    vf = O.backbone_forward(Q, image, SPEC, training, nb)
    if new_buffers is not None:
        new_buffers.update({k[len(PREFIX):]: v for k, v in nb.items()})
    pooled = vf.flatten(2).mean(-1)
    return pooled, pooled @ P["fc.weight"].t() + P["fc.bias"]


def run(state, batch, training: bool, dtype=torch.float64, frozen: bool = False):
    """One forward + CE backward: (pooled, logits, loss, grads by name, updated buffers).  frozen: only fc.* get
    gradients (the linear probe)."""
    P = {}
    for k, v in state.items():
        if O.is_buffer(k):
            P[k] = v.clone().to(dtype) if v.is_floating_point() else v.clone()
        else:
            P[k] = v.clone().to(dtype).requires_grad_(not frozen or k.startswith("fc."))
    new_buffers = {}
    pooled, logits = cnn_forward(P, batch["image"].to(dtype), training, new_buffers if training else None)
    loss = F.cross_entropy(logits, batch["label"])
    loss.backward()
    grads = {k: v.grad for k, v in P.items() if not O.is_buffer(k) and v.grad is not None}
    return pooled.detach(), logits.detach(), loss.detach(), grads, new_buffers


def probe_step(feats, label, weight, bias):
    """One iteration of clf_linear.py's loop on a frozen eval-mode backbone, given its pooled features: CE loss of
    fc = (weight, bias) and the fc gradients, in float64."""
    w = weight.detach().double().cpu().requires_grad_(True)
    b = bias.detach().double().cpu().requires_grad_(True)
    loss = F.cross_entropy(feats @ w.t() + b, label)
    loss.backward()
    return loss.detach(), w.grad, b.grad
