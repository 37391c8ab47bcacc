"""CPU oracle of the classification pretext models -- TEST INFRASTRUCTURE, NOT PRODUCT.

Plain restatement of virtex/models/classification.py:43-108 over a LinearTextualHead (virtex/modules/textual_heads.py:
46-95) on top of the ResNet of `oracle.virtex_oracle`: global average pool, one linear layer, log_softmax, and per image
the mean of -logprobs over the UNIQUE labels that are not ignored (NaN for an image without such a label), averaged over
the batch.  Pinned against the reference's own TokenClassificationModel / MultiLabelClassificationModel by the fixtures
that scripts/make_classification_golden.py writes (tests/test_classification_cpu.py)."""
from collections import OrderedDict
from typing import Dict, List, Optional

import torch
import torch.nn.functional as F

from oracle import virtex_oracle as O

TOKEN_IGNORE = [0, 1, 2, 3]   # [UNK], [SOS], [EOS], [MASK] of the base config's DATA.*_INDEX
MULTILABEL_IGNORE = [0]       # COCO background
SPEC = O.Spec(hidden=128, layers=1, heads=2, ffn=256, caption_backward=False)  # only its backbone is used


def synth_classification_state(vocab: int, seed: int = 0, bn3_gain: float = 0.25) -> "OrderedDict[str, torch.Tensor]":
    """Backbone of `O.synth_state` (randomised BN) + `textual.output.*` drawn like nn.Linear's default init."""
    state = OrderedDict((k, v) for k, v in O.synth_state(SPEC, seed, bn3_gain=bn3_gain).items() if k.startswith("visual."))
    g = torch.Generator().manual_seed(5000 + seed)
    bound = 1.0 / SPEC.visual_feature_size ** 0.5
    state["textual.output.weight"] = (torch.rand(vocab, SPEC.visual_feature_size, generator=g) * 2 - 1) * bound
    state["textual.output.bias"] = (torch.rand(vocab, generator=g) * 2 - 1) * bound
    return state


def synth_label_batch(batch_size: int, seed: int = 0, vocab: int = 10000, ignore: List[int] = TOKEN_IGNORE,
                      max_labels: int = 12, image_size: int = 96, empty_rows=()) -> Dict[str, torch.Tensor]:
    """Images + `labels` [B, max_labels] right-padded with 0 (the collate's padding id, always ignored).  Every row
    has a ragged length, a duplicated label and an ignored id among its labels; rows in `empty_rows` hold ignored ids
    only, so their set of targets is empty.  `caption_tokens` repeats `labels` (what log_predictions prints)."""
    g = torch.Generator().manual_seed(2000 + seed)
    image = torch.randn(batch_size, 3, image_size, image_size, generator=g)
    labels = torch.zeros(batch_size, max_labels, dtype=torch.int64)
    for b in range(batch_size):
        n = int(torch.randint(4, max_labels + 1, (1,), generator=g))
        if b == 0:
            n = max_labels
        row = torch.randint(0, vocab, (n,), generator=g)
        row[1] = row[0]                                                     # a duplicate counts once
        row[2] = ignore[int(torch.randint(0, len(ignore), (1,), generator=g))]  # an ignored id
        if b in empty_rows:
            row = torch.tensor(ignore, dtype=torch.int64)[torch.randint(0, len(ignore), (n,), generator=g)]
        labels[b, :n] = row
    return {"image_id": torch.arange(batch_size), "image": image, "labels": labels, "caption_tokens": labels.clone()}


def khot_loss_rows(logits: torch.Tensor, labels: torch.Tensor, ignore: List[int]) -> torch.Tensor:
    """Per-image loss -mean_{u in U_b} log_softmax(logits_b)[u]: NaN where U_b is empty (mean over an empty set)."""
    logprobs = F.log_softmax(logits, dim=1)
    rows = []
    for b in range(logits.shape[0]):
        unique = sorted(set(labels[b].tolist()) - set(ignore))
        rows.append(-logprobs[b, unique].mean())
    return torch.stack(rows)


def classification_forward(P, batch, ignore: List[int], training: bool = True, new_buffers=None,
                           return_logits: bool = False) -> Dict[str, torch.Tensor]:
    vf = O.backbone_forward(P, batch["image"], SPEC, training, new_buffers)
    logits = vf.flatten(2).mean(-1) @ P["textual.output.weight"].t() + P["textual.output.bias"]
    loss = khot_loss_rows(logits, batch["labels"], ignore).mean()
    out = {"loss": loss, "loss_components": {"classification": loss.detach().clone()}}
    if not training:
        out["predictions"] = F.log_softmax(logits, dim=1).topk(10, dim=1).indices
    if return_logits:
        out["logits"] = logits
    return out


def loss_and_grads(state, batch, ignore: List[int], dtype=torch.float64):
    """One training-mode forward + backward -> (output dict, gradients by name)."""
    P = {k: (v.clone().to(dtype).requires_grad_(True) if not O.is_buffer(k)
             else (v.clone().to(dtype) if v.is_floating_point() else v.clone())) for k, v in state.items()}
    b = dict(batch, image=batch["image"].to(dtype))
    out = classification_forward(P, b, ignore, training=True, new_buffers={}, return_logits=True)
    out["loss"].backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in P.items() if not O.is_buffer(k)}
    return {k: (v.detach() if torch.is_tensor(v) else v) for k, v in out.items()}, grads


def eval_forward(state, batch, ignore: List[int], dtype=torch.float64):
    P = O.cast_state(state, dtype)
    with torch.no_grad():
        return classification_forward(P, dict(batch, image=batch["image"].to(dtype)), ignore, training=False,
                                      return_logits=True)


def grad_summary(grads: Dict[str, torch.Tensor], names: Optional[List[str]] = None):
    names = sorted(grads) if names is None else names
    return {"names": names,
            "norm": torch.tensor([grads[n].double().norm().item() for n in names], dtype=torch.float64),
            "sum": torch.tensor([grads[n].double().sum().item() for n in names], dtype=torch.float64)}


# the two fixtures: (file stem, vocabulary, ignored ids, state seed, batch seed)
CASES = {
    "token_classification": ("token_classification_r50_b3", 10000, TOKEN_IGNORE, 41, 51),
    "multilabel_classification": ("multilabel_classification_r50_b3", 81, MULTILABEL_IGNORE, 42, 52),
}
EMPTY_ROW = 1  # the row emptied in the fixtures' second batch
