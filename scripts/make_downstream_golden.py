"""Write tests/golden/downstream_r50_fc10.pt by running the UNMODIFIED reference's torchvision ResNet-50 (the
`visual.cnn` of its TorchvisionVisualBackbone, from a checkout named by $VIRTEX_REFERENCE_ROOT) with an `fc` head on the
CPU in float64, the way scripts/clf_linear.py and scripts/clf_voc07.py call it:

    VIRTEX_REFERENCE_ROOT=/path/to/virtex python scripts/make_downstream_golden.py

Parameters, running statistics (randomised, so that the BN fold is exercised) and batches come from seeds in
tests/downstream_oracle.py, so only outputs are stored: per case, the eval-mode pooled features, logits, CE loss and fc
gradients of a frozen backbone; the train-mode logits, loss, fc gradients, sampled conv / BN gradients and sampled
updated running statistics.  Large tensors are stored as their first 64 elements and their norm."""
import os
import sys
import warnings

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shim  # noqa: E402
from tests import downstream_oracle as DO  # noqa: E402

N_SAMPLE = 64


def reference_cnn(state):
    from virtex.modules.visual_backbones import TorchvisionVisualBackbone
    cnn = TorchvisionVisualBackbone("resnet50", visual_feature_size=2048).cnn
    cnn.fc = nn.Linear(2048, DO.NUM_CLASSES)
    cnn = cnn.double()
    cnn.load_state_dict({k: (v.double() if v.is_floating_point() else v) for k, v in state.items()}, strict=True)
    return cnn


def sample(t):
    return t.detach().flatten()[:N_SAMPLE].clone()


def run_case(case):
    state, batch = DO.case_inputs(case)
    image = batch["image"].double()
    out = {}
    # eval mode, frozen backbone (the linear probe / VOC07 features)
    cnn = reference_cnn(state).eval()
    for name, p in cnn.named_parameters():
        p.requires_grad = "fc" in name
    logits = cnn(image)
    loss = nn.CrossEntropyLoss()(logits, batch["label"])
    loss.backward()
    ev = {"logits": logits.detach().clone(), "loss": loss.detach().clone(),
          "fc.weight.grad": sample(cnn.fc.weight.grad), "fc.weight.grad_norm": cnn.fc.weight.grad.norm().clone(),
          "fc.bias.grad": cnn.fc.bias.grad.clone()}
    cnn.fc = nn.Identity()  # the VOC07 feature extractor
    with torch.no_grad():
        ev["pooled"] = cnn(image).float()  # (stored in fp32 to keep the fixture small)
    out["eval"] = ev
    # train mode, every parameter trains (fine-tuning)
    cnn = reference_cnn(state).train()
    logits = cnn(image)
    loss = nn.CrossEntropyLoss()(logits, batch["label"])
    loss.backward()
    named = dict(cnn.named_parameters())
    buffers = dict(cnn.named_buffers())
    tr = {"logits": logits.detach().clone(), "loss": loss.detach().clone(),
          "fc.weight.grad": sample(named["fc.weight"].grad), "fc.weight.grad_norm": named["fc.weight"].grad.norm().clone(),
          "fc.bias.grad": named["fc.bias"].grad.clone()}
    for k in DO.CONV_PROBES:
        tr[k + ".grad"] = sample(named[k].grad)
        tr[k + ".grad_norm"] = named[k].grad.norm().detach().clone()
    for k in DO.BN_PROBES:
        for leaf in ("weight", "bias"):
            tr[f"{k}.{leaf}.grad"] = sample(named[f"{k}.{leaf}"].grad)
        for leaf in ("running_mean", "running_var"):
            tr[f"{k}.{leaf}"] = sample(buffers[f"{k}.{leaf}"])
        tr[f"{k}.num_batches_tracked"] = buffers[f"{k}.num_batches_tracked"].clone()
    out["train"] = tr
    print(f"{case}: eval loss {out['eval']['loss'].item():.9f} train loss {tr['loss'].item():.9f}", flush=True)
    return out


def main():
    if not ref_shim.available():
        raise SystemExit("reference tree not found: set VIRTEX_REFERENCE_ROOT to a checkout of the reference")
    warnings.filterwarnings("ignore")
    ref_shim.install()
    torch.manual_seed(0)
    out = {case: run_case(case) for case in DO.CASES}
    torch.save(out, os.path.join(ROOT, "tests", "golden", DO.GOLDEN))


if __name__ == "__main__":
    main()
