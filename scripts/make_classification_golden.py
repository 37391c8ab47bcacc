"""Write tests/golden/{token,multilabel}_classification_r50_b3.pt by running the UNMODIFIED reference's
TokenClassificationModel / MultiLabelClassificationModel (a checkout named by $VIRTEX_REFERENCE_ROOT) on the CPU:

    VIRTEX_REFERENCE_ROOT=/path/to/virtex python scripts/make_classification_golden.py

Inputs come from tests/classification_oracle.py (synthetic weights and labels from seeds), so only the reference's
outputs are stored: float64 and float32 runs of the training loss and gradient summaries, the same for a batch with an
image whose labels are all ignored (NaN loss), and the eval loss and top-10 predictions."""
import os
import sys
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shim, virtex_oracle as O  # noqa: E402
from tests import classification_oracle as CO  # noqa: E402

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")


def reference_model(name, vocab, ignore):
    from virtex.models import MultiLabelClassificationModel, TokenClassificationModel
    from virtex.modules.textual_heads import LinearTextualHead
    from virtex.modules.visual_backbones import TorchvisionVisualBackbone
    cls = TokenClassificationModel if name == "token_classification" else MultiLabelClassificationModel
    return cls(TorchvisionVisualBackbone("resnet50", visual_feature_size=2048),
               LinearTextualHead(visual_feature_size=2048, vocab_size=vocab), ignore_indices=ignore)


def train_record(model, state, batch, dtype):
    model.load_state_dict(O.cast_state(state, dtype), strict=True)
    model.train()
    model.zero_grad(set_to_none=True)
    res = model(dict(batch, image=batch["image"].to(dtype)))
    res["loss"].backward()
    named = dict(model.named_parameters())
    grads = {k: (p.grad if p.grad is not None else torch.zeros_like(p)) for k, p in named.items()}
    return {"loss": res["loss"].detach().double(), "grads": CO.grad_summary(grads),
            "grad_probe": {k: grads[k].detach().flatten()[:64].clone()
                           for k in ("visual.cnn.conv1.weight", "visual.cnn.layer4.2.conv3.weight",
                                     "textual.output.weight", "textual.output.bias")}}


def run_case(name):
    stem, vocab, ignore, seed, batch_seed = CO.CASES[name]
    state = CO.synth_classification_state(vocab, seed)
    batch = CO.synth_label_batch(3, seed=batch_seed, vocab=vocab, ignore=ignore)
    empty = CO.synth_label_batch(3, seed=batch_seed, vocab=vocab, ignore=ignore, empty_rows=(CO.EMPTY_ROW,))
    out = {"name": name, "vocab": vocab, "ignore": ignore, "seed": seed, "batch_seed": batch_seed}
    for tag, dtype in (("f64", torch.float64), ("f32", torch.float32)):
        model = reference_model(name, vocab, ignore).to(dtype)
        rec = train_record(model, state, batch, dtype)
        rec["empty_row"] = train_record(model, state, empty, dtype)
        model.load_state_dict(O.cast_state(state, dtype), strict=True)
        model.eval()
        with torch.no_grad():
            ev = model(dict(batch, image=batch["image"].to(dtype)))
        rec["eval_loss"] = ev["loss"].double()
        rec["eval_predictions"] = ev["predictions"].clone()
        out[tag] = rec
        print(f"{name} [{tag}] loss {rec['loss'].item():.9f} empty-row loss {rec['empty_row']['loss'].item()} "
              f"eval {rec['eval_loss'].item():.9f}", flush=True)
    torch.save(out, os.path.join(GOLDEN_DIR, stem + ".pt"))


def main():
    if not ref_shim.available():
        raise SystemExit("reference tree not found: set VIRTEX_REFERENCE_ROOT to a checkout of the reference")
    warnings.filterwarnings("ignore")
    ref_shim.install()
    torch.manual_seed(0)
    for name in (sys.argv[1:] or list(CO.CASES)):
        run_case(name)


if __name__ == "__main__":
    main()
