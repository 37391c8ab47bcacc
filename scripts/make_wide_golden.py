"""Write tests/golden/r50w2x_l1_h128_post_b2.pt by running the UNMODIFIED reference (a checkout named by
$VIRTEX_REFERENCE_ROOT) on the CPU:

    VIRTEX_REFERENCE_ROOT=/path/to/virtex python scripts/make_wide_golden.py

The wide sibling of oracle/make_golden.py's cases: the reference's VirTexModel with
TorchvisionVisualBackbone("wide_resnet50_2") (the R_50W2X backbone ablation) and a small post-norm head, batch 2, in
float64 and float32, with weights from oracle/virtex_oracle.py.  Only the reference's outputs are stored, in the layout
of the other model fixtures: training loss and its components, gradient norms / sums / probes, BN buffers, and the
eval-mode loss, predictions, logits and features."""
import os
import sys
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shim, virtex_oracle as O  # noqa: E402
from oracle.make_golden import build_reference_model, grad_summary  # noqa: E402

NAME = "r50w2x_l1_h128_post_b2"
SPEC = dict(backbone="wide_resnet50_2", hidden=128, layers=1, heads=2, ffn=256)  # O.Spec(**SPEC)
BATCH = dict(batch_size=2, seed=5, ragged=False)
SEED = 5
PROBES = ("visual.cnn.conv1.weight", "visual.cnn.layer4.2.conv3.weight", "textual.embedding.words.weight",
          "textual.visual_projection.weight", "backward_textual.transformer.layers.0.self_attn.in_proj_weight")


def main():
    if not ref_shim.available():
        raise SystemExit("reference tree not found: set VIRTEX_REFERENCE_ROOT to a checkout of the reference")
    warnings.filterwarnings("ignore")
    ref_shim.install()
    torch.manual_seed(0)
    spec = O.Spec(**SPEC)
    state = O.synth_state(spec, SEED)
    batch = O.synth_batch(max_len=spec.max_len, vocab=spec.vocab, **BATCH)
    out = {"spec": SPEC, "batch": BATCH, "seed": SEED}
    for tag, dtype in (("f64", torch.float64), ("f32", torch.float32)):
        model = build_reference_model(spec)
        model.load_state_dict(O.to_reference_state_dict(state, spec), strict=True)
        model = model.to(dtype)
        b = dict(batch, image=batch["image"].to(dtype))
        model.train()
        res = model(b)
        res["loss"].backward()
        named = dict(model.named_parameters())
        grads = {k: named[k].grad for k in state if not O.is_buffer(k)}
        bufs = dict(model.named_buffers())
        rec = {"loss": res["loss"].detach().double(),
               "loss_forward": res["loss_components"]["captioning_forward"].double(),
               "loss_backward": res["loss_components"]["captioning_backward"].double(),
               "grads": grad_summary(grads),
               "grad_probe": {k: grads[k].detach().flatten()[:64].clone() for k in PROBES},
               "bn_running_mean_layer4": bufs["visual.cnn.layer4.2.bn3.running_mean"].clone(),
               "bn_running_var_stem": bufs["visual.cnn.bn1.running_var"].clone(),
               "num_batches_tracked": bufs["visual.cnn.bn1.num_batches_tracked"].clone()}
        # eval-mode pass with the original buffers
        model.load_state_dict(O.to_reference_state_dict(O.cast_state(state, dtype), spec), strict=True)
        model.eval()
        with torch.no_grad():
            ev = model(b)
            vf = model.visual(b["image"])
            logits = model.textual(vf, b["caption_tokens"], b["caption_lengths"])
        rec.update(eval_loss=ev["loss"].double(), eval_predictions=ev["predictions"].clone(),
                   eval_logits_slice=logits[:, :, :48].clone(), eval_logits_max=logits.max(dim=-1).values.clone(),
                   eval_visual_slice=vf[:, :32].clone())
        out[tag] = rec
        print(f"{NAME} [{tag}] loss {rec['loss'].item():.9f} eval {rec['eval_loss'].item():.9f}", flush=True)
    torch.save(out, os.path.join(ROOT, "tests", "golden", NAME + ".pt"))


if __name__ == "__main__":
    main()
