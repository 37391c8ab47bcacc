"""Write tests/golden/captioning_beam_search.pt by running the UNMODIFIED reference's captioning model with its
AutoRegressiveBeamSearch (a checkout named by $VIRTEX_REFERENCE_ROOT) on the CPU in float64:

    VIRTEX_REFERENCE_ROOT=/path/to/virtex python scripts/make_captioning_golden.py

States, images and search settings are the cases of tests/captioning_oracle.py.  Per case the fixture holds the
reference's `model.eval(); model({"image": x})["predictions"]`, every beam and its score from `decoder.search(...,
only_return_best=False)`, and -- from the float64 restatement in tests/captioning_oracle.py driven by the reference's
own `decoding_step`, after checking that it reproduces the reference's beams and scores exactly -- the node and image
gaps of every step."""
import functools
import os
import sys
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shim, virtex_oracle as O  # noqa: E402
from tests import captioning_oracle as C  # noqa: E402


def reference_model(case):
    from virtex.models import ForwardCaptioningModel, VirTexModel
    from virtex.modules.textual_heads import TransformerDecoderTextualHead
    from virtex.modules.visual_backbones import TorchvisionVisualBackbone
    from virtex.utils.beam_search import AutoRegressiveBeamSearch

    c, spec = C.CASES[case], C.case_spec(case)
    visual = TorchvisionVisualBackbone(spec.backbone, visual_feature_size=spec.visual_feature_size)
    textual = TransformerDecoderTextualHead(
        visual_feature_size=spec.visual_feature_size, vocab_size=spec.vocab, hidden_size=spec.hidden,
        num_layers=spec.layers, attention_heads=spec.heads, feedforward_size=spec.ffn, dropout=0.1,
        norm_first=spec.norm_first, mask_future_positions=True, max_caption_length=spec.max_len, padding_idx=spec.pad)
    decoder = AutoRegressiveBeamSearch(C.EOS, max_steps=c["max_steps"], beam_size=c["beam"])
    cls = VirTexModel if spec.caption_backward else ForwardCaptioningModel
    model = cls(visual, textual, sos_index=C.SOS, eos_index=C.EOS, decoder=decoder).double()
    sd = O.to_reference_state_dict(C.case_state(case), spec)
    model.load_state_dict({k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}, strict=True)
    return model.eval()


def run_case(case):
    c = C.CASES[case]
    model = reference_model(case)
    image = C.case_image(case).double()
    with torch.no_grad():
        predictions = model({"image": image})["predictions"]
        features = model.visual(image)
        step = functools.partial(model.decoding_step, features)
        start = features.new_full((c["B"],), C.SOS).long()
        beams, scores = model.decoder.search(start, step, only_return_best=False)
        mine = C.beam_search(step, c["B"], c["beam"], c["max_steps"])
    assert torch.equal(mine["predictions"], beams) and torch.equal(mine["scores"], scores), case
    # the early return of beam size 1 (beam_search.py:111-117) skips the best-beam selection: (B, 1, 1) there
    predictions = predictions.reshape(c["B"], -1)
    assert torch.equal(predictions, beams[:, 0]), case
    out = {"predictions": predictions, "beams": beams, "scores": scores,
           "node_gaps": mine["node_gaps"], "image_gaps": mine["image_gaps"]}
    print(f"{case}: L {predictions.shape[1]}, best scores {scores[:, 0].tolist()}, "
          f"decisive images {C.decisive(mine, c['beam'], 0.1).tolist()}", flush=True)
    return out


def main():
    if not ref_shim.available():
        raise SystemExit("reference tree not found: set VIRTEX_REFERENCE_ROOT to a checkout of the reference")
    warnings.filterwarnings("ignore")
    ref_shim.install()
    torch.manual_seed(0)
    out = {case: run_case(case) for case in C.CASES}
    torch.save(out, os.path.join(ROOT, "tests", "golden", C.GOLDEN))


if __name__ == "__main__":
    main()
