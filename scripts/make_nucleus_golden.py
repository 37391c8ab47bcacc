"""Write tests/golden/captioning_nucleus_sampling.pt by running the UNMODIFIED reference's captioning model with its
AutoRegressiveNucleusSampling (a checkout named by $VIRTEX_REFERENCE_ROOT) on the CPU in float64:

    VIRTEX_REFERENCE_ROOT=/path/to/virtex python scripts/make_nucleus_golden.py

States, images and sampler settings are the cases of tests/nucleus_oracle.py.  Per case the fixture holds the
reference's `model.eval(); model({"image": x})["predictions"]` after `torch.manual_seed(case["rng"])`, and -- from the
float64 restatement in tests/nucleus_oracle.py driven by the reference's own `decoding_step` with a generator of the same
seed, after checking that it reproduces the reference's captions exactly -- the nucleus size, cut margin and
banned-alone flag of every step and row."""
import functools
import os
import sys
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shim, virtex_oracle as O  # noqa: E402
from tests import nucleus_oracle as N  # noqa: E402


def reference_model(case):
    from virtex.models import ForwardCaptioningModel, VirTexModel
    from virtex.modules.textual_heads import TransformerDecoderTextualHead
    from virtex.modules.visual_backbones import TorchvisionVisualBackbone
    from virtex.utils.nucleus_sampling import AutoRegressiveNucleusSampling

    c, spec = N.CASES[case], N.case_spec(case)
    visual = TorchvisionVisualBackbone(spec.backbone, visual_feature_size=spec.visual_feature_size)
    textual = TransformerDecoderTextualHead(
        visual_feature_size=spec.visual_feature_size, vocab_size=spec.vocab, hidden_size=spec.hidden,
        num_layers=spec.layers, attention_heads=spec.heads, feedforward_size=spec.ffn, dropout=0.1,
        norm_first=spec.norm_first, mask_future_positions=True, max_caption_length=spec.max_len, padding_idx=spec.pad)
    decoder = AutoRegressiveNucleusSampling(N.EOS, max_steps=c["max_steps"], nucleus_size=c["p"])
    cls = VirTexModel if spec.caption_backward else ForwardCaptioningModel
    model = cls(visual, textual, sos_index=N.SOS, eos_index=N.EOS, decoder=decoder).double()
    sd = O.to_reference_state_dict(N.case_state(case), spec)
    model.load_state_dict({k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}, strict=True)
    return model.eval()


def run_case(case):
    c = N.CASES[case]
    model = reference_model(case)
    image = N.case_image(case).double()
    with torch.no_grad():
        torch.manual_seed(c["rng"])
        predictions = model({"image": image})["predictions"]
        features = model.visual(image)
        step = functools.partial(model.decoding_step, features)
        mine = N.nucleus_sampling(step, c["B"], c["p"], c["max_steps"], torch.Generator().manual_seed(c["rng"]))
    assert torch.equal(mine["predictions"], predictions), case
    out = {"predictions": predictions, "sizes": mine["sizes"], "margins": mine["margins"],
           "banned_alone": mine["banned_alone"]}
    print(f"{case}: L {predictions.shape[1]}, nucleus sizes {[s.tolist() for s in mine['sizes']][:4]} ..., smallest "
          f"margin {min(float(m.min()) for m in mine['margins']):.2e}, banned-alone rows "
          f"{sum(int(a.sum()) for a in mine['banned_alone'])}", flush=True)
    return out


def main():
    if not ref_shim.available():
        raise SystemExit("reference tree not found: set VIRTEX_REFERENCE_ROOT to a checkout of the reference")
    warnings.filterwarnings("ignore")
    ref_shim.install()
    out = {case: run_case(case) for case in N.CASES}
    torch.save(out, os.path.join(ROOT, "tests", "golden", N.GOLDEN))


if __name__ == "__main__":
    main()
