"""Write tests/golden/trainer_adamw_r50_l1_h128_6steps.pt by running the UNMODIFIED reference's factories and loop body
(a checkout named by $VIRTEX_REFERENCE_ROOT) with OPTIM.OPTIMIZER_NAME adamw on the CPU:

    VIRTEX_REFERENCE_ROOT=/path/to/virtex python scripts/make_adamw_golden.py

The AdamW sibling of the SGD trainer fixture of oracle/make_golden.py: the same model, weights and batches, small
learning rates, and 6 steps so that the run crosses the Lookahead k = 5 boundary.  Only the reference's outputs are
stored: losses, gradient norms, final parameter norms and probes, and the stem's BN running variance."""
import os
import sys
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shim, virtex_oracle as O  # noqa: E402
from tests import adamw_oracle as AO  # noqa: E402

GOLDEN = os.path.join(ROOT, "tests", "golden", "trainer_adamw_r50_l1_h128_6steps.pt")


def main():
    if not ref_shim.available():
        raise SystemExit("reference tree not found: set VIRTEX_REFERENCE_ROOT to a checkout of the reference")
    warnings.filterwarnings("ignore")
    ref_shim.install()
    torch.manual_seed(0)
    from virtex.config import Config
    from virtex.factories import LRSchedulerFactory, OptimizerFactory, PretrainingModelFactory

    cfg = Config(os.path.join(ref_shim.REFERENCE_ROOT, "configs", "_base_bicaptioning_R_50_L1_H1024.yaml"),
                 AO.CONFIG_OVERRIDES)
    spec_kw = dict(hidden=128, layers=1, heads=2, ffn=256)
    spec = O.Spec(**spec_kw)
    state = O.synth_state(spec, 3)
    model = PretrainingModelFactory.from_config(cfg)
    model.load_state_dict(O.to_reference_state_dict(state, spec), strict=True)
    optimizer = OptimizerFactory.from_config(cfg, model.named_parameters())
    assert type(optimizer.optimizer).__name__ == "AdamW", optimizer
    scheduler = LRSchedulerFactory.from_config(cfg, optimizer)
    model.train()
    losses, norms = [], []
    for it in range(6):  # scripts/pretrain_virtex.py:145-163 (AMP disabled on CPU)
        batch = O.synth_batch(2, seed=10 + it)
        optimizer.zero_grad()
        out = model(batch)
        out["loss"].backward()
        norms.append(float(torch.nn.utils.clip_grad_norm_(model.parameters(), cfg.OPTIM.CLIP_GRAD_NORM)))
        optimizer.step()
        scheduler.step()
        losses.append(out["loss"].item())
        print(f"adamw trainer step {it} loss {losses[-1]:.6f} gnorm {norms[-1]:.4f}", flush=True)
    named = dict(model.named_parameters())
    final = {k: named[k].detach().double().norm().item() for k in state if not O.is_buffer(k)}
    bufs = dict(model.named_buffers())
    torch.save({"losses": torch.tensor(losses, dtype=torch.float64),
                "grad_norms": torch.tensor(norms, dtype=torch.float64),
                "final_param_norms": final,
                "final_probe": {k: named[k].detach().flatten()[:64].clone() for k in
                                ("visual.cnn.conv1.weight", "textual.embedding.words.weight",
                                 "textual.transformer.layers.0.linear1.weight")},
                "final_bn_running_var_stem": bufs["visual.cnn.bn1.running_var"].clone(),
                "spec": spec_kw, "seed": 3, "optim": dict(AO.OPTIM)},
               GOLDEN)


if __name__ == "__main__":
    main()
