"""Generate tests/golden/*.pt by running the UNMODIFIED reference (a checkout named by $VIRTEX_REFERENCE_ROOT).

    python -m oracle.make_golden

Every fixture is produced from (spec, seed) through `oracle.virtex_oracle.synth_state/synth_batch`, so only the
reference's *outputs* are stored (small files).  Ground truth is the reference run in float64 (its own float32 run
differs from float64 by ~2e-2 in backbone gradients at batch 2 -- batch-norm over 98 samples through 16 blocks is
ill-conditioned -- so float32-vs-float32 comparisons cannot pin anything tighter than that); float32 outputs are
stored as well.
"""
import os
import sys
import warnings

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import ref_shim, virtex_oracle as O  # noqa: E402

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden")

CASES = {
    # name: (spec kwargs, batch kwargs, state seed)
    "r50_l1_h1024_post_b2": (dict(), dict(batch_size=2, seed=0, ragged=False), 0),
    "r50_l2_h256_pre_b3_ragged": (dict(hidden=256, layers=2, heads=4, ffn=512, norm_first=True),
                                  dict(batch_size=3, seed=1, ragged=True), 1),
    "r50_l1_h128_post_b4_ragged": (dict(hidden=128, layers=1, heads=2, ffn=256), dict(batch_size=4, seed=2, ragged=True), 2),
    # the architectures of BASELINE.json configs #4 / #5 (SURVEY 8: C4 = R50-L4-H1024, C5 = R101-L1-H2048)
    "r50_l4_h1024_post_b2_ragged": (dict(layers=4), dict(batch_size=2, seed=3, ragged=True), 3),
    "r101_l1_h2048_post_b2": (dict(backbone="resnet101", hidden=2048, heads=32, ffn=8192),
                              dict(batch_size=2, seed=4, ragged=False), 4),
}


def build_reference_model(spec: O.Spec):
    from virtex.models import VirTexModel
    from virtex.modules.textual_heads import TransformerDecoderTextualHead
    from virtex.modules.visual_backbones import TorchvisionVisualBackbone

    visual = TorchvisionVisualBackbone(spec.backbone, visual_feature_size=spec.visual_feature_size)
    textual = TransformerDecoderTextualHead(
        visual_feature_size=spec.visual_feature_size, vocab_size=spec.vocab, hidden_size=spec.hidden,
        num_layers=spec.layers, attention_heads=spec.heads, feedforward_size=spec.ffn, dropout=0.0,
        norm_first=spec.norm_first, mask_future_positions=True, max_caption_length=spec.max_len,
        padding_idx=spec.pad)
    return VirTexModel(visual, textual)


def grad_summary(grads):
    names = sorted(grads)
    return {"names": names,
            "norm": torch.tensor([grads[n].double().norm().item() for n in names], dtype=torch.float64),
            "sum": torch.tensor([grads[n].double().sum().item() for n in names], dtype=torch.float64)}


def run_case(name, spec_kw, batch_kw, seed):
    spec = O.Spec(**spec_kw)
    state = O.synth_state(spec, seed)
    batch = O.synth_batch(max_len=spec.max_len, vocab=spec.vocab, **batch_kw)
    out = {"spec": spec_kw, "batch": batch_kw, "seed": seed}
    for tag, dtype in (("f64", torch.float64), ("f32", torch.float32)):
        model = build_reference_model(spec)
        model.load_state_dict(O.to_reference_state_dict(state, spec), strict=True)
        model = model.to(dtype)
        b = dict(batch)
        b["image"] = batch["image"].to(dtype)
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
               "grad_probe": {k: grads[k].detach().flatten()[:64].clone() for k in
                              ("visual.cnn.conv1.weight", "visual.cnn.layer4.2.conv3.weight",
                               "textual.embedding.words.weight", "textual.visual_projection.weight",
                               "backward_textual.transformer.layers.0.self_attn.in_proj_weight")},
               "bn_running_mean_layer4": bufs["visual.cnn.layer4.2.bn3.running_mean"].clone(),
               "bn_running_var_stem": bufs["visual.cnn.bn1.running_var"].clone(),
               "num_batches_tracked": bufs["visual.cnn.bn1.num_batches_tracked"].clone()}
        # eval-mode pass with the ORIGINAL buffers (reload the state)
        model.load_state_dict(O.to_reference_state_dict(O.cast_state(state, dtype), spec), strict=True)
        model.eval()
        with torch.no_grad():
            ev = model(b)
            vf = model.visual(b["image"])
            logits = model.textual(vf, b["caption_tokens"], b["caption_lengths"])
        rec["eval_loss"] = ev["loss"].double()
        rec["eval_predictions"] = ev["predictions"].clone()
        rec["eval_logits_slice"] = logits[:, :, :48].clone()
        rec["eval_logits_max"] = logits.max(dim=-1).values.clone()
        rec["eval_visual_slice"] = vf[:, :32].clone()
        out[tag] = rec
        print(f"{name} [{tag}] loss {rec['loss'].item():.9f} eval {rec['eval_loss'].item():.9f}", flush=True)
    torch.save(out, os.path.join(GOLDEN_DIR, name + ".pt"))


def run_masked_lm_case():
    """The masked-LM sibling (virtex/models/masked_lm.py:35-86) through the reference's own MaskedLMModel and a head
    built with mask_future_positions=False: loss, gradient summaries, eval predictions."""
    from virtex.models import MaskedLMModel
    from virtex.modules.textual_heads import TransformerDecoderTextualHead
    from virtex.modules.visual_backbones import TorchvisionVisualBackbone
    spec_kw = dict(hidden=128, layers=1, heads=2, ffn=256, caption_backward=False, mask_future=False)
    spec = O.Spec(**spec_kw)
    state = O.synth_state(spec, 31)
    batch = O.synth_masked_batch(3, seed=21)
    out = {"spec": spec_kw, "seed": 31, "batch_seed": 21}
    for tag, dtype in (("f64", torch.float64), ("f32", torch.float32)):
        visual = TorchvisionVisualBackbone(spec.backbone, visual_feature_size=spec.visual_feature_size)
        textual = TransformerDecoderTextualHead(
            visual_feature_size=spec.visual_feature_size, vocab_size=spec.vocab, hidden_size=spec.hidden,
            num_layers=spec.layers, attention_heads=spec.heads, feedforward_size=spec.ffn, dropout=0.0,
            norm_first=False, mask_future_positions=False, max_caption_length=spec.max_len, padding_idx=spec.pad)
        model = MaskedLMModel(visual, textual)
        sd = {k: v for k, v in O.to_reference_state_dict(state, spec).items() if not k.startswith("backward_textual.")}
        model.load_state_dict(sd, strict=True)
        model = model.to(dtype)
        b = dict(batch)
        b["image"] = batch["image"].to(dtype)
        model.train()
        res = model(b)
        res["loss"].backward()
        named = dict(model.named_parameters())
        grads = {k: named[k].grad for k in named}
        rec = {"loss": res["loss"].detach().double(), "grads": grad_summary(grads)}
        model.load_state_dict({k: (v.to(dtype) if v.is_floating_point() else v) for k, v in sd.items()}, strict=True)
        model.eval()
        with torch.no_grad():
            ev = model(b)
        rec["eval_loss"] = ev["loss"].double()
        rec["eval_predictions"] = ev["predictions"].clone()
        out[tag] = rec
        print(f"masked_lm [{tag}] loss {rec['loss'].item():.9f} eval {rec['eval_loss'].item():.9f}", flush=True)
    torch.save(out, os.path.join(GOLDEN_DIR, "masked_lm_r50_l1_h128_b3.pt"))


def run_trainer_case():
    """6 optimiser steps (crosses the Lookahead k=5 boundary) through the reference's own factories + loop body."""
    from virtex.config import Config
    from virtex.factories import LRSchedulerFactory, OptimizerFactory, PretrainingModelFactory

    over = ["MODEL.TEXTUAL.NAME", "transdec_postnorm::L1_H128_A2_F256", "MODEL.TEXTUAL.DROPOUT", 0.0,
            "OPTIM.WARMUP_STEPS", 3, "OPTIM.NUM_ITERATIONS", 20, "OPTIM.BATCH_SIZE", 2, "OPTIM.CNN_LR", 0.005]
    cfg = Config(os.path.join(ref_shim.REFERENCE_ROOT, "configs", "_base_bicaptioning_R_50_L1_H1024.yaml"), over)
    spec = O.Spec(hidden=128, layers=1, heads=2, ffn=256)
    state = O.synth_state(spec, 3)
    model = PretrainingModelFactory.from_config(cfg)
    model.load_state_dict(O.to_reference_state_dict(state, spec), strict=True)
    optimizer = OptimizerFactory.from_config(cfg, model.named_parameters())
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
        print(f"trainer step {it} loss {losses[-1]:.6f} gnorm {norms[-1]:.4f}", flush=True)
    named = dict(model.named_parameters())
    final = {k: named[k].detach().double().norm().item() for k in state if not O.is_buffer(k)}
    bufs = dict(model.named_buffers())
    torch.save({"losses": torch.tensor(losses, dtype=torch.float64), "grad_norms": torch.tensor(norms, dtype=torch.float64),
                "final_param_norms": final,
                "final_probe": {k: named[k].detach().flatten()[:64].clone() for k in
                                ("visual.cnn.conv1.weight", "textual.embedding.words.weight",
                                 "textual.transformer.layers.0.linear1.weight")},
                "final_bn_running_var_stem": bufs["visual.cnn.bn1.running_var"].clone(),
                "spec": dict(hidden=128, layers=1, heads=2, ffn=256), "seed": 3,
                "optim": dict(warmup_steps=3, num_iterations=20, cnn_lr=0.005)},
               os.path.join(GOLDEN_DIR, "trainer_r50_l1_h128_6steps.pt"))


def main():
    if not ref_shim.available():
        raise SystemExit("reference tree not found: set VIRTEX_REFERENCE_ROOT to a checkout of the reference")
    warnings.filterwarnings("ignore")
    ref_shim.install()
    os.makedirs(GOLDEN_DIR, exist_ok=True)
    torch.manual_seed(0)
    only = sys.argv[1:]
    for name, (spec_kw, batch_kw, seed) in CASES.items():
        if not only or name in only:
            run_case(name, spec_kw, batch_kw, seed)
    if not only or "masked_lm" in only:
        run_masked_lm_case()
    if not only or "trainer" in only:
        run_trainer_case()


if __name__ == "__main__":
    main()
