"""Wide ResNet-50-2 / 101-2 backbones (the reference's R_50W2X ablation, `torchvision::wide_resnet50_2`) on the CPU:
the parameter tree against torchvision's, the shipped config and the factories, the float64 oracle against the
reference's own VirTexModel (tests/golden/r50w2x_l1_h128_post_b2.pt, written by scripts/make_wide_golden.py), and a dry run
of the engine's schedule for a wide model.  The oracle's parameter inventory is checked here against torchvision's for
every ResNet it states, basic-block ones included."""
import os

import pytest
import torch
import torchvision
from torch import nn

from oracle import virtex_oracle as O
from tests.test_engine_dryrun import _check_gemm, _model, _run


def _tv_backbone_sd(name):
    tv = getattr(torchvision.models, name)(weights=None)
    return {k: v for k, v in tv.state_dict().items() if not k.startswith("fc.")}


# -------------------------------------------------------------------------------------------------------- state dict
@pytest.mark.parametrize("name,n_keys", [("wide_resnet50_2", 318), ("wide_resnet101_2", 624)])
def test_state_dict_matches_torchvision_and_loads_both_ways(name, n_keys):
    from virtex_b200.modules import ResNetParams
    ours = ResNetParams(name)
    ref = _tv_backbone_sd(name)
    sd = ours.state_dict()
    assert len(sd) == len(ref) == n_keys
    assert list(sd) == list(ref)
    assert {k: tuple(v.shape) for k, v in sd.items()} == {k: tuple(v.shape) for k, v in ref.items()}
    # inner width = planes * 128 / 64, output width 4 * planes
    assert tuple(sd["layer1.0.conv2.weight"].shape) == (128, 128, 3, 3)
    assert tuple(sd["layer4.0.conv1.weight"].shape) == (1024, 1024, 1, 1)
    assert tuple(sd["layer4.2.conv3.weight"].shape) == (2048, 1024, 1, 1)
    ours.load_state_dict(ref, strict=True)
    assert torch.equal(ours.layer3[1].conv2.weight, ref["layer3.1.conv2.weight"])
    # the reverse: torchvision's model loads ours strictly once an fc is assigned
    ours.fc = nn.Linear(2048, 1000)
    tv = getattr(torchvision.models, name)(weights=None)
    tv.load_state_dict(ours.state_dict(), strict=True)
    assert torch.equal(tv.layer4[2].conv3.weight, ours.layer4[2].conv3.weight)


def test_resnet50_tree_is_unchanged():
    from virtex_b200.modules import ResNetParams
    sd = ResNetParams("resnet50").state_dict()
    ref = _tv_backbone_sd("resnet50")
    assert len(sd) == 318 and {k: tuple(v.shape) for k, v in sd.items()} == {k: tuple(v.shape) for k, v in ref.items()}
    assert tuple(sd["layer1.0.conv2.weight"].shape) == (64, 64, 3, 3)


def test_grouped_backbones_are_still_rejected():
    from virtex_b200.modules import ResNetParams
    with pytest.raises(KeyError, match="unsupported torchvision backbone"):
        ResNetParams("resnext50_32x4d")


# ------------------------------------------------------------------------------------------------ config / factories
def test_config_factory_and_optimizer_groups():
    from virtex_b200.config import Config
    from virtex_b200.factories import OptimizerFactory, PretrainingModelFactory
    cfg = Config("backbone_ablations/bicaptioning_R_50W2X_L1_H1024.yaml")
    assert cfg.MODEL.VISUAL.NAME == "torchvision::wide_resnet50_2"
    assert cfg.MODEL.TEXTUAL.NAME == "transdec_postnorm::L1_H1024_A16_F4096"
    model = PretrainingModelFactory.from_config(cfg)
    assert tuple(model.visual.cnn.layer2[0].conv2.weight.shape) == (256, 256, 3, 3)
    # a reference checkpoint of this config (TorchvisionVisualBackbone("wide_resnet50_2")) loads strictly
    spec = O.Spec(backbone="wide_resnet50_2")
    state = O.synth_state(spec, 0)
    model.load_state_dict(O.to_reference_state_dict(state, spec), strict=True)
    assert torch.equal(model.visual.cnn.layer4[0].conv2.weight, state["visual.cnn.layer4.0.conv2.weight"])
    named = list(model.named_parameters())
    opt = OptimizerFactory.from_config(cfg, named)
    groups = opt.param_groups if hasattr(opt, "param_groups") else opt.optimizer.param_groups
    assert len(groups) == len(named)
    for (name, _), group in zip(named, groups):
        assert group["lr"] == (cfg.OPTIM.CNN_LR if "cnn" in name else cfg.OPTIM.LR), name


# ------------------------------------------------------------------------------------------ oracle vs the reference
def _load(golden_dir):
    g = torch.load(os.path.join(golden_dir, "r50w2x_l1_h128_post_b2.pt"), weights_only=False)
    spec = O.Spec(**g["spec"])
    batch = O.synth_batch(max_len=spec.max_len, vocab=spec.vocab, **g["batch"])
    return g, spec, O.synth_state(spec, g["seed"]), batch


def test_oracle_train_forward_backward_f64(golden_dir):
    """float64 oracle == float64 reference VirTexModel with TorchvisionVisualBackbone("wide_resnet50_2")."""
    g, spec, state, batch = _load(golden_dir)
    assert spec.backbone == "wide_resnet50_2"
    out, grads, bufs = O.loss_and_grads(state, batch, spec, dtype=torch.float64)
    ref = g["f64"]
    assert abs(out["loss"].item() - ref["loss"].item()) < 1e-9
    assert abs(out["loss_components"]["captioning_forward"].item() - ref["loss_forward"].item()) < 1e-9
    assert abs(out["loss_components"]["captioning_backward"].item() - ref["loss_backward"].item()) < 1e-9
    names = ref["grads"]["names"]
    assert sorted(grads) == names
    norm = torch.tensor([grads[n].norm().item() for n in names], dtype=torch.float64)
    ssum = torch.tensor([grads[n].sum().item() for n in names], dtype=torch.float64)
    assert torch.allclose(norm, ref["grads"]["norm"], rtol=1e-7, atol=1e-12)
    assert ((ssum - ref["grads"]["sum"]).abs() <= 1e-6 * ref["grads"]["sum"].abs() + 1e-9 * (1 + norm)).all()
    for k, probe in ref["grad_probe"].items():
        assert torch.allclose(grads[k].flatten()[:64], probe, rtol=1e-7, atol=1e-12), k
    assert torch.allclose(bufs["visual.cnn.layer4.2.bn3.running_mean"], ref["bn_running_mean_layer4"], rtol=1e-9)
    assert torch.allclose(bufs["visual.cnn.bn1.running_var"], ref["bn_running_var_stem"], rtol=1e-9)


def test_oracle_train_loss_f32(golden_dir):
    g, spec, state, batch = _load(golden_dir)
    with torch.no_grad():
        out = O.model_forward(state, batch, spec, training=True)
    for tag in ("f32", "f64"):
        assert abs(out["loss"].item() - g[tag]["loss"].item()) < 2e-6 * g[tag]["loss"].item()


def test_oracle_eval_logits_and_argmax(golden_dir):
    g, spec, state, batch = _load(golden_dir)
    st64 = O.cast_state(state, torch.float64)
    b64 = dict(batch, image=batch["image"].double())
    with torch.no_grad():
        out = O.model_forward(st64, b64, spec, training=False, return_logits=True)
        out32 = O.model_forward(state, batch, spec, training=False)
    ref = g["f64"]
    assert abs(out["loss"].item() - ref["eval_loss"].item()) < 1e-9
    assert torch.equal(out["predictions"], ref["eval_predictions"])
    assert torch.allclose(out["logits"][:, :, :48], ref["eval_logits_slice"], rtol=1e-8, atol=1e-10)
    assert torch.allclose(out["logits"].max(-1).values, ref["eval_logits_max"], rtol=1e-8, atol=1e-10)
    assert torch.allclose(out["visual_features"][:, :32], ref["eval_visual_slice"], rtol=1e-8, atol=1e-10)
    assert torch.equal(out32["predictions"], g["f32"]["eval_predictions"])


@pytest.mark.parametrize("backbone", list(O._RESNET_LAYERS))
def test_oracle_backbone_shapes_are_torchvisions(backbone):
    shapes = O.backbone_param_shapes(O.Spec(backbone=backbone))
    tv = _tv_backbone_sd(backbone)
    assert list(shapes) == ["visual.cnn." + k for k in tv]
    assert {k[len("visual.cnn."):]: v for k, v in shapes.items()} == {k: tuple(v.shape) for k, v in tv.items()}


def test_wide_synth_state_covers_the_reference_key_set():
    spec = O.Spec(backbone="wide_resnet50_2", hidden=128, layers=1, heads=2, ffn=256)
    state = O.synth_state(spec, 0, bn3_gain=0.25)
    shapes = {**O.backbone_param_shapes(spec), **O.head_param_shapes(spec)}
    assert list(state) == list(shapes) and all(tuple(state[k].shape) == shapes[k] for k in state)
    assert torch.equal(state["textual.embedding.words.weight"],
                       O.synth_state(O.Spec(hidden=128, layers=1, heads=2, ffn=256), 0)["textual.embedding.words.weight"])
    assert float(state["visual.cnn.layer1.0.bn3.weight"].max()) <= 1.5 * 0.25


# --------------------------------------------------------------------------------------------------------- dry run
@pytest.fixture
def wide_dry(monkeypatch):
    """The launchers of virtex_b200.engine replaced by recorders that check every GEMM (tests/test_engine_dryrun.py)
    and keep its operands, so that each GEMM can be traced to the weight it reads."""
    from virtex_b200 import engine as E, ops
    calls = []

    def fake_call(name, *args):
        assert len(args) == len(ops._PROTOS[name]), name
        calls.append((name, args))

    def fake_gemm(A, B, D, M, N, K, **kw):
        _check_gemm(A, B, D, M, N, K, **{k: v for k, v in kw.items() if k not in ("col_scale", "col_shift")})
        calls.append(("gemm", (A, B, D, M, N, K, kw)))

    monkeypatch.setattr(E, "call", fake_call)
    monkeypatch.setattr(E, "gemm", fake_gemm)
    monkeypatch.setattr(E, "_stream", lambda: 0)
    monkeypatch.setattr(E, "_require_cuda", lambda dev: None)
    monkeypatch.setattr(ops, "num_sms", lambda: 132)
    return calls


def test_engine_schedule_of_a_wide_model(wide_dry):
    spec = O.Spec(backbone="wide_resnet50_2", hidden=128, layers=1, heads=2, ffn=256)
    model = _model(spec)
    batch = O.synth_batch(2, seed=0)
    eng = _run(model, batch)               # training forward + backward
    eng.backbone_infer(batch["image"])     # eval forward with folded BN
    bn = eng._bn_names()
    assert eng.ws.flat["bn_slab"].numel() == 4 * sum(C for _, C in bn)
    assert dict(bn)["visual.cnn.layer1.0.bn2"] == 128 and dict(bn)["visual.cnn.layer1.0.bn3"] == 256
    # trace every GEMM's B operand to the weight (or packed weight layout) it reads
    by_ptr = {eng.W(n).data_ptr(): n for n in eng.arena.names}
    by_ptr.update({t.data_ptr(): k for k, t in eng._packed.items()})
    gemms = [c[1] for c in wide_dry if c[0] == "gemm"]
    assert not [g for g in gemms if g[6].get("conv_mode", 0) == 4]  # conv_mode 4 is for 64-channel 3x3 convs only
    seen = {"conv2": 0, "conv3": 0}
    for name, blk in eng.blocks:
        width, C4 = blk.conv1.weight.shape[0], blk.conv3.weight.shape[0]
        planes = C4 // 4
        assert width == 2 * planes
        for A, B, D, M, N, K, kw in gemms:
            src = by_ptr.get(B.data_ptr())
            if src == name + ".conv2.weight":              # conv2 fprop (training and eval)
                assert (N, K) == (width, 9 * width) and kw.get("conv_mode") == 1
                seen["conv2"] += 1
            elif src == name + ".conv3.weight" and not kw.get("b_mn"):  # conv3 fprop
                assert (N, K) == (C4, width)
                seen["conv3"] += 1
            elif src == name + ".conv3.weight":            # conv3 dgrad
                assert (N, K) == (width, C4)
    assert seen == {"conv2": 2 * len(eng.blocks), "conv3": 2 * len(eng.blocks)}
    # conv2 wgrads: split-K implicit (conv_mode 2) into [width, 9 * width]
    wg = [g for g in gemms if g[6].get("conv_mode") == 2 and g[6].get("conv_taps", 0) != 1]
    assert sorted({(g[3], g[4]) for g in wg}) == [(w, 9 * w) for w in (128, 256, 512, 1024)]
    assert len(wg) == len(eng.blocks)
    # the 3x3 unpack jobs of every bucket read the conv_mode 2 layout (kind 2), never the transposed one (kind 3)
    for layer in ("layer1", "layer2", "layer3", "layer4"):
        rows = eng._unpack_rows("rest" if layer == "layer1" else layer, True)
        assert all(r[8] == 2 for r in rows if r[5] == 3), layer
