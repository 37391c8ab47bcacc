"""ResNet-18 / ResNet-34 backbones (`torchvision::resnet18` / `resnet34` with MODEL.VISUAL.FEATURE_SIZE 512) on the
CPU: the parameter tree against torchvision's, the config and the factories, the float64 oracle against the
reference's own VirTexModel (tests/golden/r18_l1_h128_post_b2.pt, written by scripts/make_basic_golden.py), and a dry
run of the engine's basic-block schedule (training forward, backward and the folded-BN eval forward)."""
import os

import pytest
import torch
import torchvision
from torch import nn

from oracle import virtex_oracle as O
from tests.test_engine_dryrun import _check_gemm, _model, _run

BF16 = torch.bfloat16


def _tv_backbone_sd(name):
    tv = getattr(torchvision.models, name)(weights=None)
    return {k: v for k, v in tv.state_dict().items() if not k.startswith("fc.")}


# -------------------------------------------------------------------------------------------------------- state dict
@pytest.mark.parametrize("name,n_keys", [("resnet18", 120), ("resnet34", 216)])
def test_state_dict_matches_torchvision_and_loads_both_ways(name, n_keys):
    from virtex_b200.modules import BasicBlock, ResNetParams
    ours = ResNetParams(name)
    assert ours.out_channels == 512 and all(isinstance(b, BasicBlock) for b in ours.layer3)
    ref = _tv_backbone_sd(name)
    sd = ours.state_dict()
    assert len(sd) == len(ref) == n_keys
    assert list(sd) == list(ref)
    assert {k: tuple(v.shape) for k, v in sd.items()} == {k: tuple(v.shape) for k, v in ref.items()}
    assert tuple(sd["layer2.0.conv1.weight"].shape) == (128, 64, 3, 3)
    assert tuple(sd["layer4.0.downsample.0.weight"].shape) == (512, 256, 1, 1)
    assert "layer1.0.downsample.0.weight" not in sd
    ours.load_state_dict(ref, strict=True)
    assert torch.equal(ours.layer3[1].conv2.weight, ref["layer3.1.conv2.weight"])
    # the reverse: torchvision's model loads ours strictly once an fc is assigned
    ours.fc = nn.Linear(512, 1000)
    tv = getattr(torchvision.models, name)(weights=None)
    tv.load_state_dict(ours.state_dict(), strict=True)
    assert torch.equal(tv.layer4[1].conv2.weight, ours.layer4[1].conv2.weight)
    assert torch.equal(tv.fc.weight, ours.fc.weight)


@pytest.mark.parametrize("name", ["resnet18", "resnet34"])
def test_init_is_torchvisions_with_zero_init_residual(name):
    from virtex_b200.modules import ResNetParams
    torch.manual_seed(0)
    ours = ResNetParams(name, zero_init_residual=True)
    for li in range(1, 5):
        for blk in getattr(ours, f"layer{li}"):
            assert torch.count_nonzero(blk.bn2.weight) == 0 and torch.all(blk.bn1.weight == 1)
            assert torch.all(blk.bn2.bias == 0)
            if blk.downsample is not None:
                assert torch.all(blk.downsample[1].weight == 1)
            # kaiming_normal_(fan_out): std sqrt(2 / (out_channels * 9))
            w = blk.conv2.weight
            assert abs(w.std().item() / (2.0 / (w.shape[0] * 9)) ** 0.5 - 1) < 0.1
    assert torch.count_nonzero(ResNetParams(name, zero_init_residual=False).layer1[0].bn2.weight) == 64


def test_feature_size_must_match_the_backbone():
    from virtex_b200.modules import TorchvisionVisualBackbone
    with pytest.raises(ValueError, match="MODEL.VISUAL.FEATURE_SIZE"):
        TorchvisionVisualBackbone("resnet18")               # default visual_feature_size 2048
    with pytest.raises(ValueError, match="MODEL.VISUAL.FEATURE_SIZE"):
        TorchvisionVisualBackbone("resnet34", visual_feature_size=1024)
    assert TorchvisionVisualBackbone("resnet34", visual_feature_size=512).cnn.out_channels == 512
    # bottleneck names keep their behaviour: no check of the feature size
    assert TorchvisionVisualBackbone("resnet50", visual_feature_size=512).visual_feature_size == 512


# ------------------------------------------------------------------------------------------------ config / factories
@pytest.mark.parametrize("name", ["resnet18", "resnet34"])
def test_config_factory_and_optimizer_groups(name):
    from virtex_b200.config import Config
    from virtex_b200.factories import OptimizerFactory, PretrainingModelFactory
    cfg = Config("_base_bicaptioning_R_50_L1_H1024.yaml",
                 ["MODEL.VISUAL.NAME", f"torchvision::{name}", "MODEL.VISUAL.FEATURE_SIZE", 512])
    model = PretrainingModelFactory.from_config(cfg)
    assert tuple(model.visual.cnn.layer2[0].conv1.weight.shape) == (128, 64, 3, 3)
    assert tuple(model.textual.visual_projection.weight.shape) == (1024, 512)
    spec = O.Spec(backbone=name)
    state = O.synth_state(spec, 0)
    model.load_state_dict(O.to_reference_state_dict(state, spec), strict=True)
    assert torch.equal(model.visual.cnn.layer4[0].conv1.weight, state["visual.cnn.layer4.0.conv1.weight"])
    named = list(model.named_parameters())
    opt = OptimizerFactory.from_config(cfg, named)
    groups = opt.param_groups if hasattr(opt, "param_groups") else opt.optimizer.param_groups
    assert len(groups) == len(named)
    for (pname, _), group in zip(named, groups):
        assert group["lr"] == (cfg.OPTIM.CNN_LR if "cnn" in pname else cfg.OPTIM.LR), pname
    with pytest.raises(ValueError, match="MODEL.VISUAL.FEATURE_SIZE"):
        PretrainingModelFactory.from_config(Config("_base_bicaptioning_R_50_L1_H1024.yaml",
                                                   ["MODEL.VISUAL.NAME", f"torchvision::{name}"]))


# ------------------------------------------------------------------------------------------ oracle vs the reference
def _load(golden_dir):
    g = torch.load(os.path.join(golden_dir, "r18_l1_h128_post_b2.pt"), weights_only=False)
    spec = O.Spec(**g["spec"])
    batch = O.synth_batch(max_len=spec.max_len, vocab=spec.vocab, **g["batch"])
    return g, spec, O.synth_state(spec, g["seed"]), batch


def test_oracle_train_forward_backward_f64(golden_dir):
    """float64 oracle == float64 reference VirTexModel with TorchvisionVisualBackbone("resnet18", 512)."""
    g, spec, state, batch = _load(golden_dir)
    assert spec.backbone == "resnet18"
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
    assert torch.allclose(bufs["visual.cnn.layer4.1.bn2.running_mean"], ref["bn_running_mean_layer4"], rtol=1e-9)
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
    assert out["visual_features"].shape[1] == 512
    assert abs(out["loss"].item() - ref["eval_loss"].item()) < 1e-9
    assert torch.equal(out["predictions"], ref["eval_predictions"])
    assert torch.allclose(out["logits"][:, :, :48], ref["eval_logits_slice"], rtol=1e-8, atol=1e-10)
    assert torch.allclose(out["logits"].max(-1).values, ref["eval_logits_max"], rtol=1e-8, atol=1e-10)
    assert torch.allclose(out["visual_features"][:, :32], ref["eval_visual_slice"], rtol=1e-8, atol=1e-10)
    assert torch.equal(out32["predictions"], g["f32"]["eval_predictions"])


def test_basic_synth_state_covers_the_reference_key_set():
    spec = O.Spec(backbone="resnet34", hidden=128, layers=1, heads=2, ffn=256)
    state = O.synth_state(spec, 0, bn3_gain=0.25)
    shapes = {**O.backbone_param_shapes(spec), **O.head_param_shapes(spec)}
    assert list(state) == list(shapes) and all(tuple(state[k].shape) == shapes[k] for k in state)
    assert shapes["textual.visual_projection.weight"] == (128, 512)
    assert float(state["visual.cnn.layer1.0.bn2.weight"].max()) <= 1.5 * 0.25
    assert float(state["visual.cnn.layer1.0.bn1.weight"].min()) >= 0.5


# --------------------------------------------------------------------------------------------------------- dry run
def _check_basic_gemm(A, B, D, M, N, K, **kw):
    """tests/test_engine_dryrun.py's operand checks, plus the bit masks that vtx_gemm also takes on conv_mode 1
    outputs without an output view (row m = the NHWC output pixel, [M, N/8] bytes)."""
    kw = {k: v for k, v in kw.items() if k not in ("col_scale", "col_shift")}
    rmask, bnr = kw.get("residual_mask"), kw.get("bnr")
    if kw.get("conv_mode", 0) == 1 and (rmask is not None or (bnr is not None and bnr[3] is not None)):
        assert kw.get("out_view") is None and D.dtype == BF16 and N % 32 == 0
        if rmask is not None:
            assert kw.get("residual") is not None and rmask.dtype == torch.uint8 and rmask.numel() >= M * N // 8
        if bnr is not None and bnr[3] is not None:
            assert bnr[3].dtype == torch.uint8 and bnr[3].numel() >= M * N // 8 and len(bnr) == 4
        kw = dict(kw, residual_mask=None, bnr=None if bnr is None else (*bnr[:3], None))
    _check_gemm(A, B, D, M, N, K, **kw)


@pytest.fixture
def basic_dry(monkeypatch):
    from virtex_b200 import engine as E, ops
    calls = []

    def fake_call(name, *args):
        assert len(args) == len(ops._PROTOS[name]), name
        calls.append((name, args))

    def fake_gemm(A, B, D, M, N, K, **kw):
        _check_basic_gemm(A, B, D, M, N, K, **kw)
        calls.append(("gemm", (A, B, D, M, N, K, kw)))

    monkeypatch.setattr(E, "call", fake_call)
    monkeypatch.setattr(E, "gemm", fake_gemm)
    monkeypatch.setattr(E, "_stream", lambda: 0)
    monkeypatch.setattr(E, "_require_cuda", lambda dev: None)
    monkeypatch.setattr(ops, "num_sms", lambda: 132)
    return calls


@pytest.mark.parametrize("backbone", ["resnet18", "resnet34"])
@pytest.mark.parametrize("fuse", [False, True])
def test_engine_schedule_of_a_basic_block_model(basic_dry, monkeypatch, backbone, fuse):
    from virtex_b200.engine import Engine
    if fuse:  # the previous block's bn2 sums in every identity block's conv1 dgrad
        monkeypatch.setattr(Engine, "fuse_bn3_min_rows", 0)
    spec = O.Spec(backbone=backbone, hidden=128, layers=1, heads=2, ffn=256)
    model = _model(spec)
    batch = O.synth_batch(2, seed=0)
    eng = _run(model, batch)               # training forward + backward
    n_train = len(basic_dry)
    eng.backbone_infer(batch["image"])     # eval forward with folded BN
    bn = eng._bn_names()
    nb = sum(spec.blocks)
    assert len(bn) == 1 + 2 * nb + 3 and all(not n.endswith(".bn3") for n, _ in bn)
    assert eng.ws.flat["bn_slab"].numel() == 4 * sum(C for _, C in bn)
    assert eng._tape["feat"].shape == (2 * 7 * 7, 512)
    by_ptr = {eng.W(n).data_ptr(): n for n in eng.arena.names}
    by_ptr.update({t.data_ptr(): k for k, t in eng._packed.items()})
    gemms = [c[1] for c in basic_dry[:n_train] if c[0] == "gemm"]
    infer = [c[1] for c in basic_dry[n_train:] if c[0] == "gemm"]
    ident = [(n, b) for n, b in eng.blocks if b.downsample is None]
    # every 3x3 conv: one implicit fprop in training and one in eval, reading its packed [C, 9 * Cin] weight
    for name, blk in eng.blocks:
        for conv in ("conv1", "conv2"):
            C, Cin = getattr(blk, conv).weight.shape[:2]
            fp = [g for g in gemms + infer if by_ptr.get(g[1].data_ptr()) == f"{name}.{conv}.weight"]
            assert len(fp) == 2 and all((g[4], g[5], g[6]["conv_mode"]) == (C, 9 * Cin, 1) for g in fp), (name, conv)
            assert fp[0][6]["conv_stride"] == (blk.stride if conv == "conv1" else 1)
    # wgrads: conv_mode 4 for the 64 -> 64 convs of layer1, split-K conv_mode 2 into [C, 9 * Cin] otherwise
    assert len([g for g in gemms if g[6].get("conv_mode") == 4]) == 2 * spec.blocks[0]
    wg = [g for g in gemms if g[6].get("conv_mode") == 2 and g[6].get("conv_taps", 0) != 1]
    assert len(wg) == 2 * nb - 2 * spec.blocks[0]
    assert {(g[3], g[4]) for g in wg} == {(128, 9 * 64), (128, 9 * 128), (256, 9 * 128), (256, 9 * 256),
                                          (512, 9 * 256), (512, 9 * 512)}
    # identity blocks: conv1's dgrad adds the shortcut gradient under the block's bit mask (never written), and
    # accumulates the previous identity block's bn2 sums under that block's mask when fused
    masked = [g for g in gemms if g[6].get("residual_mask") is not None]
    assert len(masked) == len(ident) and all(g[6]["conv_mode"] == 1 and g[5] == 9 * g[4] for g in masked)
    for (name, blk), g in zip(reversed(ident), masked):
        assert by_ptr[g[1].data_ptr()] == name + ".conv1.weight#dgrad"
        assert g[6]["residual_mask"].data_ptr() == eng.ws.flat[name + ".m2"].data_ptr()
    fused = [g for g in masked if g[6].get("bnr") is not None]
    prev_ident = [i for i, (n, b) in enumerate(eng.blocks) if b.downsample is None and i > 0
                  and eng.blocks[i - 1][1].downsample is None]
    assert len(fused) == (len(prev_ident) if fuse else 0)
    assert all(g[6]["bnr"][3] is not None for g in fused)
    names = [c[0] for c in basic_dry[:n_train]]
    assert names.count("vtx_bn_bwd_reduce") == 1 + nb - len(fused)
    assert names.count("vtx_bn_bwd_finalize_apply") == 1 + 2 * nb
    # downsample blocks: four parity-class dgrads of conv1 with [Cin, taps * C] slices, then the shortcut's
    for name, blk in eng.blocks:
        if blk.downsample is None:
            continue
        C, Cin = blk.conv1.weight.shape[:2]
        par = [g for g in gemms if (by_ptr.get(g[1].data_ptr()) or "").startswith(name + ".conv1.weight#dgrad_s2")]
        assert sorted(g[5] for g in par) == [C, 2 * C, 2 * C, 4 * C] and all(g[4] == Cin for g in par)
        assert all(g[6].get("out_view") is not None and g[6].get("bnr") is None for g in par)
    # eval forward: identity blocks run two GEMMs, downsample blocks three; conv2 adds the shortcut
    assert len(infer) == 1 + 2 * nb + 3
    # the 3x3 unpack jobs: transposed layout (kind 3) for layer1 only, [C, 9 * Cin] (kind 2) elsewhere
    for layer, kinds in (("rest", {3, 5}), ("layer2", {2}), ("layer3", {2}), ("layer4", {2})):
        rows = eng._unpack_rows(layer, True)
        assert {r[8] for r in rows} == kinds and len([r for r in rows if r[5] == 3]) == 2 * spec.blocks[
            {"rest": 0, "layer2": 1, "layer3": 2, "layer4": 3}[layer]]
