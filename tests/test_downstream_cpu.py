"""Downstream classification evaluations (scripts/clf_linear.py, scripts/clf_voc07.py) without a GPU: the float64 oracle
against the reference's own torchvision ResNet-50 (tests/golden/downstream_r50_fc10.pt), the torchvision-like module
surface of ResNetParams, the downstream configs with the reference's optimiser / scheduler / checkpoint code, a dry run
of Engine.backbone_infer and of ResNetParams.forward that checks every launch against its header prototype, and the
host's rejection of scale / shift epilogue combinations it does not implement."""
import ctypes
import os

import pytest
import torch
from torch import nn

from tests import downstream_oracle as DO

BF16, F32 = torch.bfloat16, torch.float32


def _golden(golden_dir):
    return torch.load(os.path.join(golden_dir, DO.GOLDEN), weights_only=False)


def _close(a, b, rtol=1e-9, atol=1e-12):
    assert torch.allclose(a.double(), b.double(), rtol=rtol, atol=atol), (a.flatten()[:4], b.flatten()[:4])


# ------------------------------------------------------------------------------------------------------ oracle vs golden
@pytest.mark.parametrize("case", list(DO.CASES))
def test_oracle_matches_the_reference_resnet(golden_dir, case):
    g = _golden(golden_dir)[case]
    state, batch = DO.case_inputs(case)
    pooled, logits, loss, grads, _ = DO.run(state, batch, training=False, frozen=True)
    ev = g["eval"]
    _close(pooled, ev["pooled"], rtol=1e-6, atol=1e-7)  # the fixture stores fp32 features
    _close(logits, ev["logits"])
    _close(loss, ev["loss"])
    _close(grads["fc.weight"].flatten()[:64], ev["fc.weight.grad"])
    _close(grads["fc.weight"].norm(), ev["fc.weight.grad_norm"])
    _close(grads["fc.bias"], ev["fc.bias.grad"])
    assert set(grads) == {"fc.weight", "fc.bias"}
    _, logits, loss, grads, nb = DO.run(state, batch, training=True)
    tr = g["train"]
    _close(logits, tr["logits"], rtol=1e-8, atol=1e-10)
    _close(loss, tr["loss"], rtol=1e-8)
    _close(grads["fc.bias"], tr["fc.bias.grad"], rtol=1e-7, atol=1e-12)
    for k in DO.CONV_PROBES:
        _close(grads[k].flatten()[:64], tr[k + ".grad"], rtol=1e-6, atol=1e-12)
        _close(grads[k].norm(), tr[k + ".grad_norm"], rtol=1e-7)
    for k in DO.BN_PROBES:
        for leaf in ("weight", "bias"):
            _close(grads[f"{k}.{leaf}"].flatten()[:64], tr[f"{k}.{leaf}.grad"], rtol=1e-6, atol=1e-12)
        for leaf in ("running_mean", "running_var"):
            _close(nb[f"{k}.{leaf}"].flatten()[:64], tr[f"{k}.{leaf}"])
        assert int(nb[f"{k}.num_batches_tracked"]) == int(tr[f"{k}.num_batches_tracked"]) == 1


# ------------------------------------------------------------------------------------------------------ module surface
def _cnn(num_classes=DO.NUM_CLASSES):
    from virtex_b200.modules import ResNetParams
    cnn = ResNetParams("resnet50")
    if num_classes:
        cnn.fc = nn.Linear(2048, num_classes)
    return cnn


def test_state_dict_interchanges_with_torchvision_resnet50_strictly():
    import torchvision
    ours = _cnn()
    tv = torchvision.models.resnet50(num_classes=DO.NUM_CLASSES)
    assert isinstance(ours.avgpool, nn.AdaptiveAvgPool2d) and ours.avgpool.output_size == (1, 1)
    assert list(ours.state_dict()) == list(tv.state_dict())
    state = DO.synth_state(3)
    ours.load_state_dict(state, strict=True)
    tv.load_state_dict(ours.state_dict(), strict=True)
    ours2 = _cnn()
    ours2.load_state_dict(tv.state_dict(), strict=True)
    for k, v in state.items():
        assert torch.equal(ours2.state_dict()[k], v), k
    # without fc (pretraining): the keys of the reference's visual.cnn, fc.* absent
    assert not any(k.startswith(("fc.", "avgpool")) for k in _cnn(0).state_dict())


def test_optimizer_grouping_scheduler_and_checkpoint_with_frozen_parameters(tmp_path):
    """clf_linear.py's set-up on the module: frozen backbone parameters stay in named_parameters()."""
    from virtex_b200.config import Config
    from virtex.factories import LRSchedulerFactory, OptimizerFactory
    from virtex.utils.checkpointing import CheckpointManager
    for name, frozen in (("imagenet_clf", True), ("inaturalist_clf", False)):
        cfg = Config(f"downstream/{name}.yaml")
        assert bool(cfg.MODEL.VISUAL.FROZEN) == frozen
        model = _cnn()
        if frozen:
            model.eval()
            for n, p in model.named_parameters():
                if "fc" not in n:
                    p.requires_grad = False
        opt = OptimizerFactory.from_config(cfg, model.named_parameters())
        assert sum(len(g["params"]) for g in opt.param_groups) == len(list(model.parameters()))
        assert all(g["lr"] == cfg.OPTIM.LR for g in opt.param_groups)
        wd = {g["weight_decay"] for g in opt.param_groups}
        assert wd == {cfg.OPTIM.WEIGHT_DECAY}, wd
        sched = LRSchedulerFactory.from_config(cfg, opt)
        model.fc.weight.grad = torch.ones_like(model.fc.weight)
        model.fc.bias.grad = torch.ones_like(model.fc.bias)
        w0 = model.fc.weight.detach().clone()
        frozen_before = model.conv1.weight.detach().clone()
        opt.step()
        sched.step()
        assert not torch.equal(model.fc.weight, w0)
        assert torch.equal(model.conv1.weight, frozen_before)
        ckpt = CheckpointManager(str(tmp_path / name), model=model, optimizer=opt, scheduler=sched)
        ckpt.step(1)
        fresh = _cnn()
        CheckpointManager(model=fresh).load(str(tmp_path / name / "checkpoint_1.pth"))
        assert torch.equal(fresh.fc.weight, model.fc.weight)
    cfg = Config("downstream/inaturalist_clf.yaml")
    assert cfg.OPTIM.LR_DECAY_NAME == "multistep" and list(cfg.OPTIM.LR_STEPS) == [119700, 153900]
    sched = LRSchedulerFactory.from_config(cfg, torch.optim.SGD([nn.Parameter(torch.zeros(1))], lr=cfg.OPTIM.LR))
    assert sched.lr_lambdas[0](119699) == 1.0 and abs(sched.lr_lambdas[0](119700) - 0.1) < 1e-12
    voc = Config("downstream/voc07_clf.yaml")
    assert voc.OPTIM.BATCH_SIZE == 128 and voc.DATA.ROOT == "datasets/VOC2007"


# ------------------------------------------------------------------------------------------------------ dry run
def _check_ss_gemm(A, B, D, M, N, K, col_scale=None, col_shift=None, act=0, residual=None, conv=None, conv_mode=0,
                   conv_stride=1, conv_taps=0, lda=None, ldb=None, bias=None, stats=None, a_mn=0, b_mn=0, tap_grid=None, **kw):
    assert A.dtype == BF16 and B.dtype == BF16 and M > 0 and N > 0 and K > 0
    assert (col_scale is None) == (col_shift is None)
    if col_scale is not None:  # the host's conditions for the scale / shift epilogue
        assert D.dtype == BF16 and bias is None and stats is None and kw.get("bnr") is None and act in (0, 1)
        assert N % 2 == 0 and conv_mode in (0, 1) and kw.get("out_view") is None and kw.get("residual_mask") is None
        for v in (col_scale, col_shift):
            assert v.dtype == F32 and v.numel() == N and v.is_contiguous() and (v.data_ptr() % 8 == 0)
        if residual is not None:
            assert residual.dtype == BF16 and residual.numel() >= M * N and residual.stride(0) % 8 == 0
    if conv_mode == 1:
        NI, H, W, C = conv
        taps = 1 if conv_taps == 1 else (tap_grid[0] * tap_grid[1] if tap_grid is not None else 9)
        Ho, Wo = (H - 1) // conv_stride + 1, (W - 1) // conv_stride + 1
        assert M == NI * Ho * Wo and K == taps * C and A.numel() >= NI * H * W * C and B.numel() >= N * K
    elif conv_mode == 0:
        lda = A.stride(0) if lda is None else lda
        ldb = B.stride(0) if ldb is None else ldb
        assert A.numel() >= ((K - 1) * lda + M if a_mn else (M - 1) * lda + K), "A too small"
        assert B.numel() >= ((K - 1) * ldb + N if b_mn else (N - 1) * ldb + K), "B too small"
    assert D.numel() >= M * N


@pytest.fixture
def dry(monkeypatch):
    from virtex_b200 import engine as E, ops
    calls = []

    def fake_call(name, *args):
        assert len(args) == len(ops._PROTOS[name]), (name, len(args), len(ops._PROTOS[name]))
        calls.append(name)

    def fake_gemm(A, B, D, M, N, K, **kw):
        _check_ss_gemm(A, B, D, M, N, K, **kw)
        calls.append(("gemm", M, N, K, kw.get("conv_mode", 0), kw.get("col_scale") is not None,
                      kw.get("residual") is not None, kw.get("act", 0)))

    monkeypatch.setattr(E, "call", fake_call)
    monkeypatch.setattr(E, "gemm", fake_gemm)
    monkeypatch.setattr(E, "_stream", lambda: 0)
    monkeypatch.setattr(E, "_require_cuda", lambda dev: None)
    monkeypatch.setattr(ops, "num_sms", lambda: 132)
    return calls


def _names(calls):
    return [c for c in calls if isinstance(c, str)]


def _gemms(calls):
    return [c for c in calls if not isinstance(c, str)]


@pytest.mark.parametrize("image_size,stem", [(224, "vtx_stem_s2d"), (200, "vtx_stem_im2col")])
def test_backbone_infer_schedule(dry, image_size, stem):
    from virtex_b200.engine import Engine, _CnnView
    cnn = _cnn(0).eval()
    eng = Engine(visual=_CnnView(cnn))
    feat, h, w = eng.backbone_infer(torch.zeros(2, 3, image_size, image_size))
    assert (h, w) == ((image_size + 31) // 32,) * 2 and tuple(feat.shape) == (2 * h * w, 2048) and feat.dtype == BF16
    names, gemms = _names(dry), _gemms(dry)
    # the eval bnp of all 53 BNs from the running statistics, then nothing of the training schedule
    assert names.count("vtx_bn_finalize") == 53
    assert stem in names and names.count("vtx_bn_relu_maxpool") == 1
    assert not any(n in names for n in ("vtx_bn_finalize_act", "vtx_bn_act", "vtx_subsample", "vtx_im2col3x3"))
    assert eng._tape is None
    # stem + conv1 / conv2 / conv3 of 16 blocks + 4 downsamples; every bottleneck GEMM applies its BN in the epilogue
    assert len(gemms) == 1 + 3 * 16 + 4
    assert not gemms[0][5] and all(g[5] for g in gemms[1:])
    assert sum(1 for g in gemms if g[6]) == 16 and all(g[7] == 1 for g in gemms if g[6])  # conv3: shortcut + ReLU
    assert sum(1 for g in gemms[1:] if g[7] == 0) == 4                                   # downsample: BN only
    assert sum(1 for g in gemms if g[4] == 1) == 16 + 3                                  # implicit 3x3 + strided 1x1
    # a second call reuses the folded parameters; a train-mode forward or a load_state_dict recomputes them
    dry.clear()
    eng.backbone_infer(torch.zeros(2, 3, image_size, image_size))
    assert _names(dry).count("vtx_bn_finalize") == 0 and "vtx_conv_w_jobs" not in _names(dry)
    dry.clear()
    eng.backbone_forward(torch.zeros(2, 3, image_size, image_size), training=True)
    eng.backbone_infer(torch.zeros(2, 3, image_size, image_size))
    assert _names(dry).count("vtx_bn_finalize") == 1 + 4 + 53  # stem + downsamples (training), then the eval fold


def test_resnet_forward_module_surface(dry):
    """fc assigned after a first forward, re-initialised in place; eval-mode gradients reach fc only; a backbone that
    still requires grad in eval mode is refused; a train-mode forward fills every gradient; load_state_dict on the
    cnn marks the engine's folded BN parameters stale."""
    cnn = _cnn(0).eval()
    image = torch.zeros(2, 3, 224, 224)
    with torch.no_grad():
        feats = cnn(image)
    assert tuple(feats.shape) == (2, 2048) and feats.dtype == F32
    with pytest.raises(RuntimeError, match="eval-mode BatchNorm"):
        cnn(image)
    for n, p in cnn.named_parameters():
        p.requires_grad = False
    cnn.fc = nn.Linear(2048, 7)
    torch.nn.init.normal_(cnn.fc.weight.data, mean=0.0, std=0.01)
    torch.nn.init.constant_(cnn.fc.bias.data, 0.0)
    dry.clear()
    with torch.autocast("cpu", dtype=torch.bfloat16):
        logits = cnn(image)
    assert tuple(logits.shape) == (2, 7) and logits.dtype == F32 and logits.requires_grad
    assert "vtx_bn_finalize" not in _names(dry)  # running statistics unchanged since the first forward
    assert _gemms(dry)[-1][1:4] == (2, 7, 2048)
    dry.clear()
    logits.sum().backward()
    assert cnn.fc.weight.grad is not None and cnn.fc.bias.grad is not None
    assert all(p.grad is None for n, p in cnn.named_parameters() if not n.startswith("fc."))
    assert _names(dry) == ["vtx_cast_bf16", "vtx_colsum"] and len(_gemms(dry)) == 1  # dlogits cast, db, dW; no dX
    # load_state_dict on the cnn itself: the next eval forward re-derives the folded BN parameters
    cnn.load_state_dict(cnn.state_dict())
    dry.clear()
    with torch.no_grad():
        cnn(image)
    assert _names(dry).count("vtx_bn_finalize") == 53
    # train mode (fine-tuning): batch statistics, and gradients for every parameter
    cnn.train()
    for p in cnn.parameters():
        p.requires_grad = True
    dry.clear()
    out = cnn(image)
    assert "vtx_bn_finalize_act" in _names(dry)
    out.sum().backward()
    assert all(p.grad is not None for p in cnn.parameters())
    assert {"vtx_group_mean_bwd", "vtx_bn_bwd_finalize_apply"} <= set(_names(dry))


def test_fc_must_be_identity_or_linear_on_the_backbone_device(dry):
    cnn = _cnn(0)
    cnn.fc = nn.Sequential(nn.Linear(2048, 3))
    with pytest.raises(TypeError):
        with torch.no_grad():
            cnn(torch.zeros(1, 3, 224, 224))


# ------------------------------------------------------------------------------------------------------ host checks
def _lib():
    from virtex_b200 import lib as L
    if not os.path.exists(L.LIB_PATH):
        pytest.skip("library not built")
    return L, L.load()


def _ss_gemm(L, **over):
    """A scale / shift GEMM whose pointers are never dereferenced: every case below is rejected by the host checks,
    which run before any device work."""
    g = L.VtxGemm()
    g.A, g.B, g.D = 0x100000, 0x200000, 0x300000
    g.col_scale, g.col_shift = 0x400000, 0x500000
    g.M, g.N, g.K = 256, 128, 64
    g.lda, g.ldb, g.ldd = 64, 64, 128
    g.split_k, g.tile_n, g.alpha, g.act = 1, 128, 1.0, 1
    for k, v in over.items():
        setattr(g, k, v)
    return g


@pytest.mark.parametrize("over", [
    dict(col_shift=0),                                       # one vector without the other
    dict(col_scale=0),
    dict(out_f32=1, ldd=128),                                # fp32 output
    dict(alpha=2.0),
    dict(bias=0x600000),
    dict(stats=0x600000, act=0),
    dict(act=2),                                             # GELU
    dict(N=127, ldd=128),                                    # N must be even (float2 column pairs)
    dict(col_scale=0x400004),                                # not 8-byte aligned
    dict(col_shift=0x500004),
    dict(residual=0x600000, ldr=128, residual_mask=0x700000),
    dict(residual=0x600008, ldr=128),                        # residual the TMA cannot stage
    dict(residual=0x600000, ldr=100),
    dict(bnr_y=0x600000, bnr_bnp=0x700000, bnr_sums=0x800000, bnr_ldy=128, act=0),
    dict(conv_mode=2),
])
def test_host_rejects_unsupported_scale_shift_epilogues(over):
    L, lib = _lib()
    g = _ss_gemm(L, **over)
    rc = lib.vtx_gemm(ctypes.byref(g), None)
    assert rc == -1, rc
    msg = lib.vtx_last_error().decode()
    assert "col_scale" in msg or "conv_mode" in msg, msg
