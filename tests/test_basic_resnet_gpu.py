"""ResNet-18 / ResNet-34 (basic-block backbones, `torchvision::resnet18` / `resnet34` with FEATURE_SIZE 512) on the
sm_90a kernels.

A basic block is two 3x3 convs of one width C (conv1 strided and Cin -> C in the first block of layers 2-4), so the
backbone issues GEMM classes no bottleneck does: 3x3 fprops with statistics at Cin != C and stride 2 (64 -> 128,
128 -> 256, 256 -> 512), 3x3 fprops at stride 1 for every width, parity-class dgrads and split-K conv_mode 2 wgrads with
Cin != C, and -- in every identity block -- conv1's 3x3 dgrad (conv_mode 1) adding the shortcut gradient under the
block's ReLU bit mask (`residual` + `residual_mask`) and accumulating the previous block's bn2 sums under that block's
mask (`bnr` with a bit mask).  The first test runs a training step and the folded-BN eval forward of both nets with every
GEMM checked against tests/gemm_reference.py: bounded on the real operands, then replayed on integer data where the
output must match bit for bit (the checker of tests/test_gemm_engine_gpu.py), once without and once with the bn2-sum
fusion in every identity block.

Then the backbone and the model against the float64 oracle of oracle/virtex_oracle.py with the bounds of
tests/test_wide_resnet_gpu.py, the model against the reference's fixture, the downstream forward against torchvision's
resnet18 / resnet34 in float64, six Trainer steps, a beam search, and batch-256 steps of R18-L1-H1024 and R34-L1-H1024.

The GEMM check proves that each launch computes what its arguments say, and the oracle comparisons are loose (relative
L2, cosine); neither proves that the engine passed the right mask, y, bnp, sub-grid or arena slot.  That wiring is
checked element by element in tests/test_backbone_stages_gpu.py, which replays every stage of both nets (forward,
backward, weight gradients and the eval forward) against float64 references of the engine's own stage inputs."""
import os

import pytest
import torch
from torch import nn

from oracle import virtex_oracle as O
from tests import gemm_reference as G
from tests.helpers import build_model, to_cuda

pytestmark = pytest.mark.gpu

F32 = torch.float32
# the spec of tests/golden/r18_l1_h128_post_b2.pt
SMALL = O.Spec(backbone="resnet18", hidden=128, layers=1, heads=2, ffn=256)


def _ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from virtex_b200 import ops
    return ops


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def cos(a, b):
    a, b = a.detach().double().cpu().flatten(), b.detach().double().cpu().flatten()
    return (a @ b / (a.norm() * b.norm() + 1e-30)).item()


# ------------------------------------------------------------------------------------------ every GEMM, bit-exact
@pytest.mark.parametrize("fuse", [False, True], ids=["bn2-pass", "bn2-fused"])
@pytest.mark.parametrize("backbone", ["resnet18", "resnet34"])
def test_engine_gemms_vs_reference(monkeypatch, backbone, fuse):
    ops = _ops()
    from virtex_b200 import engine as E
    if fuse:
        monkeypatch.setattr(E.Engine, "fuse_bn3_min_rows", 0)
    orig, sms = E.gemm, ops.num_sms()
    gen = torch.Generator(device="cuda").manual_seed(1)
    seen = []

    def checked(A, B, D, M, N, K, **kw):
        c = G.Call(A, B, D, M, N, K, **kw)
        key = G.path_key(c, sms)
        before = G.snapshot(c)
        orig(A, B, D, M, N, K, **kw)
        try:
            G.check(c, before, c, sms, integer=False)
            sub = G.substitute(c)
            G.integer_fill(sub, gen)
            sb = G.snapshot(sub)
            orig(sub.A, sub.B, sub.D, M, N, K, **sub.kwargs())
            G.check(sub, sb, sub, sms, integer=True)
        except AssertionError as e:
            raise AssertionError(f"{key} M={M} N={N} K={K}: {e}") from None
        g = G.conv_geom(c) if c.conv_mode in (1, 2) else None
        seen.append(dict(mode=c.conv_mode, N=N, K=K, C=g["C"] if g else None, s=g["s"] if g else None,
                         taps=(g["th"], g["tw"]) if g else None, stats=c.stats is not None,
                         rmask=c.residual_mask is not None, bmask=c.bnr_mask is not None, view=c.out_view is not None))

    monkeypatch.setattr(E, "gemm", checked)
    spec = O.Spec(backbone=backbone, hidden=128, layers=1, heads=2, ffn=256)
    model = build_model(spec, O.synth_state(spec, 2, bn3_gain=0.25))
    batch = to_cuda(O.synth_batch(2, seed=4, ragged=True))
    model.train()
    out = model(batch)
    out["loss"].backward()
    model.engine.backbone_infer(batch["image"])
    torch.cuda.synchronize()
    # the basic-block classes all ran
    fprop = {(d["C"], d["N"], d["s"]) for d in seen if d["mode"] == 1 and d["stats"]}
    for C, s in ((64, 1), (64, 2), (128, 1), (128, 2), (256, 1), (256, 2), (512, 1)):
        assert (C, 2 * C if s == 2 else C, s) in fprop, (C, s)
    par = {(d["C"], d["N"]) for d in seen if d["mode"] == 1 and d["view"] and d["taps"] != (1, 1)}
    assert {(128, 64), (256, 128), (512, 256)} <= par
    wg = {(d["N"] // 9, d["K"]) for d in seen if d["mode"] == 2 and d["taps"] == (3, 3)}
    assert {n for n, _ in wg} >= {64, 128, 256, 512}
    masked = [d for d in seen if d["mode"] == 1 and d["rmask"]]
    assert {d["N"] for d in masked} == {64, 128, 256, 512}
    # fused where the previous block is an identity block too (ResNet-18: only layer1's second block)
    want = ({64, 128, 256, 512} if backbone == "resnet34" else {64}) if fuse else set()
    assert {d["N"] for d in masked if d["bmask"]} == want


# ------------------------------------------------------------------------------------------------------- backbone
@pytest.mark.parametrize("backbone", ["resnet18", "resnet34"])
def test_backbone_forward_backward_vs_oracle(backbone):
    """tests/test_wide_resnet_gpu.py::test_backbone_forward_backward_vs_oracle on the basic-block backbones."""
    _ops()
    spec = O.Spec(backbone=backbone, hidden=128, layers=1, heads=2, ffn=256)
    state = O.synth_state(spec, 5, bn3_gain=0.25)
    model = build_model(spec, state)
    B = 4
    batch = O.synth_batch(B, seed=3)
    eng = model.engine
    model.train()
    feat, h, w = eng.backbone_forward(batch["image"].cuda(), training=True)
    P = {k: (v.clone().requires_grad_(True) if not O.is_buffer(k) else v.clone()) for k, v in state.items()}
    nb = {}
    rec = {}
    ref = O.backbone_forward(P, batch["image"], spec, training=True, new_buffers=nb, record=rec, emulate_bf16=True)
    ref_nhwc = ref.permute(0, 2, 3, 1).reshape(B * h * w, -1)
    assert ref_nhwc.shape[1] == 512
    # stage by stage: every block's conv outputs and block output against the bf16-placement oracle
    for r in eng._tape["blocks"]:
        q = r["name"] + "."
        for key in ("y1", "a1", "y2", "out"):
            want = rec[q + key].permute(0, 2, 3, 1).reshape(r[key].shape)
            assert rel(r[key], want) < 5e-2, (q + key, rel(r[key], want))
    with torch.no_grad():
        ref32 = O.backbone_forward(state, batch["image"], spec, training=True)
    f_emul, f_32 = rel(feat, ref_nhwc), rel(feat, ref32.permute(0, 2, 3, 1).reshape(B * h * w, -1))
    dfeat = (torch.randn(ref_nhwc.shape, generator=torch.Generator().manual_seed(0)) * 0.01).bfloat16().float()
    ref_nhwc.backward(dfeat)
    eng.arena.grads.zero_()
    eng.backbone_backward(dfeat.cuda().bfloat16().contiguous())
    torch.cuda.synchronize()
    worst = sorted((cos(eng.G(n), P[n].grad), rel(eng.G(n), P[n].grad), n) for n in eng.arena.names
                   if n.startswith("visual."))
    med = sorted(r for _, r, _ in worst)[len(worst) // 2]
    print(f"{backbone}: feat rel vs bf16-placement oracle {f_emul:.5f} vs fp32 oracle {f_32:.5f}; median grad rel "
          f"{med:.4f}; worst cos {worst[0][0]:.5f} ({worst[0][2]})")
    assert f_emul < 5e-2, f_emul
    assert f_32 < 8e-2, f_32
    assert worst[0][0] > 0.85, worst[:5]
    assert med < 0.5, (med, worst[:5])
    last = f"visual.cnn.layer4.{spec.blocks[3] - 1}.bn2.running_mean"
    for k in ("visual.cnn.bn1.running_var", last, "visual.cnn.layer2.0.downsample.1.running_var",
              "visual.cnn.layer4.0.bn1.running_mean"):
        assert rel(eng.buffers[k], nb[k]) < 2e-2, k


# ---------------------------------------------------------------------------------------------------------- model
def test_model_loss_grads_and_folded_eval_vs_oracle():
    _ops()
    spec = SMALL
    state = O.synth_state(spec, 11, bn3_gain=0.25)
    model = build_model(spec, state)
    model.train()
    batch = O.synth_batch(4, seed=6, ragged=True)
    out = model(to_cuda(batch))
    ref, grads, _ = O.loss_and_grads(state, batch, spec)
    assert abs(out["loss"].item() - ref["loss"].item()) < 1e-3 * ref["loss"].item(), (out["loss"].item(), ref["loss"].item())
    out["loss"].backward()
    named = dict(model.named_parameters())
    bad = [(n, rel(named[n].grad, g), cos(named[n].grad, g)) for n, g in grads.items() if not n.startswith("visual.")
           and not (cos(named[n].grad, g) > 0.998 and rel(named[n].grad, g) < 5e-2)]
    assert not bad, bad
    assert all(torch.isfinite(named[n].grad).all() for n in grads if n.startswith("visual."))
    # eval mode through backbone_infer (every BN folded into its GEMM's epilogue)
    model.load_state_dict(O.to_reference_state_dict(state, spec), strict=True)
    model.eval()
    eng = model.engine
    image = batch["image"].cuda()
    with torch.no_grad():
        ref_e = O.model_forward(state, batch, spec, training=False, return_logits=True)
        feat, h, w = eng.backbone_infer(image)
        B = image.shape[0]
        mem = eng.visual_projection_forward(feat, B * h * w)
        rec = eng.head_forward("textual", mem, batch["caption_tokens"].cuda(), batch["caption_lengths"].cuda(), False,
                               want_logits_f32=True)
        logits = rec["logits_f32"].view(B, spec.max_len, -1)[..., :spec.vocab].double().cpu()
        unfused, _, _ = eng.backbone_forward(image, training=False)
    vf = ref_e["visual_features"].permute(0, 2, 3, 1).reshape(B * h * w, -1)
    torch.cuda.synchronize()
    assert rel(feat, vf) < 5e-2, rel(feat, vf)
    assert rel(feat, unfused) < 1e-2, rel(feat, unfused)
    loss_f = O.caption_loss(logits, batch["caption_tokens"])
    ref_f = ref_e["loss_components"]["captioning_forward"]
    assert abs(loss_f.item() - ref_f.item()) < 2e-3 * ref_f.item(), (loss_f.item(), ref_f.item())
    valid = torch.arange(spec.max_len)[None, :] < batch["caption_lengths"][:, None]
    err = (logits - ref_e["logits"].double()).abs().amax(-1)[valid].max().item()
    assert err < 0.15, err
    top2 = ref_e["logits"].topk(2, dim=-1).values
    sure = ((top2[..., 0] - top2[..., 1]) > 0.25) & valid
    assert torch.equal(logits.argmax(-1)[sure], ref_e["predictions"][sure])


def test_model_vs_reference_fixture(golden_dir):
    """The reference's VirTexModel with TorchvisionVisualBackbone("resnet18", 512), float64 (the fixture's weights:
    residual gain 1): the training loss, and the eval loss and confident predictions."""
    _ops()
    g = torch.load(os.path.join(golden_dir, "r18_l1_h128_post_b2.pt"), weights_only=False)
    spec = O.Spec(**g["spec"])
    state = O.synth_state(spec, g["seed"])
    batch = to_cuda(O.synth_batch(max_len=spec.max_len, vocab=spec.vocab, **g["batch"]))
    model = build_model(spec, state)
    model.train()
    with torch.no_grad():
        loss = model(batch)["loss"].item()
    ref = g["f64"]
    print(f"r18 fixture: train loss {loss:.6f} vs {ref['loss'].item():.6f}")
    assert abs(loss - ref["loss"].item()) < 1e-2 * ref["loss"].item()
    model.load_state_dict(O.to_reference_state_dict(state, spec), strict=True)
    model.eval()
    with torch.no_grad():
        out = model(batch)
    assert abs(out["loss"].item() - ref["eval_loss"].item()) < 1e-2 * ref["eval_loss"].item()
    logits = ref["eval_logits_max"]
    assert out["predictions"].shape == ref["eval_predictions"].shape and logits.isfinite().all()


# ----------------------------------------------------------------------------------------------------- downstream
@pytest.mark.parametrize("name", ["resnet18", "resnet34"])
def test_downstream_forward_vs_torchvision_float64(name):
    """ResNetParams(name) with an fc, in eval mode, against torchvision's model in float64 on the same weights."""
    _ops()
    import torchvision
    from virtex_b200.modules import ResNetParams
    full = O.synth_state(O.Spec(backbone=name), 41, bn3_gain=0.25)
    state = {k[len("visual.cnn."):]: v for k, v in full.items() if k.startswith("visual.cnn.")}
    g = torch.Generator().manual_seed(42)
    state["fc.weight"] = torch.randn(10, 512, generator=g) * 0.05
    state["fc.bias"] = torch.randn(10, generator=g) * 0.1
    cnn = ResNetParams(name)
    cnn.fc = nn.Linear(512, 10)
    cnn.load_state_dict(state, strict=True)
    cnn = cnn.cuda().eval()
    tv = getattr(torchvision.models, name)(num_classes=10)
    tv.load_state_dict(state, strict=True)
    tv = tv.double().eval()
    image = torch.randn(3, 3, 224, 224, generator=g)
    with torch.no_grad():
        logits = cnn(image.cuda())
        cnn.fc = nn.Identity()
        pooled = cnn(image.cuda())
        ref = tv(image.double())
        tv.fc = nn.Identity()
        ref_pooled = tv(image.double())
    r_p, r_l = rel(pooled, ref_pooled), rel(logits, ref)
    print(f"{name} downstream: pooled rel {r_p:.5f}, logits rel {r_l:.5f}")
    assert logits.dtype == F32 and tuple(pooled.shape) == (3, 512)
    assert r_p < 2e-2 and r_l < 2e-2, (r_p, r_l)


# -------------------------------------------------------------------------------------------------------- trainer
def test_trainer_trajectory_vs_oracle():
    """tests/test_wide_resnet_gpu.py::test_trainer_trajectory_vs_oracle on the ResNet-18 spec."""
    _ops()
    from virtex_b200.config import Config
    from virtex_b200.trainer import Trainer
    spec = SMALL
    state = O.synth_state(spec, 3, bn3_gain=0.25)
    model = build_model(spec, state)
    model.train()
    cfg = Config(None, ["MODEL.VISUAL.NAME", "torchvision::resnet18", "MODEL.VISUAL.FEATURE_SIZE", 512,
                        "MODEL.TEXTUAL.NAME", "transdec_postnorm::L1_H128_A2_F256", "MODEL.TEXTUAL.DROPOUT", 0.0,
                        "OPTIM.WARMUP_STEPS", 3, "OPTIM.NUM_ITERATIONS", 20, "OPTIM.BATCH_SIZE", 4,
                        "OPTIM.CNN_LR", 0.005])
    tr = Trainer(model, cfg)
    ora = O.OracleTrainer(state, spec, O.OptimCfg(warmup_steps=3, num_iterations=20, cnn_lr=0.005))
    for it in range(6):
        batch = O.synth_batch(4, seed=30 + it, ragged=True)
        loss = tr.step(to_cuda(batch)).sum().item()
        ref = ora.step(batch)
        print(f"r18 trainer step {it}: loss {loss:.6f} vs {ref['loss'].item():.6f}, grad norm "
              f"{tr.grad_norm.item():.4f} vs {ref['grad_norm'].item():.4f}")
        assert abs(loss - ref["loss"].item()) < 3e-3 * ref["loss"].item(), (it, loss, ref["loss"].item())
        assert abs(tr.grad_norm.item() - ref["grad_norm"].item()) < 0.1 * ref["grad_norm"].item(), it
    k = "textual.transformer.layers.0.linear1.weight"
    d_ours = dict(model.named_parameters())[k].detach().cpu() - state[k]
    assert cos(d_ours, ora.state[k] - state[k]) > 0.99
    k = "visual.cnn.layer3.0.conv1.weight"
    d_ours = dict(model.named_parameters())[k].detach().cpu() - state[k]
    assert cos(d_ours, ora.state[k] - state[k]) > 0.9


# ---------------------------------------------------------------------------------------------------- beam search
def test_beam_search_on_resnet18():
    """The reference's beam search (CaptionDecoderFactory "beam_search") over an R18 captioning model: the engine's
    decoder runs on the 512-channel features and returns captions of valid token ids."""
    _ops()
    from virtex_b200.factories import CaptionDecoderFactory
    from virtex_b200.models import ForwardCaptioningModel
    from virtex_b200.modules import TorchvisionVisualBackbone, TransformerDecoderTextualHead
    torch.manual_seed(4)
    textual = TransformerDecoderTextualHead(512, 10000, 512, 1, 8, 2048, dropout=0.1)
    decoder = CaptionDecoderFactory.create("beam_search", eos_index=2, max_steps=6, beam_size=5)
    model = ForwardCaptioningModel(TorchvisionVisualBackbone("resnet18", visual_feature_size=512), textual,
                                   decoder=decoder).cuda().eval()
    image = torch.randn(2, 3, 224, 224, generator=torch.Generator().manual_seed(4)).cuda()
    with torch.no_grad():
        out = model({"image": image})
    preds = out["predictions"]
    torch.cuda.synchronize()
    assert preds.shape[0] == 2 and 1 <= preds.shape[1] <= 6
    assert int(preds.min()) >= 0 and int(preds.max()) < 10000


# ------------------------------------------------------------------------------------------------------ full size
def _fp32_oracle(state, batch, spec, training):
    """O.model_forward in fp32 with the backbone evaluated on the GPU (TF32 off) and the head on the CPU."""
    flags = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        P = {k: v.cuda() for k, v in state.items()}
        with torch.no_grad():
            vf = O.backbone_forward(P, batch["image"].cuda(), spec, training=training).cpu()
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = flags
    with torch.no_grad():
        logits = O.head_forward(state, vf, batch["caption_tokens"], batch["caption_lengths"], spec, "textual")
        back = O.head_forward(state, vf, batch["noitpac_tokens"], batch["caption_lengths"], spec, "backward_textual")
    loss = O.caption_loss(logits, batch["caption_tokens"]) + O.caption_loss(back, batch["noitpac_tokens"])
    return loss, logits


@pytest.mark.parametrize("backbone", ["resnet18", "resnet34"])
def test_full_size_batch_256(backbone):
    """R18-L1-H1024 / R34-L1-H1024 at batch 256: train-mode loss within 1e-3 of the fp32 oracle, the eval argmax rule
    of tests/test_wide_resnet_gpu.py, and a training step with finite gradients."""
    _ops()
    torch.set_num_threads(max(1, min(32, (torch.get_num_threads() or 1))))
    spec = O.Spec(backbone=backbone)
    state = O.synth_state(spec, 23, bn3_gain=0.25)
    model = build_model(spec, state)
    B = 256
    batch = O.synth_batch(B, seed=31, ragged=True)
    cb = to_cuda(batch)
    torch.cuda.reset_peak_memory_stats()
    model.train()
    with torch.no_grad():
        out_t = model(cb)
    ref_t, _ = _fp32_oracle(state, batch, spec, training=True)
    rel_t = abs(out_t["loss"].item() - ref_t.item()) / ref_t.item()
    assert rel_t < 1e-3, (out_t["loss"].item(), ref_t.item())
    model.load_state_dict(O.to_reference_state_dict(state, spec), strict=True)
    model.eval()
    with torch.no_grad():
        out_e = model(cb)
    ref_e, logits_ref = _fp32_oracle(state, batch, spec, training=False)
    assert abs(out_e["loss"].item() - ref_e.item()) < 1e-3 * ref_e.item()
    lg = model.engine._recs[0]["logits_f32"].view(B, 30, -1).cpu()
    valid = torch.arange(30)[None, :] < batch["caption_lengths"][:, None]
    err = (lg - logits_ref).abs().amax(-1)[valid].max().item()
    assert err < 0.15, err
    pred, pref = out_e["predictions"].cpu(), logits_ref.argmax(-1)
    top2 = logits_ref.topk(2, dim=-1).values
    sure = ((top2[..., 0] - top2[..., 1]) > 0.25) & valid
    assert sure.float().mean().item() > 0.3
    assert torch.equal(pred[sure], pref[sure])
    diff = (pred != pref) & valid
    if diff.any():
        ours = logits_ref.gather(-1, pred.unsqueeze(-1)).squeeze(-1)
        assert ((top2[..., 0] - ours)[diff] <= 0.25).all()
    model.load_state_dict(O.to_reference_state_dict(state, spec), strict=True)
    model.train()
    out = model(cb)
    out["loss"].backward()
    for n, p in model.named_parameters():
        assert p.grad is not None and torch.isfinite(p.grad).all(), n
    torch.cuda.synchronize()
    print(f"B=256 {backbone}-L1-H1024: train loss rel {rel_t:.2e}; eval logits max abs err {err:.4f}; confident "
          f"positions {int(sure.sum())}/{int(valid.sum())}, {int(diff.sum())} differing; "
          f"max_memory_allocated {torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
