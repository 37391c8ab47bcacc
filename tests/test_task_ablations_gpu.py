"""The task ablations on the H100: the masked-LM collate kernel bit-exact against its host replay
(tests/masked_lm_oracle.py, whose distribution tests/test_task_ablations_cpu.py pins to the reference's), pipeline-built
masked-LM batches through MaskedLMModel against the float64 oracle, Trainer.step on masked_lm against the autograd loop
body, the classification batches of the pipeline, and one full-size masked_lm_R_50_L1_H2048 step."""
import numpy as np
import pytest
import torch

from oracle import virtex_oracle as O
from tests import masked_lm_oracle as MO

pytestmark = pytest.mark.gpu


def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def cos(a, b):
    a, b = a.detach().double().cpu().flatten(), b.detach().double().cpu().flatten()
    return (a @ b / (a.norm() * b.norm() + 1e-30)).item()


def _ragged(B, seed, vocab):
    """B captions of random lengths, with lengths 0, 1, 2, 3, 30 and 45 (trimmed) among them."""
    g = np.random.default_rng(seed)
    out = []
    for b in range(B):
        n = [0, 1, 2, 3, 30, 45][b] if b < 6 else int(g.integers(0, 46))
        row = [int(x) for x in g.integers(4, vocab, n)]
        if n:
            row[0] = MO.SOS
        if n > 1:
            row[-1] = MO.EOS
        out.append(row)
    return out


def _stage(lists):
    offs = np.zeros(len(lists) + 1, np.int64)
    offs[1:] = np.cumsum([len(t) for t in lists])
    flat = np.array([x for t in lists for x in t] or [0], np.int64)
    return torch.from_numpy(flat).cuda(), torch.from_numpy(offs).cuda()


def _collate(lists, seed_t, vocab, mask_prob=0.85, replace_prob=0.10, max_len=MO.MAX_LEN):
    from virtex_b200 import ops
    flat, offs = _stage(lists)
    B = len(lists)
    T = int(min(max_len, max(len(t) for t in lists)))
    cap = torch.empty(B, T, dtype=torch.int64, device="cuda")
    lab, lens = torch.empty_like(cap), torch.empty(B, dtype=torch.int64, device="cuda")
    ops.call("vtx_collate_masked_lm", flat.data_ptr(), offs.data_ptr(), cap.data_ptr(), lab.data_ptr(), lens.data_ptr(),
             B, T, max_len, MO.UNK, MO.MASK, vocab, 0.15, mask_prob, replace_prob, seed_t.data_ptr(), ops._stream())
    torch.cuda.synchronize()
    return cap.cpu().numpy(), lab.cpu().numpy(), lens.cpu().numpy()


def _seed_tensor(seed):
    return torch.tensor([seed - (1 << 64) if seed >= 1 << 63 else seed], dtype=torch.int64, device="cuda")


# ----------------------------------------------------------------------------------------------------------- kernel
@pytest.mark.parametrize("vocab", [10000, 81])
@pytest.mark.parametrize("seed", [0, 1, 0xDEADBEEF, (1 << 63) + 12345])
@pytest.mark.parametrize("mask_prob", [0.85, 0.80])
def test_collate_masked_lm_matches_the_host_replay(vocab, seed, mask_prob):
    _need_cuda()
    lists = _ragged(256, seed % 1000 + vocab, vocab)
    cap, lab, lens = _collate(lists, _seed_tensor(seed), vocab, mask_prob=mask_prob)
    rcap, rlab, rlens = MO.device_masking(lists, seed, vocab=vocab, mask_prob=mask_prob)
    assert np.array_equal(lens, rlens)
    assert np.array_equal(cap, rcap)
    assert np.array_equal(lab, rlab)
    assert (lab != MO.UNK).sum() > 256  # the batch masks something


def test_device_drawn_seed_differs_per_call_and_follows_manual_seed():
    _need_cuda()
    from virtex_b200.data_gpu import GpuInputPipeline
    pipe = GpuInputPipeline("cuda", task="masked_lm")
    g = np.random.default_rng(0)
    images = [g.integers(0, 256, (240, 260, 3), dtype=np.uint8) for _ in range(8)]
    params = [pipe.val_params(240, 260) for _ in images]
    lists = _ragged(8, 11, MO.VOCAB)
    torch.manual_seed(5)
    a = pipe(images, params, lists)
    b = pipe(images, params, lists)
    torch.manual_seed(5)
    c = pipe(images, params, lists)
    assert set(a) == {"image", "_image_u8", "caption_tokens", "masked_labels", "caption_lengths"}
    assert not torch.equal(a["masked_labels"], b["masked_labels"]) or not torch.equal(a["caption_tokens"],
                                                                                      b["caption_tokens"])
    for k in ("caption_tokens", "masked_labels", "caption_lengths", "image"):
        assert torch.equal(a[k], c[k]), k
    # an explicit seed is the host replay's
    d = pipe(images, params, lists, seed=77)
    rcap, rlab, _ = MO.device_masking(lists, 77)
    assert np.array_equal(d["caption_tokens"].cpu().numpy(), rcap)
    assert np.array_equal(d["masked_labels"].cpu().numpy(), rlab)


def test_collate_masked_lm_rejects_bad_arguments():
    _need_cuda()
    from virtex_b200 import lib as L, ops
    x = torch.zeros(4096, dtype=torch.int64, device="cuda")
    p = x.data_ptr()
    good = dict(T=30, vocab=10, prop=0.15, mp=0.85, rp=0.1)
    for bad in (dict(T=1025), dict(vocab=0), dict(prop=1.5), dict(mp=-0.1), dict(rp=float("nan"))):
        a = dict(good, **bad)
        with pytest.raises(L.VtxError, match="collate_masked_lm"):
            ops.call("vtx_collate_masked_lm", p, p, p, p, p, 2, a["T"], 2000, 0, 3, a["vocab"], a["prop"], a["mp"],
                     a["rp"], p, ops._stream())


# ------------------------------------------------------------------------------------------------------------ model
SMALL = O.Spec(hidden=128, layers=1, heads=2, ffn=256, caption_backward=False, mask_future=False)
ZERO_SEED = 21594  # with _zero_lists(): caption 0, position 21 is replaced by the id 0 (found by the host replay)


def _zero_lists():
    g = np.random.default_rng(7)
    out = []
    for n in (30, 22, 13, 9):
        row = [int(x) for x in g.integers(4, 10000, n)]
        row[0], row[-1] = MO.SOS, MO.EOS
        out.append(row)
    return out


def _images(B, seed):
    g = np.random.default_rng(seed)
    return [g.integers(0, 256, (230 + 7 * b, 250, 3), dtype=np.uint8) for b in range(B)]


def _pipe_batch(pipe, lists, seed, img_seed=0):
    images = _images(len(lists), img_seed)
    return pipe(images, [pipe.val_params(*im.shape[:2]) for im in images], lists, seed=seed)


def _masked_lm_model(state):
    from virtex_b200.models import MaskedLMModel
    from virtex_b200.modules import TorchvisionVisualBackbone, TransformerDecoderTextualHead
    textual = TransformerDecoderTextualHead(2048, SMALL.vocab, 128, 1, 2, 256, dropout=0.0, mask_future_positions=False)
    model = MaskedLMModel(TorchvisionVisualBackbone("resnet50", 2048), textual)
    sd = {k: v for k, v in O.to_reference_state_dict(state, SMALL).items() if not k.startswith("backward_textual.")}
    model.load_state_dict(sd, strict=True)
    return model.cuda().train()


def test_pipeline_masked_lm_batch_through_the_model_vs_oracle():
    """Loss 1e-3 relative, head gradients cos > 0.998 and rel < 5e-2 (test_masked_lm_model_vs_oracle's tolerances),
    on a batch whose masking wrote the id 0 inside a caption: its embedding is zeroed, its key stays visible."""
    _need_cuda()
    from virtex_b200.data_gpu import GpuInputPipeline
    lists = _zero_lists()
    rcap, _, _ = MO.device_masking(lists, ZERO_SEED)
    assert rcap[0, 21] == 0 and lists[0][21] != 0
    pipe = GpuInputPipeline("cuda", task="masked_lm")
    batch = _pipe_batch(pipe, lists, ZERO_SEED)
    assert batch["caption_tokens"][0, 21].item() == 0 and batch["caption_lengths"][0].item() == 30
    state = O.synth_state(SMALL, 31, bn3_gain=0.25)
    model = _masked_lm_model(state)
    out = model(batch)
    cpu = {k: batch[k].cpu() for k in ("image", "caption_tokens", "masked_labels", "caption_lengths")}
    ref, grads, _ = O.loss_and_grads(state, cpu, SMALL)
    assert abs(out["loss"].item() - ref["loss"].item()) < 1e-3 * ref["loss"].item(), (out["loss"].item(),
                                                                                      ref["loss"].item())
    out["loss"].backward()
    bad = []
    for name, p in model.named_parameters():
        if name.startswith("visual."):
            continue
        r, c = rel(p.grad, grads[name]), cos(p.grad, grads[name])
        if not (c > 0.998 and r < 5e-2):
            bad.append((name, r, c))
    assert not bad, bad


def _mlm_config(optimizer):
    from virtex_b200.config import Config
    return Config("task_ablations/masked_lm_R_50_L1_H2048.yaml",
                  ["MODEL.TEXTUAL.NAME", "transdec_postnorm::L1_H128_A2_F256", "MODEL.TEXTUAL.DROPOUT", 0.0,
                   "OPTIM.OPTIMIZER_NAME", optimizer, "OPTIM.WARMUP_STEPS", 0, "OPTIM.NUM_ITERATIONS", 100,
                   "OPTIM.LR", 0.01 if optimizer == "sgd" else 1e-4, "OPTIM.CNN_LR", 0.002 if optimizer == "sgd" else 1e-5,
                   "OPTIM.LOOKAHEAD.STEPS", 2])


@pytest.mark.parametrize("optimizer", ["sgd", "adamw"])
def test_trainer_steps_match_the_autograd_loop(optimizer):
    """Four Trainer.step calls on pipeline-built masked-LM batches against model -> loss.backward() -> clip ->
    OptimizerFactory step (Lookahead every 2) -> LR schedule on a twin."""
    _need_cuda()
    from virtex_b200.data_gpu import GpuInputPipeline
    from virtex_b200.factories import LRSchedulerFactory, OptimizerFactory, PretrainingModelFactory
    from virtex_b200.models import MaskedLMModel
    from virtex_b200.trainer import Trainer
    cfg = _mlm_config(optimizer)
    state = O.synth_state(SMALL, 41, bn3_gain=0.25)
    sd = {k: v for k, v in O.to_reference_state_dict(state, SMALL).items() if not k.startswith("backward_textual.")}
    models = []
    for _ in range(2):
        m = PretrainingModelFactory.from_config(cfg)
        assert isinstance(m, MaskedLMModel)
        m.load_state_dict(sd, strict=True)
        models.append(m.cuda().train())
    trainer = Trainer(models[0], cfg)
    ref = models[1]
    opt = OptimizerFactory.from_config(cfg, ref.named_parameters())
    sched = LRSchedulerFactory.from_config(cfg, opt)
    pipe = GpuInputPipeline.from_config(cfg, "cuda")
    assert pipe.task == "masked_lm" and (pipe.mask_probability, pipe.replace_probability) == (0.85, 0.10)
    for it in range(4):
        batch = _pipe_batch(pipe, _ragged(6, 90 + it, 10000)[4:] + _zero_lists(), seed=1000 + it, img_seed=it)
        loss = trainer.step(batch)
        opt.zero_grad()
        out = ref(batch)
        out["loss"].backward()
        torch.nn.utils.clip_grad_norm_(ref.parameters(), cfg.OPTIM.CLIP_GRAD_NORM)
        opt.step()
        sched.step()
        assert loss[1].item() == 0.0
        assert abs(loss[0].item() - out["loss"].item()) < 1e-3 * out["loss"].item(), (it, loss[0].item(),
                                                                                      out["loss"].item())
    torch.cuda.synchronize()
    a, b = dict(models[0].named_parameters()), dict(ref.named_parameters())
    for name in ("textual.output.bias", "textual.embedding.words.weight", "textual.transformer.layers.0.linear1.weight"):
        d_a, d_b = a[name].detach().cpu() - sd[name], b[name].detach().cpu() - sd[name]
        assert d_b.norm() > 0 and rel(d_a, d_b) < 5e-2, (name, rel(d_a, d_b))
    for name in ("visual.cnn.conv1.weight", "visual.cnn.layer4.2.conv3.weight"):
        d_a = a[name].detach().cpu() - sd[name]
        assert torch.isfinite(d_a).all() and d_a.norm() > 0, name


# --------------------------------------------------------------------------------------------------- classification
@pytest.mark.parametrize("name", ["token_classification", "multilabel_classification"])
def test_classification_batches_equal_pad_sequence_and_drive_the_trainer(name):
    _need_cuda()
    from torch.nn.utils.rnn import pad_sequence
    from tests import classification_oracle as CO
    from virtex_b200.config import Config
    from virtex_b200.data_gpu import GpuInputPipeline
    from virtex_b200.factories import PretrainingModelFactory
    from virtex_b200.trainer import Trainer
    cfg = Config(f"task_ablations/{name}_R_50.yaml", ["OPTIM.WARMUP_STEPS", 0])
    pipe = GpuInputPipeline.from_config(cfg, "cuda")
    g = np.random.default_rng(3)
    if name == "token_classification":
        # every caption has a token besides [SOS] / [EOS]: an image with none has an empty label set and a NaN loss
        lists = [[MO.SOS] + [int(x) for x in g.integers(4, 10000, n)] + [MO.EOS] for n in (3, 40, 12, 1, 28)]
        want = pad_sequence([torch.tensor(t[:30]) for t in lists], batch_first=True, padding_value=cfg.DATA.UNK_INDEX)
    else:  # category lists: never trimmed, padded with 0
        lists = [[int(x) for x in g.choice(np.arange(1, 81), n, replace=False)] for n in (3, 1, 35, 7, 2)]
        want = pad_sequence([torch.tensor(t) for t in lists], batch_first=True, padding_value=0)
    batch = _pipe_batch(pipe, lists, seed=None)
    assert set(batch) == {"image", "_image_u8", "labels"}
    assert torch.equal(batch["labels"].cpu(), want)
    model = PretrainingModelFactory.from_config(cfg)
    model.load_state_dict(CO.synth_classification_state(cfg.DATA.VOCAB_SIZE, 5), strict=True)
    model = model.cuda().train()
    with torch.no_grad():
        before = model(batch)["loss"].item()
    trainer = Trainer(model, cfg)
    loss = trainer.step(batch)
    assert loss[1].item() == 0.0 and abs(loss[0].item() - before) < 1e-3 * abs(before), (loss[0].item(), before)
    after = trainer.step(batch)[0].item()
    assert np.isfinite(after)


def test_captioning_batch_is_unchanged_by_the_task_argument():
    _need_cuda()
    from virtex_b200.data_gpu import GpuInputPipeline
    lists = _ragged(16, 5, 10000)
    lists[0] = [1, 5, 2]  # no empty batch-maximum
    a = _pipe_batch(GpuInputPipeline("cuda"), lists, seed=None)
    b = _pipe_batch(GpuInputPipeline("cuda", task="captioning", vocab_size=81), lists, seed=3)
    assert set(a) == set(b) == {"image", "_image_u8", "caption_tokens", "noitpac_tokens", "caption_lengths"}
    for k in a:
        assert torch.equal(a[k], b[k]), k


# --------------------------------------------------------------------------------------------------------- full size
def test_full_size_masked_lm_step_at_batch_256():
    """masked_lm_R_50_L1_H2048 as shipped, batch 256 of pipeline-built 224 x 224 images and captions: one Trainer.step
    gives a finite loss; the peak device memory of the step is printed."""
    _need_cuda()
    from virtex_b200.config import Config
    from virtex_b200.data_gpu import GpuInputPipeline
    from virtex_b200.factories import PretrainingModelFactory
    from virtex_b200.trainer import Trainer
    cfg = Config("task_ablations/masked_lm_R_50_L1_H2048.yaml")
    torch.manual_seed(0)
    model = PretrainingModelFactory.from_config(cfg).cuda().train()
    trainer = Trainer(model, cfg)
    pipe = GpuInputPipeline.from_config(cfg, "cuda")
    g = np.random.default_rng(1)
    B = 256
    images = [g.integers(0, 256, (256, 256, 3), dtype=np.uint8) for _ in range(B)]
    lists = [[MO.SOS] + [int(x) for x in g.integers(4, 10000, int(g.integers(6, 40)))] + [MO.EOS] for _ in range(B)]
    params = [pipe.sample_train_params(g, 256, 256) for _ in range(B)]
    batch = pipe(images, params, lists)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    loss = trainer.step(batch)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    print(f"masked_lm_R_50_L1_H2048 batch {B}: loss {loss[0].item():.4f}, peak allocated {peak:.2f} GiB")
    assert torch.isfinite(loss[0]) and loss[1].item() == 0.0
    assert (batch["masked_labels"] != 0).sum() >= B  # every caption of >= 3 tokens has a label
