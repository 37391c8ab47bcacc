"""The attention kernels past 32 queries and 64 keys (head.cu's long kernels behind vtx_attn_fwd / _bwd), and the model
at the crops and caption lengths that reach them.

  * kernel cases: float64 references on the same bf16 inputs with the bounds of tests/test_head_kernels_gpu.py (same
    two bf16 roundings: 1 ulp plus the flip floor; plain float64: relative L2 <= 1e-2), at p = 0 and p = 0.1 with the
    dropout mask replayed on the host (tests/attention_replica.py), through strided q / k / v views as the engine passes
    them (packed qkv, ld 3H; packed kv, ld 2H) and a padded ldo;
  * the dropout mask element by element, determinism of two launches;
  * the engine's head sublayer by sublayer against float64 (tests/test_head_stages_gpu.py's replay) at 100 keys;
  * the whole model against oracle/virtex_oracle.py at crop 288 and 40 tokens; a full-size batch-256 step at crop 384
    and 64 tokens; decoding_step at crop 320.
"""
import copy
import time

import numpy as np
import pytest
import torch

from oracle import virtex_oracle as O
from tests import attention_replica as AR
from tests import dropout_replica as R
from tests import head_stages as S
from tests.helpers import build_model, to_cuda
from tests.test_head_kernels_gpu import _allowed, _flip_floor, _heads, _rb, assert_bf16, assert_f32, rel

pytestmark = pytest.mark.gpu

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
DEV = "cuda"
SEEDS = (1, 2 ** 64 - 1)


def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _s():
    return torch.cuda.current_stream().cuda_stream


def _seed(s):
    return torch.tensor([R.as_i64(s)], dtype=torch.int64, device=DEV)


def _inputs(B, A, Tq, Tk, causal, g, lengths=None):
    """Strided bf16 views as the engine passes them and the caption lengths (1 and Tq included when B allows)."""
    H = A * 64
    if causal:
        qkv = torch.randn(B * Tq, 3 * H, generator=g).to(BF16).to(DEV)
        q, k, v = qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:]
    else:
        q = torch.randn(B * Tq, H, generator=g).to(BF16).to(DEV)
        kv = torch.randn(B * Tk, 2 * H, generator=g).to(BF16).to(DEV)
        k, v = kv[:, :H], kv[:, H:]
    if lengths is None:
        lengths = torch.randint(1, Tq + 1, (B,), generator=g)
        lengths[0] = Tq
        if B > 1:
            lengths[1] = 1
    dout = torch.randn(B * Tq, H, generator=g).to(BF16).to(DEV)
    return q, k, v, dout, lengths.to(DEV)


def _launch(ops, q, k, v, dout, lengths, B, A, Tq, Tk, causal, p, sd, site, ldo):
    """vtx_attn_fwd then vtx_attn_bwd into sentinel-filled buffers -> (out, lse, dq, dk, dv) with their padding."""
    H = A * 64
    Qs, _ = AR.attn_rows(Tq, Tk)
    out = torch.full((B * Tq, ldo), -777.0, dtype=BF16, device=DEV)
    lse = torch.full((B * A * Qs + 5,), -777.0, device=DEV)
    lp = lengths.data_ptr() if causal else 0
    ops.call("vtx_attn_fwd", q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
             out.data_ptr(), ldo, lse.data_ptr(), B, A, Tq, Tk, lp, causal, p, sd.data_ptr(), site, _s())
    dq = torch.full((B * Tq, q.stride(0)), -777.0, dtype=BF16, device=DEV)
    dkv = torch.full((B * Tk, 2 * H), -777.0, dtype=BF16, device=DEV)
    ops.call("vtx_attn_bwd", q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
             dout.data_ptr(), H, lse.data_ptr(), dq.data_ptr(), dq.stride(0), dkv.data_ptr(), 2 * H,
             dkv[:, H:].data_ptr(), 2 * H, B, A, Tq, Tk, lp, causal, p, sd.data_ptr(), site, _s())
    return out, lse, dq, dkv


KERNEL_CASES = [  # (Tq, Tk, causal, B, A)
    (33, 33, 1, 5, 3), (32, 65, 0, 5, 3), (48, 48, 2, 5, 3),
    (64, 64, 1, 64, 1), (100, 100, 1, 100, 1),               # every length 1 .. T
    (30, 81, 0, 4, 3), (30, 100, 0, 4, 3), (30, 144, 0, 4, 3), (1, 400, 0, 6, 2),
    (1024, 1024, 1, 2, 1), (30, 1024, 0, 2, 2),
]


@pytest.mark.parametrize("Tq,Tk,causal,B,A", KERNEL_CASES)
def test_long_attention_forward_backward(Tq, Tk, causal, B, A):
    """O, LSE, dQ, dK, dV against float64 (same roundings and plain), p = 0 and 0.1; nothing outside the written rows
    and columns changes (LSE rows Tq .. Qs of each (b, h), the ld padding of O)."""
    _need_cuda()
    from virtex_b200 import ops
    H = A * 64
    g = torch.Generator().manual_seed(Tq * 1000 + Tk + causal)
    lengths = None
    if B == Tq and causal:   # ragged: one caption of every length 1 .. T
        lengths = torch.randperm(Tq, generator=g) + 1
    q, k, v, dout, lengths = _inputs(B, A, Tq, Tk, causal, g, lengths)
    Qs, _ = AR.attn_rows(Tq, Tk)
    ldo = H + 64
    ok = _allowed(B, Tq, Tk, causal, lengths)
    q4, k4, v4, do4 = _heads(q, B, Tq, A), _heads(k, B, Tk, A), _heads(v, B, Tk, A), _heads(dout, B, Tq, A)
    s = (q4 @ k4.transpose(-1, -2) * 0.125).masked_fill(~ok, float("-inf"))
    lse_ref = torch.logsumexp(s, -1)
    P = torch.softmax(s, -1)
    pu = torch.exp(s - s.amax(-1, keepdim=True))
    psum = pu.sum(-1, keepdim=True)
    for p in (0.0, 0.1):
        for seed in (SEEDS if p else SEEDS[:1]):
            site = 1032
            tag = f"B={B} A={A} Tq={Tq} Tk={Tk} causal={causal} p={p} seed={seed}"
            Mk = torch.from_numpy(AR.attn_scale(seed, site, B, A, Tq, Tk, p)).to(DEV, F64)
            out, lse, dq, dkv = _launch(ops, q, k, v, dout, lengths, B, A, Tq, Tk, causal, p, _seed(seed), site, ldo)
            lk = lse[:B * A * Qs].view(B, A, Qs)
            assert_f32(lk[..., :Tq], lse_ref, "lse " + tag, scale=lse_ref.abs().max().item() + 1.0)
            assert (lk[..., Tq:] == -777).all() and (lse[B * A * Qs:] == -777).all(), "lse padding rows written"
            assert (out[:, H:] == -777).all(), "out ld padding written"
            o_k = _heads(out[:, :H], B, Tq, A)
            pd = _rb(pu * Mk)
            assert_bf16(o_k, pd @ v4 / psum, _flip_floor(pd / psum, v4), "out (same roundings) " + tag)
            assert rel(o_k, (P * Mk) @ v4) <= 1e-2, ("out vs float64", tag)
            dq4, dk4, dv4 = _heads(dq[:, :H], B, Tq, A), _heads(dkv[:, :H], B, Tk, A), _heads(dkv[:, H:], B, Tk, A)
            if q.stride(0) > H:
                assert (dq[:, H:] == -777).all(), "dq ld padding written"
            dP = do4 @ v4.transpose(-1, -2) * Mk
            D = (P * dP).sum(-1, keepdim=True)
            dS = P * (dP - D) * 0.125
            dSr, pdb = _rb(dS), _rb(P * Mk)
            dPmag = do4.abs() @ v4.abs().transpose(-1, -2) * Mk
            dSmag = P * ((dPmag + (P * dPmag).sum(-1, keepdim=True)) * 0.125)
            fl_q = _flip_floor(dSr, k4) + 2.0 ** -16 * (dSmag @ k4.abs())
            fl_k = _flip_floor(dSr.transpose(-1, -2), q4) + 2.0 ** -16 * (dSmag.transpose(-1, -2) @ q4.abs())
            assert_bf16(dq4, dSr @ k4, fl_q, "dq (same roundings) " + tag)
            assert_bf16(dk4, dSr.transpose(-1, -2) @ q4, fl_k, "dk (same roundings) " + tag)
            assert_bf16(dv4, pdb.transpose(-1, -2) @ do4, _flip_floor(pdb.transpose(-1, -2), do4),
                        "dv (same roundings) " + tag)
            del fl_q, fl_k
            qa, ka, va = (t.clone().requires_grad_(True) for t in (q4, k4, v4))
            sa = (qa @ ka.transpose(-1, -2) * 0.125).masked_fill(~ok, float("-inf"))
            ((torch.softmax(sa, -1) * Mk) @ va).backward(do4)
            for name, got, ref in (("dq", dq4, qa.grad), ("dk", dk4, ka.grad), ("dv", dv4, va.grad)):
                assert rel(got, ref) <= 1e-2, (name, rel(got, ref), tag)
    torch.cuda.empty_cache()


@pytest.mark.parametrize("B,A,Tq,Tk", [(3, 2, 33, 33), (2, 3, 32, 65), (2, 2, 48, 100), (2, 1, 30, 400),
                                      (1, 2, 70, 1024)])
def test_long_attention_dropout_mask_element_by_element(B, A, Tq, Tk):
    """Q = K = 0 (equal scores) and V = the one-hot rows e_(j - w0) for the keys j of one 64-key window w0, zero
    elsewhere: out row i of head h, column c, is the dropped probability of key w0 + c, bf16(1/(1-p)) / Tk where the
    replay keeps it and 0 where it drops it.  Every window of keys is checked, at two seeds and two sites."""
    _need_cuda()
    from virtex_b200 import ops
    p = 0.1
    ik = float(R.inv_keep(p))
    Hh = A * 64
    kept = (torch.tensor(ik, dtype=F32).to(BF16).float() * torch.tensor(1.0 / Tk, dtype=F32)).to(BF16).to(DEV)
    q = torch.zeros(B * Tq, Hh, dtype=BF16, device=DEV)
    k = torch.zeros(B * Tk, Hh, dtype=BF16, device=DEV)
    Qs, _ = AR.attn_rows(Tq, Tk)
    lse = torch.empty(B * A * Qs, device=DEV)
    for seed in SEEDS:
        for site in (14, 2045):
            msk = torch.from_numpy(AR.attn_scale(seed, site, B, A, Tq, Tk, p)).to(DEV)
            for w0 in range(0, Tk, 64):
                n = min(64, Tk - w0)
                v = torch.zeros(B, Tk, A, 64, dtype=BF16, device=DEV)
                v[:, w0 + torch.arange(n), :, torch.arange(n)] = 1
                o = torch.empty(B * Tq, Hh, dtype=BF16, device=DEV)
                ops.call("vtx_attn_fwd", q.data_ptr(), Hh, k.data_ptr(), Hh, v.view(B * Tk, Hh).data_ptr(), Hh,
                         o.data_ptr(), Hh, lse.data_ptr(), B, A, Tq, Tk, 0, 0, p, _seed(seed).data_ptr(), site, _s())
                got = o.view(B, Tq, A, 64).permute(0, 2, 1, 3)[..., :n]
                m = msk[..., w0:w0 + n]
                assert torch.equal(got != 0, m != 0), ("mask", seed, site, w0)
                assert (got[m != 0] == kept).all(), ("kept values", seed, site, w0)
                assert (o.view(B, Tq, A, 64)[..., n:] == 0).all()


@pytest.mark.parametrize("Tq,Tk,causal", [(100, 100, 1), (30, 400, 0), (64, 64, 2)])
def test_long_attention_is_deterministic(Tq, Tk, causal):
    """Two launches on the same inputs give bit-identical O, LSE and gradients (no atomics, fixed reduction order)."""
    _need_cuda()
    from virtex_b200 import ops
    B, A = 16, 4
    g = torch.Generator().manual_seed(5)
    q, k, v, dout, lengths = _inputs(B, A, Tq, Tk, causal, g)
    runs = [_launch(ops, q, k, v, dout, lengths, B, A, Tq, Tk, causal, 0.1, _seed(77), 31, A * 64) for _ in range(2)]
    for a, b in zip(*runs):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16)) if a.dtype == BF16 else torch.equal(a, b)


def test_long_attention_rejects_shapes_past_the_limit():
    _need_cuda()
    from virtex_b200 import ops
    from virtex_b200.engine import ATTN_MAX_T
    x = torch.zeros(8, 64, dtype=BF16, device=DEV)
    lse = torch.zeros(64, device=DEV)
    for Tq, Tk in ((ATTN_MAX_T + 1, 8), (8, ATTN_MAX_T + 1), (0, 8)):
        with pytest.raises(RuntimeError, match="unsupported shape"):
            ops.call("vtx_attn_fwd", x.data_ptr(), 64, x.data_ptr(), 64, x.data_ptr(), 64, x.data_ptr(), 64,
                     lse.data_ptr(), 1, 1, Tq, Tk, 0, 0, 0.0, 0, 0, _s())


# ------------------------------------------------------------------------------------------------ sublayer replay
REPLAY_CASES = [  # (hidden, layers, heads, ffn, norm_first, task, B, T)
    pytest.param(512, 1, 8, 2048, False, "bicap", 3, 48, id="L1-H512-bicap-T48"),
    pytest.param(512, 2, 8, 2048, True, "cap", 3, 48, id="L2-H512-prenorm-cap-T48"),
    pytest.param(512, 1, 8, 2048, False, "mlm", 3, 64, id="L1-H512-mlm-T64"),
]


@pytest.mark.parametrize("H,L,A,Fd,norm_first,task,B,T", REPLAY_CASES)
def test_head_stages_replay_at_100_keys(H, L, A, Fd, norm_first, task, B, T, monkeypatch):
    """tests/test_head_stages_gpu.py's stage-by-stage replay of Engine.forward / backward with a 10 x 10 feature grid
    (100 cross-attention keys) and T = 48 or 64 tokens, dropout 0.1: every attention launch runs the long kernels."""
    _need_cuda()
    from tests.test_head_stages_gpu import PAD, SEED, WGRAD_INFO, Replay, _batch, _finish_totals
    from virtex_b200.engine import Engine
    from virtex_b200.modules import TransformerDecoderTextualHead
    # the replay reads attention masks through tests/dropout_replica.attn_scale, whose layout covers Tq <= 32 and
    # Tk <= 64 only: give it the kernels' layout at every shape
    monkeypatch.setattr(R, "attn_scale", AR.attn_scale)
    t0 = time.time()
    V, Cv, Sk = 10000, 2048, 100
    torch.manual_seed(H + L + B + T)
    g = torch.Generator().manual_seed(H * 10 + L + B + T)
    textual = TransformerDecoderTextualHead(visual_feature_size=Cv, vocab_size=V, hidden_size=H, num_layers=L,
                                            attention_heads=A, feedforward_size=Fd, dropout=0.1, norm_first=norm_first,
                                            mask_future_positions=task != "mlm", max_caption_length=T,
                                            padding_idx=PAD)
    with torch.no_grad():
        for n, p in textual.named_parameters():
            if p.dim() == 1:
                p.copy_((1.0 if n.endswith("weight") and "norm" in n else 0.0) + 0.1 * torch.randn(p.shape, generator=g))
        textual.embedding.words.weight[PAD] = 0.02 * torch.randn(H, generator=g)
    backward = None
    if task == "bicap":
        backward = copy.deepcopy(textual)
        with torch.no_grad():
            for p in backward.transformer.parameters():
                p.add_(0.01 * torch.randn(p.shape, generator=g))
        backward.visual_projection = textual.visual_projection
        backward.embedding = textual.embedding
        backward.output = textual.output
    textual.cuda()
    if backward is not None:
        backward.cuda()
    eng = Engine(None, textual, backward)
    eng.prepare_weights()
    eng.seed.fill_(R.as_i64(SEED))
    tokens, noitpac, lengths, labels = (t.cuda() if t is not None else None for t in _batch(B, T, V, task, g))
    feat = (torch.randn(B * Sk, Cv, generator=g).abs() * 0.5).to(BF16).cuda()
    rp = Replay(eng, f"{task} L{L} H{H} B={B} T={T} Sk={Sk} norm_first={int(norm_first)}", tokens, noitpac, lengths,
                labels, feat, None)
    rp.B, rp.T = B, T
    rp.install(monkeypatch)
    rp.cross_seen = 0
    got_dfeat = []
    monkeypatch.setattr(eng, "backbone_forward", lambda image, training: (feat, 10, 10))
    monkeypatch.setattr(eng, "backbone_backward", lambda dfeat, cb=None: got_dfeat.append(dfeat))
    orig_vp = eng.visual_projection_forward

    def vp(f, S_):
        mem = orig_vp(f, S_)
        rp.check_mem(mem)
        return mem
    monkeypatch.setattr(eng, "visual_projection_forward", vp)
    image = torch.empty(B, 1, 320, 320, device="cuda")
    with torch.no_grad():
        eng.forward(image, tokens, noitpac, lengths, training=True, with_grad=True, labels=labels)
        eng.backward()
        assert len(got_dfeat) == 1
        rp.on_feature_grad(got_dfeat[0])
        assert rp.cross_seen == L * (2 if backward is not None else 1)
        _finish_totals(rp)
        rp.check_kept()
        torch.cuda.synchronize()
    rp.report(WGRAD_INFO)
    print(f"wall time {time.time() - t0:.1f} s")


# ------------------------------------------------------------------------------------------------ whole model
def _cos(a, b):
    a, b = a.detach().double().cpu().flatten(), b.detach().double().cpu().flatten()
    return (a @ b / (a.norm() * b.norm() + 1e-30)).item()


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-20)).item()


SPEC_288 = dict(hidden=128, layers=1, heads=2, ffn=256, max_len=40)


def test_model_at_crop_288_and_40_tokens_vs_oracle():
    """Crop 288 (a 9 x 9 grid: 81 cross-attention keys) and 40 tokens, p = 0: training loss within 1e-3 relative of the
    fp32 oracle, head gradients cos > 0.998 and rel < 5e-2 (test_gpu_parity's bounds); eval argmax equal to the
    oracle's wherever its top-2 margin exceeds the bf16 noise floor (0.25)."""
    _need_cuda()
    spec = O.Spec(**SPEC_288)
    state = O.synth_state(spec, 11, bn3_gain=0.25)
    model = build_model(spec, state)
    model.train()
    batch = O.synth_batch(4, seed=6, ragged=True, max_len=40, image_size=288)
    out = model(to_cuda(batch))
    ref, grads, _ = O.loss_and_grads(state, batch, spec)
    assert abs(out["loss"].item() - ref["loss"].item()) < 1e-3 * ref["loss"].item(), (out["loss"].item(),
                                                                                      ref["loss"].item())
    out["loss"].backward()
    named = dict(model.named_parameters())
    bad = [(n, _rel(named[n].grad, gr), _cos(named[n].grad, gr)) for n, gr in grads.items()
           if not n.startswith("visual.") and not (_cos(named[n].grad, gr) > 0.998 and _rel(named[n].grad, gr) < 5e-2)]
    assert not bad, bad
    model.eval()
    with torch.no_grad():
        out = model(to_cuda(batch))
        ref = O.model_forward(state, batch, spec, training=False, return_logits=True)
    assert abs(out["loss"].item() - ref["loss"].item()) < 2e-3 * ref["loss"].item()
    pred, pref = out["predictions"].cpu(), ref["predictions"]
    top2 = ref["logits"].topk(2, dim=-1).values
    confident = (top2[..., 0] - top2[..., 1]) > 0.25
    assert torch.equal(pred[confident], pref[confident])


def test_trainer_step_at_crop_288_and_40_tokens_vs_autograd():
    """Two Trainer.step calls against model -> loss.backward() -> clip -> OptimizerFactory step on a twin, at crop 288
    and MAX_CAPTION_LENGTH 40 (Config overrides): losses within 1e-3 relative, head updates within 5e-2."""
    _need_cuda()
    from virtex_b200.config import Config
    from virtex_b200.factories import LRSchedulerFactory, OptimizerFactory
    from virtex_b200.trainer import Trainer
    spec = O.Spec(**SPEC_288)
    cfg = Config(None, ["MODEL.TEXTUAL.NAME", "transdec_postnorm::L1_H128_A2_F256", "MODEL.TEXTUAL.DROPOUT", 0.0,
                        "DATA.IMAGE_CROP_SIZE", 288, "DATA.MAX_CAPTION_LENGTH", 40, "OPTIM.WARMUP_STEPS", 0,
                        "OPTIM.NUM_ITERATIONS", 100, "OPTIM.BATCH_SIZE", 4])
    state = O.synth_state(spec, 3, bn3_gain=0.25)
    model, twin = build_model(spec, state).train(), build_model(spec, state).train()
    trainer = Trainer(model, cfg)
    opt = OptimizerFactory.from_config(cfg, twin.named_parameters())
    sched = LRSchedulerFactory.from_config(cfg, opt)
    for it in range(2):
        batch = to_cuda(O.synth_batch(4, seed=30 + it, ragged=True, max_len=40, image_size=288))
        loss = trainer.step(batch).sum().item()
        opt.zero_grad()
        out = twin(batch)
        out["loss"].backward()
        torch.nn.utils.clip_grad_norm_(twin.parameters(), cfg.OPTIM.CLIP_GRAD_NORM)
        opt.step()
        sched.step()
        assert abs(loss - out["loss"].item()) < 1e-3 * out["loss"].item(), (it, loss, out["loss"].item())
    torch.cuda.synchronize()
    a, b = dict(model.named_parameters()), dict(twin.named_parameters())
    for name in ("textual.output.bias", "textual.transformer.layers.0.linear1.weight",
                 "textual.transformer.layers.0.multihead_attn.in_proj_weight"):
        d_a, d_b = a[name].detach().cpu() - state[name], b[name].detach().cpu() - state[name]
        assert d_b.norm() > 0 and _rel(d_a, d_b) < 5e-2, (name, _rel(d_a, d_b))


@pytest.mark.parametrize("config,task", [(None, "captioning"), ("task_ablations/masked_lm_R_50_L1_H2048.yaml",
                                                                "masked_lm")])
def test_full_size_step_at_crop_384_and_64_tokens(config, task):
    """R50-L1-H1024 at DATA.IMAGE_CROP_SIZE 384 (144 keys) and MAX_CAPTION_LENGTH 64, batch 256 built by
    GpuInputPipeline.from_config: one Trainer.step gives a finite loss; the peak device memory is printed."""
    _need_cuda()
    from tests import masked_lm_oracle as MO
    from virtex_b200.config import Config
    from virtex_b200.data_gpu import GpuInputPipeline
    from virtex_b200.factories import PretrainingModelFactory
    from virtex_b200.trainer import Trainer
    cfg = Config(config, ["MODEL.TEXTUAL.NAME", "transdec_postnorm::L1_H1024_A16_F4096", "DATA.IMAGE_CROP_SIZE", 384,
                          "DATA.MAX_CAPTION_LENGTH", 64])
    torch.manual_seed(0)
    model = PretrainingModelFactory.from_config(cfg).cuda().train()
    trainer = Trainer(model, cfg)
    pipe = GpuInputPipeline.from_config(cfg, "cuda")
    assert pipe.task == task and pipe.S == 384 and pipe.max_len == 64
    g = np.random.default_rng(2)
    B = 256
    images = [g.integers(0, 256, (400, 420, 3), dtype=np.uint8) for _ in range(B)]
    lists = [[MO.SOS] + [int(x) for x in g.integers(4, 10000, int(g.integers(6, 80)))] + [MO.EOS] for _ in range(B)]
    params = [pipe.sample_train_params(g, 400, 420) for _ in range(B)]
    batch = pipe(images, params, lists)
    assert tuple(batch["image"].shape) == (B, 3, 384, 384) and batch["caption_tokens"].shape[1] == 64
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    loss = trainer.step(batch)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    print(f"{task} R50-L1-H1024 crop 384, T 64, batch {B}: loss {loss.sum().item():.4f}, peak allocated {peak:.2f} GiB")
    assert torch.isfinite(loss).all()


def test_decoding_step_at_crop_320_vs_float64_head():
    """model.decoding_step on 10 x 10 features (a 320 x 320 image: 100 cross-attention keys) against the float64 head
    of tests/head_stages.py on the bf16 features: the next-token logits of every partial caption within 2e-2 relative
    L2 (bf16 activations and weights through two layers)."""
    _need_cuda()
    from virtex_b200.models import ForwardCaptioningModel
    from virtex_b200.modules import TorchvisionVisualBackbone, TransformerDecoderTextualHead
    torch.manual_seed(4)
    textual = TransformerDecoderTextualHead(2048, 1000, 256, 2, 4, 1024, dropout=0.1, max_caption_length=30)
    model = ForwardCaptioningModel(TorchvisionVisualBackbone("resnet50", 2048), textual).cuda().eval()
    feats = torch.randn(2, 2048, 10, 10, device=DEV).abs() * 0.5
    g = torch.Generator().manual_seed(9)
    partial = torch.randint(4, 1000, (6, 7), generator=g)
    partial[:, 0] = 1
    with torch.no_grad():
        got = model.decoding_step(feats, partial.cuda())
    assert tuple(got.shape) == (6, 1000)
    P = {"textual." + n: p.detach().to(F64) for n, p in textual.named_parameters()}
    f = feats.repeat_interleave(3, 0).permute(0, 2, 3, 1).reshape(6, 100, 2048).to(BF16).to(F64)
    vals, _, _ = S.head_forward_backward(P, "textual.", f, partial.cuda(), torch.full((6,), 7, device=DEV), 0, 4,
                                         False, 1)
    ref = vals["logits"][:, -1]
    assert _rel(got, ref) < 2e-2, _rel(got, ref)
