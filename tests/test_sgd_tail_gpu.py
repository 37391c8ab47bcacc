"""The fused SGD optimiser tail on the H100, element by element against float64 (tests/sgd_tail.py, pinned to
clip_grad_norm_ / Lookahead(SGD) / LambdaLR by tests/test_sgd_tail_cpu.py):

  * kernels: vtx_sumsq, vtx_clip_coef and vtx_sgd_step against sumsq64 / clip64 / sgd64 within bounds derived from
    their fp32 operation sequence; the bf16 mirror bit-exact; everything outside the segments bit-identical;
  * Trainer replay: every step of a Trainer re-done in float64 from its own gradient arena, with lr / wd from the
    reference recipe's param groups and schedule, the packed conv-weight layouts checked against a fresh re-pack, and
    the host-side Lookahead / momentum / iteration state; SGD resume from a checkpoint; a two-rank step emulated in
    one process;
  * the gradient-bucket contract of Engine.backward(bucket_cb=...): a bucket's range is final when its tag fires.
"""
import struct

import pytest
import torch

from oracle import virtex_oracle as O
from tests import classification_oracle as CO
from tests import sgd_tail as T

pytestmark = pytest.mark.gpu


def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _call(name, *args):
    from virtex_b200.ops import _stream, call
    call(name, *args, _stream())


def _num_sms():
    from virtex_b200 import ops
    return ops.num_sms()


def _seg_blob(segs, dev="cuda"):
    return torch.frombuffer(bytearray(b"".join(struct.pack("<qqff", *s) for s in segs)), dtype=torch.uint8).to(dev)


# ------------------------------------------------------------------------------------------------------------ kernels
@pytest.mark.parametrize("n", [1, 3, 4, 5, 255, 1021, 3 * 65536 + 13, 5_000_011])
def test_sumsq_kernel_against_float64(n):
    """Magnitudes spread over 1e-20 ... 1e3 with zeros among them, the n % 4 scalar tail at 1e3; the largest n takes
    more than one sweep of the 8 * SMs blocks.  Into a zeroed and into a preset `out`."""
    _need_cuda()
    gen = torch.Generator(device="cuda").manual_seed(n)
    mag = 10.0 ** (torch.rand(n, generator=gen, device="cuda", dtype=torch.float64) * 23.0 - 20.0)
    x = (torch.randn(n, generator=gen, device="cuda", dtype=torch.float64).sign() * mag).float()
    x[torch.rand(n, generator=gen, device="cuda") < 0.1] = 0.0
    x[4 * (n // 4):] = 1e3  # a kernel that skips its scalar tail is off by 1e6 per element
    assert x.data_ptr() % 16 == 0
    s64 = T.sumsq64(x)
    for preset in (0.0, 0.75 * s64):
        out = torch.tensor([preset], dtype=torch.float32, device="cuda")
        p32 = out.item()
        _call("vtx_sumsq", x.data_ptr(), n, out.data_ptr())
        torch.cuda.synchronize()
        err = abs(out.item() - (p32 + s64))
        assert err <= T.sumsq_bound(n, s64, _num_sms(), p32), (n, preset, err)


def test_sumsq_kernel_of_nothing_leaves_out_untouched():
    _need_cuda()
    x = torch.ones(8, device="cuda")
    out = torch.tensor([1.2345], device="cuda")
    _call("vtx_sumsq", x.data_ptr(), 0, out.data_ptr())
    torch.cuda.synchronize()
    assert out.item() == torch.tensor(1.2345).item()


@pytest.mark.parametrize("world", [1, 2, 8])
def test_clip_coef_kernel_against_float64(world):
    """Norms below, at and above max_norm, a zero and a huge sum of squares within the bound of clip64; an inf norm
    gives the coefficient 0 and a NaN norm a NaN coefficient (torch.clamp keeps it); max_norm <= 0 does not clip."""
    _need_cuda()
    max_norm = 10.0
    ctl = torch.empty(2, device="cuda")
    for s in (0.0, (0.5 * max_norm * world) ** 2, (max_norm * world) ** 2, (2.0 * max_norm * world) ** 2, 1e30,
              float("inf"), float("nan")):
        ssq = torch.tensor([s], dtype=torch.float32, device="cuda")
        ctl.fill_(-7.0)
        _call("vtx_clip_coef", ssq.data_ptr(), world, max_norm, ctl.data_ptr())
        torch.cuda.synchronize()
        c, nrm = ctl.tolist()
        coef, norm = T.clip64(float(ssq.item()), world, max_norm)
        if s != s:
            assert c != c and nrm != nrm, (world, c, nrm)
            continue
        if s == float("inf"):
            assert c == 0.0 and nrm == float("inf"), (world, c, nrm)
            continue
        dcoef, dnorm = T.clip_bound(coef, norm, 0.0, s)
        assert abs(c - coef) <= dcoef and abs(nrm - norm) <= dnorm, (world, s, c, coef, nrm, norm)
    for m in (0.0, -1.0):
        for s in (4e6, float("nan")):
            ssq = torch.tensor([s], dtype=torch.float32, device="cuda")
            _call("vtx_clip_coef", ssq.data_ptr(), world, m, ctl.data_ptr())
            torch.cuda.synchronize()
            assert ctl[0].item() == 1.0 / world, (world, m, s)


# (begin, end, lr, wd): a 3-chunk tensor with a 13-element tail, a wd = 0 tensor, a gap, a short odd tensor, a gap
_TENSORS = [(0, 2 * 65536 + 13, 0.2, 1e-4), (2 * 65536 + 13, 200_000, 1e-3, 0.0), (210_000, 210_777, 5e-3, 1e-2),
            (211_000, 300_000, 1e-3, 1e-4)]
_N = 300_017


def _arenas(seed):
    gen = torch.Generator(device="cuda").manual_seed(seed)
    p = torch.randn(_N, generator=gen, device="cuda")
    g = torch.randn(_N, generator=gen, device="cuda")
    g *= torch.logspace(-9, 0, _N, device="cuda")[torch.randperm(_N, generator=gen, device="cuda")]
    m = torch.randn(_N, generator=gen, device="cuda") * 0.1  # non-zero even on the first step: it must be ignored
    slow = torch.randn(_N, generator=gen, device="cuda")
    bf = torch.full((_N,), 7.0, device="cuda", dtype=torch.bfloat16)
    return p, g, m, slow, bf


@pytest.mark.parametrize("step", ["first", "steady", "lookahead", "lookahead_without_slow"])
@pytest.mark.parametrize("world,max_norm", [(1, 1e6), (2, 1.0)], ids=["unclipped", "clipped-world2"])
def test_sgd_step_kernel_against_float64(step, world, max_norm):
    """vtx_sumsq -> vtx_clip_coef -> vtx_sgd_step on ragged 64 Ki chunks with a wd = 0 group and gaps standing for
    frozen tensors: parameters, momentum and slow weights within the derived bound of sgd64, slow == p bit-exactly
    after a Lookahead step, the bf16 mirror == bf16(p), and every element outside the segments (parameter, momentum,
    slow weight, mirror) bit-identical.  do_la with slow = nullptr is a plain step."""
    _need_cuda()
    p, g, m, slow, bf = _arenas(11)
    segs = [(c, min(e, c + 65536), lr, wd) for b, e, lr, wd in _TENSORS for c in range(b, e, 65536)]
    blob = _seg_blob(segs)
    p0, m0, s0, bf0 = p.clone(), m.clone(), slow.clone(), bf.clone()
    first = step == "first"
    do_la = step.startswith("lookahead")
    use_slow = step != "lookahead_without_slow"
    sumsq = torch.zeros(1, device="cuda")
    ctl = torch.zeros(2, device="cuda")
    _call("vtx_sumsq", g.data_ptr(), _N, sumsq.data_ptr())
    _call("vtx_clip_coef", sumsq.data_ptr(), world, max_norm, ctl.data_ptr())
    mult, alpha = 0.37, 0.5
    hyper = torch.tensor([mult, float(first), float(do_la), 0.0], device="cuda")
    _call("vtx_sgd_step", p.data_ptr(), g.data_ptr(), m.data_ptr(), slow.data_ptr() if use_slow else 0, bf.data_ptr(),
          blob.data_ptr(), len(segs), ctl.data_ptr(), hyper.data_ptr(), 0.9, alpha)
    torch.cuda.synchronize()
    # the kernel sees the summed gradient of `world` ranks: the mean is g / world
    gm = g.double() / world
    s64 = T.sumsq64(gm)
    coef, norm = T.clip64(s64, 1, max_norm)
    dcoef, dnorm = T.clip_bound(coef, norm, T.sumsq_bound(_N, s64, _num_sms()), s64)
    assert (coef < 1.0) == (max_norm == 1.0)
    assert abs(ctl[0].item() * world - coef) <= dcoef and abs(ctl[1].item() - norm) <= dnorm, (ctl.tolist(), coef)
    inside = torch.zeros(_N, dtype=torch.bool, device="cuda")
    for b, e, lr, wd in _TENSORS:
        inside[b:e] = True
        args = (p0[b:e], gm[b:e], m0[b:e], s0[b:e] if use_slow else None, lr, wd, mult)
        rp, rm, _ = T.sgd64(*args, coef, first, do_la, alpha)
        tol_p, tol_m = T.sgd_tol(*args, coef, dcoef, first, do_la, alpha)
        err_p, err_m = (p[b:e].double() - rp).abs(), (m[b:e].double() - rm).abs()
        assert (err_p <= tol_p).all(), (b, e, (err_p / tol_p).max().item())
        assert (err_m <= tol_m).all(), (b, e, (err_m / tol_m).max().item())
        if do_la and use_slow:
            assert torch.equal(slow[b:e], p[b:e]), (b, e)
        assert torch.equal(bf[b:e], p[b:e].bfloat16()), (b, e)
    out = ~inside
    for x, x0 in ((p, p0), (m, m0), (slow, s0), (bf, bf0)):
        assert torch.equal(x[out], x0[out])
    if not (do_la and use_slow):
        assert torch.equal(slow, s0)


@pytest.mark.parametrize("optimizer", ["sgd", "adamw"])
def test_nan_gradient_norm_makes_every_updated_parameter_nan(optimizer):
    """One NaN gradient element makes the norm NaN; clip_grad_norm_ then multiplies every gradient by NaN, so a torch
    step writes NaN into every parameter.  The fused tail does the same (a clamp that dropped the NaN would run the
    step unclipped on every finite element); elements outside the segments stay untouched."""
    _need_cuda()
    p, g, m, slow, bf = _arenas(5)
    g[123_456] = float("nan")
    segs = [(c, min(e, c + 65536), lr, wd) for b, e, lr, wd in _TENSORS for c in range(b, e, 65536)]
    blob = _seg_blob(segs)
    p0 = p.clone()
    sumsq = torch.zeros(1, device="cuda")
    ctl = torch.zeros(2, device="cuda")
    _call("vtx_sumsq", g.data_ptr(), _N, sumsq.data_ptr())
    _call("vtx_clip_coef", sumsq.data_ptr(), 1, 10.0, ctl.data_ptr())
    if optimizer == "sgd":
        hyper = torch.tensor([1.0, 0.0, 0.0, 0.0], device="cuda")
        _call("vtx_sgd_step", p.data_ptr(), g.data_ptr(), m.data_ptr(), slow.data_ptr(), bf.data_ptr(), blob.data_ptr(),
              len(segs), ctl.data_ptr(), hyper.data_ptr(), 0.9, 0.5)
    else:
        v = m * m
        hyper = torch.tensor([1.0, 10.0, 3.0, 0.0], device="cuda")
        _call("vtx_adamw_step", p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), slow.data_ptr(), bf.data_ptr(),
              blob.data_ptr(), len(segs), ctl.data_ptr(), hyper.data_ptr(), 0.9, 0.999, 1e-8, 0.5)
    torch.cuda.synchronize()
    assert ctl[0].isnan() and ctl[1].isnan()
    inside = torch.zeros(_N, dtype=torch.bool, device="cuda")
    for b, e, _, _ in _TENSORS:
        inside[b:e] = True
    assert p[inside].isnan().all() and bf[inside].isnan().all()
    assert torch.equal(p[~inside], p0[~inside])


# ------------------------------------------------------------------------------------------------------------- models
_HEAD = ["MODEL.TEXTUAL.NAME", "transdec_postnorm::L1_H128_A2_F256", "MODEL.TEXTUAL.DROPOUT", 0.0]
_R50 = O.Spec(hidden=128, layers=1, heads=2, ffn=256)
_R18 = O.Spec(backbone="resnet18", hidden=128, layers=1, heads=2, ffn=256)
_ONE_WAY = {"captioning": O.Spec(hidden=128, layers=1, heads=2, ffn=256, caption_backward=False),
            "masked_lm": O.Spec(hidden=128, layers=1, heads=2, ffn=256, caption_backward=False, mask_future=False)}


def _masked_lm_batch(B, seed, mask_index):
    """A captioning batch whose tokens are masked at ~30% of the caption positions (always position 1), with the
    original tokens as `masked_labels` and 0 (ignored) elsewhere."""
    batch = O.synth_batch(B, seed=seed, ragged=True)
    tok = batch["caption_tokens"]
    g = torch.Generator().manual_seed(seed)
    pick = (torch.rand(tok.shape, generator=g) < 0.3) & (tok != 0)
    pick[:, 1] = True
    batch["masked_labels"] = torch.where(pick, tok, torch.zeros_like(tok))
    batch["caption_tokens"] = torch.where(pick, torch.full_like(tok, mask_index), tok)
    return batch


def _model(kind, *extra):
    """(model on the GPU in train mode, config, batch(seed, B)) of one case, with synthetic weights so that every
    gradient of the backbone is non-zero."""
    from virtex_b200.config import Config
    from virtex_b200.factories import PretrainingModelFactory
    if kind == "token_classification":
        cfg = Config("task_ablations/token_classification_R_50.yaml", list(extra))
        sd = CO.synth_classification_state(cfg.DATA.VOCAB_SIZE, 5)

        def batch(seed, B=4):
            return CO.synth_label_batch(B, seed=seed, vocab=cfg.DATA.VOCAB_SIZE, ignore=CO.TOKEN_IGNORE, image_size=224)
    elif kind in _ONE_WAY:
        spec = _ONE_WAY[kind]
        cfg = Config(f"task_ablations/{kind}_R_50_L1_H2048.yaml", _HEAD + list(extra))
        sd = {k: v for k, v in O.to_reference_state_dict(O.synth_state(spec, 7, bn3_gain=0.25), spec).items()
              if not k.startswith("backward_textual.")}

        def batch(seed, B=4):
            if kind == "masked_lm":
                return _masked_lm_batch(B, seed, cfg.DATA.MASK_INDEX)
            return O.synth_batch(B, seed=seed, ragged=True)
    else:
        r18 = kind == "r18"
        spec = _R18 if r18 else _R50
        cfg = Config(None, _HEAD + (["MODEL.VISUAL.NAME", "torchvision::resnet18", "MODEL.VISUAL.FEATURE_SIZE", 512]
                                    if r18 else []) + list(extra))
        state = O.synth_state(spec, 7, bn3_gain=0.25)
        sd = O.to_reference_state_dict(state, spec)

        def batch(seed, B=4):
            return O.synth_batch(B, seed=seed, ragged=True)
    model = PretrainingModelFactory.from_config(cfg)
    model.load_state_dict(sd, strict=True)

    def cuda_batch(seed, B=4):
        return {k: v.cuda() for k, v in batch(seed, B).items()}
    return model.cuda().train(), cfg, cuda_batch


# ----------------------------------------------------------------------------------------------------- Trainer replay
def _check_step(tr, hp, snap, it, first, do_la, world=1):
    """One finished optimiser step of `tr` against sgd64 on its own gradient arena (the mean over `world` summed
    rank gradients), from the state `snap` = (params, momentum, slow, mirror) before it.  Returns whether it clipped."""
    lr, wd, trainable, schedule = hp
    a, eng, O_ = tr.arena, tr.engine, tr.config.OPTIM
    p0, m0, s0, w0 = snap
    gm = a.grads.double() / world
    s64 = T.sumsq64(gm)
    coef, norm = T.clip64(s64, 1, float(O_.CLIP_GRAD_NORM))
    dcoef, dnorm = T.clip_bound(coef, norm, T.sumsq_bound(a.total, s64, _num_sms()), s64)
    assert abs(tr.grad_norm.item() - norm) <= dnorm, (it, tr.grad_norm.item(), norm)
    assert abs(tr.ctl[0].item() * world - coef) <= dcoef, (it, tr.ctl[0].item(), coef)
    alpha, mu, mult = float(O_.LOOKAHEAD.ALPHA), float(O_.SGD_MOMENTUM), schedule(it)
    args = (p0, gm, m0, s0, lr, wd, mult)
    rp, rm, _ = T.sgd64(*args, coef, first, do_la, alpha, mu)
    tol_p, tol_m = T.sgd_tol(*args, coef, dcoef, first, do_la, alpha, mu)
    t, o = trainable, ~trainable
    err_p, err_m = (a.params.double() - rp)[t].abs(), (tr.mom.double() - rm)[t].abs()
    assert (err_p <= tol_p[t]).all(), (it, (err_p / tol_p[t]).max().item())
    assert (err_m <= tol_m[t]).all(), (it, (err_m / tol_m[t]).max().item())
    if do_la:
        assert torch.equal(tr.slow[t], a.params[t]), it
    else:
        assert torch.equal(tr.slow, s0), it
    assert torch.equal(a.mirror[t], a.params[t].bfloat16()), it
    for x, x0 in ((a.params, p0), (tr.mom, m0), (tr.slow, s0), (a.mirror, w0)):
        assert torch.equal(x[o], x0[o]), it  # padding and frozen tensors
    # the packed k > 1 conv-weight layouts the next forward reads were re-packed from the updated parameters
    packed = {k: v.clone() for k, v in eng._packed.items()}
    mirror = a.mirror.clone()
    eng.mark_weights_dirty()
    eng.prepare_weights()
    torch.cuda.synchronize()
    assert packed.keys() == eng._packed.keys()
    for k, v in packed.items():
        assert torch.equal(eng._packed[k], v), (it, k)
    assert torch.equal(a.mirror, mirror), it
    return coef < 1.0


def _snapshot(tr):
    return tr.arena.params.clone(), tr.mom.clone(), tr.slow.clone(), tr.arena.mirror.clone()


def _replay(tr, hp, batches, it0=0, k0=0, first=True):
    """Trainer.step on each batch, each step checked by _check_step; Lookahead every LOOKAHEAD.STEPS steps counted
    from k0.  Returns the clipped flags of the steps."""
    K = int(tr.config.OPTIM.LOOKAHEAD.STEPS)
    k, clipped = k0, []
    for j, batch in enumerate(batches):
        it = it0 + j
        snap = _snapshot(tr)
        tr.step(batch)
        torch.cuda.synchronize()
        k += 1
        do_la = k >= K
        k = 0 if do_la else k
        clipped.append(_check_step(tr, hp, snap, it, first and j == 0, do_la))
        assert tr._k_counter == k and tr.momentum_ready and tr.iteration == it + 1, (it, tr._k_counter, k)
    return clipped


def _grad_norm(model, batch):
    _forward(model, batch)
    model.engine.backward(zero_grads=True)
    return T.sumsq64(model.engine.arena.grads) ** 0.5


_OPTIM = ["OPTIM.WARMUP_STEPS", 3, "OPTIM.NUM_ITERATIONS", 20, "OPTIM.CNN_LR", 0.005, "OPTIM.LOOKAHEAD.STEPS", 3]
_REPLAYS = {
    # 7 steps: warm-up ends after step 3, Lookahead at steps 3 and 6
    "r50-clip10": ("r50", 7, _OPTIM),
    "r50-clip-small": ("r50", 7, _OPTIM),  # CLIP_GRAD_NORM set from the batches' gradient norms
    "r18-multistep": ("r18", 7, ["OPTIM.LR_DECAY_NAME", "multistep", "OPTIM.LR_STEPS", [4, 6], "OPTIM.LR_GAMMA", 0.1,
                                 "OPTIM.WARMUP_STEPS", 2, "OPTIM.NUM_ITERATIONS", 20, "OPTIM.CNN_LR", 0.005,
                                 "OPTIM.LOOKAHEAD.STEPS", 3]),
    "r50-frozen": ("r50", 4, _OPTIM + ["MODEL.VISUAL.FROZEN", True]),
    "token-classification": ("token_classification", 4, ["OPTIM.WARMUP_STEPS", 2, "OPTIM.NUM_ITERATIONS", 20,
                                                         "OPTIM.LOOKAHEAD.STEPS", 3]),
}


@pytest.mark.parametrize("case", list(_REPLAYS))
def test_trainer_steps_replayed_in_float64(case):
    """Every Trainer.step: the gradient norm and clip coefficient within the sumsq bound; parameters, momentum and
    slow weights element by element within the bound of sgd64 with the recipe's lr / wd and schedule; the mirror
    bit-exact; padding and frozen elements bit-identical; the packed layouts equal to a fresh re-pack; the host's
    Lookahead counter, momentum flag and iteration."""
    _need_cuda()
    from virtex_b200.config import Config
    from virtex_b200.trainer import Trainer
    kind, steps, extra = _REPLAYS[case]
    model, cfg, batch = _model(kind, *extra)
    batches = [batch(30 + i) for i in range(steps)]
    if case == "r50-clip-small":
        # max_norm at the median of the batches' gradient norms at the initial weights, so that some steps clip and
        # some do not (the small learning rates of these steps move the norms far less than the batches do)
        norms = sorted(_grad_norm(model, b) for b in batches)
        cfg = Config(None, _HEAD + extra + ["OPTIM.CLIP_GRAD_NORM", norms[steps // 2]])
    tr = Trainer(model, cfg)
    hp = T.arena_hparams(model, cfg)
    if case == "r50-frozen":
        assert not hp[2][tr.arena.offsets["visual.cnn.conv1.weight"]]
    clipped = _replay(tr, hp, batches)
    if case == "r50-clip-small":
        assert any(clipped) and not all(clipped), (clipped, norms)


def test_trainer_resumes_sgd_from_a_checkpoint(tmp_path):
    """3 steps -> CheckpointManager -> a fresh model and Trainer (parameters perturbed before the load) -> load: the
    parameters and momentum equal the saved ones bit for bit, the slow weights restart from the loaded parameters with
    the k counter at 0, and the next 3 steps are sgd64 with the loaded momentum (not a first step)."""
    _need_cuda()
    from virtex_b200.checkpointing import CheckpointManager
    from virtex_b200.trainer import Trainer
    m_b, cfg, batch = _model("r50", *_OPTIM)
    tr_b = Trainer(m_b, cfg)
    hp = T.arena_hparams(m_b, cfg)
    _replay(tr_b, hp, [batch(50 + i) for i in range(3)])
    CheckpointManager(str(tmp_path), model=m_b, optimizer=tr_b.optimizer, scheduler=tr_b.scheduler).step(3)
    m_c, _, _ = _model("r50", *_OPTIM)
    tr_c = Trainer(m_c, cfg)
    a = tr_c.arena
    with torch.no_grad():
        for p in m_c.parameters():
            p.add_(0.01)
    tr_c.engine.mark_weights_dirty()
    tr_c.step(batch(49))  # a step of its own: momentum, Lookahead counter and iteration all move before the load
    mgr = CheckpointManager(str(tmp_path), model=m_c, optimizer=tr_c.optimizer, scheduler=tr_c.scheduler)
    assert mgr.load(str(tmp_path / "checkpoint_3.pth")) == 3 and not mgr.not_loaded
    assert torch.equal(a.params, tr_b.arena.params) and torch.equal(tr_c.mom, tr_b.mom)
    assert torch.equal(tr_c.slow, a.params) and tr_c._k_counter == 0
    assert tr_c.momentum_ready and tr_c.iteration == 3
    tr_c.engine.mark_weights_dirty()
    _replay(tr_c, T.arena_hparams(m_c, cfg), [batch(50 + i) for i in range(3, 6)], it0=3, k0=0, first=False)


def test_two_rank_step_emulated_in_one_process():
    """Backward on two shards through one engine, the arena set to g0 + g1 in fp32 (what NCCL's SUM leaves on both
    ranks), tr.world = 2: the step equals sgd64 on the mean gradient with the norm of the mean, and leaves the summed
    gradients untouched.  Two steps: the first (momentum := gradient) and a steady one."""
    _need_cuda()
    from virtex_b200.trainer import Trainer
    model, cfg, batch = _model("r50", *(_OPTIM[2:] + ["OPTIM.WARMUP_STEPS", 0]))
    tr = Trainer(model, cfg)
    hp = T.arena_hparams(model, cfg)
    eng, a = tr.engine, tr.arena
    tr.world = 2  # stands in for a two-rank process group: only the clip reads the world size in optimizer_step
    for it in range(2):
        parts = []
        for shard in (batch(70 + 2 * it, B=2), batch(71 + 2 * it, B=3)):
            eng.forward(shard["image"], shard["caption_tokens"], shard["noitpac_tokens"], shard["caption_lengths"],
                        training=True, with_grad=True)
            eng.backward(zero_grads=True)
            parts.append(a.grads.clone())
        a.grads.copy_(parts[0] + parts[1])
        snap = _snapshot(tr)
        tr.optimizer_step()
        torch.cuda.synchronize()
        assert torch.equal(a.grads, parts[0] + parts[1])
        _check_step(tr, hp, snap, it, it == 0, False, world=2)
    assert tr._k_counter == 2 and tr.iteration == 2


# ----------------------------------------------------------------------------------------------- bucket contract
def _forward(model, batch):
    """The forward of Trainer.step for each model kind."""
    eng = model.engine
    if eng.classify:
        eng.forward(batch["image"], None, None, None, training=True, with_grad=True, labels=batch["labels"])
    elif "masked_labels" in batch:
        tok = batch["caption_tokens"]
        eng.forward(batch["image"], tok, tok, batch["caption_lengths"], training=True, with_grad=True,
                    labels=batch["masked_labels"])
    else:
        eng.forward(batch["image"], batch["caption_tokens"],
                    batch["noitpac_tokens"] if model.caption_backward else batch["caption_tokens"],
                    batch["caption_lengths"], training=True, with_grad=True)


def _bucket_of(name):
    """The bucket a parameter belongs to by its name: backward-direction decoder, the backbone's layer4 / layer3 /
    layer2, the stem and layer1, and everything else of the head."""
    if name.startswith("backward_textual."):
        return "head_b"
    if name.startswith("visual."):
        layer = name.split(".")[2]
        return layer if layer in ("layer2", "layer3", "layer4") else "rest"
    return "head"


_ALL = ("head_b", "head", "layer4", "layer3", "layer2", "rest")
_ONE_HEAD = _ALL[1:]
_BUCKETS = {  # kind, dynamic GEMM schedule, fused bn3 reductions forced on / off (None: the default), config, tags
    "r50-static-fused": ("r50", False, True, [], _ALL),
    "r50-static-unfused": ("r50", False, False, [], _ALL),
    "r50-dynamic-fused": ("r50", True, True, [], _ALL),
    "r50-dynamic-unfused": ("r50", True, False, [], _ALL),
    "r18": ("r18", False, None, [], _ALL),
    "captioning": ("captioning", False, None, [], _ONE_HEAD),
    "masked-lm": ("masked_lm", False, None, [], _ONE_HEAD),
    "token-classification": ("token_classification", False, None, [], _ONE_HEAD),
    "r50-frozen": ("r50", False, None, ["MODEL.VISUAL.FROZEN", True], ("head_b", "head", "rest")),
}


@pytest.mark.parametrize("case", list(_BUCKETS))
def test_bucket_ranges_are_final_when_their_tag_fires(case):
    """Engine.backward(bucket_cb=cb), cb cloning the tag's range of the real arena on the current stream: each tag
    fires once, in BUCKET_ORDER, exactly the model kind's tags; every clone equals the final gradients bit for bit
    (nothing lands in a range after its tag); the ranges are disjoint and every trainable tensor lies in exactly one
    fired range, the one its name says."""
    _need_cuda()
    from virtex_b200 import ops
    from virtex_b200.trainer import BUCKET_ORDER, bucket_ranges
    kind, dynamic, fused, extra, want = _BUCKETS[case]
    model, _, batch = _model(kind, *extra)
    eng, a = model.engine, model.engine.arena
    if fused is not None:
        eng.fuse_bn3_min_rows = 0 if fused else 1 << 40
    ranges = bucket_ranges(a.names, a.offsets, a.numels)
    fired, snaps = [], {}

    def cb(tag):
        fired.append(tag)
        r = ranges[tag]
        snaps[tag] = None if r is None else a.grads[r[0]:r[1]].clone()

    b = batch(3)
    ops.set_dynamic_gemm_schedule(dynamic)
    try:
        _forward(model, b)
        eng.backward(zero_grads=True, bucket_cb=cb)
        torch.cuda.synchronize()
    finally:
        ops.set_dynamic_gemm_schedule(False)
    assert tuple(fired) == want and list(want) == [t for t in BUCKET_ORDER if t in want], fired
    for tag in fired:
        r = ranges[tag]
        assert r is not None, tag
        final = a.grads[r[0]:r[1]]
        assert final.abs().sum() > 0 or case == "r50-frozen" and tag == "rest", tag
        assert torch.equal(snaps[tag], final), (tag, (snaps[tag] != final).sum().item())
    spans = sorted(r for r in ranges.values() if r is not None)
    assert all(e0 <= b1 for (_, e0), (b1, _) in zip(spans, spans[1:])), spans
    for n in a.names:
        if not a._param_objs[n].requires_grad:
            continue
        o, e = a.offsets[n], a.offsets[n] + a.numels[n]
        touching = [t for t in fired if ranges[t][0] < e and o < ranges[t][1]]
        assert touching == [_bucket_of(n)], (n, touching)
        r = ranges[touching[0]]
        assert r[0] <= o and e <= r[1], n
