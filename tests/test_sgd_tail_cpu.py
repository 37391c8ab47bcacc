"""The float64 references of the fused SGD tail (tests/sgd_tail.py) against the reference recipe in float64:
torch.nn.utils.clip_grad_norm_ -> OptimizerFactory's Lookahead(SGD) -> LRSchedulerFactory's LambdaLR."""
import math

import pytest
import torch

from tests import sgd_tail as T

# one tensor per param-group kind: CNN lr, NO_DECAY (a transformer norm), and plain lr with weight decay
SHAPES = {"visual.cnn.conv1.weight": (4, 3, 3, 3), "textual.transformer.layers.0.norm1.weight": (16,),
          "textual.output.weight": (10, 8)}
GRAD_SCALES = [0.1, 5.0, 0.3, 20.0, 1.0, 50.0, 0.01]  # norms from ~1 to ~500 around max_norm 10


def _config():
    from virtex_b200.config import Config
    return Config(None, ["OPTIM.WARMUP_STEPS", 2, "OPTIM.NUM_ITERATIONS", 10, "OPTIM.LR_DECAY_NAME", "cosine",
                         "OPTIM.LOOKAHEAD.STEPS", 3, "OPTIM.CLIP_GRAD_NORM", 10.0])


def _params(seed):
    g = torch.Generator().manual_seed(seed)
    return [(n, torch.nn.Parameter(torch.randn(s, generator=g, dtype=torch.float64))) for n, s in SHAPES.items()]


def test_sgd64_chain_matches_clip_lookahead_sgd_and_lambda_lr():
    """7 steps across the end of warm-up into cosine decay, with Lookahead k = 3 (two slow-weight updates) and
    clipped and unclipped steps: clip64 -> sgd64 on flat vectors equals the float64 torch loop to 1e-12."""
    from virtex_b200.factories import LRSchedulerFactory, OptimizerFactory, param_group_hparams
    cfg = _config()
    O = cfg.OPTIM
    named = _params(0)
    opt = OptimizerFactory.from_config(cfg, named)
    sched = LRSchedulerFactory.from_config(cfg, opt)
    schedule = T.Schedule(LRSchedulerFactory.from_config(cfg, OptimizerFactory.from_config(cfg, _params(0))))
    flat = torch.cat([p.detach().flatten() for _, p in named]).clone()
    lr = torch.cat([torch.full((p.numel(),), param_group_hparams(cfg, n)[0], dtype=torch.float64) for n, p in named])
    wd = torch.cat([torch.full((p.numel(),), param_group_hparams(cfg, n)[1], dtype=torch.float64) for n, p in named])
    assert len(set(lr.tolist())) == 2 and set(wd.tolist()) == {0.0, O.WEIGHT_DECAY}
    mom, slow = torch.zeros_like(flat), flat.clone()
    gen = torch.Generator().manual_seed(1)
    clipped, la_steps, k = [], [], 0
    for it, scale in enumerate(GRAD_SCALES):
        grads = [torch.randn(p.shape, generator=gen, dtype=torch.float64) * scale for _, p in named]
        for (_, p), g in zip(named, grads):
            p.grad = g.clone()
        norm_t = torch.nn.utils.clip_grad_norm_([p for _, p in named], O.CLIP_GRAD_NORM)
        opt.step()
        sched.step()
        gflat = torch.cat([g.flatten() for g in grads])
        coef, norm = T.clip64(T.sumsq64(gflat), 1, O.CLIP_GRAD_NORM)
        assert abs(norm - norm_t.item()) <= 1e-12 * norm
        clipped.append(coef < 1.0)
        k += 1
        do_la = k >= O.LOOKAHEAD.STEPS
        k = 0 if do_la else k
        la_steps += [it] if do_la else []
        flat, mom, slow = T.sgd64(flat, gflat, mom, slow, lr, wd, schedule(it), coef, it == 0, do_la,
                                  O.LOOKAHEAD.ALPHA, O.SGD_MOMENTUM)
        ref = torch.cat([p.detach().flatten() for _, p in named])
        assert torch.allclose(flat, ref, rtol=1e-12, atol=1e-15), (it, (flat - ref).abs().max().item())
        ref_m = torch.cat([opt.optimizer.state[p]["momentum_buffer"].flatten() for _, p in named])
        assert torch.allclose(mom, ref_m, rtol=1e-12, atol=1e-15), it
        ref_s = torch.cat([opt.state[p]["slow_params"].flatten() for _, p in named])
        assert torch.allclose(slow, ref_s, rtol=1e-12, atol=1e-15), it
    assert any(clipped) and not all(clipped)
    assert la_steps == [2, 5]
    assert schedule(0) == 0.0 and schedule(2) == 1.0 and 0.0 < schedule(6) < 1.0  # warm-up, then cosine decay


def _torch_clip(grads, max_norm):
    ps = [torch.nn.Parameter(torch.zeros_like(g)) for g in grads]
    for p, g in zip(ps, grads):
        p.grad = g.clone()
    norm = torch.nn.utils.clip_grad_norm_(ps, max_norm).item()
    return [p.grad for p in ps], norm


@pytest.mark.parametrize("case", ["zero", "at_max_norm", "clipped", "inf", "nan"])
def test_clip64_edges_match_clip_grad_norm(case):
    """norm 0 (coefficient 1), a norm of exactly max_norm (still scaled by max_norm / (max_norm + 1e-6)), an inf
    norm (coefficient 0: finite gradients become 0, inf ones NaN) and a NaN norm (the NaN propagates into every
    gradient), each as clip_grad_norm_ has them."""
    g = {"zero": [0.0, 0.0, 0.0], "at_max_norm": [6.0, 8.0, 0.0], "clipped": [60.0, -80.0, 1.0],
         "inf": [math.inf, 1.0, -2.0], "nan": [math.nan, 1.0, -2.0]}[case]
    g = torch.tensor(g, dtype=torch.float64)
    out, norm_t = _torch_clip([g[:2], g[2:]], 10.0)
    coef, norm = T.clip64(T.sumsq64(g), 1, 10.0)
    out = torch.cat(out)
    assert (math.isnan(norm) and math.isnan(norm_t)) or norm == pytest.approx(norm_t, rel=1e-15)
    if case == "nan":
        assert math.isnan(coef) and out.isnan().all()
        return
    assert torch.allclose(g * coef, out, rtol=1e-15, atol=0.0, equal_nan=True)
    want = {"zero": 1.0, "at_max_norm": 10.0 / (10.0 + 1e-6), "inf": 0.0}.get(case)
    if want is not None:
        assert coef == want
    if case == "inf":
        assert out[0].isnan() and (out[1:] == 0).all()


@pytest.mark.parametrize("world", [2, 8])
def test_clip64_of_summed_gradients_is_the_clip_of_their_mean(world):
    """Over `world` summed gradients, clip64's norm is the norm of the mean gradient and coef * sum equals
    clip_grad_norm_ applied to the mean (what DistributedDataParallel's averaged gradients see)."""
    gen = torch.Generator().manual_seed(world)
    for scale in (0.1, 100.0):  # unclipped and clipped
        gsum = torch.randn(50, generator=gen, dtype=torch.float64) * scale * world
        out, norm_t = _torch_clip([gsum / world], 10.0)
        coef, norm = T.clip64(T.sumsq64(gsum), world, 10.0)
        assert norm == pytest.approx(norm_t, rel=1e-14)
        assert torch.allclose(gsum * coef, out[0], rtol=1e-14, atol=0.0)


def test_clip64_without_a_positive_max_norm_does_not_clip():
    """max_norm <= 0 disables clipping in the fused tail (coefficient 1 / world); clip_grad_norm_ would instead scale
    every gradient by max_norm / norm <= 0."""
    for m in (0.0, -1.0):
        assert T.clip64(400.0, 1, m) == (1.0, 20.0)
        assert T.clip64(400.0, 2, m) == (0.5, 10.0)


def test_sumsq_bound_counts_the_launch():
    """The bound grows with the terms per thread and with the blocks of the launch: n = 5 is one float4 and a scalar
    tail in one block (k = 4 + 1 + 1); 5 000 011 elements on 132 SMs cap the grid at 1056 blocks with 5 float4
    iterations per thread."""
    assert T.sumsq_bound(0, 1.0, 132) == 0.0
    assert T.sumsq_bound(5, 1.0, 132) == T.U * (6 + 10 + 1)
    assert T.sumsq_bound(5_000_011, 1.0, 132) == T.U * (20 + 1 + 1 + 10 + 1056)
    assert T.sumsq_bound(5, 1.0, 132, preset=3.0) == 4.0 * T.sumsq_bound(5, 1.0, 132)
