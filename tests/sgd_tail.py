"""Float64 references of the fused SGD optimiser tail -- TEST INFRASTRUCTURE, NOT PRODUCT.

The tail every shipped config runs (virtex_b200/csrc/optim.cu, Trainer.optimizer_step):
    sumsq = sum g^2 (vtx_sumsq) -> clip coefficient and norm (vtx_clip_coef) -> SGD with momentum and per-tensor
    lr / wd (vtx_sgd_step) -> Lookahead every k steps -> bf16 mirror
`sumsq64`, `clip64` and `sgd64` restate it in float64 with the semantics of torch.nn.utils.clip_grad_norm_,
torch.optim.SGD and virtex_b200.optim.Lookahead (pinned to them by tests/test_sgd_tail_cpu.py).  The error bounds are
derived from the kernels' operation sequence in fp32 (u = 2^-24 per rounding, first order), not fitted to
measurements.  `arena_hparams` builds the per-element lr / wd and the per-iteration lr multiplier from the reference
recipe (OptimizerFactory's param groups and LRSchedulerFactory on a twin model), not from the trainer's segment table
or schedule function, so that those are checked rather than restated.
"""
import math
import warnings

import torch

U = 2.0 ** -24  # unit roundoff of fp32
F64 = torch.float64


# ------------------------------------------------------------------------------------------------------- global norm
def sumsq64(g) -> float:
    """Sum of squares of a gradient (arena) in float64."""
    return float((g.double() ** 2).sum())


def sumsq_bound(n: int, sumsq: float, num_sms: int, preset: float = 0.0) -> float:
    """Absolute error bound of vtx_sumsq on n elements with exact sum of squares `sumsq`, added to `*out = preset`.

    u * (k + 10 + nblocks) * (sumsq + preset): k covers one thread's sequential sum -- four squares per float4
    iteration, its share of the n % 4 scalar tail, and the rounding of the squares themselves; 10 covers the two
    5-level warp trees; every block adds its partial sum to `out` with one float atomic.  The launch shape is the
    wrapper's: min(ceil(n/4 / 256), 8 * SMs) blocks of 256 threads, at least one."""
    if n == 0:
        return 0.0
    n4 = n // 4
    blocks = min(max(1, -(-n4 // 256)), 8 * num_sms)
    threads = blocks * 256
    k = 4 * -(-n4 // threads) + -(-(n - 4 * n4) // threads) + 1
    return U * (k + 10 + blocks) * (sumsq + abs(preset))


def clip64(sumsq: float, world: int, max_norm: float):
    """(coef, norm) of the clip over `world` summed gradients: norm = sqrt(sumsq) / world is the norm of the mean
    gradient and coef the scale the step applies to the SUM, min(1, max_norm / (norm + 1e-6)) / world.

    Non-finite norms follow clip_grad_norm_'s torch.clamp(coef, max=1): an inf norm gives 0 and a NaN norm a NaN
    coefficient.  max_norm <= 0 disables clipping (coefficient 1 / world), which is where the fused tail departs from
    clip_grad_norm_ (that would scale every gradient by max_norm / norm <= 0)."""
    norm = math.sqrt(sumsq) / world
    c = max_norm / (norm + 1e-6) if max_norm > 0 else 1.0
    if c > 1.0:  # a NaN compares false and stays NaN
        c = 1.0
    return c / world, norm


def clip_bound(coef: float, norm: float, sumsq_err: float, sumsq: float):
    """(|d coef|, |d norm|) bounds of vtx_clip_coef fed a sum of squares within `sumsq_err` of the exact `sumsq`.
    e = sumsq_err / sumsq relative error of the sum halves under the sqrt; then the norm takes the sqrt's rounding,
    1/world's and the product's (3u); the coefficient adds 1e-6f's and the sum's, max_norm's and the division's, and
    1/world's and the last product's (8u).  One more u each covers the second-order terms."""
    e = sumsq_err / sumsq if sumsq > 0 else 0.0
    return abs(coef) * (0.5 * e + 9 * U), norm * (0.5 * e + 4 * U)


# --------------------------------------------------------------------------------------------------------------- SGD
def _f64(x, like):
    return x.to(device=like.device, dtype=F64) if torch.is_tensor(x) else x


def sgd64(p, g, m, slow, lr, wd, mult, coef, first, do_la, alpha, momentum=0.9):
    """One step of torch.optim.SGD(momentum, dampening 0) on the clipped gradient g * coef with per-tensor lr * mult
    and weight decay (lr / wd scalars or per-element vectors), then, when do_la, Lookahead's
    `p <- alpha p + (1 - alpha) slow; slow <- p`.  The first step sets the momentum buffer to the gradient.
    Returns float64 (p, m, slow)."""
    p, g, m = p.double(), g.double(), m.double()
    lr, wd = _f64(lr, p), _f64(wd, p)
    d = g * coef + wd * p
    m1 = d if first else momentum * m + d
    p1 = p - (lr * mult) * m1
    s1 = slow.double() if slow is not None else None
    if do_la and slow is not None:
        p1 = alpha * p1 + (1.0 - alpha) * s1
        s1 = p1
    return p1, m1, s1


def sgd_tol(p, g, m, slow, lr, wd, mult, coef, dcoef, first, do_la, alpha, momentum=0.9):
    """Per-element bounds (tol_p, tol_m) of the fp32 sgd_step_kernel against sgd64, from its operation sequence.

    gg = g * c + wd * w: the product, fp32 wd, the sum (one rounding less under FMA contraction): 3u of
        A_g = |g c| + |wd w|, plus |g| |d coef| from the fp32 clip coefficient;
    m = mu * m0 + gg: fp32 mu, the product and the sum: 4u of A_m = A_g + mu |m0| (A_g on the first step);
    w1 = w - lr' m with lr' = fp32(fp32(lr) * fp32(mult)) (3u): lr' times m's error, lr's 3u, the product and the
        difference: 9u of A_p = |w| + lr A_m, plus lr |g| |d coef|;
    Lookahead alpha w1 + (1 - alpha) slow: alpha times w1's error, fp32 alpha and 1 - alpha, two products and a sum:
        4u of |w1| + |slow|."""
    p, g, m = p.double(), g.double(), m.double()
    lr_t, wd_t = _f64(lr, p) * mult, _f64(wd, p)
    a_g = (g * coef).abs() + (wd_t * p).abs()
    a_m = a_g if first else a_g + momentum * m.abs()
    tol_m = 4 * U * a_m + g.abs() * dcoef
    a_p = p.abs() + lr_t * a_m
    tol_p = 9 * U * a_p + lr_t * g.abs() * dcoef
    if do_la and slow is not None:
        w1 = sgd64(p, g, m, None, lr, wd, mult, coef, first, False, alpha, momentum)[0]
        tol_p = alpha * tol_p + 4 * U * (w1.abs() + slow.double().abs())
    return tol_p, tol_m


# ---------------------------------------------------------------------------------------------- the recipe's groups
class Schedule:
    """Lr multiplier of iteration i: the LambdaLR of LRSchedulerFactory stepped i times, as the reference loop does
    (scheduler.step() after every optimizer.step())."""

    def __init__(self, sched):
        self.sched = sched
        self.mults = []
        self._j = next(i for i, b in enumerate(sched.base_lrs) if b != 0)

    def __call__(self, i: int) -> float:
        while len(self.mults) <= i:
            if self.mults:
                with warnings.catch_warnings():  # the twin optimiser never steps: only its schedule is read
                    warnings.simplefilter("ignore", UserWarning)
                    self.sched.step()
            self.mults.append(self.sched.get_last_lr()[self._j] / self.sched.base_lrs[self._j])
        return self.mults[i]


def arena_hparams(model, cfg):
    """(lr, wd, trainable, schedule) of a model's parameter arena: float64 per-element base lr and weight decay from
    the param groups `OptimizerFactory.from_config` builds for a twin model of the same config (0 outside every
    trainable tensor), the bool mask of trainable elements, and the `Schedule` of LRSchedulerFactory on them."""
    from virtex_b200.factories import LRSchedulerFactory, OptimizerFactory, PretrainingModelFactory
    twin = PretrainingModelFactory.from_config(cfg)
    opt = OptimizerFactory.from_config(cfg, twin.named_parameters())
    sched = LRSchedulerFactory.from_config(cfg, opt)
    names = {id(p): n for n, p in twin.named_parameters()}
    a = model.engine.arena
    dev = a.params.device
    lr = torch.zeros(a.total, dtype=F64, device=dev)
    wd = torch.zeros_like(lr)
    trainable = torch.zeros(a.total, dtype=torch.bool, device=dev)
    seen = set()
    for grp in opt.param_groups:
        (p,) = grp["params"]
        if not p.requires_grad:  # torch.optim.SGD skips a parameter that never has a gradient
            continue
        n = names[id(p)]
        o, k = a.offsets[n], a.numels[n]
        lr[o:o + k], wd[o:o + k] = grp["initial_lr"], grp["weight_decay"]
        trainable[o:o + k] = True
        seen.add(n)
    assert seen == {n for n in a.names if a._param_objs[n].requires_grad}, "twin and arena disagree on parameters"
    return lr, wd, trainable, Schedule(sched)
