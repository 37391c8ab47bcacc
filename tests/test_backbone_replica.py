"""CPU checks of tests/backbone_replica.py against plain Python loops over exact rational arithmetic (fractions): the
rounding helpers, the ReLU bit-mask layout, the max-pool slot rule and the BatchNorm finalize arithmetic."""
import math
import random
from fractions import Fraction

import numpy as np
import torch

from tests import backbone_replica as R

F64 = torch.float64


def _round(v, mant_bits, emin=-126):
    """Exact Fraction -> nearest binary float with `mant_bits` significant bits and fp32's exponent range (ties to
    even)."""
    if v == 0:
        return 0.0
    sign, v = (-1 if v < 0 else 1), abs(v)
    e = v.numerator.bit_length() - v.denominator.bit_length()
    if Fraction(2) ** e > v:
        e -= 1
    e = max(e, emin)
    ulp = Fraction(2) ** (e - (mant_bits - 1))
    q = v / ulp
    fl = q.numerator // q.denominator
    rem = q - fl
    if rem > Fraction(1, 2) or (rem == Fraction(1, 2) and fl % 2 == 1):
        fl += 1
    if fl * ulp >= Fraction(2) ** 128:  # fp32 and bf16 share the exponent range: FLT_MAX rounds to inf in bf16
        return sign * math.inf
    return sign * float(fl * ulp)


def r32(v):
    return _round(Fraction(v), 24)


def rbf(v):
    return _round(Fraction(v), 8)


def _t(xs):
    return torch.tensor(xs, dtype=F64)


def _rand_bf16(rng, n, lo=-20, hi=20):
    return [rbf(rng.uniform(1, 2) * rng.choice((-1, 1)) * 2.0 ** rng.randint(lo, hi)) for _ in range(n)]


def _rand_f32(rng, n, lo=-20, hi=20):
    return [r32(rng.uniform(1, 2) * rng.choice((-1, 1)) * 2.0 ** rng.randint(lo, hi)) for _ in range(n)]


def test_f32_and_bf16_rounding_match_exact_rounding():
    rng = random.Random(1)
    xs = _rand_f32(rng, 3000, -140, 60) + [0.0, -0.0, 2.0 ** -149, -(2.0 ** -130), float(np.finfo(np.float32).max)]
    # bf16 ties: 1 + 2^-8 lies halfway between 1 and 1 + 2^-7 (even: 1), 1 + 3 * 2^-8 between 1 + 2^-7 and 1 + 2^-6
    # (even: 1 + 2^-6); the same at negative values and in the subnormal range
    ties = [1 + 2.0 ** -8, 1 + 3 * 2.0 ** -8, -(1 + 2.0 ** -8), -(1 + 3 * 2.0 ** -8), 3 * 2.0 ** -134, 2.0 ** -134]
    got = R.bf16(_t(xs + ties)).tolist()
    want = [rbf(x) for x in xs + ties]
    assert got == want
    assert got[-6:] == [1.0, 1 + 2.0 ** -6, -1.0, -(1 + 2.0 ** -6), 2.0 ** -132, 0.0]
    # torch's own conversion agrees for finite fp32 input (the layout test on the GPU compares with it)
    assert R.bf16(_t(xs)).tolist() == torch.tensor(xs, dtype=torch.float32).bfloat16().double().tolist()
    ds = [rng.uniform(-1, 1) * 2.0 ** rng.randint(-30, 30) for _ in range(2000)]
    assert R.f32(_t(ds)).tolist() == [r32(d) for d in ds]


def test_fma_f32_rounds_once_including_float64_midpoints():
    rng = random.Random(2)
    n = 4000
    a = _rand_bf16(rng, n, -10, 10)
    b = _rand_f32(rng, n, -10, 10)
    c = _rand_f32(rng, n, -30, 30)
    # products of 32 significant bits that put the exact sum 2^-54 off the fp32 midpoint of c: float64 rounds that
    # sum onto the midpoint, and rounding it again would go to the even neighbour on the wrong side in the cases below
    hard = [(130.0, 16519105 * 2.0 ** -55, 1.0), (151.0, 14221746 * 2.0 ** -55, 1 + 2.0 ** -23),
            (-130.0, 16519105 * 2.0 ** -55, -1.0), (151.0, -14221746 * 2.0 ** -55, -(1 + 2.0 ** -23))]
    for x, y, z in hard:
        assert r32(Fraction(x) * Fraction(y) + Fraction(z)) != float(np.float32(x * y + z))
    a += [h[0] for h in hard]
    b += [h[1] for h in hard]
    c += [h[2] for h in hard]
    got = R.fma_f32(_t(a), _t(b), _t(c)).tolist()
    want = [r32(Fraction(x) * Fraction(y) + Fraction(z)) for x, y, z in zip(a, b, c)]
    assert got == want


def test_relu_mask_layout():
    rng = random.Random(3)
    M, C = 5, 40
    keep = [[rng.random() < 0.5 for _ in range(C)] for _ in range(M)]
    bits = R.pack_mask(torch.tensor(keep))
    assert bits.dtype == torch.uint8 and tuple(bits.shape) == (M, C // 8)
    for m in range(M):
        for g in range(C // 8):
            assert int(bits[m, g]) == sum(1 << j for j in range(8) if keep[m][8 * g + j])
    assert R.unpack_mask(bits, C).tolist() == keep


def test_bn_act_replica():
    rng = random.Random(4)
    M, C = 6, 16
    y = [_rand_bf16(rng, C, -3, 3) for _ in range(M)]
    res = [_rand_bf16(rng, C, -3, 3) for _ in range(M)]
    sc, sh, sc2, sh2 = (_rand_f32(rng, C, -3, 3) for _ in range(4))
    for mode in ("plain", "res", "res_bn"):
        for relu in (False, True):
            kw = {}
            if mode != "plain":
                kw["res"] = _t(res)
            if mode == "res_bn":
                kw["scale_r"], kw["shift_r"] = _t(sc2), _t(sh2)
            pre, out = R.bn_act(_t(y), _t(sc), _t(sh), relu=relu, **kw)
            for m in range(M):
                for c in range(C):
                    v = r32(Fraction(y[m][c]) * Fraction(sc[c]) + Fraction(sh[c]))
                    if mode == "res":
                        v = r32(Fraction(v) + Fraction(res[m][c]))
                    if mode == "res_bn":
                        v = r32(Fraction(v) + Fraction(r32(Fraction(res[m][c]) * Fraction(sc2[c]) + Fraction(sh2[c]))))
                    assert pre[m, c].item() == v
                    assert out[m, c].item() == rbf(max(v, 0.0) if relu else v)


def _pool_loops(act, N, H, W, C):
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    out, idx = {}, {}
    for n in range(N):
        for ph in range(Ho):
            for pw in range(Wo):
                for c in range(C):
                    best, bi = -math.inf, 0
                    for kh in range(3):
                        for kw in range(3):
                            h, w = 2 * ph - 1 + kh, 2 * pw - 1 + kw
                            if 0 <= h < H and 0 <= w < W and act[n][h][w][c] > best:
                                best, bi = act[n][h][w][c], kh * 3 + kw
                    out[n, ph, pw, c], idx[n, ph, pw, c] = best, bi
    return out, idx


def test_maxpool_replica_first_maximum_and_scatter():
    rng = random.Random(5)
    C = 3
    for N, H, W in ((2, 5, 7), (1, 1, 1), (1, 2, 3), (1, 4, 4), (1, 7, 9)):
        # post-ReLU values: many exact zeros (ties) and a few repeated positive values
        act = [[[[rng.choice((0.0, 0.0, 0.0, 0.5, 0.75, rbf(rng.random()))) for _ in range(C)] for _ in range(W)]
                for _ in range(H)] for _ in range(N)]
        out, idx = R.maxpool_fwd(torch.tensor(act, dtype=F64))
        ref_out, ref_idx = _pool_loops(act, N, H, W, C)
        Ho, Wo = R.pool_extent(H, W)
        assert tuple(out.shape) == (N, Ho, Wo, C)
        for k, v in ref_out.items():
            assert out[k].item() == v and int(idx[k]) == ref_idx[k], (N, H, W, k)
        dpool = [[[[rng.randint(-64, 64) / 64 for _ in range(C)] for _ in range(Wo)] for _ in range(Ho)] for _ in range(N)]
        da = R.maxpool_bwd(torch.tensor(dpool, dtype=F64), idx, H, W)
        ref = [[[[0.0] * C for _ in range(W)] for _ in range(H)] for _ in range(N)]
        for (n, ph, pw, c), s in ref_idx.items():
            ref[n][2 * ph - 1 + s // 3][2 * pw - 1 + s % 3][c] += dpool[n][ph][pw][c]
        assert da.tolist() == ref


def test_bn_finalize_replica():
    rng = random.Random(6)
    C = 7
    for count in (1.0, 2.0, 7.0, 1001.0, 3211264.0):
        s1 = _rand_f32(rng, C, -4, 20)
        s2 = [r32(abs(x) * x / count * rng.choice((0.5, 1.0, 1.001, 1.5))) for x in s1]  # incl. var < 0 -> clamp
        gamma, beta, rm = (_rand_f32(rng, C, -2, 2) for _ in range(3))
        rv = [abs(x) for x in _rand_f32(rng, C, -2, 2)]
        mean, var, invstd_ref, rm2, rv2 = R.bn_finalize(_t([s1, s2]), count, _t(gamma), _t(beta), _t(rm), _t(rv), 0.1,
                                                        1e-5, True)
        m, e = Fraction(r32(0.1)), Fraction(r32(1e-5))
        for c in range(C):
            mu = r32(Fraction(s1[c]) / Fraction(count))
            q = r32(Fraction(s2[c]) / Fraction(count))
            v = max(r32(q - Fraction(mu) * Fraction(mu)), 0.0)
            assert mean[c].item() == mu and var[c].item() == v
            one_m = r32(1 - m)
            assert rm2[c].item() == r32(Fraction(mu) * m + Fraction(r32(Fraction(rm[c]) * Fraction(one_m))))
            unb = r32(Fraction(count) / max(Fraction(r32(count - 1)), Fraction(1)))
            t = r32(Fraction(r32(Fraction(v) * m)) * Fraction(unb))
            assert rv2[c].item() == r32(Fraction(one_m) * Fraction(rv[c]) + Fraction(t))
            assert invstd_ref[c].item() == 1.0 / math.sqrt(r32(Fraction(v) + e))
        invstd = R.f32(invstd_ref)
        sc, sh = R.bn_scale_shift(_t(gamma), _t(beta), mean, invstd)
        for c in range(C):
            s = r32(Fraction(gamma[c]) * Fraction(invstd[c].item()))
            assert sc[c].item() == s
            assert sh[c].item() == r32(Fraction(beta[c]) - Fraction(s) * Fraction(mean[c].item()))
    # eval mode reads the running buffers and leaves them alone
    rm, rv = _t([0.5, -1.25]), _t([2.0, 0.0])
    mean, var, invstd_ref, rm2, rv2 = R.bn_finalize(None, 0.0, None, None, rm, rv, 0.1, 1e-5, False)
    assert torch.equal(mean, rm) and torch.equal(var, rv) and torch.equal(rm2, rm) and torch.equal(rv2, rv)
    assert invstd_ref.tolist() == [1 / math.sqrt(r32(2.0 + Fraction(r32(1e-5)))), 1 / math.sqrt(r32(1e-5))]
