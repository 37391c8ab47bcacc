"""Stand-alone tests of the textual-head kernels (virtex_b200/csrc/head.cu) against float64 references, at p = 0 and
at p = 0.1 with the dropout masks replayed on the host (tests/dropout_replica.py).

Every kernel is called through the C ABI (virtex_b200.ops.call) on the same bf16 / fp32 tensors the reference reads.
Dropout cases run at seeds 1, 2^63 + 5 and 2^64 - 1 (the device reads the seed word as a uint64; it is stored in an
int64 tensor, so the two large seeds go in as their two's-complement values).  Outputs start as a sentinel so that
nothing outside the written region may change; accumulated gradients start non-zero so that they must add.

Tolerances, from each kernel's rounding points:
  * fp32 outputs and fp32 sums: 1e-5 of the largest magnitude of the float64 value (of its terms, for sums);
  * bf16 outputs: within 1 bf16 ulp of the float64 value, plus a floor of 1e-5 of the tensor's magnitude for the fp32
    cancellation before the rounding (LayerNorm backward, the centring of the LN forward);
  * GELU: the p = 0 output within 1 ulp of the float64 GELU (plus |u| 2^-22, the fp32 error of 1 + erf that
    cancels for u << 0), the p = 0.1 output equal to the p = 0 output times the mask, rounded as the kernel rounds;
    the backward within 1 ulp of float64 dh * mask * gelu'(u) plus |dh| 2^-20;
  * attention: the kernel rounds the unnormalised dropped probabilities (forward, and dV in backward) and dS (dQ, dK)
    to bf16 before its MMAs.  It is compared with a float64 reference that applies the same two roundings: 1 ulp, plus
    2^-7 of the largest term of each output's sum (the fp32 probabilities can round to the neighbouring bf16 value
    where float64 does not: at most 2 such flips are allowed per output) and 2^-16 of the sum of the term magnitudes
    (fp32 accumulation).  It is also compared with the plain float64 reference at relative L2 error <= 1e-2;
  * cross entropy: loss 1e-5 relative; dlogits 1 ulp plus 2^-20 / count (fp32 softmax near 1) and 2^-120 (the
    flush-to-zero of the fast exp).
A wrong dropout mask moves about 10 % of the elements by O(1): far outside every bound.
"""
import pytest
import torch

from tests import dropout_replica as R

pytestmark = pytest.mark.gpu

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
DEV = "cuda"
SEEDS = (1, 2 ** 63 + 5, 2 ** 64 - 1)
PS = (0.0, 0.1)
HS = (128, 256, 512, 768, 1024, 2048)


def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _ops():
    from virtex_b200 import ops
    return ops


def _s():
    return torch.cuda.current_stream().cuda_stream


def _p(t):
    return 0 if t is None else t.data_ptr()


def _seed(s):
    return torch.tensor([R.as_i64(s)], dtype=torch.int64, device=DEV)


def _flat_scale(seed, site, shape, p):
    return torch.from_numpy(R.flat_scale(seed, site, shape, p)).to(DEV, F64)


def _rb(x):
    """float64 -> nearest bf16 value (as float64)."""
    return x.to(BF16).to(F64)


def ulp_bf16(x):
    ax = x.abs()
    e = torch.floor(torch.log2(ax))
    return torch.exp2(e - 7).nan_to_num(0.0).clamp_min(2.0 ** -133)


def assert_bf16(out, ref, floor=0.0, what=""):
    """bf16 `out` within 1 bf16 ulp of the float64 `ref` (+ `floor`, scalar or tensor)."""
    err = (out.to(F64) - ref).abs()
    tol = ulp_bf16(ref) + floor
    bad = ~(err <= tol)
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.numel()} elements beyond tolerance; worst err/tol "
                           f"{(err / tol).max().item():.3g}")


def assert_f32(out, ref, what="", rtol=1e-5, scale=None):
    """fp32 `out` against float64 `ref`: max error <= rtol * (largest |ref| or the given scale)."""
    err = (out.to(F64) - ref).abs().max().item()
    s = ref.abs().max().item() if scale is None else float(scale)
    assert err <= rtol * s, f"{what}: max error {err:.3g} > {rtol:g} * {s:.3g}"


def rel(a, b):
    a, b = a.to(F64), b.to(F64)
    return ((a - b).norm() / (b.norm() + 1e-300)).item()


# ------------------------------------------------------------------------------------------------ replica vs device
def test_replica_matches_device_masks_bit_for_bit():
    """The kept / dropped pattern of four kernels equals the host replica's, at 3 seeds and 2 sites each."""
    _need_cuda()
    ops = _ops()
    p = 0.1
    ik = float(R.inv_keep(p))
    for seed in SEEDS:
        sd = _seed(seed)
        for site in (14, 1045):
            # GELU + dropout on u = 1: gelu(1) != 0, so h == 0 exactly where dropped
            M, Fd = 61, 264
            u = torch.ones(M, Fd, dtype=BF16, device=DEV)
            h = torch.empty_like(u)
            ops.call("vtx_gelu_dropout_fwd", u.data_ptr(), h.data_ptr(), M * Fd, p, sd.data_ptr(), site, _s())
            sc = _flat_scale(seed, site, (M, Fd), p)
            assert torch.equal(h != 0, sc != 0), ("gelu", seed, site)
            # residual add, ln = 0, res = 0, branch = 1: z is the scale itself
            M, H = 77, 384
            res = torch.zeros(M, H, device=DEV)
            br = torch.ones(M, H, dtype=BF16, device=DEV)
            z = torch.empty(M, H, device=DEV)
            ops.call("vtx_add_ln_fwd", res.data_ptr(), br.data_ptr(), 0, 0, z.data_ptr(), 0, 0, 0, M, H, 0.0, p,
                     sd.data_ptr(), site, 0, _s())
            assert torch.equal(z.to(F64), _flat_scale(seed, site, (M, H), p)), ("add_ln", seed, site)
            # embedding with gamma = 1, beta = 0.5: out == 0 exactly where dropped (no token is the pad)
            V, T, B, H = 50, 30, 3, 256
            g = torch.Generator().manual_seed(seed % 1000 + site)
            tokens = torch.randint(1, V, (B * T,), generator=g).to(DEV)
            words, pos = torch.randn(V, H, generator=g).to(DEV), torch.randn(T, H, generator=g).to(DEV)
            gamma, beta = torch.ones(H, device=DEV), torch.full((H,), 0.5, device=DEV)
            z, st = torch.empty(B * T, H, device=DEV), torch.empty(B * T, 2, device=DEV)
            out, ob = torch.empty(B * T, H, device=DEV), torch.empty(B * T, H, dtype=BF16, device=DEV)
            ops.call("vtx_embed_fwd", tokens.data_ptr(), words.data_ptr(), pos.data_ptr(), gamma.data_ptr(),
                     beta.data_ptr(), z.data_ptr(), st.data_ptr(), out.data_ptr(), ob.data_ptr(), B * T, T, H, 0, 1e-8,
                     p, sd.data_ptr(), site, _s())
            sc = _flat_scale(seed, site, (B * T, H), p)
            assert torch.equal(out != 0, sc != 0), ("embed", seed, site)
            # attention with equal scores (Q = K = 0) and V = the first Tk rows of I_64: out row i of head h is the
            # dropped probability row, bf16(1/(1-p)) / Tk where kept and 0 where dropped
            for B, A, Tq, Tk in ((3, 2, 30, 49), (2, 3, 32, 64)):
                Hh = A * 64
                q = torch.zeros(B * Tq, Hh, dtype=BF16, device=DEV)
                k = torch.zeros(B * Tk, Hh, dtype=BF16, device=DEV)
                v = torch.zeros(B, Tk, A, 64, dtype=BF16, device=DEV)
                v[:, torch.arange(Tk), :, torch.arange(Tk)] = 1
                v = v.view(B * Tk, Hh)
                o = torch.empty(B * Tq, Hh, dtype=BF16, device=DEV)
                lse = torch.empty(B * A * 32, device=DEV)
                ops.call("vtx_attn_fwd", q.data_ptr(), Hh, k.data_ptr(), Hh, v.data_ptr(), Hh, o.data_ptr(), Hh,
                         lse.data_ptr(), B, A, Tq, Tk, 0, 0, p, sd.data_ptr(), site, _s())
                got = o.view(B, Tq, A, 64).permute(0, 2, 1, 3)[..., :Tk]
                msk = torch.from_numpy(R.attn_scale(seed, site, B, A, Tq, Tk, p)).to(DEV)
                assert torch.equal(got != 0, msk != 0), ("attn", seed, site, Tk)
                # the kernel multiplies the bf16 probability by the fp32 reciprocal of the row sum (= Tk)
                kept = (torch.tensor(ik, dtype=F32).to(BF16).float() * torch.tensor(1.0 / Tk, dtype=F32)).to(BF16)
                assert (got[msk != 0] == kept.to(DEV)).all(), ("attn kept values", seed, site, Tk)
                assert (o.view(B, Tq, A, 64)[..., Tk:] == 0).all()


# ------------------------------------------------------------------------------------------------ embedding
def _embed_case(ops, H, M, T, tokens, words, pos, gamma, beta, p, seed, site, variant):
    V = words.shape[0]
    pad = 0
    sd = _seed(seed)
    tok = tokens[:M]
    sc = _flat_scale(seed, site, (M, H), p)
    # ---- forward: outputs one row larger than M, filled with a sentinel
    z = torch.full((M + 1, H), -777.0, device=DEV)
    st = torch.full((M + 1, 2), -777.0, device=DEV)
    out = torch.full((M + 1, H), -777.0, device=DEV)
    ob = torch.full((M + 1, H), -777.0, dtype=BF16, device=DEV)
    ops.call("vtx_embed_fwd", tok.data_ptr(), words.data_ptr(), pos.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
             z.data_ptr(), st.data_ptr(), out.data_ptr(), ob.data_ptr(), M, T, H, pad, 1e-8, p, sd.data_ptr(), site, _s())
    t = torch.arange(M, device=DEV) % T
    w64 = words.to(F64).requires_grad_(True)
    p64 = pos.to(F64).requires_grad_(True)
    g64 = gamma.to(F64).requires_grad_(True)
    b64 = beta.to(F64).requires_grad_(True)
    zr = w64[tok] + p64[t]
    mean = zr.mean(-1, keepdim=True)
    rstd = (((zr - mean) ** 2).mean(-1, keepdim=True) + 1e-8).rsqrt()
    y = ((zr - mean) * rstd * g64 + b64) * sc * (tok != pad).to(F64)[:, None]
    tag = f"H={H} M={M} p={p} seed={seed}"
    assert_f32(z[:M], zr.detach(), "z " + tag)
    assert_f32(st[:M, 0], mean.detach()[:, 0], "mean " + tag, scale=zr.detach().abs().max())
    assert_f32(st[:M, 1], rstd.detach()[:, 0], "rstd " + tag)
    assert_f32(out[:M], y.detach(), "out " + tag)
    assert_bf16(ob[:M], y.detach(), 1e-5 * y.detach().abs().max().item(), "out_bf " + tag)
    assert (z[M] == -777).all() and (st[M] == -777).all() and (out[M] == -777).all() and (ob[M] == -777).all()
    # ---- backward: upstream dy_a (fp32) and / or dy_b (bf16), gradients accumulate into non-zero buffers
    g = torch.Generator().manual_seed(H + M + site)
    dy_a = torch.randn(M, H, generator=g).to(DEV) if variant != "b" else None
    dy_b = torch.randn(M, H, generator=g).to(BF16).to(DEV) if variant != "a" else None
    up = torch.zeros(M, H, dtype=F64, device=DEV)
    for d in (dy_a, dy_b):
        if d is not None:
            up += d.to(F64)
    y.backward(up)
    init = {n: (torch.randn(shape, generator=g) * 0.25).to(DEV) for n, shape in
            (("words", (V, H)), ("pos", (pos.shape[0], H)), ("gamma", (H,)), ("beta", (H,)))}
    dw, dp, dg, db = (init[n].clone() for n in ("words", "pos", "gamma", "beta"))
    ops.call("vtx_embed_bwd", _p(dy_a), _p(dy_b), tok.data_ptr(), z.data_ptr(), st.data_ptr(), gamma.data_ptr(),
             dw.data_ptr(), dp.data_ptr(), dg.data_ptr(), db.data_ptr(), M, T, H, pad, p, sd.data_ptr(), site, _s())
    for name, got, ref in (("d_words", dw, w64.grad), ("d_pos", dp, p64.grad), ("d_gamma", dg, g64.grad),
                           ("d_beta", db, b64.grad)):
        i64 = init[name[2:]].to(F64)
        assert_f32(got, i64 + ref, f"{name} {tag} dy={variant}", scale=max(ref.abs().max().item(), 1.0))
    present = torch.zeros(V, dtype=torch.bool, device=DEV)
    present[tok[tok != pad]] = True
    assert torch.equal(dw[~present], init["words"][~present]), "d_words rows of absent tokens changed"


@pytest.mark.parametrize("H", HS)
def test_embedding_forward_backward(H):
    """vtx_embed_fwd / _bwd: gather + LayerNorm(1e-8) + dropout + pad mask, and the scatter of its gradient; caption
    rows of pad tokens, one token repeated in many rows (colliding d_words scatter), token V - 1, and an M that is not
    a multiple of T (the generic backward kernel at every width)."""
    _need_cuda()
    ops = _ops()
    V, T, B = 1000, 30, 9
    g = torch.Generator().manual_seed(H)
    tokens = torch.randint(1, V, (B, T), generator=g)
    tokens[0, 20:] = 0                         # trailing padding
    tokens[2] = 0                              # a row of pad tokens only
    tokens[3] = 7                              # one token in many rows
    tokens[5, ::3] = 7
    tokens[6, 4] = V - 1
    tokens[8, -1] = V - 1
    tokens = tokens.view(-1).to(DEV)
    words = (torch.randn(V, H, generator=g) * 0.8).to(DEV)
    pos = (torch.randn(T, H, generator=g) * 0.5 + 0.3).to(DEV)
    gamma = (1 + 0.2 * torch.randn(H, generator=g)).to(DEV)
    beta = (0.1 * torch.randn(H, generator=g)).to(DEV)
    for M in (B * T, B * T - 7):
        for p in PS:
            for i, seed in enumerate(SEEDS):
                _embed_case(ops, H, M, T, tokens, words, pos, gamma, beta, p, seed, 1000 + 5 * i, ("ab", "b", "a")[i])


# ------------------------------------------------------------------------------------------------ add + LayerNorm
def _ln_ref(z64, gamma, beta):
    mean = z64.mean(-1, keepdim=True)
    rstd = (((z64 - mean) ** 2).mean(-1, keepdim=True) + 1e-5).rsqrt()
    return (z64 - mean) * rstd * gamma.to(F64) + beta.to(F64), mean, rstd


@pytest.mark.parametrize("H", HS)
def test_add_layernorm_forward_backward(H):
    """vtx_add_ln_fwd / vtx_ln_bwd in every combination the engine issues, M = 7683 rows (more than one grid sweep of
    the capped backward grid, not a multiple of 4 warps): post-norm (res, branch, ln = 1); the pre-norm `norm` (no
    branch) and `residual` (ln = 0); ln_bwd with dy_a only, dy_b only and both; d_skip aliasing d_res as the pre-norm
    backward passes them; d_res = NULL; d_branch at p > 0."""
    _need_cuda()
    ops = _ops()
    M = 7683
    g = torch.Generator().manual_seed(H + 1)
    res = torch.randn(M, H, generator=g).to(DEV)
    branch = (torch.randn(M, H, generator=g) * 0.7).to(BF16).to(DEV)
    gamma = (1 + 0.2 * torch.randn(H, generator=g)).to(DEV)
    beta = (0.1 * torch.randn(H, generator=g)).to(DEV)
    dy_a_all = torch.randn(M, H, generator=g).to(DEV)
    dy_b_all = torch.randn(M, H, generator=g).to(BF16).to(DEV)
    SENT = -777.0
    for p in PS:
        for i, seed in enumerate(SEEDS):
            sd = _seed(seed)
            site = 21 + 1000 * i
            tag = f"H={H} p={p} seed={seed}"
            sc = _flat_scale(seed, site, (M, H), p)
            zref = res.to(F64) + branch.to(F64) * sc
            yref, mref, rref = _ln_ref(zref, gamma, beta)
            # ---- post-norm forward
            z = torch.full((M + 1, H), SENT, device=DEV)
            st = torch.full((M + 1, 2), SENT, device=DEV)
            out = torch.full((M + 1, H), SENT, device=DEV)
            ob = torch.full((M + 1, H), SENT, dtype=BF16, device=DEV)
            ops.call("vtx_add_ln_fwd", res.data_ptr(), branch.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                     z.data_ptr(), st.data_ptr(), out.data_ptr(), ob.data_ptr(), M, H, 1e-5, p, sd.data_ptr(), site, 1,
                     _s())
            assert_f32(z[:M], zref, "z " + tag)
            assert_f32(st[:M, 0], mref[:, 0], "mean " + tag, scale=zref.abs().max())
            assert_f32(st[:M, 1], rref[:, 0], "rstd " + tag)
            assert_f32(out[:M], yref, "out " + tag)
            assert_bf16(ob[:M], yref, 1e-5 * yref.abs().max().item(), "out_bf " + tag)
            assert all((t[M] == SENT).all() for t in (z, st, out, ob))
            # ---- pre-norm `norm`: LN of the residual stream, no branch, bf16 output only
            zn = torch.full((M, H), SENT, device=DEV)
            stn = torch.full((M, 2), SENT, device=DEV)
            nb = torch.full((M + 1, H), SENT, dtype=BF16, device=DEV)
            ops.call("vtx_add_ln_fwd", res.data_ptr(), 0, gamma.data_ptr(), beta.data_ptr(), zn.data_ptr(),
                     stn.data_ptr(), 0, nb.data_ptr(), M, H, 1e-5, p, sd.data_ptr(), site, 1, _s())
            ynref, _, _ = _ln_ref(res.to(F64), gamma, beta)
            assert torch.equal(zn, res)
            assert_bf16(nb[:M], ynref, 1e-5 * ynref.abs().max().item(), "norm out_bf " + tag)
            assert (nb[M] == SENT).all()
            # ---- pre-norm `residual`: z = res + dropout(branch), ln = 0, nothing else written
            zr = torch.full((M + 1, H), SENT, device=DEV)
            ops.call("vtx_add_ln_fwd", res.data_ptr(), branch.data_ptr(), 0, 0, zr.data_ptr(), 0, 0, 0, M, H, 0.0, p,
                     sd.data_ptr(), site, 0, _s())
            assert_f32(zr[:M], zref, "residual z " + tag)
            assert (zr[M] == SENT).all()
            # ---- post-norm backward, dy_a / dy_b / both by seed
            variant = ("ab", "a", "b")[i]
            dy_a = dy_a_all if "a" in variant else None
            dy_b = dy_b_all if "b" in variant else None
            up = sum(d.to(F64) for d in (dy_a, dy_b) if d is not None)
            zk = z[:M].to(F64).requires_grad_(True)
            g64, b64 = gamma.to(F64).requires_grad_(True), beta.to(F64).requires_grad_(True)
            y, _, _ = _ln_ref(zk, g64, b64)
            y.backward(up)
            dz = zk.grad
            dz_floor = 1e-5 * dz.abs().max().item()
            g0, b0 = (0.25 * torch.randn(H, generator=g)).to(DEV), (0.25 * torch.randn(H, generator=g)).to(DEV)
            dg, db = g0.clone(), b0.clone()
            dres = torch.full((M + 1, H), SENT, device=DEV)
            dbr = torch.full((M + 1, H), SENT, dtype=BF16, device=DEV)
            ops.call("vtx_ln_bwd", _p(dy_a), _p(dy_b), z.data_ptr(), st.data_ptr(), gamma.data_ptr(), 0, dres.data_ptr(),
                     dbr.data_ptr(), dg.data_ptr(), db.data_ptr(), M, H, p, sd.data_ptr(), site, 1, _s())
            assert_f32(dres[:M], dz, f"d_res {tag} dy={variant}")
            assert_bf16(dbr[:M], dz * sc, dz_floor, f"d_branch {tag} dy={variant}")
            assert_f32(dg, g0.to(F64) + g64.grad, f"d_gamma {tag}", scale=g64.grad.abs().max())
            assert_f32(db, b0.to(F64) + b64.grad, f"d_beta {tag}", scale=b64.grad.abs().max())
            assert (dres[M] == SENT).all() and (dbr[M] == SENT).all()
            # ---- d_res = NULL: only d_branch (and dgamma / dbeta)
            dbr2 = torch.full((M, H), SENT, dtype=BF16, device=DEV)
            dg2, db2 = g0.clone(), b0.clone()
            ops.call("vtx_ln_bwd", _p(dy_a), _p(dy_b), z.data_ptr(), st.data_ptr(), gamma.data_ptr(), 0, 0,
                     dbr2.data_ptr(), dg2.data_ptr(), db2.data_ptr(), M, H, p, sd.data_ptr(), site, 1, _s())
            assert torch.equal(dbr2, dbr[:M]), "d_branch with d_res = NULL " + tag
            assert_f32(dg2, g0.to(F64) + g64.grad, "d_gamma, d_res = NULL " + tag, scale=g64.grad.abs().max())
            # ---- pre-norm norm_bwd: g += LN_backward(dn), d_skip and d_res the same buffer, p = 0 as the engine passes
            zk2 = zn.to(F64).requires_grad_(True)
            g64b = gamma.to(F64).requires_grad_(True)
            y2, _, _ = _ln_ref(zk2, g64b, beta)
            y2.backward(dy_b_all.to(F64))
            gbuf = dy_a_all.clone()
            dg3, db3 = g0.clone(), b0.clone()
            ops.call("vtx_ln_bwd", 0, dy_b_all.data_ptr(), zn.data_ptr(), stn.data_ptr(), gamma.data_ptr(),
                     gbuf.data_ptr(), gbuf.data_ptr(), 0, dg3.data_ptr(), db3.data_ptr(), M, H, 0.0, sd.data_ptr(), 0, 1,
                     _s())
            assert_f32(gbuf, dy_a_all.to(F64) + zk2.grad, "aliased d_skip == d_res " + tag,
                       scale=max(zk2.grad.abs().max().item(), dy_a_all.abs().max().item()))
            assert_f32(dg3, g0.to(F64) + g64b.grad, "d_gamma (norm_bwd) " + tag, scale=g64b.grad.abs().max())
            # ---- pre-norm branch_grad: ln = 0, d_res = NULL, d_branch = g * mask
            dbr3 = torch.full((M + 1, H), SENT, dtype=BF16, device=DEV)
            ops.call("vtx_ln_bwd", dy_a_all.data_ptr(), 0, 0, 0, 0, 0, 0, dbr3.data_ptr(), 0, 0, M, H, p, sd.data_ptr(),
                     site, 0, _s())
            assert_bf16(dbr3[:M], dy_a_all.to(F64) * sc, 0.0, "branch_grad " + tag)
            assert (dbr3[M] == SENT).all()


# ------------------------------------------------------------------------------------------------ attention
ATTN_CASES = [(30, 30, 1), (30, 49, 0), (30, 30, 2), (32, 64, 0), (1, 1, 1), (17, 33, 0), (32, 32, 2)]


def _allowed(B, Tq, Tk, causal, lengths):
    i = torch.arange(Tq, device=DEV)[:, None]
    j = torch.arange(Tk, device=DEV)[None, :]
    L = lengths.view(B, 1, 1)
    if causal == 1:
        ok = (j <= i)[None] & (j[None] < L)
    elif causal == 2:
        ok = (j[None] < L).expand(B, Tq, Tk)
    else:
        ok = torch.ones(B, Tq, Tk, dtype=torch.bool, device=DEV)
    return ok[:, None]                                                      # [B, 1, Tq, Tk]


def _heads(x, B, T, A):
    return x.to(F64).reshape(B, T, A, 64).transpose(1, 2)                   # [B, A, T, 64]


def _flip_floor(a, b):
    """Bound for an output sum_k a[..., i, k] b[..., k, d] whose bf16-rounded terms may flip: 2^-7 of the largest term
    (two flips) + 2^-16 of the sum of magnitudes (fp32 accumulation)."""
    terms = a.abs()[..., :, :, None] * b.abs()[..., None, :, :]
    return 2.0 ** -7 * terms.amax(-2) + 2.0 ** -16 * terms.sum(-2)


@pytest.mark.parametrize("Tq,Tk,causal", ATTN_CASES)
def test_attention_forward_backward(Tq, Tk, causal):
    """vtx_attn_fwd / _bwd against float64 softmax(mask(Q K^T / 8)) * M / (1 - p) . V and its autograd, with ragged
    lengths that include 1 and Tq, B * heads that leave partial CTAs in both kernels (80 and 21 units: 4 warps per
    forward CTA, 3 per backward CTA) and the engine's leading dimensions (packed qkv / dqkv with ld 3H, kv / dkv with
    ld 2H, one output with ldo > H)."""
    _need_cuda()
    ops = _ops()
    self_attn = causal != 0
    for B, A in ((5, 16), (7, 3)):
        H = A * 64
        g = torch.Generator().manual_seed(Tq * 100 + Tk + B)
        if self_attn:
            qkv = torch.randn(B * Tq, 3 * H, generator=g).to(BF16).to(DEV)
            q, k, v = qkv[:, :H], qkv[:, H:2 * H], qkv[:, 2 * H:]
            ldq = ldk = ldv = 3 * H
        else:
            q = torch.randn(B * Tq, H, generator=g).to(BF16).to(DEV)
            kv = torch.randn(B * Tk, 2 * H, generator=g).to(BF16).to(DEV)
            k, v = kv[:, :H], kv[:, H:]
            ldq, ldk, ldv = H, 2 * H, 2 * H
        lengths = torch.randint(1, Tq + 1, (B,), generator=g)
        lengths[0] = Tq
        lengths[1] = 1
        lengths = lengths.to(DEV)
        ldo = H + 64 if (Tq, Tk) == (17, 33) else H
        dout = torch.randn(B * Tq, H, generator=g).to(BF16).to(DEV)
        ok = _allowed(B, Tq, Tk, causal, lengths)
        q4, k4, v4, do4 = _heads(q, B, Tq, A), _heads(k, B, Tk, A), _heads(v, B, Tk, A), _heads(dout, B, Tq, A)
        s = (q4 @ k4.transpose(-1, -2) * 0.125).masked_fill(~ok, float("-inf"))
        lse_ref = torch.logsumexp(s, -1)
        P = torch.softmax(s, -1)
        mx = s.amax(-1, keepdim=True)
        pu = torch.exp(s - mx)
        psum = pu.sum(-1, keepdim=True)
        for p in PS:
            for i, seed in enumerate(SEEDS):
                site = 30 + 1000 * i + 2 * (i % 2)
                tag = f"B={B} A={A} Tq={Tq} Tk={Tk} causal={causal} p={p} seed={seed}"
                sd = _seed(seed)
                Mk = torch.from_numpy(R.attn_scale(seed, site, B, A, Tq, Tk, p)).to(DEV, F64)
                # ---- forward
                out = torch.full((B * Tq, ldo), -777.0, dtype=BF16, device=DEV)
                lse = torch.full((B * A * 32 + 5,), -777.0, device=DEV)
                ops.call("vtx_attn_fwd", q.data_ptr(), ldq, k.data_ptr(), ldk, v.data_ptr(), ldv, out.data_ptr(), ldo,
                         lse.data_ptr(), B, A, Tq, Tk, _p(lengths) if causal else 0, causal, p, sd.data_ptr(), site, _s())
                lk = lse[:B * A * 32].view(B, A, 32)
                assert_f32(lk[..., :Tq], lse_ref, "lse " + tag, scale=lse_ref.abs().max().item() + 1.0)
                assert (lk[..., Tq:] == -777).all() and (lse[B * A * 32:] == -777).all(), "lse padding rows written"
                assert (out[:, H:] == -777).all(), "out ld padding written"
                o_k = _heads(out[:, :H], B, Tq, A)
                pd = _rb(pu * Mk)
                o_same = pd @ v4 / psum
                assert_bf16(o_k, o_same, _flip_floor(pd / psum, v4), "out (same roundings) " + tag)
                o_plain = (P * Mk) @ v4
                assert rel(o_k, o_plain) <= 1e-2, ("out vs float64", rel(o_k, o_plain), tag)
                # ---- backward
                if self_attn:
                    dqkv = torch.full((B * Tq, 3 * H), -777.0, dtype=BF16, device=DEV)
                    dq, dk, dv = dqkv[:, :H], dqkv[:, H:2 * H], dqkv[:, 2 * H:]
                    lddq = lddk = lddv = 3 * H
                else:
                    dq = torch.full((B * Tq, H), -777.0, dtype=BF16, device=DEV)
                    dkv = torch.full((B * Tk, 2 * H), -777.0, dtype=BF16, device=DEV)
                    dk, dv = dkv[:, :H], dkv[:, H:]
                    lddq, lddk, lddv = H, 2 * H, 2 * H
                ops.call("vtx_attn_bwd", q.data_ptr(), ldq, k.data_ptr(), ldk, v.data_ptr(), ldv, dout.data_ptr(), H,
                         lse.data_ptr(), dq.data_ptr(), lddq, dk.data_ptr(), lddk, dv.data_ptr(), lddv, B, A, Tq, Tk,
                         _p(lengths) if causal else 0, causal, p, sd.data_ptr(), site, _s())
                dq4, dk4, dv4 = _heads(dq, B, Tq, A), _heads(dk, B, Tk, A), _heads(dv, B, Tk, A)
                # same roundings: Pd and dS rounded to bf16 before the products
                dPd = do4 @ v4.transpose(-1, -2)
                dP = dPd * Mk
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
                # plain float64 autograd
                qa, ka, va = (t.clone().requires_grad_(True) for t in (q4, k4, v4))
                sa = (qa @ ka.transpose(-1, -2) * 0.125).masked_fill(~ok, float("-inf"))
                ((torch.softmax(sa, -1) * Mk) @ va).backward(do4)
                for name, got, ref in (("dq", dq4, qa.grad), ("dk", dk4, ka.grad), ("dv", dv4, va.grad)):
                    assert rel(got, ref) <= 1e-2, (name, rel(got, ref), tag)


# ------------------------------------------------------------------------------------------------ GELU + dropout
def _all_finite_bf16():
    bits = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16)
    u = bits.view(BF16)
    return u[torch.isfinite(u.float())]


def test_gelu_dropout_every_finite_bf16_input():
    """vtx_gelu_dropout_fwd / _bwd on every finite bf16 value (tiled past one grid sweep), p = 0 and 0.1."""
    _need_cuda()
    ops = _ops()
    u0 = _all_finite_bf16()
    n0 = u0.numel()
    reps = 40
    u = u0.repeat(reps)
    u = torch.cat([u, torch.zeros((-u.numel()) % 8, dtype=BF16)]).to(DEV)
    n = u.numel()
    g = torch.Generator().manual_seed(3)
    dh = torch.randn(n, generator=g).to(BF16).to(DEV)
    u64 = u.to(F64)
    gelu64 = 0.5 * u64 * (1 + torch.erf(u64 / 2 ** 0.5))
    dgelu64 = 0.5 * (1 + torch.erf(u64 / 2 ** 0.5)) + u64 * torch.exp(-0.5 * u64 * u64) / (2 * torch.pi) ** 0.5
    h0 = None
    for p in PS:
        for i, seed in enumerate(SEEDS):
            site = 14 + 1000 * i
            sd = _seed(seed)
            sc = _flat_scale(seed, site, (n,), p)
            h = torch.full((n + 8,), -777.0, dtype=BF16, device=DEV)
            ops.call("vtx_gelu_dropout_fwd", u.data_ptr(), h.data_ptr(), n, p, sd.data_ptr(), site, _s())
            assert (h[n:] == -777).all()
            h = h[:n]
            if p == 0:
                assert_bf16(h, gelu64, u64.abs() * 2.0 ** -22, f"gelu fwd seed={seed}")
                h0 = h.clone()
            else:
                # the kernel scales the bf16-rounded GELU by the fp32 1/(1-p) and rounds again
                want = (h0.float() * torch.from_numpy(R.flat_scale(seed, site, (n,), p)).to(DEV)).to(BF16)
                assert torch.equal(h, want), f"gelu fwd p={p} seed={seed}: {int((h != want).sum())} elements differ"
            du = torch.full((n + 8,), -777.0, dtype=BF16, device=DEV)
            ops.call("vtx_gelu_dropout_bwd", dh.data_ptr(), u.data_ptr(), du.data_ptr(), n, p, sd.data_ptr(), site, _s())
            assert (du[n:] == -777).all()
            ref = dh.to(F64) * sc * dgelu64
            assert_bf16(du[:n], ref, (dh.to(F64) * sc).abs() * 2.0 ** -20, f"gelu bwd p={p} seed={seed}")
            # in place over dh, as the engine calls it
            dh2 = dh.clone()
            ops.call("vtx_gelu_dropout_bwd", dh2.data_ptr(), u.data_ptr(), dh2.data_ptr(), n, p, sd.data_ptr(), site,
                     _s())
            assert torch.equal(dh2, du[:n])
    assert n0 == 65536 - 2 * 128             # every finite bf16 value was covered (not the 2 x 128 inf / NaN codes)


# ------------------------------------------------------------------------------------------------ cross entropy
@pytest.mark.parametrize("V", [1000, 10000, 10240, 10248, 16384])
def test_count_valid_and_cross_entropy(V):
    """vtx_count_valid + vtx_cross_entropy against float64 log-softmax: ldl > V, shift 1 (next-token targets) and 0
    (one label per position), rows whose target is the pad, logits of magnitude up to 80.  V <= 10240 runs the
    register kernel, above it the generic one."""
    _need_cuda()
    ops = _ops()
    B, T, pad = 4, 30, 0
    ldl = V + 24
    g = torch.Generator().manual_seed(V)
    base = (torch.randn(B * T, ldl, generator=g) * 12).clamp(-80, 80)
    base[3, :V] = -80.0
    base[3, 5] = 80.0
    base[7, :V:2] = 80.0
    base[11, V - 1] = 80.0
    tokens = torch.randint(1, V, (B, T), generator=g)
    tokens[0, 25:] = pad
    tokens[1, 3] = pad
    tokens[2, 4] = V - 1
    tokens[2, 5] = 0
    tokens = tokens.to(DEV)
    for shift in (1, 0):
        for write_grad in (1, 0):
            logits = base.to(BF16).to(DEV)
            lg0 = logits.clone()
            if shift:
                tgt = torch.cat([tokens[:, 1:], torch.full((B, 1), pad, device=DEV)], 1).reshape(-1)
            else:
                tgt = tokens.reshape(-1)
            valid = tgt != pad
            n = int(valid.sum())
            count = torch.full((1,), 3.0, device=DEV)
            ops.call("vtx_count_valid", tokens.data_ptr(), B, T, pad, shift, count.data_ptr(), _s())
            assert count.item() == 3.0 + n, (count.item(), n)       # accumulates
            count.fill_(0)
            ops.call("vtx_count_valid", tokens.data_ptr(), B, T, pad, shift, count.data_ptr(), _s())
            loss = torch.full((1,), 0.5, device=DEV)
            ops.call("vtx_cross_entropy", logits.data_ptr(), ldl, tokens.data_ptr(), B, T, V, pad, shift,
                     count.data_ptr(), loss.data_ptr(), write_grad, _s())
            z = lg0[:, :V].to(F64)
            lse = torch.logsumexp(z, -1)
            nll = lse - z.gather(1, tgt.clamp_min(0)[:, None])[:, 0]
            ref = (nll * valid).sum() / n
            tag = f"V={V} shift={shift} write_grad={write_grad}"
            assert abs(loss.item() - 0.5 - ref.item()) <= 1e-5 * abs(ref.item()) + 1e-6, (loss.item() - 0.5, ref.item(),
                                                                                           tag)
            assert torch.equal(logits[:, V:], lg0[:, V:]), "columns >= V written " + tag
            if not write_grad:
                assert torch.equal(logits, lg0)
                continue
            d = (torch.softmax(z, -1) - torch.nn.functional.one_hot(tgt, V).to(F64)) / n * valid[:, None]
            assert_bf16(logits[:, :V], d, 2.0 ** -20 / n + 2.0 ** -120, "dlogits " + tag)
            assert (logits[~valid, :V] == 0).all()


def test_cross_entropy_all_pad_batch():
    """A batch without a single target: the kernels give loss += 0 and zero gradient rows (count = 0 is clamped to 1
    in the division); torch's token-mean cross entropy would give NaN (0 / 0).  This pins the kernels' behaviour."""
    _need_cuda()
    ops = _ops()
    B, T = 3, 30
    tokens = torch.zeros(B, T, dtype=torch.int64, device=DEV)
    tokens[:, 0] = 1                                 # [SOS] only: no next-token target anywhere
    for shift, V in ((1, 1000), (0, 16384)):     # the register and the generic kernel
        toks = tokens if shift else torch.zeros_like(tokens)
        logits = torch.randn(B * T, V).to(BF16).to(DEV)
        count = torch.zeros(1, device=DEV)
        loss = torch.full((1,), 0.25, device=DEV)
        ops.call("vtx_count_valid", toks.data_ptr(), B, T, 0, shift, count.data_ptr(), _s())
        assert count.item() == 0
        ops.call("vtx_cross_entropy", logits.data_ptr(), V, toks.data_ptr(), B, T, V, 0, shift, count.data_ptr(),
                 loss.data_ptr(), 1, _s())
        assert loss.item() == 0.25
        assert (logits == 0).all()


# ------------------------------------------------------------------------------------------------ colsum / argmax
@pytest.mark.parametrize("M", [1, 7, 63, 64, 65, 7683])
def test_colsum(M):
    """out[n] += sum_m X[m, n] over bf16 X with ld > N: the row-lane kernel (M >= 64, N % 8 == 0, including its
    m + 24 < m1 tail) and the generic one."""
    _need_cuda()
    ops = _ops()
    for N in (8, 81, 1024, 3072, 10000):
        ld = (N + 7) // 8 * 8 + 16
        g = torch.Generator().manual_seed(M * 7 + N)
        X = (torch.randn(M, ld, generator=g) + 0.25).to(BF16).to(DEV)
        init = torch.randn(N + 4, generator=g).to(DEV)
        out = init.clone()
        ops.call("vtx_colsum", X.data_ptr(), ld, M, N, out.data_ptr(), _s())
        x = X[:, :N].to(F64)
        ref = init[:N].to(F64) + x.sum(0)
        tol = 1e-5 * (x.abs().sum(0) + init[:N].to(F64).abs())
        err = (out[:N].to(F64) - ref).abs()
        assert (err <= tol).all(), (M, N, (err / tol).max().item())
        assert torch.equal(out[N:], init[N:])


def test_argmax_rows():
    """First-index argmax of fp32 rows with ld > N: ties anywhere in the row (across threads and warps), an all -inf
    row, the maximum in the last column, N in {1, 255, 257, 10000}."""
    _need_cuda()
    ops = _ops()
    for N in (1, 255, 257, 10000):
        M, ld = 9, N + 3
        g = torch.Generator().manual_seed(N)
        X = torch.randn(M, ld, generator=g)
        X[:, N:] = 1e30                               # beyond N: must never be picked
        X[1, :N] = float("-inf")
        if N > 1:
            X[2, :N] = 0.5
            X[3, N - 1] = 50.0
            X[4, [N // 2, N - 1]] = 60.0
            X[5, [1, N // 3, N - 1]] = 70.0
            X[6, :N] = torch.randint(0, 3, (N,), generator=g).float()
        X = X.to(DEV)
        out = torch.full((M + 1,), -5, dtype=torch.int64, device=DEV)
        ops.call("vtx_argmax_rows", X.data_ptr(), ld, M, N, out.data_ptr(), _s())
        ref = torch.argmax(X[:, :N].cpu().to(F64), 1)   # torch: the first maximal index
        assert torch.equal(out[:M].cpu(), ref), (N, out[:M].tolist(), ref.tolist())
        assert out[M].item() == -5
