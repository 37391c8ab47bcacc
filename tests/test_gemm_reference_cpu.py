"""The float64 GEMM reference of tests/gemm_reference.py on the CPU: against independent torch formulas at small
shapes, its checker against simulated kernel outputs with and without planted faults, and a census of the kernel paths
every GEMM of the shipped workloads takes (dry run of the engine, tests/test_engine_dryrun.py's recorder pattern)."""
import pytest
import torch
import torch.nn.functional as F

from tests import gemm_reference as G

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
SMS = 132   # H100 SXM


def _rnd(*shape, seed=0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)).to(BF16)


def _ref(c):
    """Whole float64 product of a call (no epilogue), [M, N]."""
    out = torch.zeros(c.M, c.N, dtype=F64)
    for r0, r1, acc in G.acc_chunks(c):
        out[r0:r1] = acc
    return out


def _nchw(x):
    return x.double().permute(0, 3, 1, 2)


# ----------------------------------------------------------------------------------- reference vs torch formulas
@pytest.mark.parametrize("stride,taps", [(1, 0), (2, 0), (2, 1)])
def test_fprop_and_wgrad_match_conv2d(stride, taps):
    NI, H, W, C, Co = 2, 7, 6, 64, 128
    x, w = _rnd(NI, H, W, C, seed=1), _rnd(Co, 3, 3, C, seed=2)
    k = 1 if taps == 1 else 3
    wk = w[:, 1:2, 1:2] if taps == 1 else w
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    M = NI * Ho * Wo
    y = torch.empty(M, Co, dtype=BF16)
    c = G.Call(x, wk.reshape(Co, -1).contiguous(), y, M, Co, k * k * C, lda=C, conv=(NI, H, W, C), conv_mode=1,
               conv_stride=stride, conv_taps=taps)
    want = F.conv2d(_nchw(x), _nchw(wk), stride=stride, padding=0 if taps == 1 else 1)
    assert torch.allclose(_ref(c), want.permute(0, 2, 3, 1).reshape(M, Co), rtol=1e-12, atol=1e-9)
    dy = _rnd(NI, Ho, Wo, Co, seed=3)
    dw = torch.zeros(Co, k * k * C)
    c = G.Call(dy, x, dw, Co, k * k * C, M, lda=Co, ldb=C, atomic=True, split_k=2, out_f32=True, conv=(NI, H, W, C),
               conv_mode=2, conv_stride=stride, conv_taps=taps)
    want = torch.nn.grad.conv2d_weight(_nchw(x), (Co, C, k, k), _nchw(dy), stride=stride, padding=0 if taps == 1 else 1)
    assert torch.allclose(_ref(c), want.permute(0, 2, 3, 1).reshape(Co, -1), rtol=1e-12, atol=1e-9)


def test_mode4_is_the_transpose_of_mode2():
    NI, H, W, C = 2, 5, 9, 64
    x, dy = _rnd(NI, H, W, C, seed=4), _rnd(NI, H, W, C, seed=5)
    c2 = G.Call(dy, x, torch.zeros(C, 9 * C), C, 9 * C, NI * H * W, lda=C, ldb=C, atomic=True, out_f32=True,
                conv=(NI, H, W, C), conv_mode=2)
    c4 = G.Call(dy, x, torch.zeros(9 * C, C), 9 * C, C, NI * H * W, lda=C, ldb=C, ldd=C, atomic=True, out_f32=True,
                conv=(NI, H, W, C), conv_mode=4)
    assert torch.equal(_ref(c4), _ref(c2).t())


@pytest.mark.parametrize("ph,pw", [(0, 0), (0, 1), (1, 0), (1, 1)])
def test_parity_class_dgrad_matches_conv_autograd(ph, pw):
    """A stride-2 3x3 dgrad as the engine splits it: parity class (ph, pw) of the input gradient is a (1+ph) x (1+pw)
    tap grid over dy whose tap (a, b) uses kernel element (ph + 1 - 2a, pw + 1 - 2b), written through an output view."""
    NI, H, W, C, Co = 2, 7, 8, 64, 64
    x = _nchw(_rnd(NI, H, W, C, seed=6)).requires_grad_(True)
    w = _rnd(Co, 3, 3, C, seed=7)
    y = F.conv2d(x, _nchw(w), stride=2, padding=1)
    dy = _rnd(NI, y.shape[2], y.shape[3], Co, seed=8)
    y.backward(_nchw(dy))
    dx = x.grad.permute(0, 2, 3, 1)                       # [NI, H, W, C]
    th, tw = 1 + ph, 1 + pw
    Hn, Wn = dy.shape[1], dy.shape[2]
    # dgrad weights of the class: [C_in, (a, b, co)]
    wt = torch.stack([torch.stack([w[:, ph + 1 - 2 * a, pw + 1 - 2 * b, :] for b in range(tw)]) for a in range(th)])
    wt = wt.permute(3, 0, 1, 2).reshape(C, th * tw * Co).contiguous()
    Hs, Ws = (H - ph + 1) // 2, (W - pw + 1) // 2
    D = torch.full((NI, H, W, C), 7.0, dtype=BF16)
    voff = (ph * W + pw) * C * 2
    c = G.Call(dy, wt, D, NI * Hn * Wn, C, th * tw * Co, lda=Co, conv=(NI, Hn, Wn, Co), conv_mode=1,
               tap_grid=(th, tw, 0), d_ptr=D.data_ptr() + voff, out_view=(Hs, Ws, 2 * C, 2 * W * C, H * W * C))
    flat = torch.zeros(D.numel(), dtype=F64)
    for r0, r1, acc in G.acc_chunks(c):
        idx, ok = G.out_index(c, r0, r1)
        flat[idx[ok].reshape(-1)] = acc[ok].reshape(-1)
    got = flat.view(NI, H, W, C)[:, ph::2, pw::2]
    assert torch.allclose(got, dx[:, ph::2, pw::2], rtol=1e-12, atol=1e-9)


def test_stem_matches_the_7x7_stride2_conv():
    """conv_mode 5 over the space-to-depth view S of the header equals the 7x7/2/pad-3 conv of the image; conv_mode 6
    equals its weight gradient (both in the packed k = a*64 + b*16 + (r*2+q)*3 + c layout)."""
    NI, H, W = 2, 32, 32
    img = torch.randn(NI, 3, H, W, generator=torch.Generator().manual_seed(9)).to(BF16).double()
    w = torch.randn(64, 3, 7, 7, generator=torch.Generator().manual_seed(10)).to(BF16).double()
    Ho, Wo = H // 2, W // 2
    S = torch.zeros(NI, Ho + 3, Wo + 3, 16, dtype=F64)
    wp = torch.zeros(64, 256, dtype=F64)
    for r in range(2):
        for q in range(2):
            for ch in range(3):
                for i in range(Ho + 3):
                    for j in range(Wo + 3):
                        y, x = 2 * i + r - 3, 2 * j + q - 3
                        if 0 <= y < H and 0 <= x < W:
                            S[:, i, j, (r * 2 + q) * 3 + ch] = img[:, ch, y, x]
                for a in range(4):
                    for b in range(4):
                        kh, kw = 2 * a + r, 2 * b + q
                        if kh < 7 and kw < 7:
                            wp[:, a * 64 + b * 16 + (r * 2 + q) * 3 + ch] = w[:, ch, kh, kw]
    S, wp = S.to(BF16), wp.to(BF16)
    M = NI * Ho * Wo
    c = G.Call(S, wp, torch.empty(M, 64, dtype=BF16), M, 64, 256, lda=64, ldb=256, conv=(NI, Ho, Wo, 64), conv_mode=5)
    want = F.conv2d(img, w, stride=2, padding=3)
    assert torch.allclose(_ref(c), want.permute(0, 2, 3, 1).reshape(M, 64), rtol=1e-12, atol=1e-9)
    dy = _rnd(NI, Ho, Wo, 64, seed=11)
    c = G.Call(dy, S, torch.zeros(64, 256), 64, 256, M, lda=64, ldb=64, atomic=True, out_f32=True,
               conv=(NI, Ho, Wo, 64), conv_mode=6)
    dw = torch.nn.grad.conv2d_weight(img, (64, 3, 7, 7), _nchw(dy), stride=2, padding=3)
    got = _ref(c)
    for r in range(2):
        for q in range(2):
            for a in range(4):
                for b in range(4):
                    kh, kw = 2 * a + r, 2 * b + q
                    cols = [a * 64 + b * 16 + (r * 2 + q) * 3 + ch for ch in range(3)]
                    if kh < 7 and kw < 7:
                        assert torch.allclose(got[:, cols], dw[:, :, kh, kw], rtol=1e-12, atol=1e-9)


# ------------------------------------------------------------------------------------------- checker sensitivity
def _simulate(c, before, integer, fault=None):
    """What a correct kernel writes for call c: the reference rounded to the output type (real data: through fp32,
    the accumulator), written through the call's output map, with the statistics of the written D.  `fault(c, r0, r1,
    val, idx)` may alter the values about to be written."""
    Df = G._flat(c.D)
    sums = torch.zeros(2, c.N, dtype=F64)
    for r0, r1, acc in G.acc_chunks(before):
        v, _, _ = G.epilogue(before, r0, r1, acc)
        val = G.activation(v, c.act)
        idx, ok = G.out_index(c, r0, r1)
        if c.atomic:
            val = val + G._flat(before.D)[idx].double()
        if fault is not None:
            val, ok = fault(c, r0, r1, val, ok)
        q = val.float()
        if not c.out_f32:
            q = q.to(BF16)
        Df[idx[ok]] = q[ok].to(Df.dtype)
        d = Df[idx[ok]].double()
        sums += torch.stack([d.sum(0), (d * d).sum(0)])
    if c.stats is not None:
        c.stats.view(2, -1)[:, :c.N] += sums.float()


def _fill_real(c, seed):
    g = torch.Generator().manual_seed(seed)
    for t in c.tensors().values():
        f = G._flat(t)
        if t.dtype == torch.uint8:
            f.copy_(torch.randint(0, 256, f.shape, generator=g).to(torch.uint8))
        else:
            f.copy_(torch.randn(f.shape, generator=g).to(t.dtype))


def _case(kind):
    """Small calls, each with the feature a planted fault targets (ragged M = 300: the last row tile is partial)."""
    M, N, K = 300, 128, 256
    A, B = torch.empty(M, K, dtype=BF16), torch.empty(N, K, dtype=BF16)
    D = torch.empty(M, N, dtype=BF16)
    if kind == "conv":
        NI, H, W, C = 2, 6, 5, 64
        return G.Call(torch.empty(NI, H, W, C, dtype=BF16), torch.empty(64, 9 * C, dtype=BF16),
                      torch.empty(NI * H * W, 64, dtype=BF16), NI * H * W, 64, 9 * C, lda=C, conv=(NI, H, W, C),
                      conv_mode=1)
    if kind == "splitk":
        return G.Call(torch.empty(K, M, dtype=BF16), torch.empty(K, N, dtype=BF16), torch.empty(M, N), M, N, K,
                      a_mn=1, b_mn=1, atomic=True, split_k=2, out_f32=True)
    if kind == "bias":
        return G.Call(A, torch.empty(320, K, dtype=BF16), torch.empty(M, 320, dtype=BF16), M, 320, K,
                      bias=torch.empty(320))
    if kind == "residual":
        return G.Call(A, B, D, M, N, K, residual=torch.empty(M, N, dtype=BF16))
    if kind == "mask":
        return G.Call(A, B, D, M, N, K, residual=torch.empty(M, N, dtype=BF16),
                      residual_mask=torch.empty(M, N // 8, dtype=torch.uint8))
    return G.Call(A, B, D, M, N, K, stats=torch.empty(2, N))


def _drop_kblock(c, r0, r1, val, ok):
    A = G._mat(c.A, c.M, c.K, c.lda, c.a_mn).double()[:128, 64:128]
    Bm = G._mat(c.B, c.N, c.K, c.ldb, c.b_mn).double()[:128, 64:128]
    val = val.clone()
    val[:128, :128] -= A @ Bm.t()
    return val, ok


def _tap_off(c, r0, r1, val, ok):
    """The left tap column of output column 0 reads input column 0 instead of the zero padding."""
    NI, H, W, C = c.conv
    x = c.A.double()
    Wt = G._mat(c.B, c.N, c.K, c.ldb, 0).double()
    val = val.view(NI, H, W, -1).clone()
    for a in range(3):
        for h in range(H):
            hh = h + a - 1
            if 0 <= hh < H:
                val[:, h, 0] += x[:, hh, 0] @ Wt[:, (a * 3) * C:(a * 3 + 1) * C].t()
    return val.view(NI * H * W, -1), ok


def _ragged_unwritten(c, r0, r1, val, ok):
    ok = ok.clone()
    ok[256 - r0:] = False
    return val, ok


def _neighbour_residual(c, r0, r1, val, ok):
    res = c.residual.double()
    val = val.clone()
    val[5] += res[6] - res[5]
    return val, ok


def _split_twice(c, r0, r1, val, ok):
    A = G._mat(c.A, c.M, c.K, c.lda, c.a_mn).double()[:, 128:]
    Bm = G._mat(c.B, c.N, c.K, c.ldb, c.b_mn).double()[:, 128:]
    return val + A @ Bm.t(), ok


def _bias_block_missing(c, r0, r1, val, ok):
    val = val.clone()
    val[:, 128:256] -= c.bias.double()[128:256]
    return val, ok


def _mask_wrong_byte(c, r0, r1, val, ok):
    """Row 3 reads its residual mask bits from the next byte (the next 8 columns' bits)."""
    res = c.residual.double()[3]
    bits = G._bits(c.residual_mask, 0, c.M, c.N)[3]
    wrong = torch.roll(bits.view(-1, 8), -1, 0).reshape(-1)
    val = val.clone()
    val[3] += res * (wrong.double() - bits.double())
    return val, ok


FAULTS = {
    "k-block dropped": ("plain", _drop_kblock),
    "border tap one pixel off": ("conv", _tap_off),
    "ragged last row tile unwritten": ("plain", _ragged_unwritten),
    "neighbouring row's residual": ("residual", _neighbour_residual),
    "split-K partial added twice": ("splitk", _split_twice),
    "column block without bias": ("bias", _bias_block_missing),
    "mask bit from the wrong byte": ("mask", _mask_wrong_byte),
}


@pytest.mark.parametrize("integer", [True, False], ids=["integer", "real"])
@pytest.mark.parametrize("fault", list(FAULTS))
def test_checker_passes_a_correct_output_and_catches_each_fault(fault, integer):
    kind, plant = FAULTS[fault]
    c = _case(kind)
    if integer:
        G.integer_fill(c, torch.Generator().manual_seed(1))
    else:
        _fill_real(c, 2)
    D0 = G._flat(c.D).clone()
    before = G.snapshot(c)
    _simulate(c, before, integer)
    G.check(c, before, c, SMS, integer=integer)
    G._flat(c.D).copy_(D0)
    before = G.snapshot(c)
    _simulate(c, before, integer, plant)
    if integer or fault not in ("border tap one pixel off", "mask bit from the wrong byte"):
        with pytest.raises(AssertionError):
            G.check(c, before, c, SMS, integer=integer)


def test_statistics_are_checked():
    c = _case("plain")
    G.integer_fill(c, torch.Generator().manual_seed(3))
    before = G.snapshot(c)
    _simulate(c, before, True)
    G.check(c, before, c, SMS, integer=True)
    c.stats[1, 7] += 1.0
    with pytest.raises(AssertionError):
        G.check(c, before, c, SMS, integer=True)


# ------------------------------------------------------------------------------------------------------ census
def census(monkeypatch, sms, workloads=None):
    """Path keys of every GEMM of the workloads, from a dry run of the engine on the CPU at `sms` SMs."""
    from virtex_b200 import engine as E, ops
    from tests.test_engine_dryrun import _check_gemm
    keys = set()

    def fake_gemm(A, B, D, M, N, K, col_scale=None, col_shift=None, **kw):
        _check_gemm(A, B, D, M, N, K, **kw)
        c = G.Call(A, B, D, M, N, K, col_scale=col_scale, col_shift=col_shift, **kw)
        expressible(c)
        keys.add(G.path_key(c, sms))

    with monkeypatch.context() as m:
        m.setattr(E, "call", lambda name, *args: None)
        m.setattr(E, "gemm", fake_gemm)
        m.setattr(E, "_stream", lambda: 0)
        m.setattr(E, "_require_cuda", lambda dev: None)
        m.setattr(ops, "num_sms", lambda: sms)
        m.setattr(ops, "set_dynamic_gemm_schedule", lambda on: None)
        for name, run in (workloads or list(G.WORKLOADS.items()) + [G.BATCH_256]):
            run("cpu")
    return keys


def expressible(c):
    """The reference's assumptions about a call hold: every epilogue term it models, nothing it does not."""
    assert c.act in (0, 1, 2) and c.conv_mode in (0, 1, 2, 4, 5, 6)
    if c.conv_mode != 0:
        g = G.conv_geom(c)
        HW = g["Ho"] * g["Wo"] * g["NI"]
        if c.conv_mode in (1, 5):
            assert c.M == HW and c.K == g["th"] * g["tw"] * g["C"]
        elif c.conv_mode == 4:
            assert c.M == 9 * g["C"] and c.K == HW
        else:
            assert c.N == g["th"] * g["tw"] * g["C"] and c.K == HW
    if c.out_view is not None:
        oh, ow, sw, sh, sn = c.out_view
        g = G.conv_geom(c)
        last = c.d_off + (g["NI"] - 1) * sn + (oh - 1) * sh + (ow - 1) * sw + c.N
        assert c.conv_mode == 1 and last <= c.D.numel()
    if not c.out_f32 and c.N % 8:   # bf16 rows are stored in 16-byte chunks: D's rows must own the padding
        assert c.D.dim() == 2 and c.D.stride(0) == c.ldd and c.D.shape[1] >= (c.N + 7) // 8 * 8
    if c.ss:
        assert c.bias is None and c.stats is None and c.bnr_y is None and c.out_view is None
    if c.bnr_y is not None:
        assert c.stats is None and c.bias is None and not c.out_f32 and c.split_k == 1


# The kernel paths of the shipped workloads at 132 SMs (H100 SXM); 24 of them appear only in the batch-256 step (sched_chunk
# 4, 256-wide tiles of the large convs, the bn3 reductions fused into conv1 dgrads).  An engine change that routes a GEMM onto a path
# not listed here has to extend the table -- and so gets its path checked by tests/test_gemm_engine_gpu.py.
EXPECTED = {
    'm0 gemm bn128 ls f32 rtma0 bp1 bnr=- ss0 view0 ch1',
    'm0 gemm bn128 ls f32+= rtma0 bp0 bnr=- ss0 view0 ch1',
    'm0 gemm bn128 pp bf16 rtma0 bp0 bnr=- ss0 view0 ch1',
    'm0 gemm bn128 pp bf16 rtma0 bp0 bnr=- ss0 view0 ch4',
    'm0 gemm bn128 pp bf16 rtma0 bp0 bnr=- ss1 view0 ch1',
    'm0 gemm bn128 pp bf16 rtma0 bp0 bnr=y ss0 view0 ch1',
    'm0 gemm bn128 pp bf16 rtma0 bp1 bnr=- ss0 view0 ch1',
    'm0 gemm bn128 pp bf16 rtma1 bp0 bnr=- ss0 view0 ch1',
    'm0 gemm bn128 pp bf16 rtma1 bp0 bnr=- ss1 view0 ch1',
    'm0 gemm bn192 ls f32+= rtma0 bp0 bnr=- ss0 view0 ch1',
    'm0 gemm bn256 ls bf16 rtma0 bp0 bnr=- ss0 view0 ch1',
    'm0 gemm bn256 ls bf16 rtma0 bp0 bnr=- ss0 view0 ch2',
    'm0 gemm bn256 ls bf16 rtma0 bp0 bnr=- ss0 view0 ch4',
    'm0 gemm bn256 ls bf16 rtma0 bp0 bnr=y ss0 view0 ch1',
    'm0 gemm bn256 ls bf16 rtma0 bp1 bnr=- ss0 view0 ch1',
    'm0 gemm bn256 ls bf16 rtma0 bp1 bnr=- ss0 view0 ch2',
    'm0 gemm bn256 ls bf16 rtma1 bp0 bnr=- ss0 view0 ch1',
    'm0 gemm bn256 ls bf16 rtma1 bp0 bnr=- ss0 view0 ch2',
    'm0 gemm bn256 ls bf16 rtma1 bp0 bnr=- ss0 view0 ch4',
    'm0 gemm bn256 ls bf16 rtma1 bp0 bnr=bits ss0 view0 ch1',
    'm0 gemm bn256 ls bf16 rtma1 bp0 bnr=bits ss0 view0 ch2',
    'm0 gemm bn256 ls bf16 rtma1 bp0 bnr=bits ss0 view0 ch4',
    'm0 gemm bn256 ls f32+= rtma0 bp0 bnr=- ss0 view0 ch1',
    'm0 gemm bn64 ls f32 rtma0 bp1 bnr=- ss0 view0 ch1',
    'm0 gemm bn64 ls f32+= rtma0 bp0 bnr=- ss0 view0 ch1',
    'm0 gemm bn64 pp bf16 rtma0 bp0 bnr=- ss0 view0 ch1',
    'm0 gemm bn64 pp bf16 rtma0 bp0 bnr=- ss0 view0 ch4',
    'm0 gemm bn64 pp bf16 rtma0 bp0 bnr=- ss1 view0 ch1',
    'm0 gemm bn64 pp bf16 rtma0 bp0 bnr=y ss0 view0 ch1',
    'm0 gemm bn64 pp bf16 rtma0 bp0 bnr=y ss0 view0 ch4',
    'm0 gemm bn64 pp bf16 rtma1 bp0 bnr=- ss0 view0 ch1',
    'm0 gemm bn64 pp bf16 rtma1 bp0 bnr=- ss0 view0 ch4',
    'm1 s1/1x1p0 bn128 pp bf16 rtma0 bp0 bnr=y ss0 view1 ch1',
    'm1 s1/1x1p0 bn128 pp bf16 rtma1 bp0 bnr=- ss0 view1 ch1',
    'm1 s1/1x1p0 bn256 ls bf16 rtma0 bp0 bnr=y ss0 view1 ch1',
    'm1 s1/1x1p0 bn256 ls bf16 rtma1 bp0 bnr=- ss0 view1 ch1',
    'm1 s1/1x2p0 bn128 pp bf16 rtma0 bp0 bnr=y ss0 view1 ch1',
    'm1 s1/1x2p0 bn256 ls bf16 rtma0 bp0 bnr=y ss0 view1 ch1',
    'm1 s1/2x1p0 bn128 pp bf16 rtma0 bp0 bnr=y ss0 view1 ch1',
    'm1 s1/2x1p0 bn256 ls bf16 rtma0 bp0 bnr=y ss0 view1 ch1',
    'm1 s1/2x2p0 bn128 pp bf16 rtma0 bp0 bnr=y ss0 view1 ch1',
    'm1 s1/2x2p0 bn256 ls bf16 rtma0 bp0 bnr=y ss0 view1 ch1',
    'm1 s1/3x3p1 bn128 pp bf16 rtma0 bp0 bnr=- ss0 view0 ch1',
    'm1 s1/3x3p1 bn128 pp bf16 rtma0 bp0 bnr=- ss1 view0 ch1',
    'm1 s1/3x3p1 bn128 pp bf16 rtma0 bp0 bnr=y ss0 view0 ch1',
    'm1 s1/3x3p1 bn256 ls bf16 rtma0 bp0 bnr=- ss0 view0 ch1',
    'm1 s1/3x3p1 bn256 ls bf16 rtma0 bp0 bnr=y ss0 view0 ch1',
    'm1 s1/3x3p1 bn64 pp bf16 rtma0 bp0 bnr=- ss0 view0 ch1',
    'm1 s1/3x3p1 bn64 pp bf16 rtma0 bp0 bnr=- ss0 view0 ch4',
    'm1 s1/3x3p1 bn64 pp bf16 rtma0 bp0 bnr=- ss1 view0 ch1',
    'm1 s1/3x3p1 bn64 pp bf16 rtma0 bp0 bnr=y ss0 view0 ch1',
    'm1 s1/3x3p1 bn64 pp bf16 rtma0 bp0 bnr=y ss0 view0 ch4',
    'm1 s2/1x1p0 bn128 pp bf16 rtma0 bp0 bnr=- ss0 view0 ch1',
    'm1 s2/1x1p0 bn128 pp bf16 rtma0 bp0 bnr=- ss0 view0 ch2',
    'm1 s2/1x1p0 bn128 pp bf16 rtma0 bp0 bnr=- ss1 view0 ch1',
    'm1 s2/1x1p0 bn256 ls bf16 rtma0 bp0 bnr=- ss0 view0 ch1',
    'm1 s2/1x1p0 bn256 ls bf16 rtma0 bp0 bnr=- ss0 view0 ch2',
    'm1 s2/3x3p1 bn128 pp bf16 rtma0 bp0 bnr=- ss0 view0 ch1',
    'm1 s2/3x3p1 bn128 pp bf16 rtma0 bp0 bnr=- ss1 view0 ch1',
    'm1 s2/3x3p1 bn256 ls bf16 rtma0 bp0 bnr=- ss0 view0 ch1',
    'm2 s1/3x3p1 bn128 ls f32+= rtma0 bp0 bnr=- ss0 view0 ch1',
    'm2 s1/3x3p1 bn256 ls f32+= rtma0 bp0 bnr=- ss0 view0 ch1',
    'm2 s2/1x1p0 bn128 ls f32+= rtma0 bp0 bnr=- ss0 view0 ch1',
    'm2 s2/1x1p0 bn256 ls f32+= rtma0 bp0 bnr=- ss0 view0 ch1',
    'm2 s2/3x3p1 bn128 ls f32+= rtma0 bp0 bnr=- ss0 view0 ch1',
    'm2 s2/3x3p1 bn256 ls f32+= rtma0 bp0 bnr=- ss0 view0 ch1',
    'm4 s1/3x3p1 bn256 ls f32+= rtma0 bp0 bnr=- ss0 view0 ch1',
    'm5 stem bn64 pp bf16 rtma0 bp0 bnr=- ss0 view0 ch1',
    'm5 stem bn64 pp bf16 rtma0 bp0 bnr=- ss0 view0 ch2',
    'm5 stem bn64 pp bf16 rtma0 bp0 bnr=- ss0 view0 ch4',
    'm6 stem bn256 ls f32+= rtma0 bp0 bnr=- ss0 view0 ch1',
}


def test_census_of_the_shipped_workloads(monkeypatch):
    keys = census(monkeypatch, SMS)
    assert keys == EXPECTED, (sorted(keys - EXPECTED), sorted(EXPECTED - keys))
