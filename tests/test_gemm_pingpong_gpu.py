"""The two consumer schedules of the GEMM (csrc/gemm_tc.cu) compute the same bits.  A bf16 output at most 128 columns
wide runs the ping-pong schedule; asking for 256-wide tiles (tile_n = 256) runs the same problem in lockstep.  Every
output element sees the same K order in both, so bf16 outputs must match exactly; the BN statistics / BN-backward sums
are reduced in another order and match to fp32 rounding.  Covers odd tile counts per CTA (one warpgroup gets one more
tile), a single tile (the second warpgroup only sees the end marker), several column blocks, the TMA-staged residual
with and without its mask, the fused BN-backward sums and the implicit 3x3 convolution, under both tile schedules."""
import pytest
import torch

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16


def _ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from virtex_b200 import ops
    return ops


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def _pack_mask(keep):
    M, C = keep.shape
    w = (1 << torch.arange(8, device=keep.device)).to(torch.int32)
    return (keep.view(M, C // 8, 8).to(torch.int32) * w).sum(-1).to(torch.uint8).contiguous()


@pytest.fixture(params=["static", "dynamic"])
def schedule(request):
    ops = _ops()
    ops.set_dynamic_gemm_schedule(request.param == "dynamic")
    yield request.param
    ops.set_dynamic_gemm_schedule(False)


def _both(fn):
    """fn(tile_n) -> tuple of tensors: ping-pong (tile_n = 0) and lockstep (tile_n = 256) results."""
    return fn(0), fn(256)


@pytest.mark.parametrize("M,N,K", [
    (60000, 64, 64),     # 469 tiles: odd count per CTA, one k-block
    (19077, 128, 576),   # ragged last row tile, nine k-blocks
    (100, 64, 256),      # one tile: the second warpgroup only sees the end marker
    (30011, 96, 128),    # partial column tile
    (9000, 128, 1024),   # long K
])
def test_pingpong_matches_lockstep_bit_for_bit(M, N, K, schedule):
    ops = _ops()
    g = torch.Generator().manual_seed(M + N + K)
    A = (torch.randn(M, K, generator=g) * 0.5).bfloat16().cuda()
    B = (torch.randn(N, K, generator=g) * 0.5).bfloat16().cuda()
    Bt = B.t().contiguous()
    bias = torch.randn(N, generator=g).cuda()
    R = torch.randn(M, N, generator=g).bfloat16().cuda()
    keep = (torch.rand(M, N, generator=g) > 0.5).cuda()
    ref = A.float() @ B.float().t()

    def run(tile_n):
        out = []
        D = torch.empty(M, N, dtype=BF16, device="cuda")
        st = torch.zeros(2, N, device="cuda")
        ops.gemm(A, B, D, M, N, K, stats=st, tile_n=tile_n)
        out += [D, st]
        D = torch.empty(M, N, dtype=BF16, device="cuda")
        ops.gemm(A, Bt, D, M, N, K, b_mn=1, bias=bias, act=2, tile_n=tile_n)
        out.append(D)
        D = torch.empty(M, N, dtype=BF16, device="cuda")
        ops.gemm(A, B, D, M, N, K, residual=R, tile_n=tile_n)
        out.append(D)
        if N % 32 == 0:
            D = torch.empty(M, N, dtype=BF16, device="cuda")
            ops.gemm(A, B, D, M, N, K, residual=R, residual_mask=_pack_mask(keep), tile_n=tile_n)
            out.append(D)
        return out

    pp, ls = _both(run)
    assert rel(pp[0], ref) < 4e-3
    assert rel(pp[1][0], pp[0].double().sum(0)) < 1e-4 and rel(pp[1][1], (pp[0].double() ** 2).sum(0)) < 1e-4
    assert rel(pp[1], ls[1]) < 1e-5
    for a, b in zip(pp[:1] + pp[2:], ls[:1] + ls[2:]):
        assert torch.equal(a, b)


@pytest.mark.parametrize("M,N,K", [(20000, 64, 256), (5001, 128, 512)])
def test_pingpong_fused_bn_backward_sums_match_lockstep(M, N, K, schedule):
    ops = _ops()
    g = torch.Generator().manual_seed(M + N)
    A = (torch.randn(M, K, generator=g) * 0.5).bfloat16().cuda()
    Bt = (torch.randn(K, N, generator=g) * 0.1).bfloat16().cuda()
    y = (torch.randn(M, N, generator=g) * 1.5).bfloat16().cuda()
    mean = torch.randn(N, generator=g) * 0.5
    invstd = torch.rand(N, generator=g) + 0.5
    sc = (torch.rand(N, generator=g) + 0.5) * invstd
    bnp = torch.stack([mean, invstd, sc, torch.randn(N, generator=g) * 0.3 - mean * sc]).contiguous().cuda()
    R = torch.randn(M, N, generator=g).bfloat16().cuda()

    def run(tile_n):
        D = torch.empty(M, N, dtype=BF16, device="cuda")
        sums = torch.zeros(2, N, device="cuda")
        ops.gemm(A, Bt, D, M, N, K, b_mn=1, residual=R, bnr=(y, bnp, sums, None), tile_n=tile_n)
        return D, sums

    (dp, sp), (dl, sl) = _both(run)
    assert torch.equal(dp, dl)
    dz = dp.double() * ((y.float() * bnp[2] + bnp[3]) > 0).double()
    xhat = (y.double() - bnp[0].double()) * bnp[1].double()
    assert rel(sp[0], dz.sum(0)) < 1e-4 and rel(sp[1], (dz * xhat).sum(0)) < 1e-4
    assert rel(sp, sl) < 1e-5


@pytest.mark.parametrize("NI,H,W,C,Cout", [(8, 56, 56, 64, 64), (6, 28, 28, 128, 128)])
def test_pingpong_implicit_conv_matches_lockstep(NI, H, W, C, Cout, schedule):
    ops = _ops()
    g = torch.Generator().manual_seed(H + C)
    x = (torch.randn(NI, H, W, C, generator=g) * 0.5).bfloat16().cuda()
    wt = (torch.randn(Cout, 3, 3, C, generator=g) * 0.1).bfloat16().cuda().reshape(Cout, 9 * C).contiguous()
    M, K = NI * H * W, 9 * C

    def run(tile_n):
        D = torch.empty(M, Cout, dtype=BF16, device="cuda")
        st = torch.zeros(2, Cout, device="cuda")
        ops.gemm(x, wt, D, M, Cout, K, lda=C, stats=st, conv=(NI, H, W, C), conv_mode=1, tile_n=tile_n)
        return D, st

    (dp, sp), (dl, sl) = _both(run)
    ref = torch.nn.functional.conv2d(x.permute(0, 3, 1, 2).float(),
                                     wt.reshape(Cout, 3, 3, C).permute(0, 3, 1, 2).float(), padding=1)
    assert rel(dp, ref.permute(0, 2, 3, 1).reshape(M, Cout)) < 4e-3
    assert torch.equal(dp, dl)
    assert rel(sp, sl) < 1e-5
