"""The masked-residual 1x1 dgrads of the identity bottlenecks, dx = dy1 . W1 + m3 (.) dOut (optionally with the previous
block's BN-backward sums over dx), run on a streaming kernel of their own (csrc/gemm_resid.cu) when K <= 256 and the
tile width is left to vtx_gemm.  Covers the four batch-256 ResNet-50 shapes and ragged ones (row counts that are no
multiple of any tile, every N of the stages), with and without the sums:
  * integer operands: D and the sums equal the float64 reference bit for bit;
  * real data: D within the VtxGemm bound and equal, bit for bit, to the persistent kernel (tile_n = 256 keeps that
    route), the sums within the reference's bound;
  * the calls really take the streaming kernel (kernel names in a profiler trace), and the others the persistent one."""
import pytest
import torch

from tests import gemm_reference as G

pytestmark = pytest.mark.gpu

BF16 = torch.bfloat16

SHAPES = [
    (802816, 256, 64),    # layer1, batch 256
    (200704, 512, 128),   # layer2
    (50176, 1024, 256),   # layer3: 64-column blocks
    (12544, 2048, 512),   # layer4 (K > 256: the persistent kernel)
    (1000, 256, 64),      # ragged: 15.6 row tiles
    (30011, 512, 128),
    (4097, 1024, 64),
    (777, 2048, 128),
    (3001, 1024, 256),
]


def _ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from virtex_b200 import ops
    return ops


def _streams(K):
    return K <= 256


def _call(M, N, K, bnr, seed, tile_n=0):
    g = torch.Generator().manual_seed(seed)
    dy1 = (torch.randn(M, K, generator=g) * 0.5).bfloat16().cuda()
    w1 = (torch.randn(K, N, generator=g) * 0.1).bfloat16().cuda()
    dout = torch.randn(M, N, generator=g).bfloat16().cuda()
    m3 = torch.randint(0, 256, (M, N // 8), generator=g, dtype=torch.uint8).cuda()
    D = torch.empty(M, N, dtype=BF16, device="cuda")
    b = None
    if bnr:
        y = (torch.randn(M, N, generator=g) * 1.5).bfloat16().cuda()
        mean = torch.randn(N, generator=g) * 0.5
        invstd = torch.rand(N, generator=g) + 0.5
        sc = (torch.rand(N, generator=g) + 0.5) * invstd
        bnp = torch.stack([mean, invstd, sc, torch.randn(N, generator=g) * 0.3 - mean * sc]).contiguous().cuda()
        mb = torch.randint(0, 256, (M, N // 8), generator=g, dtype=torch.uint8).cuda()
        b = (y, bnp, torch.zeros(2, N, device="cuda"), mb)
    return G.Call(dy1, w1, D, M, N, K, b_mn=1, residual=dout, residual_mask=m3, bnr=b, tile_n=tile_n)


def _run(ops, c):
    ops.gemm(c.A, c.B, c.D, c.M, c.N, c.K, **c.kwargs())


@pytest.mark.parametrize("bnr", [False, True], ids=["plain", "bnr"])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_real_data_matches_reference_and_persistent_route(M, N, K, bnr):
    ops = _ops()
    sms = ops.num_sms()
    c = _call(M, N, K, bnr, M + N + K)
    before = G.snapshot(c)
    _run(ops, c)
    torch.cuda.synchronize()
    G.check(c, before, c, sms, integer=False)
    ref = G.Call(c.A, c.B, torch.empty_like(c.D), M, N, K, b_mn=1, residual=c.residual, residual_mask=c.residual_mask,
                 bnr=None if not bnr else (c.bnr_y, c.bnr_bnp, torch.zeros_like(c.bnr_sums), c.bnr_mask), tile_n=256)
    _run(ops, ref)
    torch.cuda.synchronize()
    assert torch.equal(c.D, ref.D)


@pytest.mark.parametrize("bnr", [False, True], ids=["plain", "bnr"])
@pytest.mark.parametrize("M,N,K", SHAPES)
def test_integer_operands_bit_exact(M, N, K, bnr):
    ops = _ops()
    c = _call(M, N, K, bnr, 7 * M + N)
    G.integer_fill(c, torch.Generator(device="cuda").manual_seed(M + K))
    before = G.snapshot(c)
    _run(ops, c)
    torch.cuda.synchronize()
    G.check(c, before, c, ops.num_sms(), integer=True)


@pytest.mark.parametrize("M,N,K", [(30011, 512, 128), (1000, 256, 64), (3001, 1024, 256), (2000, 2048, 512)])
def test_route_taken(M, N, K):
    """With and without the sums, tile_n = 0 runs the streaming kernel where it serves the call (K <= 256) and the
    persistent one otherwise; tile_n = 256 always runs the persistent one.  One profiler session over all four calls."""
    ops = _ops()
    calls = [_call(M, N, K, bnr, 3, tile_n=tile_n) for tile_n in (0, 256) for bnr in (False, True)]
    for c in calls:
        _run(ops, c)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA], acc_events=True) as prof:
        for c in calls:
            _run(ops, c)
            torch.cuda.synchronize()
    names = [e.name for e in prof.events() if "_kernel" in e.name]
    streaming = sum("resid_dgrad_kernel" in k for k in names)
    persistent = sum("gemm_wgmma_kernel" in k for k in names)
    want_streaming = 2 if _streams(K) else 0
    assert (streaming, persistent) == (want_streaming, 4 - want_streaming), names
