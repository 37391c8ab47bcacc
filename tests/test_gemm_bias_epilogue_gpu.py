"""The bias epilogue of the GEMM (csrc/gemm_tc.cu) rounds fp32(acc + bias) to bf16, bit for bit.

A bf16 GEMM with `bias=` and, on the same operands with the same tile width, an fp32-output GEMM without one must
satisfy D_bias == (D_f32 + bias).bfloat16() exactly: every output element keeps its K order in both schedules, and the
bias is added to the fp32 accumulator before the one rounding to bf16.  Covers every tile width (64 / 128 wide bf16
tiles run the ping-pong schedule, 192 / 256 lockstep; fp32 outputs always run lockstep), ragged last row tiles, N not a
multiple of the tile width, a bias that is a slice of a larger vector, and biases that take the general epilogue loop:
one not 8-byte aligned and one of odd length."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _bias_gemm_vs_f32(M, N, K, tile_n, bias_offset=0, ldd=None):
    _need_cuda()
    from virtex_b200 import ops
    g = torch.Generator().manual_seed(M * 7 + N * 3 + K + tile_n + bias_offset)
    A = (torch.randn(M, K, generator=g) * 0.5).bfloat16().cuda()
    B = (torch.randn(N, K, generator=g) * 0.1).bfloat16().cuda()
    full = torch.randn(N + bias_offset + 3, generator=g).cuda()
    bias = full[bias_offset:bias_offset + N]
    ldd = N if ldd is None else ldd
    D = torch.full((M, ldd), float("nan"), dtype=torch.bfloat16, device="cuda")
    D32 = torch.full((M, ldd), float("nan"), device="cuda")
    ops.gemm(A, B, D, M, N, K, ldd=ldd, bias=bias, tile_n=tile_n)
    ops.gemm(A, B, D32, M, N, K, ldd=ldd, tile_n=tile_n)
    torch.cuda.synchronize()
    D, D32 = D[:, :N], D32[:, :N]
    ref = (D32 + bias).bfloat16()
    assert torch.equal(D, ref), f"{(D.float() != ref.float()).sum().item()} elements differ"
    # and the GEMM itself is right
    prod = A.float() @ B.float().t()
    assert ((D32 - prod).norm() / prod.norm()).item() < 1e-5


@pytest.mark.parametrize("M,N,K,tile_n", [
    (1000, 256, 256, 64),       # ping-pong, ragged last row tile
    (1000, 256, 320, 128),      # ping-pong
    (1000, 384, 256, 192),      # lockstep
    (1000, 512, 256, 256),      # lockstep
    (777, 200, 192, 64),        # last column tile 8 wide
    (777, 1000, 128, 128),      # last column tile 104 wide
    (1025, 1000, 128, 192),     # last column tile 40 wide
    (7680, 10000, 1024, 256),   # the vocabulary projection: last column tile 16 wide
])
def test_bias_epilogue_matches_f32_plus_bias(M, N, K, tile_n):
    _bias_gemm_vs_f32(M, N, K, tile_n)


@pytest.mark.parametrize("tile_n", [64, 256])
def test_bias_slice_at_an_offset(tile_n):
    # like the cross-attention projections' bias[H:]: 8-byte aligned, so the compact loop runs
    _bias_gemm_vs_f32(600, 320, 192, tile_n, bias_offset=320)


@pytest.mark.parametrize("tile_n", [64, 128, 256])
def test_bias_not_8_byte_aligned_takes_the_general_loop(tile_n):
    _bias_gemm_vs_f32(600, 320, 192, tile_n, bias_offset=1)


@pytest.mark.parametrize("tile_n", [64, 256])
def test_bias_of_odd_length_takes_the_general_loop(tile_n):
    _bias_gemm_vs_f32(600, 301, 192, tile_n, ldd=304)
