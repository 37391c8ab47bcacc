"""Developer check of the wgmma GEMM against torch on the GPU."""
import ctypes
import sys
import time

import torch

sys.path.insert(0, ".")
from virtex_b200 import lib as L  # noqa: E402

lib = L.load()
dev = torch.device("cuda:0")
torch.manual_seed(0)


def gemm(A, B, M, N, K, a_mn=0, b_mn=0, out_f32=False, bias=None, act=0, residual=None, stats=None, atomic=False,
         split_k=1, tile_n=0, D=None, conv=None, conv_mode=0):
    if D is None:
        D = torch.full((M, N), float("nan"), device=dev, dtype=torch.float32 if out_f32 else torch.bfloat16)
    g = L.VtxGemm()
    g.A, g.B, g.D = A.data_ptr(), B.data_ptr(), D.data_ptr()
    g.bias = L.ptr(bias)
    g.residual = L.ptr(residual)
    g.stats = L.ptr(stats)
    g.lda = A.stride(0) if conv_mode == 0 else A.shape[-1]
    g.ldb = B.stride(0) if conv_mode != 2 else B.shape[-1]
    g.ldd = D.stride(0)
    g.ldr = residual.stride(0) if residual is not None else 0
    g.M, g.N, g.K = M, N, K
    g.a_mn, g.b_mn = a_mn, b_mn
    g.out_f32, g.atomic, g.act, g.split_k, g.tile_n = int(out_f32), int(atomic), act, split_k, tile_n
    g.alpha = 1.0
    if conv is not None:
        g.conv_n, g.conv_h, g.conv_w, g.conv_c = conv
    g.conv_mode = conv_mode
    L.check(lib.vtx_gemm(ctypes.byref(g), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)), "vtx_gemm")
    return D


def rel(a, b):
    return ((a.float() - b.float()).norm() / (b.float().norm() + 1e-12)).item()


ok = True


def report(name, err, tol=1e-2):
    global ok
    good = err < tol
    ok &= good
    print(f"{'PASS' if good else 'FAIL'} {name}: rel err {err:.3e}", flush=True)


def bf(*shape):
    return (torch.randn(*shape, device=dev) * 0.5).to(torch.bfloat16)


# ---- 1. plain K-major x K-major
for (M, N, K) in [(128, 64, 64), (256, 256, 128), (300, 200, 192), (7680, 1024, 1024), (98, 10000, 1024),
                  (1024, 64, 160)]:
    A, B = bf(M, K), bf(N, K)
    D = gemm(A, B, M, N, K)
    torch.cuda.synchronize()
    report(f"TN M{M} N{N} K{K}", rel(D, A.float() @ B.float().t()))

# ---- 2. epilogues
M, N, K = 512, 384, 256
A, B = bf(M, K), bf(N, K)
bias = torch.randn(N, device=dev)
res = bf(M, N)
ref = A.float() @ B.float().t()
D = gemm(A, B, M, N, K, bias=bias, act=2)
report("bias+gelu", rel(D, torch.nn.functional.gelu(ref + bias)))
D = gemm(A, B, M, N, K, residual=res, act=1)
report("residual+relu", rel(D, torch.relu(ref + res.float())))
stats = torch.zeros(2, N, device=dev)
D = gemm(A, B, M, N, K, out_f32=True)
report("f32 out", rel(D, ref), 1e-5)
D = gemm(A, B, M, N, K, stats=stats)
rb = D.float()
report("stats sum", rel(stats[0], rb.sum(0)), 1e-4)
report("stats sumsq", rel(stats[1], (rb * rb).sum(0)), 1e-4)
for bn_ in (64, 128, 256):
    D = gemm(A, B, M, N, K, bias=bias, tile_n=bn_)
    report(f"tile_n {bn_}", rel(D, ref + bias))
D = gemm(A[:, :96].contiguous(), B[:, :96].contiguous(), M, 200, 96, bias=bias[:200])
report("N tail 200, K 96", rel(D, (A[:, :96].float() @ B[:200, :96].float().t()) + bias[:200]))

# ---- 3. dgrad: B MN-major ([K, N] storage):  dX[M,Kout] = dY[M,Nred] @ W[Nred,Kout]
M, Nred, Kout = 640, 320, 448
dY, W = bf(M, Nred), bf(Nred, Kout)
D = gemm(dY, W, M, Kout, Nred, b_mn=1)
report("dgrad (B MN-major)", rel(D, dY.float() @ W.float()))

# ---- 4. wgrad: both MN-major, split-K + atomics:  dW[N,K] = dY[M,N]^T @ X[M,K]
Mred, N, K = 4096 + 37, 192, 320
dY, X = bf(Mred, N), bf(Mred, K)
out = torch.zeros(N, K, device=dev)
gemm(dY, X, N, K, Mred, a_mn=1, b_mn=1, out_f32=True, atomic=True, split_k=8, D=out)
report("wgrad (A,B MN-major, split-K)", rel(out, dY.float().t() @ X.float()), 1e-4)

# ---- 5. implicit 3x3 conv fprop / wgrad
for (NI, H, W_, C, Co) in [(4, 56, 56, 64, 64), (3, 20, 20, 64, 64), (5, 7, 7, 64, 64), (8, 28, 28, 128, 128), (33, 14, 14, 256, 256), (130, 7, 7, 512, 512),
                           (2, 14, 14, 64, 128)]:
    x = bf(NI, H, W_, C)
    w = (torch.randn(Co, 3, 3, C, device=dev) * 0.05).to(torch.bfloat16)
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), padding=1)
    ref = ref.permute(0, 2, 3, 1).reshape(-1, Co)
    D = gemm(x, w.reshape(Co, 9 * C), NI * H * W_, Co, 9 * C, conv=(NI, H, W_, C), conv_mode=1)
    report(f"conv3x3 fprop N{NI} {H}x{W_} C{C}->{Co}", rel(D, ref))
    st = torch.zeros(2, Co, device=dev)
    D = gemm(x, w.reshape(Co, 9 * C), NI * H * W_, Co, 9 * C, conv=(NI, H, W_, C), conv_mode=1, stats=st)
    report(f"   + stats sum/sumsq", max(rel(st[0], D.float().sum(0)), rel(st[1], (D.float() ** 2).sum(0))), 1e-3)
    dy = bf(NI, H, W_, Co)
    out = torch.zeros(Co, 9 * C, device=dev)
    gemm(dy, x, Co, 9 * C, NI * H * W_, out_f32=True, atomic=True, split_k=4, D=out, conv=(NI, H, W_, C),
         conv_mode=2)
    xr = x.float().permute(0, 3, 1, 2).requires_grad_(False)
    wref = torch.nn.grad.conv2d_weight(xr, (Co, C, 3, 3), dy.float().permute(0, 3, 1, 2), padding=1)
    report(f"conv3x3 wgrad N{NI} {H}x{W_}", rel(out, wref.permute(0, 2, 3, 1).reshape(Co, 9 * C)), 1e-4)
    if C == 64 and Co == 64:
        out_t = torch.zeros(9 * C, Co, device=dev)
        gemm(dy, x, 9 * C, Co, NI * H * W_, out_f32=True, atomic=True, D=out_t, conv=(NI, H, W_, C), conv_mode=4)
        report(f"   transposed wgrad (mode 4) N{NI} {H}x{W_}", rel(out_t, wref.permute(2, 3, 1, 0).reshape(9 * C, Co)), 1e-4)

# ---- 6. timing of a few representative shapes
def bench(name, fn, flops, iters=20):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    print(f"TIME {name}: {ms*1e3:.1f} us  {flops/ms/1e9:.1f} TFLOP/s", flush=True)


for (M, N, K) in [(7680, 4096, 1024), (7680, 10000, 1024), (12544, 2048, 1024), (802816, 64, 64), (802816, 256, 64),
                  (200704, 512, 128), (50176, 1024, 256), (8192, 8192, 8192)]:
    A, B = bf(M, K), bf(N, K)
    D = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    bench(f"vtx TN {M}x{N}x{K}", lambda: gemm(A, B, M, N, K, D=D), 2.0 * M * N * K)
    bench(f"torch  {M}x{N}x{K}", lambda: torch.matmul(A, B.t()), 2.0 * M * N * K)
x = bf(256, 56, 56, 64)
w = bf(64, 9 * 64)
D = torch.empty(256 * 56 * 56, 64, device=dev, dtype=torch.bfloat16)
bench("vtx conv3x3 l1", lambda: gemm(x, w, 256 * 3136, 64, 576, D=D, conv=(256, 56, 56, 64), conv_mode=1),
      2.0 * 256 * 3136 * 64 * 576)
x = bf(256, 14, 14, 256)
w = bf(256, 9 * 256)
D = torch.empty(256 * 196, 256, device=dev, dtype=torch.bfloat16)
bench("vtx conv3x3 l3", lambda: gemm(x, w, 256 * 196, 256, 2304, D=D, conv=(256, 14, 14, 256), conv_mode=1),
      2.0 * 256 * 196 * 256 * 2304)
x = bf(256, 56, 56, 64); dy = bf(256, 56, 56, 64)
out = torch.zeros(64, 576, device=dev); out_t = torch.zeros(576, 64, device=dev)
bench("vtx conv3x3 l1 wgrad mode 2", lambda: gemm(dy, x, 64, 576, 256 * 3136, out_f32=True, atomic=True, split_k=49, D=out,
                                                    conv=(256, 56, 56, 64), conv_mode=2), 2.0 * 256 * 3136 * 64 * 576)
bench("vtx conv3x3 l1 wgrad mode 4", lambda: gemm(dy, x, 576, 64, 256 * 3136, out_f32=True, atomic=True, D=out_t,
                                                    conv=(256, 56, 56, 64), conv_mode=4), 2.0 * 256 * 3136 * 64 * 576)
print("ALL OK" if ok else "SOME FAILED")
sys.exit(0 if ok else 1)
