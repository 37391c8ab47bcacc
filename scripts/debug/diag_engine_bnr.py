"""Engine-level check of every fused BN-backward reduction: after each GEMM with bnr=..., run the stand-alone
vtx_bn_bwd_reduce over the same gradient tensor and compare the sums."""
import os, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import virtex_oracle as O
from test_gpu_parity import build_model
from virtex_b200 import engine as E, ops

spec = O.Spec(hidden=128, layers=1, heads=2, ffn=256)
state = O.synth_state(spec, 5, bn3_gain=0.25)
model = build_model(spec, state)
B = int(sys.argv[1]) if len(sys.argv) > 1 else 6
batch = O.synth_batch(B, seed=3)
eng = model.engine
model.train()
orig_gemm = E.gemm
pending = {}


def rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def checked_gemm(A, Bm, D, M, N, K, **kw):
    orig_gemm(A, Bm, D, M, N, K, **kw)
    bnr = kw.get("bnr")
    if bnr is None:
        return
    y, bnp, sums, mbits = bnr[:4]
    key = sums.data_ptr()
    n = pending.get(key, 0) + 1
    pending[key] = n
    if kw.get("out_view") is not None and n < 4:
        return  # the four parity classes of a strided dgrad fill D together
    torch.cuda.synchronize()
    Mfull = D.shape[0]
    ref = torch.zeros(2, N, device="cuda")
    ops.call("vtx_bn_bwd_reduce", D.data_ptr(), ops._p(mbits), y.data_ptr(), bnp.data_ptr(), 0, 0, ref.data_ptr(), 0, Mfull, N,
             int(mbits is None), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    r0, r1 = rel(sums[:N], ref[0]), rel(sums[N:2 * N], ref[1])
    flag = "" if max(r0, r1) < 1e-4 else "   <<<<<< MISMATCH"
    print(f"bnr M={M} N={N} K={K} mode={kw.get('conv_mode', 0)} view={kw.get('out_view') is not None} mask={'bits' if mbits is not None else 'y'} "
          f"res={kw.get('residual') is not None}: rel sum_dz {r0:.2e} sum_dz_xhat {r1:.2e}{flag}", flush=True)
    if flag:
        d = (sums.view(2, N) - ref).abs()
        bad = (d[1] > 1e-3 * ref[1].abs().max()).nonzero().flatten().tolist()
        print("      bad columns:", bad[:32], "of", len(bad))


E.gemm = checked_gemm
eng.fuse_bn_reduce, eng.fuse_bn3_min_rows = True, 0
for dynamic in (False, True):
    ops.set_dynamic_gemm_schedule(dynamic)
    print(f"=== batch {B}, {'dynamic' if dynamic else 'static'} tile schedule")
    pending.clear()
    feat, h, w = eng.backbone_forward(batch["image"].cuda(), training=True)
    dfeat = (torch.randn(feat.shape, generator=torch.Generator().manual_seed(0)) * 0.01).bfloat16().cuda()
    eng.arena.grads.zero_()
    eng.backbone_backward(dfeat)
    torch.cuda.synchronize()
