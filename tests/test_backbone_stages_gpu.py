"""The engine's backbone forward, backward and eval forward replayed stage by stage against the float64 references of
tests/backbone_stages.py, element by element, from the engine's own inputs of each stage.

Every reference is a function of tensors the engine produced (its block inputs, conv outputs, BN statistics, ReLU bit
masks, incoming gradients) and of the modules' parameters rounded to bf16 by torch, never of the engine's bf16 mirror or
packed weight layouts.  So no ReLU mask can flip between the engine and the reference, and each stage is held to the
bound of a single launch: which packed weight slice a launch reads, the parity-class sub-grids of the stride-2 dgrads,
which block's bit mask and bnp a fused reduction reads, where the downsample gradient lands and which arena slot receives
each gradient are all checked at once.  Bottleneck blocks (ResNet-50 / 101, Wide ResNet-50-2) and basic blocks
(ResNet-18 / 34: conv1 3x3 strided, conv2 3x3, both weight gradients through the fp32 scratch and its unpack jobs; the
identity blocks' conv1 dgrad adding the shortcut gradient under the block's bit mask and accumulating the previous
block's bn2 sums under that block's mask) run through the same harness, dispatched on the tape's `basic` flag.

Capture, without changing the engine: `eng._bn_fwd` / `eng._bn_act_fwd` / `eng._bn_bwd` are wrapped as instance
attributes (statistics and running buffers before, bnp after; dA before, dy after, the arena's BN gradients before and
after); `engine.gemm` and `engine.call` are patched to record the sequential depth of every fused BN reduction and
weight-gradient launch, to read the eval forward's shared `inf.*` buffers and the max-pool gradient's input, which are
identified by their workspace name.  The forward tape stays intact until the next forward and is read directly.  Each
stage is checked as soon as its inputs exist; only the float64 weight-gradient references are kept to the end.

Bounds (tests/backbone_stages.py): bit equality for the BN finalize (mean, scale, shift from the device's invstd,
running buffers), BN apply, ReLU bit masks and max pool; 4 fp32 ulp for rsqrtf; the GEMM bound of
tests/gemm_reference.py for conv outputs, dgrads, the outgoing gradient and weight gradients; the BN-backward dy and
sums bounds of tests/test_backbone_kernels_gpu.py for dy, dgamma and dbeta.

Power: each case prints one row per stage kind (run with -s): the worst err / bound and, for bf16 stages, the median of
bound / |ref| (weight gradients: the largest bound over the RMS of the reference), under a title that names the deepest
weight-gradient launch.  Each case asserts that the bounds are informative: median bound / |ref| <= BF16_INFO for every
bf16 stage and max bound <= its case's limit * RMS for every weight gradient.  Set from runs on an H100 SXM (80 GB,
default 700 W power limit); the bottleneck cases:
  * bf16 stages: median bound / |ref| at most 0.0139 (the strided downsample of resnet101 at B = 1; about 1 bf16 ulp
    plus the accumulation term), BF16_INFO = 2^-6.  The worst err / bound of any bf16 stage was 0.5: half an ulp, the
    final rounding;
  * weight gradients at B <= 3: max bound / RMS at most 0.0070 (the stem at B = 1), WGRAD_INFO = 2^-7;
  * weight gradients at B = 256: the reductions run over up to 3.2 M rows, and the worst-case bound grows with
    sum |terms|, about sqrt(rows) times |ref|: max bound / RMS 0.57 (stem), worst err / bound 0.027.  That case is held
    to WGRAD_INFO_B256 = 1, enough to catch a missing image tile, a wrong arena slot or a wrong operand; the small
    cases carry the tight check of the same launches.
The basic-block cases (ResNet-18 / 34) and the bottleneck at a 288 crop, each case 1-2.5 s on the same machine (the
figures move in the third digit between runs):
  * bf16 stages: median bound / |ref| at most 0.0112 (the identity blocks' dx: the shortcut term added to the
    bf16-rounded conv1 dgrad tile, two ulps) and 0.0127 for resnet50 at 288 (its stride-1 transition dx); worst
    err / bound 0.5 in every case;
  * weight gradients, max bound / RMS: 0.0023 (r18-b2-224), 0.0026 (r34-b2-224-fused-bn2-dynamic), 0.0050
    (r18-b2-320), 0.0044 (r50-b2-288), all under WGRAD_INFO; 0.67 at B = 256 (r34-b256-224-dynamic, basic conv1),
    worst err / bound 0.027, under WGRAD_INFO_B256;
  * r18-b3-199x230-fused: 0.0118 (layer2.0's strided conv1; its downsample 0.0093).  Not looser data: the launch is
    deeper.  Its wgrad reads the 25 x 29 output grid in boxes of 64 positions, and no power-of-two w x h box tiles a
    29-wide grid without waste, so the kernel takes 1 x 1 x 64 boxes (one position of up to 64 images; three here):
    725 k-blocks in 8 splits, L = 4 * 91 + 8 = 372 against 42 for the same conv at 224 x 224 at B = 2.  The bound
    scales with L + 2; that case is held to WGRAD_INFO_DEEP = 2^-6, and its bound stays 85 times below the RMS.
    resnet50 at the same extents stays under WGRAD_INFO (0.0070, its downsample) and keeps that limit.
"""
import pytest
import torch

from oracle import virtex_oracle as O
from tests import backbone_replica as R
from tests import backbone_stages as S
from tests import gemm_reference as G
from tests.helpers import build_model

pytestmark = pytest.mark.gpu

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
BF16_INFO = 2.0 ** -6
WGRAD_INFO = 2.0 ** -7
WGRAD_INFO_DEEP = 2.0 ** -6
WGRAD_INFO_B256 = 1.0


def _d(t):
    return t.to(F64)


class _Row:
    def __init__(self, info):
        self.info, self.n, self.worst, self.power = info, 0, 0.0, []


class Replay:
    """Wraps one engine's backbone and checks every stage it runs."""

    def __init__(self, eng, image, sub_every=16):
        self.eng, self.image = eng, image
        self.B = B = image.shape[0]
        self.sms = eng_sms()
        sub = sorted({0, B - 1} | set(range(0, B, sub_every)))
        self.sub = None if len(sub) == B else torch.tensor(sub, device="cuda")
        self.P = {"visual." + n: p for n, p in eng.visual.named_parameters()}
        self.recs = {}
        self.rows = {}
        self.wref = {}          # weight name -> (float64 reference, mag)
        self.wdepth = {}        # D pointer of an accumulating GEMM -> its sequential depth
        self.bnr_depth = {}     # BN-sums pointer -> depth of the fused reductions into it
        self.fwd = {}           # BN name -> (stats, running mean, running var) before its finalize
        self.pending = None     # (block name, dx reference, bound): checked when the next stage reads dx
        self.state = None       # float64 gradients of the block in flight, for its next stages
        self.dpool = None
        self.eval_state = None

    # ------------------------------------------------------------------------------------------------ reporting
    def check(self, kind, got, ref, bound=None, info="median"):
        got = _d(got)
        assert got.shape == ref.shape, (kind, tuple(got.shape), tuple(ref.shape))
        row = self.rows.setdefault(kind, _Row("exact" if bound is None else info))
        row.n += 1
        if bound is None:
            bad = got != ref
            assert not bool(bad.any()), f"{kind}: {int(bad.sum())} of {bad.numel()} elements differ (bit-exact stage)"
            return
        err = (got - ref).abs()
        ratio = err / bound
        worst = float(ratio.max())
        bad = ~(ratio <= 1.0)
        assert not bool(bad.any()), (f"{kind}: {int(bad.sum())} of {bad.numel()} beyond the bound; worst err/bound "
                                     f"{worst:.3g} at {tuple(bad.nonzero()[0].tolist())}")
        row.worst = max(row.worst, worst)
        if info == "median":
            nz = ref != 0
            q = (bound[nz] / ref[nz].abs()).flatten()
            q = q[::max(1, q.numel() // (1 << 22))]
            row.power.append(float(q.median()))
        elif info == "wgrad":
            row.power.append(float(bound.max() / ref.pow(2).mean().sqrt()))

    def report(self, title, wgrad_info):
        print(f"\n{title}\n{'stage':<22} {'checks':>6} {'err/bound':>10} {'power':>10}")
        for kind, r in sorted(self.rows.items()):
            p = "exact" if r.info == "exact" else ("-" if not r.power else f"{max(r.power):.3g}")
            print(f"{kind:<22} {r.n:>6} {r.worst:>10.3g} {p:>10}")
        for kind, r in self.rows.items():
            if r.info == "median" and r.power:
                assert max(r.power) <= BF16_INFO, (kind, "median bound / |ref|", max(r.power))
            elif r.info == "wgrad":
                assert max(r.power) <= wgrad_info, (kind, "max bound / RMS", max(r.power))

    # ------------------------------------------------------------------------------------------------ helpers
    def w(self, name):
        return _d(self.P[name].detach().to(BF16))

    def rows4(self, t, H, W, full=False):
        """[B*H*W, C] device rows -> [n, H, W, C] float64 of the checked images (all of them when full)."""
        v = t.reshape(self.B, H, W, -1)
        if self.sub is not None and not full:
            v = v[self.sub]
        return _d(v)

    def img(self, full=False):
        x = self.image.permute(0, 2, 3, 1).to(BF16)
        if self.sub is not None and not full:
            x = x[self.sub]
        return _d(x)

    def bn_vec(self, bn):
        return _d(self.P[bn + ".weight"].detach()), _d(self.P[bn + ".bias"].detach())

    # ------------------------------------------------------------------------------------------------ install
    def install(self, monkeypatch):
        from virtex_b200 import engine as E
        eng = self
        e = self.eng
        orig_gemm, orig_call = E.gemm, E.call
        orig_fwd, orig_act, orig_bwd = e._bn_fwd, e._bn_act_fwd, e._bn_bwd

        def before_fwd(bn_name, training, stats):
            if training:
                eng.fwd[bn_name] = (_d(stats.view(2, -1)), _d(e.buffers[bn_name + ".running_mean"]),
                                    _d(e.buffers[bn_name + ".running_var"]))

        def bn_fwd(y, bn_name, M, C, training, stats, key="bnp:"):
            before_fwd(bn_name, training, stats)
            return orig_fwd(y, bn_name, M, C, training, stats, key=key)

        def bn_act_fwd(y, bn_name, M, C, training, stats, out, **kw):
            before_fwd(bn_name, training, stats)
            return orig_act(y, bn_name, M, C, training, stats, out, **kw)

        def bn_bwd(dA, a, y, bnp, bn_name, M, C, dy, two=None, dz_out=None, mask_from_y=0, sums=None):
            names = [bn_name] + ([two[2]] if two is not None else [])
            for n in names:
                assert not bool(e.G(n + ".weight").any()) and not bool(e.G(n + ".bias").any()), n
            dA0 = dA.clone()
            depth = eng.bnr_depth.pop(sums.data_ptr()) if sums is not None else \
                R.reduce_depth(eng.sms, M, C, two is not None)
            orig_bwd(dA, a, y, bnp, bn_name, M, C, dy, two=two, dz_out=dz_out, mask_from_y=mask_from_y, sums=sums)
            dys = [dy.clone()] + ([two[3].clone()] if two is not None else [])
            eng.on_bn_bwd(bn_name, dA0, dys, two is not None, depth)

        def gemm(A, B, D, M, N, K, **kw):
            orig_gemm(A, B, D, M, N, K, **kw)
            bnr = kw.get("bnr")
            if bnr is not None or kw.get("atomic"):
                c = G.Call(A, B, D, M, N, K, **kw)
                if bnr is not None:
                    k = bnr[2].data_ptr()
                    eng.bnr_depth[k] = eng.bnr_depth.get(k, 0) + -(-M // 8) + 32 + G.plan(c, eng.sms)["m_tiles"]
                if kw.get("atomic"):
                    eng.wdepth[D.data_ptr()] = max(eng.wdepth.get(D.data_ptr(), 0), G.seq_depth(c, eng.sms))
            if eng.eval_state is not None:
                eng.on_eval_gemm(A, D, kw)

        def call(name, *args):
            if name == "vtx_maxpool_bwd":
                eng.on_maxpool_bwd(args[0])
            return orig_call(name, *args)

        monkeypatch.setattr(e, "_bn_fwd", bn_fwd)
        monkeypatch.setattr(e, "_bn_act_fwd", bn_act_fwd)
        monkeypatch.setattr(e, "_bn_bwd", bn_bwd)
        monkeypatch.setattr(E, "gemm", gemm)
        monkeypatch.setattr(E, "call", call)

    # ------------------------------------------------------------------------------------------------ forward
    def check_bnp(self, bn, bnp, M):
        stats, rm0, rv0 = self.fwd.pop(bn)
        gamma, beta = self.bn_vec(bn)
        mean, inv, rm, rv = S.bn_train(stats, M, gamma, beta, rm0, rv0)
        self.check("bn finalize", bnp[0], mean)
        self.check("bn invstd", bnp[1], inv, 4 * inv * 2.0 ** -23, info="-")
        sc, sh = R.bn_scale_shift(gamma, beta, mean, _d(bnp[1]))
        self.check("bn finalize", bnp[2], sc)
        self.check("bn finalize", bnp[3], sh)
        self.check("bn running buffers", self.eng.buffers[bn + ".running_mean"], rm)
        self.check("bn running buffers", self.eng.buffers[bn + ".running_var"], rv)
        return _d(bnp)

    def check_forward(self):
        tape = self.eng._tape
        st = tape["stem"]
        Ho, Wo, Hp, Wp = st["Ho"], st["Wo"], st["Hp"], st["Wp"]
        w0 = self.w("visual.cnn.conv1.weight")
        ref, mag = S.conv(self.img(), w0, 2, 3)
        K0 = 256 if st["s2d"] is not None else 160
        self.check("fwd y0 stem", self.rows4(st["y"], Ho, Wo), ref, S.bf16_bound(ref, S.gemm_err(mag, K0)))
        bnp0 = self.check_bnp("visual.cnn.bn1", st["bnp"], st["M"])
        y0 = self.rows4(st["y"], Ho, Wo)
        act = S.bn_apply(y0.reshape(-1, 64), bnp0)[1].view(y0.shape)
        pool, idx = S.maxpool(act)
        self.check("fwd maxpool", self.rows4(tape["blocks"][0]["x"], Hp, Wp), pool)
        got_idx = st["idx"].view(self.B, Hp, Wp, 64)
        got_idx = got_idx if self.sub is None else got_idx[self.sub]
        assert torch.equal(got_idx, idx), "max-pool slots"
        for rec in tape["blocks"]:
            self.check_block_forward(rec)
        assert not self.fwd, sorted(self.fwd)

    def check_block_forward(self, rec):
        name, s = rec["name"], rec["stride"]
        self.recs[name] = rec
        Hi, Wi, Ho, Wo = rec["Hin"], rec["Win"], rec["Hout"], rec["Wout"]
        x = self.rows4(rec["x"], Hi, Wi)

        def conv(kind, inp, wname, stride, pad, got, H, W):
            w = self.w(wname)
            ref, mag = S.conv(inp, w, stride, pad)
            K = w.shape[1] * w.shape[2] * w.shape[3]
            self.check(kind, self.rows4(got, H, W), ref, S.bf16_bound(ref, S.gemm_err(mag, K)))

        def act(kind, y, bnp, got, H, W, **kw):
            yv = self.rows4(y, H, W)
            pre, out = S.bn_apply(yv.reshape(-1, yv.shape[-1]), bnp, **kw)
            self.check(kind, self.rows4(got, H, W), out.view(yv.shape))
            return pre

        if rec["basic"]:
            # conv1 3x3 (stride) -> bn1 + ReLU -> conv2 3x3 -> bn2 + shortcut + ReLU, all at the output extent
            conv(f"fwd y1 basic conv1 s{s}", x, name + ".conv1.weight", s, 1, rec["y1"], Ho, Wo)
            bnp1 = self.check_bnp(name + ".bn1", rec["bnp1"], rec["Mout"])
            act("fwd a1 basic", rec["y1"], bnp1, rec["a1"], Ho, Wo)
            conv("fwd y2 basic conv2", self.rows4(rec["a1"], Ho, Wo), name + ".conv2.weight", 1, 1, rec["y2"], Ho, Wo)
            last = "2"
        else:
            conv("fwd y1 conv1", x, name + ".conv1.weight", 1, 0, rec["y1"], Hi, Wi)
            bnp1 = self.check_bnp(name + ".bn1", rec["bnp1"], rec["Min"])
            act("fwd a1", rec["y1"], bnp1, rec["a1"], Hi, Wi)
            conv(f"fwd y2 conv2 s{s}", self.rows4(rec["a1"], Hi, Wi), name + ".conv2.weight", s, 1, rec["y2"], Ho, Wo)
            bnp2 = self.check_bnp(name + ".bn2", rec["bnp2"], rec["Mout"])
            act("fwd a2", rec["y2"], bnp2, rec["a2"], Ho, Wo)
            conv("fwd y3 conv3", self.rows4(rec["a2"], Ho, Wo), name + ".conv3.weight", 1, 0, rec["y3"], Ho, Wo)
            last = "3"
        if rec["has_ds"]:
            assert s == 1 or rec["xs"] is None  # a stride-2 shortcut reads x in place (no subsampled copy)
            conv(f"fwd yd downsample s{s}", x, name + ".downsample.0.weight", s, 0, rec["yd"], Ho, Wo)
            bnpd = self.check_bnp(name + ".downsample.1", rec["bnpd"], rec["Mout"])
            res = self.rows4(rec["yd"], Ho, Wo)
        else:
            bnpd, res = None, x
        bnpo = self.check_bnp(name + ".bn" + last, rec["bnp" + last], rec["Mout"])
        pre = act("fwd block output" + (" basic" if rec["basic"] else ""), rec["y" + last], bnpo, rec["out"], Ho, Wo,
                  res=res.reshape(-1, res.shape[-1]), bnp_res=bnpd)
        m = rec["m" + last].view(self.B, Ho, Wo, -1)
        m = m if self.sub is None else m[self.sub]
        assert torch.equal(m.reshape(-1, m.shape[-1]), R.pack_mask(pre > 0)), f"{name}: ReLU bit mask m{last}"
        self.rows.setdefault(f"fwd bit mask m{last}", _Row("exact")).n += 1

    # ------------------------------------------------------------------------------------------------ backward
    def bn_stage(self, kind, bn, dA, keep, y, bnp, dy_got, M, H, W, depth):
        """dgamma / dbeta in full (the device sums the dy reference uses), dy on the checked images."""
        e = self.eng
        dgam, dbet = _d(e.G(bn + ".weight")), _d(e.G(bn + ".bias"))
        C = bnp.shape[1]
        dAf = _d(dA).view(M, C)
        yf = y.view(M, C)
        kf = keep.view(M, C) if keep is not None else None
        dz = dAf if kf is None else dAf * kf
        ref, tol = S.bn_sums(dz, yf, bnp, depth)
        del dz
        self.check("bwd dbeta", dbet, ref[0], tol[0], info="-")
        self.check("bwd dgamma", dgam, ref[1], tol[1], info="-")
        sums = torch.stack([dbet, dgam])
        dAs = self.rows4(dA, H, W)
        ks = None if keep is None else (keep.view(self.B, H, W, C) if self.sub is None else
                                        keep.view(self.B, H, W, C)[self.sub])
        _, dy, bound = S.bn_backward(dAs.reshape(-1, C), None if ks is None else ks.reshape(-1, C),
                                     self.rows4(y, H, W).reshape(-1, C), bnp, sums, M)
        self.check(kind, self.rows4(dy_got, H, W), dy.view(dAs.shape), bound.view(dAs.shape))

    def wgrad(self, wname, dy, x, k, stride, pad):
        self.wref[wname] = S.conv_wgrad(dy, x, k, k, stride, pad)

    def check_pending(self, dx):
        name, ref, bound = self.pending
        rec = self.recs[name]
        self.check("bwd dx " + ("basic " if rec["basic"] else "") +
                   ("identity" if not rec["has_ds"] else f"transition s{rec['stride']}"),
                   self.rows4(dx, rec["Hin"], rec["Win"]), ref, bound)
        self.pending = None

    def downsample_bwd(self, rec, dA, keep, dy_got, depth):
        """The downsample BN's share of a two-branch block-output BN backward, and its conv's weight gradient."""
        name, Ho, Wo = rec["name"], rec["Hout"], rec["Wout"]
        self.bn_stage("bwd dyd", name + ".downsample.1", dA, keep, rec["yd"], _d(rec["bnpd"]), dy_got, rec["Mout"],
                      Ho, Wo, depth)
        self.wgrad(name + ".downsample.0.weight", self.rows4(dy_got, Ho, Wo, full=True),
                   self.rows4(rec["x"], rec["Hin"], rec["Win"], full=True), 1, rec["stride"], 0)
        return self.rows4(dy_got, Ho, Wo)

    def on_bn_bwd(self, bn_name, dA, dys, two, depth):
        if bn_name == "visual.cnn.bn1":
            return self.on_stem_bwd(dA, dys[0], depth)
        name, which = bn_name.rsplit(".", 1)
        rec = self.recs[name]
        if rec["basic"]:
            return self.on_basic_bn_bwd(rec, which, dA, dys, two, depth)
        Hi, Wi, Ho, Wo, s = rec["Hin"], rec["Win"], rec["Hout"], rec["Wout"], rec["stride"]
        st = self.state = getattr(self, "state", None) if which != "bn3" else {}
        if which == "bn3":
            if self.pending is not None:
                self.check_pending(dA)
            keep = R.unpack_mask(rec["m3"], rec["Cout"])
            self.bn_stage("bwd dy3", bn_name, dA, keep, rec["y3"], _d(rec["bnp3"]), dys[0], rec["Mout"], Ho, Wo,
                          depth)
            full = lambda t, H, W: self.rows4(t, H, W, full=True)  # noqa: E731
            self.wgrad(name + ".conv3.weight", full(dys[0], Ho, Wo), full(rec["a2"], Ho, Wo), 1, 1, 0)
            st["dy3"] = self.rows4(dys[0], Ho, Wo)
            if two:
                st["dyd"] = self.downsample_bwd(rec, dA, keep, dys[1], depth)
            else:
                st["dOut"] = self.rows4(dA, Ho, Wo)
                k = keep.view(self.B, Ho, Wo, -1)
                st["keep3"] = k if self.sub is None else k[self.sub]
        elif which == "bn2":
            ref, mag = S.conv_dgrad(st["dy3"], self.w(name + ".conv3.weight"), 1, 0, Ho, Wo)
            self.check("bwd da2 conv3 dgrad", self.rows4(dA, Ho, Wo), ref,
                       S.bf16_bound(ref, S.gemm_err(mag, rec["Cout"])))
            bnp2 = _d(rec["bnp2"])
            keep = S.relu_keep(_d(rec["y2"]), bnp2)
            self.bn_stage("bwd dy2", bn_name, dA, keep, rec["y2"], bnp2, dys[0], rec["Mout"], Ho, Wo, depth)
            self.wgrad(name + ".conv2.weight", self.rows4(dys[0], Ho, Wo, full=True),
                       self.rows4(rec["a1"], Hi, Wi, full=True), 3, s, 1)
            st["dy2"] = self.rows4(dys[0], Ho, Wo)
        else:
            w2 = self.w(name + ".conv2.weight")
            ref, mag = S.conv_dgrad(st["dy2"], w2, s, 1, Hi, Wi)
            self.check(f"bwd da1 conv2 dgrad s{s}", self.rows4(dA, Hi, Wi), ref,
                       S.bf16_bound(ref, S.gemm_err(mag, 9 * rec["width"])))
            bnp1 = _d(rec["bnp1"])
            keep = S.relu_keep(_d(rec["y1"]), bnp1)
            self.bn_stage("bwd dy1", bn_name, dA, keep, rec["y1"], bnp1, dys[0], rec["Min"], Hi, Wi, depth)
            self.wgrad(name + ".conv1.weight", self.rows4(dys[0], Hi, Wi, full=True),
                       self.rows4(rec["x"], Hi, Wi, full=True), 1, 1, 0)
            dy1 = self.rows4(dys[0], Hi, Wi)
            w1 = self.w(name + ".conv1.weight")
            if rec["has_ds"]:
                ref, bound = S.block_dx(dy1, w1, Hi, Wi, dyd=st["dyd"], wd=self.w(name + ".downsample.0.weight"),
                                        stride=s)
            else:
                ref, bound = S.block_dx(dy1, w1, Hi, Wi, dOut=st["dOut"], keep3=st["keep3"])
            self.pending = (name, ref, bound)
            self.state = None

    def on_basic_bn_bwd(self, rec, which, dA, dys, two, depth):
        """A basic block's backward: bn2 (+ the downsample BN) from the block's output gradient, conv2's 3x3 dgrad
        da1 read by bn1, and conv1's strided 3x3 dgrad (+ shortcut) left pending for the stage that reads it."""
        name, Hi, Wi, Ho, Wo, s, C = (rec["name"], rec["Hin"], rec["Win"], rec["Hout"], rec["Wout"], rec["stride"],
                                      rec["Cout"])
        bn_name = name + "." + which
        if which == "bn2":
            if self.pending is not None:
                self.check_pending(dA)
            st = self.state = {}
            keep = R.unpack_mask(rec["m2"], C)
            self.bn_stage("bwd dy2 basic", bn_name, dA, keep, rec["y2"], _d(rec["bnp2"]), dys[0], rec["Mout"], Ho, Wo,
                          depth)
            self.wgrad(name + ".conv2.weight", self.rows4(dys[0], Ho, Wo, full=True),
                       self.rows4(rec["a1"], Ho, Wo, full=True), 3, 1, 1)
            st["dy2"] = self.rows4(dys[0], Ho, Wo)
            if two:
                st["dyd"] = self.downsample_bwd(rec, dA, keep, dys[1], depth)
            else:
                st["dOut"] = self.rows4(dA, Ho, Wo)
                k = keep.view(self.B, Ho, Wo, -1)
                st["keep2"] = k if self.sub is None else k[self.sub]
            return
        st = self.state
        ref, mag = S.conv_dgrad(st["dy2"], self.w(name + ".conv2.weight"), 1, 1, Ho, Wo)
        self.check("bwd da1 basic conv2 dgrad", self.rows4(dA, Ho, Wo), ref, S.bf16_bound(ref, S.gemm_err(mag, 9 * C)))
        bnp1 = _d(rec["bnp1"])
        keep = S.relu_keep(_d(rec["y1"]), bnp1)
        self.bn_stage("bwd dy1 basic", bn_name, dA, keep, rec["y1"], bnp1, dys[0], rec["Mout"], Ho, Wo, depth)
        self.wgrad(name + ".conv1.weight", self.rows4(dys[0], Ho, Wo, full=True),
                   self.rows4(rec["x"], Hi, Wi, full=True), 3, s, 1)
        dy1, w1 = self.rows4(dys[0], Ho, Wo), self.w(name + ".conv1.weight")
        if rec["has_ds"]:
            ref, bound = S.basic_block_dx(dy1, w1, s, Hi, Wi, dyd=st["dyd"], wd=self.w(name + ".downsample.0.weight"))
        else:
            ref, bound = S.basic_block_dx(dy1, w1, s, Hi, Wi, dOut=st["dOut"], keep2=st["keep2"])
        self.pending = (name, ref, bound)
        self.state = None

    def on_maxpool_bwd(self, ptr):
        ws = self.eng.ws.flat
        names = [n for n in ("bwd.dx0", "bwd.dx1") if n in ws and ws[n].data_ptr() == ptr]
        assert names, "the max-pool gradient does not read a block's outgoing gradient buffer"
        st = self.eng._tape["stem"]
        dpool = ws[names[0]][:self.B * st["Hp"] * st["Wp"] * 64].view(-1, 64).clone()
        self.check_pending(dpool)
        self.dpool = dpool

    def on_stem_bwd(self, da0, dy0, depth):
        st = self.eng._tape["stem"]
        Ho, Wo, Hp, Wp = st["Ho"], st["Wo"], st["Hp"], st["Wp"]
        idx = st["idx"].view(self.B, Hp, Wp, 64)
        idx = idx if self.sub is None else idx[self.sub]
        ref, bound = S.maxpool_backward(self.rows4(self.dpool, Hp, Wp), idx, Ho, Wo)
        self.check("bwd da0 maxpool", self.rows4(da0, Ho, Wo), ref, bound)
        bnp0 = _d(st["bnp"])
        keep = S.relu_keep(_d(st["y"]), bnp0)
        self.bn_stage("bwd dy0 stem", "visual.cnn.bn1", da0, keep, st["y"], bnp0, dy0, st["M"], Ho, Wo, depth)
        self.wgrad("visual.cnn.conv1.weight", self.rows4(dy0, Ho, Wo, full=True), self.img(full=True), 7, 2, 3)
        self.dpool = None

    def check_weight_grads(self):
        e = self.eng
        for wname, (ref, mag) in sorted(self.wref.items()):
            # every k > 1 conv (the stem, conv2 of a bottleneck, both 3x3 convs of a basic block) accumulates into
            # its fp32 scratch, which the unpack jobs fold into the arena; the 1x1 convs straight into the arena
            key = wname[:-len(".weight")]
            ptr = (e._dwp[key] if key in e._dwp else e.G(wname)).data_ptr()
            if "layer" not in wname:
                kind = "bwd dW stem"
            elif "downsample" in wname:
                kind = "bwd dW downsample"
            else:
                kind = "bwd dW " + ("basic " if self.recs[wname.rsplit(".", 2)[0]]["basic"] else "") + \
                    wname.split(".")[-2]
            self.check(kind, e.G(wname), ref, S.wgrad_bound(mag, self.wdepth[ptr]), info="wgrad")
        assert len(self.wref) == sum(1 for n in e.arena.names if n.startswith("visual.") and n.endswith("weight")
                                     and len(e.arena.shapes[n]) == 4)

    # ------------------------------------------------------------------------------------------------ eval forward
    def on_eval_gemm(self, A, D, kw):
        ws = self.eng.ws.flat
        names = [n for n, t in ws.items() if n.startswith("inf.") and t.data_ptr() == D.data_ptr()]
        if not names:
            return
        n = names[0]
        es = self.eval_state
        if n == "inf.stem.y":
            return
        if n == "inf.a1":
            es["bi"] += 1
            es["x"] = A
        rec = self.eng._tape["blocks"][es["bi"]]
        name, s = rec["name"], rec["stride"]
        Hi, Wi, Ho, Wo = rec["Hin"], rec["Win"], rec["Hout"], rec["Wout"]
        x = self.rows4(es["x"], Hi, Wi)

        def bnp(bn):
            return _d(ws["bnp_eval:" + bn].view(4, -1))
        if rec["basic"]:
            # conv1 3x3 (stride) with bn1 folded + ReLU, then conv2 3x3 with bn2 folded + shortcut + ReLU
            if n == "inf.a1":
                ref, bound = S.eval_conv_bn(x, self.w(name + ".conv1.weight"), s, 1, bnp(name + ".bn1"))
                self.check(f"eval a1 basic s{s}", self.rows4(D, Ho, Wo), ref, bound)
                es["a1"] = D
                return
            if n != "inf.shortcut":
                assert kw.get("residual") is not None, n
                want = es.pop("shortcut", None)
                assert kw["residual"].data_ptr() == (es["x"] if want is None else want).data_ptr(), f"{name}: shortcut"
                ref, bound = S.eval_conv_bn(self.rows4(es["a1"], Ho, Wo), self.w(name + ".conv2.weight"), 1, 1,
                                            bnp(name + ".bn2"), res=self.rows4(kw["residual"], Ho, Wo))
                self.check("eval block output basic", self.rows4(D, Ho, Wo), ref, bound)
                return
        if n == "inf.a1":
            ref, bound = S.eval_conv_bn(x, self.w(name + ".conv1.weight"), 1, 0, bnp(name + ".bn1"))
            self.check("eval a1", self.rows4(D, Hi, Wi), ref, bound)
            es["a1"] = D
        elif n == "inf.a2":
            a1 = self.rows4(es["a1"], Hi, Wi)
            ref, bound = S.eval_conv_bn(a1, self.w(name + ".conv2.weight"), s, 1, bnp(name + ".bn2"))
            self.check(f"eval a2 s{s}", self.rows4(D, Ho, Wo), ref, bound)
            es["a2"] = D
        elif n == "inf.shortcut":
            ref, bound = S.eval_conv_bn(x, self.w(name + ".downsample.0.weight"), s, 0, bnp(name + ".downsample.1"),
                                        relu=False)
            self.check(f"eval shortcut s{s}", self.rows4(D, Ho, Wo), ref, bound)
            es["shortcut"] = D
        else:
            assert kw.get("residual") is not None, n
            res = self.rows4(kw["residual"], Ho, Wo)
            want = es.pop("shortcut", None)
            assert kw["residual"].data_ptr() == (es["x"] if want is None else want).data_ptr(), f"{name}: shortcut"
            a2 = self.rows4(es["a2"], Ho, Wo)
            ref, bound = S.eval_conv_bn(a2, self.w(name + ".conv3.weight"), 1, 0, bnp(name + ".bn3"), res=res)
            self.check("eval block output", self.rows4(D, Ho, Wo), ref, bound)

    def check_eval_bnp(self):
        ws = self.eng.ws.flat
        for bn in [n[len("bnp_eval:"):] for n in ws if n.startswith("bnp_eval:")]:
            bnp = ws["bnp_eval:" + bn].view(4, -1)
            gamma, beta = self.bn_vec(bn)
            mean, inv = S.bn_eval(gamma, beta, _d(self.eng.buffers[bn + ".running_mean"]),
                                  _d(self.eng.buffers[bn + ".running_var"]))
            self.check("eval bnp", bnp[0], mean)
            self.check("bn invstd", bnp[1], inv, 4 * inv * 2.0 ** -23, info="-")
            sc, sh = R.bn_scale_shift(gamma, beta, mean, _d(bnp[1]))
            self.check("eval bnp", bnp[2], sc)
            self.check("eval bnp", bnp[3], sh)

    def run_eval(self):
        self.eval_state = {"bi": -1}
        self.eng.backbone_infer(self.image)
        assert self.eval_state["bi"] == len(self.eng.blocks) - 1
        self.eval_state = None
        self.check_eval_bnp()


def eng_sms():
    from virtex_b200 import ops
    return ops.num_sms()


def _model(backbone, seed):
    spec = O.Spec(backbone=backbone, hidden=128, layers=1, heads=2, ffn=256)
    return build_model(spec, O.synth_state(spec, seed, bn3_gain=0.25)).train()


CASES = [  # backbone, B, (H, W), fuse_bn3_min_rows (None: default), dynamic schedule, eval replay, weight-gradient
    # informativeness limit (max bound / RMS)
    pytest.param("resnet50", 2, (224, 224), None, False, True, WGRAD_INFO, id="r50-b2-224"),
    pytest.param("resnet50", 2, (224, 224), 0, True, False, WGRAD_INFO, id="r50-b2-224-fused-bn3-dynamic"),
    pytest.param("resnet50", 3, (199, 230), None, False, True, WGRAD_INFO, id="r50-b3-199x230"),
    pytest.param("wide_resnet50_2", 2, (224, 224), None, False, True, WGRAD_INFO, id="r50w2x-b2-224"),
    pytest.param("resnet101", 1, (224, 224), None, False, False, WGRAD_INFO, id="r101-b1-224"),
    pytest.param("resnet50", 256, (224, 224), None, True, False, WGRAD_INFO_B256, id="r50-b256-224-dynamic"),
    pytest.param("resnet18", 2, (224, 224), None, False, True, WGRAD_INFO, id="r18-b2-224"),
    pytest.param("resnet34", 2, (224, 224), 0, True, False, WGRAD_INFO, id="r34-b2-224-fused-bn2-dynamic"),
    pytest.param("resnet18", 3, (199, 230), 0, False, True, WGRAD_INFO_DEEP, id="r18-b3-199x230-fused"),
    pytest.param("resnet34", 256, (224, 224), None, True, False, WGRAD_INFO_B256, id="r34-b256-224-dynamic"),
    pytest.param("resnet18", 2, (320, 320), None, False, True, WGRAD_INFO, id="r18-b2-320"),
    pytest.param("resnet50", 2, (288, 288), None, False, True, WGRAD_INFO, id="r50-b2-288"),
]


@pytest.mark.parametrize("backbone,B,hw,fuse_rows,dynamic,with_eval,wgrad_info", CASES)
def test_backbone_stages_replay(backbone, B, hw, fuse_rows, dynamic, with_eval, wgrad_info, monkeypatch):
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from virtex_b200 import ops
    model = _model(backbone, seed=B + hw[1])
    eng = model.engine
    if fuse_rows is not None:
        eng.fuse_bn3_min_rows = fuse_rows
    g = torch.Generator().manual_seed(B * 7 + hw[0])
    image = torch.randn(B, 3, *hw, generator=g).cuda()
    rp = Replay(eng, image)
    rp.install(monkeypatch)
    ops.set_dynamic_gemm_schedule(dynamic)
    try:
        with torch.no_grad():
            feat, h, w = eng.backbone_forward(image, training=True)
            rp.check_forward()
            dfeat = (torch.randn(feat.shape, generator=g) * 0.01).to(BF16).cuda()
            eng.arena.grads.zero_()
            eng.backbone_backward(dfeat)
            assert rp.pending is None and rp.dpool is None
            rp.check_weight_grads()
            if with_eval:
                rp.run_eval()
        torch.cuda.synchronize()
    finally:
        ops.set_dynamic_gemm_schedule(False)
    rp.report(f"{backbone} B={B} {hw[0]}x{hw[1]} fuse_bn3_min_rows={eng.fuse_bn3_min_rows} dynamic={int(dynamic)} "
              f"deepest weight-gradient launch L={max(rp.wdepth.values())}", wgrad_info)
