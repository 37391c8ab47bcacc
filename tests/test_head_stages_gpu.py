"""The engine's textual head, forward and backward, replayed sublayer by sublayer against the float64 references of
tests/head_stages.py, element by element, from the engine's own inputs of each stage.

Every reference is a function of tensors the engine produced (the residual stream entering a sublayer, the QKV / KV
projections, the attention output, the GELU input, the incoming gradients) and of the modules' parameters -- rounded
to bf16 by torch where the engine reads its bf16 mirror, fp32 where it reads the parameter arena -- never of the mirror
itself.  The caption lengths, the mask mode, the dropout sites (tests/head_stages.site, masks from
tests/dropout_replica.py) and which parameter each stage reads are the test's own, so a key-padding length that is off
for one caption, a mask drawn at a neighbouring site, a stale workspace buffer (`hb.*` is shared by every sublayer) or
a gradient overwritten instead of accumulated each breaks a per-element bound.

Capture, without changing the engine: `_self_attn_fwd` / `_bwd`, `_cross_attn_fwd` / `_bwd`, `_ffn_fwd` / `_bwd`,
`_residual_sublayer`, `head_forward` and `head_backward` are wrapped as instance attributes; `engine.call` is patched
to see the embedding, LayerNorm-backward, GELU-backward and cross-entropy launches, and `engine.gemm` to check that
every GEMM reads the bf16 rounding of the current parameters and to record the sequential depth of every weight-
gradient launch.  Each stage is checked as soon as its inputs exist; each gradient slot's total after the step is
compared with the sum of the float64 contributions of its launches.  `Engine.forward` / `Engine.backward` run as they
are, with the backbone replaced by fixed features.

Bounds: every linear layer gets the VtxGemm bound of tests/gemm_reference.py, E + ulp_bf16(|ref| + E) with
E = (4 ceil(K / 64) + 3) 2^-22 sum |terms| (plus one ulp of the pre-residual value when a GEMM accumulates onto its
output) and (L + 2) 2^-22 sum |terms| for weight gradients of sequential depth L; LayerNorm, attention, GELU and cross
entropy get the bounds of tests/test_head_kernels_gpu.py (1 bf16 ulp plus its floors, the two-rounding attention
reference with at most 2 flips per output, 1e-5 of the magnitude for fp32 values).

Power: each case prints one row per stage kind (run with -s): worst err / bound and, for bf16 stages, the median of
bound / |ref| (weight gradients: max bound / RMS of the reference).  Asserted: median bound / |ref| <= BF16_INFO for
every bf16 stage (ATTN_INFO for the attention outputs and gradients), max bound / RMS <= WGRAD_INFO for every weight
gradient (WGRAD_INFO_B256 at B = 256).  Set from a run on an H100 SXM (80 GB, default 700 W power limit), where the ten
cases took 62 s in all (36 s of it the B = 256 case, the others 0.5 to 3.4 s each):
  * bf16 stages: median bound / |ref| at most 0.0137 (the FFN linear1 dgrad at H = 2048; the GELU + dropout output
    0.0114), BF16_INFO = 2^-6.  The worst err / bound of any stage was 0.89 (a cross-attention dv at B = 256);
  * attention: median bound / |ref| at most 0.0182 (the cross-attention dq, where the 2-flip floor of the dS rounding
    is largest against outputs that cancel), ATTN_INFO = 2^-5;
  * weight-gradient totals: max bound / RMS at most 8.1e-5 at B <= 3 (WGRAD_INFO = 2^-7) and 0.0056 at B = 256, where
    the reductions run over 7680 token rows and 12544 memory rows (WGRAD_INFO_B256 = 2^-6).
"""
import copy
import math
import time

import pytest
import torch

from tests import dropout_replica as R
from tests import gemm_reference as G
from tests import head_stages as S
from tests import test_head_kernels_gpu as K

pytestmark = pytest.mark.gpu

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
SEED = 2 ** 63 + 5
PAD = 0
STEP = 2.0 ** -22
BF16_INFO = 2.0 ** -6
ATTN_INFO = 2.0 ** -5
WGRAD_INFO = 2.0 ** -7
WGRAD_INFO_B256 = 2.0 ** -6


def _d(t):
    return t.detach().to(F64)


def ulp(x):
    return G.ulp_bf16(x)


def gemm_bound(ref, mag, K, *rounded):
    E = (4 * math.ceil(K / 64) + 3) * STEP * mag
    b = E + ulp(ref.abs() + E)
    for t in rounded:
        b = b + ulp(t.abs() + E)
    return b


class _Row:
    def __init__(self, info):
        self.info, self.n, self.worst, self.power = info, 0, 0.0, []


class Replay:
    def __init__(self, eng, case, tokens, noitpac, lengths, labels, feat, sub):
        self.eng, self.case = eng, case
        self.tok = {"textual": tokens, "backward_textual": noitpac}
        self.lengths, self.labels, self.feat = lengths, labels, feat
        self.sub = sub                       # caption indices checked element by element (None: all)
        self.mods = {"textual": eng.textual, "backward_textual": eng.backward_textual}
        self.params = {}
        for pre, mod in (("textual.", eng.textual), ("backward_textual.", eng.backward_textual)):
            if mod is not None:
                for n, p in mod.named_parameters():
                    self.params.setdefault(pre + n, p)
        self.rows = {}
        self.tot, self.totb = {}, {}         # gradient slot -> float64 sum of contributions, sum of their bounds
        self.totm = {}                       # gradient slot -> sum |terms| of its weight-gradient launches
        self.depth = {}                      # gradient slot -> deepest weight-gradient launch into it
        self.kept = []                       # (name, tensor, clone) of forward tape entries that must survive
        self.d = None
        self.sms = K._ops().num_sms()

    # ------------------------------------------------------------------------------------------------ reporting
    def check(self, kind, got, ref, bound, info="median"):
        got = _d(got)
        assert got.shape == ref.shape, (kind, tuple(got.shape), tuple(ref.shape))
        row = self.rows.setdefault(kind, _Row(info))
        row.n += 1
        err = (got - ref).abs()
        ratio = err / bound.clamp_min(1e-300) if torch.is_tensor(bound) else err / bound
        worst = float(ratio.max()) if ratio.numel() else 0.0
        bad = ~(ratio <= 1.0)
        assert not bool(bad.any()), (f"{self.case} {kind}: {int(bad.sum())} of {bad.numel()} beyond the bound; worst "
                                     f"err/bound {worst:.3g} at {tuple(bad.nonzero()[0].tolist())}")
        row.worst = max(row.worst, worst)
        if info in ("median", "attn"):
            nz = ref != 0
            b = bound if torch.is_tensor(bound) else torch.full_like(ref, bound)
            q = (b[nz] / ref[nz].abs()).flatten()
            q = q[::max(1, q.numel() // (1 << 22))]
            if q.numel():
                row.power.append(float(q.median()))
        elif info == "wgrad" and bool(ref.any()):
            b = bound if torch.is_tensor(bound) else torch.full_like(ref, bound)
            row.power.append(float(b.max() / ref.pow(2).mean().sqrt()))

    def f32(self, kind, got, ref, scale=None):
        """fp32 value within 1e-5 of the largest |ref| (or of `scale`)."""
        s = float(ref.abs().max()) if scale is None else float(scale)
        self.check(kind, got, ref, torch.full_like(ref, 1e-5 * max(s, 1e-30)), info="-")

    def bf(self, kind, got, ref, floor=0.0):
        self.check(kind, got, ref, ulp(ref) + floor)

    def report(self, wgrad_info):
        print(f"\n{self.case}\n{'stage':<30} {'checks':>6} {'err/bound':>10} {'power':>10}")
        for kind, r in sorted(self.rows.items()):
            p = "-" if not r.power else f"{max(r.power):.3g}"
            print(f"{kind:<30} {r.n:>6} {r.worst:>10.3g} {p:>10}")
        for kind, r in self.rows.items():
            if r.info in ("median", "attn") and r.power:
                lim = BF16_INFO if r.info == "median" else ATTN_INFO
                assert max(r.power) <= lim, (kind, "median bound / |ref|", max(r.power))
            elif r.info == "wgrad" and r.power:
                assert max(r.power) <= wgrad_info, (kind, "max bound / RMS", max(r.power))

    # ------------------------------------------------------------------------------------------------ helpers
    def w(self, name):
        """bf16 rounding (by torch) of the current fp32 parameter."""
        return _d(self.params[name].detach().to(BF16))

    def p32(self, name):
        return _d(self.params[name])

    def rows3(self, t, T=None):
        """[M, C] device rows -> [n, T, C] float64 of the checked captions."""
        T = self.T if T is None else T
        v = t.reshape(-1, T, t.shape[-1])
        return _d(v if self.sub is None else v[self.sub])

    def mrows(self, t):
        return self.rows3(t, self.Sk)

    def scale(self, site, shape):
        if self.p == 0:
            return None
        sc = torch.from_numpy(R.flat_scale(SEED, site, shape, self.p)).to("cuda", F64).view(-1, self.T, shape[-1])
        return sc if self.sub is None else sc[self.sub]

    def ascale(self, site, B, A, Tq, Tk):
        if self.p == 0:
            return None
        sc = torch.from_numpy(R.attn_scale(SEED, site, B, A, Tq, Tk, self.p)).to("cuda", F64)
        return sc if self.sub is None else sc[self.sub]

    def contribute(self, name, ref, bound):
        self.tot[name] = self.tot.get(name, 0) + ref
        self.totb[name] = self.totb.get(name, 0) + bound

    def wgrad(self, name, dy, x, rows=None):
        """Contribution dy^T x (+ its bias colsum) to slot `name` (rows: a row slice of a packed weight)."""
        d2, x2 = _d(dy).reshape(-1, dy.shape[-1]), _d(x).reshape(-1, x.shape[-1])
        shape = self.params[name].shape
        ref, mag = torch.zeros(shape, dtype=F64, device="cuda"), torch.zeros(shape, dtype=F64, device="cuda")
        sl = slice(None) if rows is None else rows
        ref[sl] = d2.t() @ x2
        mag[sl] = d2.abs().t() @ x2.abs()
        self.contribute(name, ref, 0)
        self.totm[name] = self.totm.get(name, 0) + mag

    def colsum(self, name, dy, rows=None):
        d2 = _d(dy).reshape(-1, dy.shape[-1])
        shape = self.params[name].shape
        ref, mag = torch.zeros(shape, dtype=F64, device="cuda"), torch.zeros(shape, dtype=F64, device="cuda")
        sl = slice(None) if rows is None else rows
        ref[sl], mag[sl] = d2.sum(0), d2.abs().sum(0)
        self.contribute(name, ref, 1e-5 * mag)

    def name_of(self, t):
        a = self.eng.arena
        off = (t.data_ptr() - a.grads.data_ptr()) // 4
        for n in a.names:
            if a.offsets[n] <= off < a.offsets[n] + a.numels[n]:
                return n
        return None

    def keep(self, name, t):
        self.kept.append((name, t, t.clone()))

    # ------------------------------------------------------------------------------------------------ install
    def install(self, monkeypatch):
        from virtex_b200 import engine as E
        rp, e = self, self.eng
        orig_gemm, orig_call = E.gemm, E.call
        orig = {n: getattr(e, n) for n in ("head_forward", "head_backward", "_residual_sublayer", "_self_attn_fwd",
                                           "_cross_attn_fwd", "_ffn_fwd", "_self_attn_bwd", "_cross_attn_bwd",
                                           "_ffn_bwd")}
        mirror = e.arena.mirror

        def gemm(A, B, D, M, N, K_, **kw):
            m0 = mirror.data_ptr()
            if m0 <= B.data_ptr() < m0 + mirror.numel() * 2:   # a weight from the bf16 mirror: fresh, by torch
                off = (B.data_ptr() - m0) // 2
                name = next(n for n in e.arena.names if e.arena.offsets[n] <= off < e.arena.offsets[n] +
                            e.arena.numels[n])
                p = e.arena.p(name).reshape(-1)
                o = off - e.arena.offsets[name]
                n_el = B.numel()
                assert torch.equal(B.reshape(-1), p[o:o + n_el].to(BF16)), f"stale bf16 mirror of {name}"
            orig_gemm(A, B, D, M, N, K_, **kw)
            if kw.get("atomic"):
                name = rp.name_of(D)
                dep = G.seq_depth(G.Call(A, B, D, M, N, K_, **kw), rp.sms)
                rp.depth[name] = max(rp.depth.get(name, 0), dep)

        def call(name, *a):
            hook = getattr(rp, "on_" + name, None)
            state = hook(True, a) if hook is not None else None
            out = orig_call(name, *a)
            if hook is not None:
                hook(False, a, state)
            return out

        def head_forward(direction, mem, tokens, lengths, training, want_logits_f32=False):
            rp.begin_forward(direction, mem, tokens, lengths, training)
            rec = orig["head_forward"](direction, mem, tokens, lengths, training, want_logits_f32)
            rp.end_forward(rec)
            return rec

        def head_backward(rec, dmem, started):
            rp.begin_backward(rec, dmem)
            out = orig["head_backward"](rec, dmem, started)
            rp.end_backward(rec)
            return out

        def residual(norm_first, norm, run, x, xb, xo, xb_out, pr, z, st, M, H, p, site):
            return rp.sublayer(orig["_residual_sublayer"], norm_first, norm, run, x, xb, xo, xb_out, pr, z, st, M, H,
                               p, site)

        def fwd(kind):
            def f(rec, lr, x, out):
                orig[f"_{kind}_fwd"](rec, lr, x, out)
                getattr(rp, f"after_{kind}_fwd")(rec, lr, x, out)
            return f

        def bwd(kind):
            def f(rec, lr, dy, dx, *a):
                st = rp.before_bwd(kind, rec, lr, dy, dx, *a)
                orig[f"_{kind}_bwd"](rec, lr, dy, dx, *a)
                getattr(rp, f"after_{kind}_bwd")(st, rec, lr, dy, dx, *a)
            return f

        monkeypatch.setattr(E, "gemm", gemm)
        monkeypatch.setattr(E, "call", call)
        monkeypatch.setattr(e, "head_forward", head_forward)
        monkeypatch.setattr(e, "head_backward", head_backward)
        monkeypatch.setattr(e, "_residual_sublayer", residual)
        for kind in ("self_attn", "cross_attn", "ffn"):
            monkeypatch.setattr(e, f"_{kind}_fwd", fwd(kind))
            monkeypatch.setattr(e, f"_{kind}_bwd", bwd(kind))

    # ------------------------------------------------------------------------------------------------ forward
    def check_mem(self, mem):
        self.Sk = mem.shape[0] // self.B
        ref, mag = S.linear(self.mrows(self.feat), self.w("textual.visual_projection.weight"),
                            self.p32("textual.visual_projection.bias"))
        self.check("fwd mem visual projection", self.mrows(mem), ref, gemm_bound(ref, mag, self.feat.shape[1]))
        self.mem = mem.clone()

    def begin_forward(self, direction, mem, tokens, lengths, training):
        self.d, self.di = direction, 0 if direction == "textual" else 1
        mod = self.mods[direction]
        self.B, self.T = tokens.shape
        self.H, self.A, self.L = mod.hidden_size, mod.attention_heads, mod.num_layers
        self.p = float(mod.dropout) if training else 0.0
        self.norm_first, self.mm = mod.norm_first, (1 if mod.mask_future_positions else 2)
        self.head = direction + "."
        assert torch.equal(tokens, self.tok[direction]) and torch.equal(lengths, self.lengths)
        assert torch.equal(mem, self.mem), "the head reads the checked visual memory"
        self.fcount = 0

    def lname(self, l):
        return f"{self.head}transformer.layers.{l}."

    def on_vtx_embed_fwd(self, before, a, state=None):
        if before:
            return
        tokens = self.tok[self.d]
        M, T, H = a[9], a[10], a[11]
        ws = self.eng.ws.flat
        z0, st0, x, xb = (ws[f"{self.d}.{k}"] for k in ("z0", "st0", "x0", "x0b"))
        n = M * H
        z0, st0, x, xb = z0[:n].view(M, H), st0[:2 * M].view(M, 2), x[:n].view(M, H), xb[:n].view(M, H)
        emb = "textual.embedding."
        tk = tokens if self.sub is None else tokens[self.sub]
        z, mean, rstd, out = S.embed_fwd(tk, self.p32(emb + "words.weight"), self.p32(emb + "positions.weight"),
                                         self.p32(emb + "layer_norm.weight"), self.p32(emb + "layer_norm.bias"), PAD,
                                         self.scale(S.site(self.di), (M, H)))
        self.f32("fwd embedding z, stats", self.rows3(z0), z)
        self.f32("fwd embedding z, stats", self.rows3(st0)[..., 0], mean, scale=z.abs().max())
        self.f32("fwd embedding z, stats", self.rows3(st0)[..., 1], rstd)
        self.f32("fwd embedding out f32", self.rows3(x), out)
        self.bf("fwd embedding out bf16", self.rows3(xb), out, 1e-5 * float(out.abs().max()))
        self.stream = (x.clone(), xb.clone())

    def sublayer(self, orig, norm_first, norm, run, x, xb, xo, xb_out, pr, z, st, M, H, p, site):
        l, i = divmod(self.fcount, 3)
        i += 1
        self.fcount += 1
        q = self.lname(l)
        assert norm == f"{q}norm{i}.", (norm, l, i)
        gamma, beta = self.p32(norm + "weight"), self.p32(norm + "bias")
        assert torch.equal(x, self.stream[0]), f"L{l} sublayer {i}: the fp32 stream is not the previous output"
        if not norm_first:
            assert torch.equal(xb, self.stream[1]), f"L{l} sublayer {i}: the bf16 input is not the previous output"
        x64 = self.rows3(x)
        box = {}

        def run2(inp, out):
            if norm_first:   # the branch's input is LN(x)
                n, _, _ = S.ln_fwd(x64, gamma, beta)
                self.bf("fwd pre-norm LN bf16", self.rows3(inp), n, 1e-5 * float(n.abs().max()))
            self.branch_in = inp
            run(inp, out)
            box["branch"] = self.rows3(out)

        res = orig(norm_first, norm, run2, x, xb, xo, xb_out, pr, z, st, M, H, p, site)
        br = box["branch"]
        sc = self.scale(S.site(self.di, l, 2 * i - 1), (M, H))
        zr = x64 + (br if sc is None else br * sc)
        if norm_first:
            self.f32("fwd residual add", self.rows3(xo), zr)
            self.stream = (xo.clone(), None)
        else:
            y, mean, rstd = S.ln_fwd(zr, gamma, beta)
            self.f32("fwd residual z, stats", self.rows3(z), zr)
            self.f32("fwd residual z, stats", self.rows3(st)[..., 0], mean, scale=zr.abs().max())
            self.f32("fwd residual z, stats", self.rows3(st)[..., 1], rstd)
            self.f32("fwd post-norm LN f32", self.rows3(xo), y)
            self.bf("fwd post-norm LN bf16", self.rows3(xb_out), y, 1e-5 * float(y.abs().max()))
            self.stream = (xo.clone(), xb_out.clone())
        return res

    def lin(self, kind, got, x64, wname, bname=None, rows=None, rounded=()):
        w = self.w(wname)
        b = self.p32(bname) if bname is not None else None
        if rows is not None:
            w, b = w[rows], (None if b is None else b[rows])
        ref, mag = S.linear(x64, w, b)
        self.check(kind, got, ref, gemm_bound(ref, mag, x64.shape[-1], *rounded))
        return ref

    def attn_fwd_check(self, kind, q, k, v, o, lengths, mm, site, Tk):
        B, A = q.shape[0], self.A
        q4, k4, v4 = S.heads(q, A), S.heads(k, A), S.heads(v, A)
        s = (q4 @ k4.transpose(-1, -2) * 0.125).masked_fill(~S.allowed(B, q.shape[1], Tk, lengths, mm, q.device),
                                                            float("-inf"))
        mx = s.amax(-1, keepdim=True)
        pu = torch.exp(s - mx)
        psum = pu.sum(-1, keepdim=True)
        Mk = self.ascale(site, self.B, A, self.T, Tk)
        pd = K._rb(pu if Mk is None else pu * Mk)
        ref = S.merge(pd @ v4 / psum)
        fl = S.merge(K._flip_floor(pd / psum, v4))
        self.check(kind, o, ref, ulp(ref) + fl, info="attn")

    def attn_bwd_check(self, kind, q, k, v, do, dq, dk, dv, lengths, mm, site, Tk):
        B, A = q.shape[0], self.A
        q4, k4, v4, do4 = S.heads(q, A), S.heads(k, A), S.heads(v, A), S.heads(do, A)
        s = (q4 @ k4.transpose(-1, -2) * 0.125).masked_fill(~S.allowed(B, q.shape[1], Tk, lengths, mm, q.device),
                                                            float("-inf"))
        P = torch.softmax(s, -1)
        Mk = self.ascale(site, self.B, A, self.T, Tk)
        Mk = torch.ones_like(P) if Mk is None else Mk
        dP = do4 @ v4.transpose(-1, -2) * Mk
        D = (P * dP).sum(-1, keepdim=True)
        dS = P * (dP - D) * 0.125
        dSr, pdb = K._rb(dS), K._rb(P * Mk)
        dPmag = do4.abs() @ v4.abs().transpose(-1, -2) * Mk
        dSmag = P * ((dPmag + (P * dPmag).sum(-1, keepdim=True)) * 0.125)
        fl_q = K._flip_floor(dSr, k4) + 2.0 ** -16 * (dSmag @ k4.abs())
        fl_k = K._flip_floor(dSr.transpose(-1, -2), q4) + 2.0 ** -16 * (dSmag.transpose(-1, -2) @ q4.abs())
        for nm, got, ref, fl in (("dq", dq, dSr @ k4, fl_q), ("dk", dk, dSr.transpose(-1, -2) @ q4, fl_k),
                                 ("dv", dv, pdb.transpose(-1, -2) @ do4, K._flip_floor(pdb.transpose(-1, -2), do4))):
            self.check(f"{kind} {nm}", got, S.merge(ref), ulp(S.merge(ref)) + S.merge(fl), info="attn")

    def sub_lengths(self):
        return self.lengths if self.sub is None else self.lengths[self.sub]

    def after_self_attn_fwd(self, rec, lr, x, out):
        l = (self.fcount - 1) // 3
        q, H = self.lname(l) + "self_attn.", self.H
        assert lr["q"] == self.lname(l)
        x64 = self.rows3(self.branch_in)
        self.lin("fwd qkv projection", self.rows3(lr["qkv"]), x64, q + "in_proj_weight", q + "in_proj_bias")
        qkv = self.rows3(lr["qkv"])
        self.attn_fwd_check("fwd self-attention", qkv[..., :H], qkv[..., H:2 * H], qkv[..., 2 * H:],
                            self.rows3(lr["o_s"]), self.sub_lengths(), self.mm, S.site(self.di, l, 0), self.T)
        self.lin("fwd attention out projection", self.rows3(out), self.rows3(lr["o_s"]), q + "out_proj.weight",
                 q + "out_proj.bias")
        self.keep("qkv", lr["qkv"])

    def after_cross_attn_fwd(self, rec, lr, x, out):
        l = (self.fcount - 1) // 3
        q, H = self.lname(l) + "multihead_attn.", self.H
        x64 = self.rows3(self.branch_in)
        self.lin("fwd cross q projection", self.rows3(lr["qc"]), x64, q + "in_proj_weight", q + "in_proj_bias",
                 rows=slice(0, H))
        self.lin("fwd cross kv projection", self.mrows(lr["kv"]), self.mrows(self.mem), q + "in_proj_weight",
                 q + "in_proj_bias", rows=slice(H, 3 * H))
        kv = self.mrows(lr["kv"])
        self.attn_fwd_check("fwd cross-attention", self.rows3(lr["qc"]), kv[..., :H], kv[..., H:],
                            self.rows3(lr["o_c"]), None, 0, S.site(self.di, l, 2), self.Sk)
        self.lin("fwd attention out projection", self.rows3(out), self.rows3(lr["o_c"]), q + "out_proj.weight",
                 q + "out_proj.bias")
        self.keep("kv", lr["kv"])

    def after_ffn_fwd(self, rec, lr, x, out):
        l = (self.fcount - 1) // 3
        q = self.lname(l)
        self.lin("fwd ffn linear1", self.rows3(lr["u"]), self.rows3(self.branch_in), q + "linear1.weight",
                 q + "linear1.bias")
        u = self.rows3(lr["u"])
        g = S.gelu(u)
        sc = self.scale(S.site(self.di, l, 4), tuple(lr["u"].shape))
        # the kernel rounds GELU(u) to bf16, scales it by the fp32 1 / (1 - p) and rounds again
        ref = g if sc is None else g * sc
        bound = ulp(ref) + u.abs() * 2.0 ** -22 + (0 if sc is None else ulp(g) * sc)
        self.check("fwd gelu dropout", self.rows3(lr["h"]), ref, bound)
        self.lin("fwd ffn linear2", self.rows3(out), self.rows3(lr["h"]), q + "linear2.weight", q + "linear2.bias")
        self.keep("h", lr["h"])

    def end_forward(self, rec):
        xb = rec["x_out_b"]
        if self.norm_first:
            fn = f"{self.head}transformer.norm."
            y, _, _ = S.ln_fwd(self.rows3(self.stream[0]), self.p32(fn + "weight"), self.p32(fn + "bias"))
            self.bf("fwd final LN bf16", self.rows3(xb), y, 1e-5 * float(y.abs().max()))
        else:
            assert torch.equal(xb, self.stream[1]), "the output projection reads the last sublayer's output"
        x64 = self.rows3(xb)
        if "logits_f32" in rec:
            lf = rec["logits_f32"]
            ref, mag = S.linear(x64, self.w("textual.embedding.words.weight"), self.p32("textual.output.bias"))
            E = (4 * math.ceil(self.H / 64) + 3) * STEP * mag
            self.check("fwd logits f32 (eval)", self.rows3(lf), ref, E, info="-")
        self.lin("fwd logits", self.rows3(rec["logits"]), x64, "textual.embedding.words.weight", "textual.output.bias")
        self.keep("x_out_b", xb)
        self.rec = rec
        self.logits0 = rec["logits"].clone()

    def on_vtx_cross_entropy(self, before, a, state=None):
        if before:
            return
        di = 0 if self.rec["direction"] == "textual" else 1
        d = self.rec["direction"]
        write = a[-2]
        lab = self.labels if (self.labels is not None and d == "textual") else None
        tgt = S.targets(self.tok[d], PAD, lab)
        n, loss, dl = S.cross_entropy(_d(self.logits0).view(self.B, self.T, -1), tgt, PAD)
        assert self.eng.count[di].item() == n
        self.f32("loss", self.eng.loss[di:di + 1], loss.view(1))
        if write:
            got = self.rec["logits"]
            self.check("cross entropy dlogits", self.rows3(got), dl if self.sub is None else dl[self.sub],
                       ulp(dl if self.sub is None else dl[self.sub]) + 2.0 ** -20 / n + 2.0 ** -120, info="-")
            self.dlog = getattr(self, "dlog", {})
            self.dlog[d] = got.clone()
        else:
            assert torch.equal(self.rec["logits"], self.logits0)

    # ------------------------------------------------------------------------------------------------ backward
    def begin_backward(self, rec, dmem):
        d = rec["direction"]
        self.begin_forward(d, rec["mem"], rec["tokens"], rec["lengths"], True)
        self.p = rec["p"]
        self.rec, self.dmem = rec, dmem
        assert torch.equal(rec["logits"], self.dlog[d]), "backward starts from this direction's dlogits"
        dl, xb = rec["logits"], rec["x_out_b"]
        self.colsum("textual.output.bias", dl)
        self.wgrad("textual.embedding.words.weight", dl, xb)
        dx, _, _, mag, _ = S.linear_bwd(self.rows3(dl), self.rows3(xb), self.w("textual.embedding.words.weight"))
        self.pend_dxb = (dx, gemm_bound(dx, mag, dl.shape[1]))
        self.cursor = [(l, i) for l in reversed(range(self.L)) for i in (3, 2, 1)]
        self.cur = None
        self.exp_a, self.exp_b = None, "dxb"   # the upstream gradient of the next LayerNorm backward

    def hb(self, name, shape, dtype=None):
        t = self.eng.ws.flat[name]
        n = 1
        for s in shape:
            n *= s
        return t[:n].view(shape)

    def first_dxb(self):
        """The output projection's dgrad, checked when its reader first runs."""
        if self.pend_dxb is not None:
            ref, bound = self.pend_dxb
            self.check("bwd output projection dgrad", self.rows3(self.hb("hb.dxb", (self.B * self.T, self.H))), ref,
                       bound)
            self.pend_dxb = None
            self.exp_b = self.hb("hb.dxb", (self.B * self.T, self.H)).clone()

    def _ptr_tensor(self, ptr, dtype):
        M, H = self.B * self.T, self.H
        for n in ("hb.dres_a", "hb.dres_b", "hb.dxb"):
            t = self.eng.ws.flat.get(n)
            if t is not None and t.data_ptr() == ptr and t.dtype == dtype:
                return t[:M * H].view(M, H)
        raise AssertionError(f"gradient pointer {ptr:#x} is not a head gradient buffer")

    def given(self, a, b):
        """Checks that the upstream pointers carry exactly the expected gradients; returns their float64 sum."""
        self.first_dxb()
        ta = self._ptr_tensor(a, F32) if a else None
        tb = self._ptr_tensor(b, BF16) if b else None
        for what, t, e in (("fp32", ta, self.exp_a), ("bf16", tb, self.exp_b)):
            assert (t is None) == (e is None), (what, "upstream gradient present / absent")
            if t is not None:
                assert torch.equal(t, e), f"stale {what} upstream gradient buffer"
        g = 0
        for t in (ta, tb):
            if t is not None:
                g = g + self.rows3(t)
        return g

    def on_vtx_ln_bwd(self, before, a, state=None):
        dy_a, dy_b, z, st, w, d_skip, d_res, d_branch, dg, db, M, H, p, seed, site, ln = a[:16]
        if before:
            if self.norm_first and ln and not d_skip and not d_branch:   # final LayerNorm
                kind, l, i = "final", None, None
            elif ln and d_skip:   # pre-norm: g += LN backward of the branch input's gradient
                kind, (l, i) = "norm", self.cur
                assert torch.equal(self._ptr_tensor(d_skip, F32), self.exp_a), "stale skip gradient"
                self.exp_a = None
            else:
                kind = "branch" if not ln else "post"
                self.cur = self.cursor.pop(0)
                l, i = self.cur
            g = self.given(dy_a, dy_b)
            dgb = {n: self.eng.G(n).clone() for n in self.norm_names(kind, l, i)}
            # the full-batch upstream gradient, read now: from the second layer down, d_res is dy_a's own buffer
            gf = self.full_g(dy_a, dy_b) if kind != "branch" else None
            return kind, l, i, g, gf, (self._ptr_tensor(d_skip, F32).clone() if d_skip else None), dgb
        kind, l, i, g, gf, skip, dgb = state
        rl = self.rec["layers"]
        if kind == "final":
            fn = f"{self.head}transformer.norm."
            zz = self.rows3(self.rec["zf"])
        elif kind != "branch":
            fn = f"{self.lname(l)}norm{i}."
            zz = self.rows3(rl[l][f"z{i}"])
        if kind == "branch":
            sc = self.scale(S.site(self.di, l, 2 * i - 1), (M, H))
            ref = g if sc is None else g * sc
            self.bf("bwd pre-norm branch gradient", self.rows3(self._bf_out(d_branch)), ref)
            self.exp_dy = self._bf_out(d_branch).clone()
            return
        gamma = self.p32(fn + "weight")
        dz, dgam, dbet = S.ln_bwd(g, zz, gamma)
        y1, _, rstd = S.ln_fwd(zz, 1.0, 0.0)
        fl = 2.0 ** -16 * (g * gamma).abs().amax(-1, keepdim=True) * rstd[..., None] * (1 + y1.abs())
        out = self._ptr_tensor(d_res, F32)
        if kind == "norm":
            ref = skip_ref = self.rows3(skip) + dz
            self.check("bwd pre-norm LN + skip", self.rows3(out), ref, fl * 4 + 2.0 ** -23 * skip_ref.abs(), info="-")
            self.exp_a, self.exp_b = out.clone(), None
        else:
            self.check("bwd LN gradient f32", self.rows3(out), dz, fl * 4, info="-")
            self.exp_a = out.clone()
            if kind == "post":
                sc = self.scale(S.site(self.di, l, 2 * i - 1), (M, H))
                ref = dz if sc is None else dz * sc
                bfo = self._bf_out(d_branch)
                self.check("bwd post-norm branch gradient", self.rows3(bfo), ref,
                           ulp(ref) + fl * 4 * (1 if sc is None else sc))
                self.exp_dy = bfo.clone()
                self.exp_b = None
            else:
                self.exp_b = None
        # the parameter gradients: this launch's own contribution, from the full batch
        zf = _d(rl[l][f"z{i}"] if kind != "final" else self.rec["zf"])
        _, dgf, dbf = S.ln_bwd(gf, zf, gamma)
        for n, ref in ((fn + "weight", dgf), (fn + "bias", dbf)):
            got = self.eng.G(n) - dgb[n].view_as(self.eng.G(n))
            mag = (gf.abs() * (1 + S.ln_fwd(zf, 1.0, 0.0)[0].abs())).reshape(-1, H).sum(0)
            b = 1e-5 * mag + 1e-5 * ref.abs().max() + 2.0 ** -14 * _d(dgb[n]).view_as(ref).abs()
            self.check("bwd LN dgamma dbeta", got, ref, b, info="-")
            self.contribute(n, ref, b)

    def full_g(self, a, b):
        g = 0
        for ptr, dt in ((a, F32), (b, BF16)):
            if ptr:
                g = g + _d(self._ptr_tensor(ptr, dt))
        return g

    def _bf_out(self, ptr):
        t = self.eng.ws.flat["hb.dbr"]
        assert t.data_ptr() == ptr
        return t[:self.B * self.T * self.H].view(-1, self.H)

    def norm_names(self, kind, l, i):
        if kind == "branch":
            return []
        fn = f"{self.head}transformer.norm." if kind == "final" else f"{self.lname(l)}norm{i}."
        return [fn + "weight", fn + "bias"]

    def before_bwd(self, kind, rec, lr, dy, dx, *a):
        l, i = self.cur
        assert i == {"ffn": 3, "cross_attn": 2, "self_attn": 1}[kind] and lr["q"] == self.lname(l)
        assert torch.equal(dy, self.exp_dy), f"L{l} {kind}: the branch gradient is not the LayerNorm's output"
        st = dict(dy=dy.clone())
        if kind == "cross_attn":
            st["dmem"] = a[0].clone()
            st["first"] = self.cross_seen == 0
            self.cross_seen += 1
        return st

    def after_ffn_bwd(self, st, rec, lr, dy, dx):
        l, _ = self.cur
        q = self.lname(l)
        dh = self.hb("hb.dh", (self.B * self.T, rec["Fd"]))
        dpre = self.gelu_in
        ref, _, _, mag, _ = S.linear_bwd(self.rows3(st["dy"]), self.rows3(lr["h"]), self.w(q + "linear2.weight"))
        self.check("bwd ffn linear2 dgrad", self.rows3(dpre), ref, gemm_bound(ref, mag, self.H))
        sc = self.scale(S.site(self.di, l, 4), tuple(dh.shape))
        dd = self.rows3(dpre) if sc is None else self.rows3(dpre) * sc
        ref = dd * S.gelu_grad(self.rows3(lr["u"]))
        self.check("bwd gelu dropout", self.rows3(dh), ref, ulp(ref) + dd.abs() * 2.0 ** -20)
        self.lin_dgrad("bwd ffn linear1 dgrad", dx, dh, q + "linear1.weight")
        self.wgrad(q + "linear2.weight", st["dy"], lr["h"])
        self.colsum(q + "linear2.bias", st["dy"])
        self.wgrad(q + "linear1.weight", dh, lr["x_f"])
        self.colsum(q + "linear1.bias", dh)
        self.exp_b = dx.clone()

    def on_vtx_gelu_dropout_bwd(self, before, a, state=None):
        if before:
            self.gelu_in = self.hb("hb.dh", (self.B * self.T, self.mods[self.d].feedforward_size)).clone()

    def lin_dgrad(self, kind, dx, dy, wname, rows=None, residual=None, rmat=None):
        w = self.w(wname) if rows is None else self.w(wname)[rows]
        y64 = self.rows3(dy) if rmat is None else rmat(dy)
        ref, mag = y64 @ w, y64.abs() @ w.abs()
        rounded = ()
        if residual is not None:
            rounded = (ref,)
            ref, mag = ref + residual, mag + residual.abs()
        got = self.rows3(dx) if rmat is None else rmat(dx)
        self.check(kind, got, ref, gemm_bound(ref, mag, w.shape[0], *rounded))

    def after_self_attn_bwd(self, st, rec, lr, dy, dx):
        l, _ = self.cur
        q, H, M = self.lname(l) + "self_attn.", self.H, self.B * self.T
        do, dqkv = self.hb("hb.do", (M, H)), self.hb("hb.dqkv", (M, 3 * H))
        self.lin_dgrad("bwd attention out dgrad", do, st["dy"], q + "out_proj.weight")
        qkv = self.rows3(lr["qkv"])
        d3 = self.rows3(dqkv)
        self.attn_bwd_check("bwd self-attention", qkv[..., :H], qkv[..., H:2 * H], qkv[..., 2 * H:], self.rows3(do),
                            d3[..., :H], d3[..., H:2 * H], d3[..., 2 * H:], self.sub_lengths(), self.mm,
                            S.site(self.di, l, 0), self.T)
        self.lin_dgrad("bwd qkv dgrad", dx, dqkv, q + "in_proj_weight")
        self.wgrad(q + "out_proj.weight", st["dy"], lr["o_s"])
        self.colsum(q + "out_proj.bias", st["dy"])
        self.wgrad(q + "in_proj_weight", dqkv, lr["x_s"])
        self.colsum(q + "in_proj_bias", dqkv)
        self.exp_b = dx.clone()

    def after_cross_attn_bwd(self, st, rec, lr, dy, dx, dmem, started):
        l, _ = self.cur
        q, H, M, Sn = self.lname(l) + "multihead_attn.", self.H, self.B * self.T, self.B * self.Sk
        do, dqc, dkv = self.hb("hb.do", (M, H)), self.hb("hb.dqc", (M, H)), self.hb("hb.dkv", (Sn, 2 * H))
        self.lin_dgrad("bwd attention out dgrad", do, st["dy"], q + "out_proj.weight")
        kv, dk2 = self.mrows(lr["kv"]), self.mrows(dkv)
        self.attn_bwd_check("bwd cross-attention", self.rows3(lr["qc"]), kv[..., :H], kv[..., H:], self.rows3(do),
                            self.rows3(dqc), dk2[..., :H], dk2[..., H:], None, 0, S.site(self.di, l, 2), self.Sk)
        self.lin_dgrad("bwd cross q dgrad", dx, dqc, q + "in_proj_weight", rows=slice(0, H))
        # dmem: overwritten by the step's first cross-attention backward, accumulated by every later one
        prev = None if st["first"] else self.mrows(st["dmem"])
        self.lin_dgrad("bwd dmem" + (" first" if st["first"] else " accumulated"), dmem, dkv, q + "in_proj_weight",
                       rows=slice(H, 3 * H), residual=prev, rmat=self.mrows)
        self.wgrad(q + "out_proj.weight", st["dy"], lr["o_c"])
        self.colsum(q + "out_proj.bias", st["dy"])
        self.wgrad(q + "in_proj_weight", dqc, lr["x_c"], rows=slice(0, H))
        self.colsum(q + "in_proj_bias", dqc, rows=slice(0, H))
        self.wgrad(q + "in_proj_weight", dkv, self.mem, rows=slice(H, 3 * H))
        self.colsum(q + "in_proj_bias", dkv, rows=slice(H, 3 * H))
        self.exp_b = dx.clone()

    def on_vtx_embed_bwd(self, before, a, state=None):
        dy_a, dy_b, tok, z0, st0, gam, dw, dp, dg, db, M, T, H, pad, p, seed, site = a[:17]
        emb = "textual.embedding."
        names = [emb + n for n in ("words.weight", "positions.weight", "layer_norm.weight", "layer_norm.bias")]
        if before:
            self.given(dy_a, dy_b)
            return {n: self.eng.G(n).clone() for n in names}
        assert pad == PAD and T == self.T and tok == self.tok[self.d].data_ptr()
        g = self.full_g(dy_a, dy_b).view(self.B, self.T, H)
        tokens = self.tok[self.d]
        z = _d(self.eng.ws.flat[f"{self.d}.z0"][:M * H]).view(self.B, self.T, H)
        sc = None if self.p == 0 else torch.from_numpy(R.flat_scale(SEED, S.site(self.di), (M, H), self.p)).to(
            "cuda", F64).view(self.B, self.T, H)
        V, P_ = self.params[emb + "words.weight"].shape[0], self.params[emb + "positions.weight"].shape[0]
        refs = S.embed_bwd(g, tokens, z, self.p32(emb + "layer_norm.weight"), PAD, V, P_, sc)
        keep = (tokens != PAD).to(F64)[..., None]
        ga = g.abs() * (1 if sc is None else sc) * keep
        zz = S.ln_fwd(z, 1.0, 0.0)[0]
        gam64 = self.p32(emb + "layer_norm.weight")
        rstd = S.ln_fwd(z, 1.0, 0.0, S.EPS_EMBED)[2][..., None]
        dzb = 2.0 ** -14 * rstd * ((ga * gam64).abs() + (ga * gam64).mean(-1, keepdim=True) * (1 + zz.abs()))
        dzb = dzb * keep
        bw = torch.zeros_like(refs[0]).index_add_(0, tokens.reshape(-1), dzb.reshape(-1, H))
        bp = torch.zeros_like(refs[1])
        bp[:T] = dzb.sum(0)
        # every atomic add rounds onto the slot's running value
        cnt = torch.zeros(V, dtype=F64, device="cuda").index_add_(0, tokens.reshape(-1), keep.reshape(-1))
        bw = bw + 2.0 ** -23 * (_d(state[names[0]]).abs() + refs[0].abs()) * (cnt[:, None] + 1)
        bp = bp + 2.0 ** -23 * (_d(state[names[1]]).abs() + refs[1].abs()) * (self.B + 1)
        bounds = (bw, bp, 1e-5 * (ga * (1 + zz.abs())).reshape(-1, H).sum(0) + 2.0 ** -14 * _d(state[names[2]]).abs(),
                  1e-5 * ga.reshape(-1, H).sum(0) + 2.0 ** -14 * _d(state[names[3]]).abs())
        for n, ref, b in zip(names, refs, bounds):
            got = self.eng.G(n) - state[n]
            self.check("bwd embedding " + n.split(".")[-2], got, ref, b, info="-")
            self.contribute(n, ref, b)
        # the pad row and the rows of absent tokens: nothing from the lookup
        present = torch.zeros(V, dtype=torch.bool, device="cuda")
        present[tokens[tokens != PAD]] = True
        assert not bool((self.eng.G(names[0]) - state[names[0]])[~present].any()), "lookup gradient outside its rows"
        assert not bool((self.eng.G(names[1]) - state[names[1]])[T:].any()), "positions rows >= T changed"

    def end_backward(self, rec):
        assert not self.cursor, self.cursor

    def on_feature_grad(self, dfeat):
        """The visual projection's backward from the final dmem (Engine.backward hands dfeat to the backbone)."""
        dmem = self.eng.ws.flat["hb.dmem"][:self.mem.numel()].view_as(self.mem)
        self.lin_dgrad("bwd dfeat", dfeat, dmem, "textual.visual_projection.weight", rmat=self.mrows)
        self.wgrad("textual.visual_projection.weight", dmem, self.feat)
        self.colsum("textual.visual_projection.bias", dmem)

    def check_kept(self):
        for name, t, c in self.kept:
            assert torch.equal(t, c), f"forward tape entry {name} changed before the next forward"


CASES = [  # id: (hidden, layers, heads, ffn, norm_first, task, B, T, training, row subsample)
    pytest.param(1024, 1, 16, 4096, False, "bicap", 3, 30, True, None, id="L1-H1024-bicap"),
    pytest.param(1024, 2, 16, 4096, False, "bicap", 2, 30, True, None, id="L2-H1024-bicap"),
    pytest.param(1024, 4, 16, 4096, False, "bicap", 2, 30, True, None, id="L4-H1024-bicap"),
    pytest.param(512, 1, 8, 2048, False, "bicap", 2, 30, True, None, id="L1-H512-bicap"),
    pytest.param(768, 1, 12, 3072, False, "bicap", 2, 17, True, None, id="L1-H768-bicap"),
    pytest.param(2048, 1, 32, 8192, False, "cap", 2, 30, True, None, id="L1-H2048-cap"),
    pytest.param(2048, 1, 32, 8192, False, "mlm", 3, 30, True, None, id="L1-H2048-mlm"),
    pytest.param(512, 2, 8, 2048, True, "bicap", 2, 30, True, None, id="L2-H512-prenorm"),
    pytest.param(1024, 1, 16, 4096, False, "bicap", 3, 30, False, None, id="L1-H1024-eval"),
    pytest.param(2048, 1, 32, 8192, False, "bicap", 256, 30, True, 16, id="L1-H2048-b256"),
]


def _batch(B, T, V, task, g):
    if B <= 3:
        lengths = torch.tensor([T, 2, max(2, T - 11)])[:B]
    else:
        lengths = torch.randint(2, T + 1, (B,), generator=g)
        lengths[0], lengths[1] = T, 2
    tokens = torch.zeros(B, T, dtype=torch.int64)
    noitpac = torch.zeros(B, T, dtype=torch.int64)
    for b in range(B):
        n = int(lengths[b])
        row = torch.randint(4, V, (n,), generator=g)
        row[0], row[-1] = 1, 2
        if n > 6:
            row[3] = PAD                      # an <unk> (= the pad id) inside the caption
        tokens[b, :n] = row
        noitpac[b, :n] = row.flip(0)
    labels = None
    if task == "mlm":
        labels = torch.zeros_like(tokens)
        for b in range(B):
            n = int(lengths[b])
            for t in range(1, n - 1, 3):
                labels[b, t] = tokens[b, t] if tokens[b, t] != PAD else 5
                tokens[b, t] = 3              # [MASK]
        tokens[0, 5] = PAD                    # a random replacement by token 0 inside the length
        labels[0, 5] = 9
    return tokens, noitpac, lengths, labels


@pytest.mark.parametrize("H,L,A,Fd,norm_first,task,B,T,training,sub_every", CASES)
def test_head_stages_replay(H, L, A, Fd, norm_first, task, B, T, training, sub_every, monkeypatch):
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from virtex_b200.engine import Engine
    from virtex_b200.modules import TransformerDecoderTextualHead
    t0 = time.time()
    V, Cv, Sk = 10000, 2048, 49
    torch.manual_seed(H + L + B)
    g = torch.Generator().manual_seed(H * 10 + L + B)
    textual = TransformerDecoderTextualHead(visual_feature_size=Cv, vocab_size=V, hidden_size=H, num_layers=L,
                                            attention_heads=A, feedforward_size=Fd, dropout=0.1, norm_first=norm_first,
                                            mask_future_positions=task != "mlm", max_caption_length=30,
                                            padding_idx=PAD)
    with torch.no_grad():
        for n, p in textual.named_parameters():
            if p.dim() == 1:   # every bias and LayerNorm parameter non-trivial
                p.copy_((1.0 if n.endswith("norm1.weight") or n.endswith("norm2.weight") or
                         n.endswith("norm3.weight") or n.endswith("layer_norm.weight") or
                         n.endswith("norm.weight") else 0.0) + 0.1 * torch.randn(p.shape, generator=g))
        textual.embedding.words.weight[PAD] = 0.02 * torch.randn(H, generator=g)
    backward = None
    if task == "bicap":
        backward = copy.deepcopy(textual)
        with torch.no_grad():
            for p in backward.transformer.parameters():
                p.add_(0.01 * torch.randn(p.shape, generator=g))
        backward.visual_projection = textual.visual_projection
        backward.embedding = textual.embedding
        backward.output = textual.output
    textual.cuda()
    if backward is not None:
        backward.cuda()
    eng = Engine(None, textual, backward)
    eng.prepare_weights()   # the bf16 mirror (in a full step, the backbone's forward refreshes it)
    eng.seed.fill_(R.as_i64(SEED))
    tokens, noitpac, lengths, labels = (t.cuda() if t is not None else None for t in _batch(B, T, V, task, g))
    feat = (torch.randn(B * Sk, Cv, generator=g).abs() * 0.5).to(BF16).cuda()
    sub = None if sub_every is None else torch.tensor(sorted({0, 1, B - 1} | set(range(0, B, sub_every))),
                                                      device="cuda")
    rp = Replay(eng, f"{task} L{L} H{H} B={B} T={T} norm_first={int(norm_first)} training={int(training)}", tokens,
                noitpac, lengths, labels, feat, sub)
    rp.B, rp.T = B, T
    rp.install(monkeypatch)
    rp.cross_seen = 0
    got_dfeat = []
    monkeypatch.setattr(eng, "backbone_forward", lambda image, training: (feat, 7, 7))
    monkeypatch.setattr(eng, "backbone_backward", lambda dfeat, cb=None: got_dfeat.append(dfeat))
    orig_vp = eng.visual_projection_forward

    def vp(f, S_):
        mem = orig_vp(f, S_)
        rp.check_mem(mem)
        return mem
    monkeypatch.setattr(eng, "visual_projection_forward", vp)
    image = torch.empty(B, 1, device="cuda")
    with torch.no_grad():
        eng.forward(image, tokens, noitpac, lengths, training=training, with_grad=training, labels=labels)
        if training:
            eng.backward()
            assert len(got_dfeat) == 1
            rp.on_feature_grad(got_dfeat[0])
            assert rp.cross_seen == L * (2 if backward is not None else 1)
            _finish_totals(rp)
            rp.check_kept()
        torch.cuda.synchronize()
    rp.report(WGRAD_INFO if B < 256 else WGRAD_INFO_B256)
    print(f"wall time {time.time() - t0:.1f} s")


def _finish_totals(rp):
    e = rp.eng
    for n in e.arena.names:
        got = e.G(n)
        if n not in rp.tot:
            assert not bool(got.any()), f"{n}: a gradient slot no launch of this step should touch changed"
            continue
        bound = rp.totb[n] + (rp.depth.get(n, 0) + 2) * STEP * rp.totm.get(n, 0)
        wg = got.dim() == 2 and "embedding" not in n
        rp.check("total " + ("dW" if wg else "db dgamma dbeta embedding"), got, rp.tot[n], bound,
                 info="wgrad" if wg else "-")
    for n in rp.totm:
        assert n in rp.depth, f"{n}: no weight-gradient launch recorded"
