"""Float64 reference of the VtxGemm contract (include/virtex_b200.h), an element-wise checker in two regimes, and a
mirror of the kernel-path selection of vtx_gemm (virtex_b200/csrc/gemm_tc.cu, `vtx_gemm`).

A call is what the engine passes to `virtex_b200.ops.gemm`: `Call(A, B, D, M, N, K, **kw)`.  The reference reads the
operands through the same pointers and leading dimensions the kernel does (`d_ptr` and the y pointer of `bnr` are kept as
element offsets into D / y), so it sees views, `ldd > N`, output sub-grids and aliased residuals exactly as the kernel.
Implicit convolutions are sums over taps of shifted float64 matmuls, chunked over images; the stem (conv_mode 5 / 6) is
a 4 x 4-tap, 16-channel, unpadded conv over the space-to-depth view S.

Regimes
  * integer: every operand a small integer, bias / residual / shift integers, scales powers of two.  When
    sum_k |a_k b_k| < 2^24 and every epilogue value of a bf16 output is at most 256 in magnitude (asserted before the
    comparison), every fp32 partial sum is exact in any order and the kernel's D must equal the reference bit for bit.
  * real data: |D - ref| <= E + ulp_bf16(|ref| + E) for bf16 outputs, E alone for fp32 outputs, with
        E = (L + 2) * 2^-22 * (sum_k |a_k b_k| * |scale| + |shift| + |bias| + |residual| + |D before| (atomic)),
        L = ceil(K_split / 16) wgmma steps + k_splits atomics.
    2^-22 per step, not the 2^-24 of one round-to-nearest addition: the tensor cores' internal rounding is not
    documented, and with 2^-23 the vocabulary weight gradient (K = 960 and 7680, accumulated onto the tied embedding's
    gradient) was measured at up to 1.06 times the bound on an H100 -- a k = 16 step rounds more than once.  Epilogues whose residual comes
    through the TMA-staged tile add it in bf16 after rounding the accumulator to bf16 (add_res_bf16x2 in gemm_tc.cu),
    a second rounding: their bound gets one more ulp_bf16(|alpha * acc + bias| + E).

BN statistics (`stats`) and the fused BN-backward sums (`bnr`) are checked against float64 sums of the kernel's own D
within (L_s + 3) * 2^-24 * (sum |term| + |value before|), exactly when that is below 2^24 in the integer regime.
L_s is the longest fp32 addition chain of the epilogue: a thread sums its rows of every tile of one column block in
registers (at most R / 8 rows: a tile has 128 rows and at least 8 row groups), the row groups are added in order (at
most 32) and every flush adds one atomic per column (at most m_tiles):  L_s = ceil(R / 8) + 32 + m_tiles, R = output
rows.  The mask of a recomputed-mask `bnr` is y * scale + shift > 0 in fp32; elements within two fp32 ulps of zero may
go either way and count into the bound.
"""
import math

import torch
import torch.nn.functional as F

BF16, F32, F64 = torch.bfloat16, torch.float32, torch.float64
KBM, KBK = 128, 64
_CHUNK = 1 << 24   # float64 elements per reference chunk


def _flat(t):
    """1-D typed view of t's whole storage."""
    return t.as_strided((t.untyped_storage().nbytes() // t.element_size(),), (1,), 0)


def _skey(t):
    return t.untyped_storage().data_ptr()


class Call:
    """One vtx_gemm call with the defaults of virtex_b200.ops.gemm resolved."""

    TENSORS = ("A", "B", "D", "bias", "residual", "stats", "residual_mask", "col_scale", "col_shift")

    def __init__(self, A, B, D, M, N, K, lda=None, ldb=None, ldd=None, a_mn=0, b_mn=0, bias=None, act=0, residual=None,
                 ldr=0, stats=None, atomic=False, split_k=1, tile_n=0, conv=None, conv_mode=0, out_f32=None,
                 residual_mask=None, conv_stride=1, conv_taps=0, tap_grid=None, out_view=None, d_ptr=None, bnr=None,
                 col_scale=None, col_shift=None):
        self.A, self.B, self.D, self.M, self.N, self.K = A, B, D, M, N, K
        self.lda = A.stride(0) if lda is None else lda
        self.ldb = B.stride(0) if ldb is None else ldb
        self.ldd = D.stride(0) if ldd is None else ldd
        self.a_mn, self.b_mn, self.bias, self.act, self.residual = a_mn, b_mn, bias, act, residual
        self.ldr = (residual.stride(0) if residual is not None else 0) if not ldr else ldr
        self.stats, self.atomic, self.split_k, self.tile_n = stats, bool(atomic), split_k, tile_n
        self.conv, self.conv_mode = conv, conv_mode
        self.out_f32 = (D.dtype == F32) if out_f32 is None else bool(out_f32)
        self.residual_mask, self.conv_stride, self.conv_taps = residual_mask, conv_stride, conv_taps
        self.tap_grid, self.out_view = tap_grid, out_view
        self.d_off = 0 if d_ptr is None else (d_ptr - D.data_ptr()) // D.element_size()
        self.has_d_ptr = d_ptr is not None
        self.bnr_y = self.bnr_bnp = self.bnr_sums = self.bnr_mask = None
        self.y_off, self.bnr_has_ptr = 0, False
        if bnr is not None:
            self.bnr_y, self.bnr_bnp, self.bnr_sums, self.bnr_mask = bnr[:4]
            if len(bnr) > 4:
                self.y_off, self.bnr_has_ptr = (bnr[4] - bnr[0].data_ptr()) // 2, True
        self.col_scale, self.col_shift = col_scale, col_shift

    # ------------------------------------------------------------------------------------------------ plumbing
    def tensors(self):
        """{role: tensor} of every tensor argument."""
        out = {r: getattr(self, r) for r in self.TENSORS if getattr(self, r) is not None}
        for r in ("bnr_y", "bnr_bnp", "bnr_sums", "bnr_mask"):
            if getattr(self, r) is not None:
                out[r] = getattr(self, r)
        return out

    def written(self):
        return [t for t in (self.D, self.stats, self.bnr_sums) if t is not None]

    def replace(self, sub):
        """A copy whose tensors t are sub(t) (same shape, strides and offset into a storage of the same layout)."""
        c = Call.__new__(Call)
        c.__dict__.update(self.__dict__)
        for r, t in self.tensors().items():
            setattr(c, r, sub(t))
        return c

    def kwargs(self):
        """Keyword arguments of virtex_b200.ops.gemm that reproduce this call (pointers from the current tensors)."""
        kw = dict(lda=self.lda, ldb=self.ldb, ldd=self.ldd, a_mn=self.a_mn, b_mn=self.b_mn, bias=self.bias,
                  act=self.act, residual=self.residual, ldr=self.ldr, stats=self.stats, atomic=self.atomic,
                  split_k=self.split_k, tile_n=self.tile_n, conv=self.conv, conv_mode=self.conv_mode,
                  out_f32=self.out_f32, residual_mask=self.residual_mask, conv_stride=self.conv_stride,
                  conv_taps=self.conv_taps, tap_grid=self.tap_grid, out_view=self.out_view,
                  col_scale=self.col_scale, col_shift=self.col_shift)
        if self.has_d_ptr:
            kw["d_ptr"] = self.D.data_ptr() + self.d_off * self.D.element_size()
        if self.bnr_y is not None:
            kw["bnr"] = (self.bnr_y, self.bnr_bnp, self.bnr_sums, self.bnr_mask)
            if self.bnr_has_ptr:
                kw["bnr"] += (self.bnr_y.data_ptr() + 2 * self.y_off,)
        return kw

    @property
    def ss(self):
        return self.col_scale is not None

    @property
    def rowwise(self):
        """D rows are output positions (plain GEMM, fprop); otherwise D is a weight gradient computed whole."""
        return self.conv_mode in (0, 1, 5)


# ------------------------------------------------------------------------------------------------- geometry
def conv_geom(c):
    """Implicit-conv geometry: input x [NI, Hin, Win, C], output grid Ho x Wo, th x tw taps reading
    (s * ho + a - pad, s * wo + b - pad); K index of tap (a, b), channel ch = (a * tw + b) * C + ch."""
    NI, Hin, Win, C = c.conv
    if c.conv_mode in (5, 6):   # space-to-depth view S [NI, Ho + 3, Wo + 3, 16]: 4 x 4 taps of 16 channels
        return dict(NI=NI, Hin=Hin + 3, Win=Win + 3, C=16, th=4, tw=4, pad=0, s=1, Ho=Hin, Wo=Win)
    s = 2 if c.conv_stride == 2 and c.conv_mode in (1, 2) else 1
    if c.conv_taps == 1 and c.conv_mode != 4:
        th = tw = 1
        pad = 0
    elif c.tap_grid is not None and c.tap_grid[0] > 0:
        th, tw, pad = c.tap_grid
    else:
        th, tw, pad = 3, 3, 1
    return dict(NI=NI, Hin=Hin, Win=Win, C=C, th=th, tw=tw, pad=pad, s=s, Ho=(Hin - 1) // s + 1, Wo=(Win - 1) // s + 1)


def _x4(t, g, base=None):
    f = _flat(t)
    return f.as_strided((g["NI"], g["Hin"], g["Win"], g["C"]), (g["Hin"] * g["Win"] * g["C"], g["Win"] * g["C"], g["C"], 1),
                        t.storage_offset() if base is None else base)


def _mat(t, rows, cols, ld, mn):
    """Logical [rows, cols] operand stored [rows, cols] (mn = 0) or [cols, rows] (mn = 1) with leading dimension ld."""
    f = _flat(t)
    if not mn:
        return f.as_strided((rows, cols), (ld, 1), t.storage_offset())
    return f.as_strided((cols, rows), (ld, 1), t.storage_offset()).t()


def _shifted(xp, g, a, b):
    """[n, Ho, Wo, C] view of the padded chunk xp at tap (a, b)."""
    s = g["s"]
    return xp[:, a:a + s * (g["Ho"] - 1) + 1:s, b:b + s * (g["Wo"] - 1) + 1:s]


def _pad(x, g):
    p, e = g["pad"], g["th"] + g["s"]
    return F.pad(x, (0, 0, p, e, p, e))


def _img_chunk(g, per_img):
    return max(1, _CHUNK // max(1, per_img))


def acc_chunks(c, absval=False):
    """Yields (r0, r1, acc): float64 sum_k A[m, k] B[n, k] of logical rows [r0, r1) (all rows of a weight gradient at
    once), over |A| and |B| when absval."""
    f = (lambda t: t.double().abs()) if absval else (lambda t: t.double())
    M, N, K = c.M, c.N, c.K
    if c.conv_mode == 0:
        A = _mat(c.A, M, K, c.lda, c.a_mn)
        Bt = f(_mat(c.B, N, K, c.ldb, c.b_mn)).t()
        step = max(1, _CHUNK // max(N, K))
        for r0 in range(0, M, step):
            r1 = min(M, r0 + step)
            yield r0, r1, f(A[r0:r1]) @ Bt
        return
    g = conv_geom(c)
    C, taps, HW = g["C"], [(a, b) for a in range(g["th"]) for b in range(g["tw"])], g["Ho"] * g["Wo"]
    if c.conv_mode in (1, 5):
        x = _x4(c.A, g)
        W = f(_mat(c.B, N, K, c.ldb, 0))
        step = _img_chunk(g, g["Hin"] * g["Win"] * C * 2 + HW * N)
        for n0 in range(0, g["NI"], step):
            n1 = min(g["NI"], n0 + step)
            xp = _pad(f(x[n0:n1]), g)
            acc = torch.zeros((n1 - n0) * HW, N, dtype=F64, device=x.device)
            for i, (a, b) in enumerate(taps):
                acc += _shifted(xp, g, a, b).reshape(-1, C) @ W[:, i * C:(i + 1) * C].t()
            yield n0 * HW, n1 * HW, acc
        return
    # weight gradients: dy [NI, Ho, Wo, Co] (rows of Co contiguous), x = B
    Co = N if c.conv_mode == 4 else M
    dy = _flat(c.A).as_strided((g["NI"], HW, Co), (HW * Co, Co, 1), c.A.storage_offset())
    x = _x4(c.B, g)
    acc = torch.zeros(Co, len(taps) * C, dtype=F64, device=x.device)
    step = _img_chunk(g, g["Hin"] * g["Win"] * C * 2 + HW * Co)
    for n0 in range(0, g["NI"], step):
        n1 = min(g["NI"], n0 + step)
        xp = _pad(f(x[n0:n1]), g)
        d = f(dy[n0:n1]).reshape(-1, Co).t()
        for i, (a, b) in enumerate(taps):
            acc[:, i * C:(i + 1) * C] += d @ _shifted(xp, g, a, b).reshape(-1, C)
    yield 0, M, (acc.t() if c.conv_mode == 4 else acc)


def _row_index(c, r0, r1, base, ld, view_strides):
    """Element index (into the flat storage) of logical (m, n), m in [r0, r1), and the mask of rows inside the output."""
    dev = c.D.device
    m = torch.arange(r0, r1, device=dev)
    n = torch.arange(c.N, device=dev)
    if c.out_view is None or not c.rowwise:
        return base + m[:, None] * ld + n[None, :], torch.ones(r1 - r0, dtype=torch.bool, device=dev)
    g = conv_geom(c)
    oh, ow, sw, sh, sn = view_strides
    img, rem = m // (g["Ho"] * g["Wo"]), m % (g["Ho"] * g["Wo"])
    ho, wo = rem // g["Wo"], rem % g["Wo"]
    ok = (ho < oh) & (wo < ow)
    return base + (img * sn + ho * sh + wo * sw)[:, None] + n[None, :], ok


def out_index(c, r0, r1):
    v = c.out_view
    return _row_index(c, r0, r1, c.D.storage_offset() + c.d_off, c.ldd, None if v is None else v)


def _bits(t, r0, r1, N):
    """[r1 - r0, N] bool of the [M, N / 8] bit mask t (bit n % 8 of byte (m * N + n) / 8)."""
    f = _flat(t)
    byte = f[t.storage_offset() + r0 * (N // 8):t.storage_offset() + r1 * (N // 8)].view(r1 - r0, N // 8).long()
    return ((byte[:, :, None] >> torch.arange(8, device=t.device)) & 1).reshape(r1 - r0, N).bool()


def _vec(t, N):
    return t.reshape(-1)[:N].double()


def epilogue(c, r0, r1, acc, absval=False):
    """(value before the activation and the store, pre-residual part, the residual added) of rows [r0, r1)."""
    f = (lambda t: t.double().abs()) if absval else (lambda t: t.double())
    N = c.N
    if c.ss:
        pre = acc * (_vec(c.col_scale, N).abs() if absval else _vec(c.col_scale, N)) + f(_vec(c.col_shift, N))
    else:
        pre = acc + (f(_vec(c.bias, N)) if c.bias is not None else 0.0)
    res = None
    if c.residual is not None and c.rowwise:
        if c.out_view is not None:
            idx, ok = _row_index(c, r0, r1, c.residual.storage_offset(), c.ldr, c.out_view)
            idx = torch.where(ok[:, None], idx, torch.zeros_like(idx))
        else:
            idx, ok = _row_index(c, r0, r1, c.residual.storage_offset(), c.ldr, None)
        res = f(_flat(c.residual)[idx])
        if c.residual_mask is not None:
            res = res * _bits(c.residual_mask, r0, r1, N)
    return (pre if res is None else pre + res), pre, res


def activation(v, act):
    if act == 1:
        return v.clamp_min(0.0)
    if act == 2:
        return 0.5 * v * (1.0 + torch.erf(v / math.sqrt(2.0)))
    return v


def ulp_bf16(x):
    """Spacing of bf16 numbers at |x| (the smallest normal spacing below 2^-126)."""
    e = torch.frexp(x.abs().clamp_min(2.0 ** -126))[1]
    return torch.ldexp(torch.ones_like(x), (e - 8).to(torch.int32))


# ------------------------------------------------------------------------------------------------ path mirror
def choose_box(H, W, positions):
    best, bw, bh = -1.0, 1, 1
    w = 1
    while w <= positions:
        h = 1
        while w * h <= positions:
            if not (w > 2 * W or h > 2 * H):
                tw, th = (W + w - 1) // w, (H + h - 1) // h
                score = (W * H) / (tw * w * th * h) * 1000.0 + w * 0.01 + h * 0.0001
                if score > best:
                    best, bw, bh = score, w, h
            h <<= 1
        w <<= 1
    return bw, bh, positions // (bw * bh)


def plan(c, sms):
    """The launch vtx_gemm makes of this call (the selection logic of gemm_tc.cu, vtx_gemm)."""
    M, N, split_k, mode = c.M, c.N, c.split_k if c.split_k > 1 else 1, c.conv_mode
    if mode == 4:
        M, N, split_k = c.N, c.M, sms // 3
    kmode = {0: 0, 1: 1, 5: 1, 2: 2, 4: 2, 6: 2}[mode]
    b_mn = c.b_mn if kmode == 0 else (0 if kmode == 1 else 1)
    bn = c.tile_n
    if bn == 0:
        gran = 64 if b_mn else 16
        bn = 256 if N >= 256 else (N + gran - 1) // gran * gran
        if bn == 256 and split_k == 1:
            mt = (M + KBM - 1) // KBM
            t256 = mt * ((N + 255) // 256)
            if t256 < 100 or (t256 < sms and N % 256 != 0 and N <= 2048):
                bn = 128
            elif t256 < 3 * sms and kmode <= 1:
                best_cost, best_bn = 0, 256
                for cand in (256, 192, 128):
                    cost = ((mt * ((N + cand - 1) // cand) + sms - 1) // sms) * (cand + 64)
                    if best_cost == 0 or cost < best_cost:
                        best_cost, best_bn = cost, cand
                bn = best_bn
    bn = 64 if bn <= 64 else 128 if bn <= 128 else 192 if bn <= 192 else 256
    n_tiles = (N + bn - 1) // bn
    if kmode == 0:
        m_tiles, kb_total = (M + KBM - 1) // KBM, (c.K + KBK - 1) // KBK
    else:
        g = conv_geom(c)
        bw, bh, bnn = choose_box(g["Ho"], g["Wo"], 128 if kmode == 1 else 64)
        boxes = ((g["Wo"] + bw - 1) // bw) * ((g["Ho"] + bh - 1) // bh) * ((g["NI"] + bnn - 1) // bnn)
        if kmode == 1:
            m_tiles, kb_total = boxes, g["th"] * g["tw"] * g["C"] // 64
        else:
            m_tiles, kb_total = (M + KBM - 1) // KBM, boxes
    k_splits = min(split_k, kb_total)
    kbps = (kb_total + k_splits - 1) // k_splits
    k_splits = (kb_total + kbps - 1) // kbps
    total = m_tiles * n_tiles * k_splits
    grid = min(total, sms)
    res = c.residual
    res_tma = (not c.out_f32 and res is not None and c.ldr % 8 == 0 and res.data_ptr() % 16 == 0 and c.bias is None
               and (c.act == 0 or c.ss))
    return dict(kmode=kmode, bn=bn, pingpong=bn <= 128 and not c.out_f32, n_tiles=n_tiles, m_tiles=m_tiles,
                kb_total=kb_total, k_splits=k_splits, kb_per_split=kbps,
                sched_chunk=4 if total >= 32 * grid else 2 if total >= 12 * grid else 1, res_tma=res_tma,
                bias_pairs=c.bias is not None and N % 2 == 0 and c.bias.data_ptr() % 8 == 0)


def path_key(c, sms):
    """Name of the kernel path a call takes: mode, stride / taps, tile width, ping-pong or lockstep, output kind,
    TMA-staged residual, paired bias loads, fused BN-backward reduction (recomputed or bit mask), folded scale / shift,
    output view, tiles per schedule fetch."""
    p = plan(c, sms)
    if c.conv_mode == 0:
        geo = "gemm"
    elif c.conv_mode in (5, 6):
        geo = "stem"
    else:
        g = conv_geom(c)
        geo = f"s{g['s']}/{g['th']}x{g['tw']}p{g['pad']}"
    out = "f32+=" if c.atomic else "f32" if c.out_f32 else "bf16"
    bnr = "-" if c.bnr_y is None else "y" if c.bnr_mask is None else "bits"
    return (f"m{c.conv_mode} {geo} bn{p['bn']} {'pp' if p['pingpong'] else 'ls'} {out} rtma{int(p['res_tma'])} "
            f"bp{int(p['bias_pairs'])} bnr={bnr} ss{int(c.ss)} view{int(c.out_view is not None)} ch{p['sched_chunk']}")


def seq_depth(c, sms):
    """L: sequential fp32 depth of one output element (wgmma K = 16 steps of one split plus one atomic per split)."""
    p = plan(c, sms)
    return 4 * p["kb_per_split"] + p["k_splits"]


# ------------------------------------------------------------------------------------------------ checker
class Report:
    def __init__(self):
        self.worst = 0.0        # max |D - ref| / bound (real data) or the number of mismatches (integer)
        self.where = None

    def note(self, r, where):
        if r > self.worst:
            self.worst, self.where = r, where


def _sums_bound(c, p, R, terms_abs, before, exact):
    Ls = -(-R // 8) + 32 + p["m_tiles"]
    mag = terms_abs + before.abs()
    if exact and bool((mag < 2.0 ** 24).all()):
        return torch.zeros_like(mag)
    return (Ls + 3) * 2.0 ** -24 * mag


def check(c, before, after, sms, integer):
    """Compares the call's outputs in `after` (a Call over the storages after the launch) with the float64 reference of
    the operands in `before` (a Call over snapshots taken before it).  Returns the worst ratio |D - ref| / bound (real
    data) or 0.0 (integer regime: any mismatch raises).  Raises AssertionError on a violation."""
    p = plan(c, sms)
    L = seq_depth(c, sms)
    N = c.N
    rep = Report()
    bf = not c.out_f32
    Dflat, Dflat0 = _flat(after.D), _flat(before.D)
    written = []
    st_s = st_q = st_sa = st_qa = None
    R = 0
    want_stats, want_bnr = c.stats is not None, c.bnr_y is not None
    if want_bnr:
        bnp = _flat(before.bnr_bnp)[before.bnr_bnp.storage_offset():before.bnr_bnp.storage_offset() + 4 * N].double()
        mean, invstd, scale, shift = bnp.view(4, N)
    for (r0, r1, acc), (_, _, mag) in zip(acc_chunks(before), acc_chunks(before, absval=True)):
        v, pre, res = epilogue(before, r0, r1, acc)
        vmag, _, _ = epilogue(before, r0, r1, mag, absval=True)
        if integer:
            assert c.act != 2, "GELU has no integer regime"
            lim = 256.0 if bf else 2.0 ** 24
            assert float(mag.max()) < 2.0 ** 24 and float(vmag.max()) <= lim, ("integer precondition", float(vmag.max()))
        ref = activation(v, c.act)
        idx, ok = out_index(after, r0, r1)
        idx, ref, vmag, pre = idx[ok], ref[ok], vmag[ok], pre[ok]
        got = Dflat[idx].double()
        if c.atomic:
            d0 = Dflat0[idx].double()
            ref = ref + d0
            vmag = vmag + d0.abs()
        if integer:
            bad = got != ref
            if bool(bad.any()):
                i = int(bad.nonzero()[0, 0]) if bad.dim() == 1 else tuple(bad.nonzero()[0].tolist())
                raise AssertionError(f"integer regime: {int(bad.sum())} of {bad.numel()} elements differ; first at "
                                     f"row {r0} + {i}: got {float(got[i])} want {float(ref[i])}")
        else:
            E = (L + 2) * 2.0 ** -22 * vmag
            bound = E + ulp_bf16(ref.abs() + E) if bf else E
            if bf and p["res_tma"] and not c.ss:
                bound = bound + ulp_bf16(pre.abs() + E)
            ratio = (got - ref).abs() / bound.clamp_min(1e-300)
            rep.note(float(ratio.max()), r0)
            assert float(ratio.max()) <= 1.0, (f"real-data bound exceeded: worst ratio {float(ratio.max()):.3g} in rows "
                                                f"from {r0}", float((got - ref).abs().max()))
        written.append(idx.reshape(-1))
        if want_stats or want_bnr:
            R += int(ok.sum())
            d = got   # the kernel's own D of the valid rows
            if want_stats:
                terms = (d, d * d)
            else:
                yidx, _ = _row_index(before, r0, r1, before.bnr_y.storage_offset() + before.y_off,
                                     before.bnr_y.stride(0), c.out_view)
                y = _flat(before.bnr_y)[yidx[ok]].double()
                if c.bnr_mask is not None:
                    on = _bits(before.bnr_mask, r0, r1, N)[ok]
                    unsure = torch.zeros_like(on)
                else:
                    z = y * scale + shift
                    on = z > 0
                    unsure = z.abs() <= 2.0 ** -22 * ((y * scale).abs() + shift.abs())
                    assert not (integer and bool(unsure.any()))
                dz = d * on
                xh = (y - mean) * invstd
                terms = (dz, dz * xh)
                sl = (d.abs() * unsure, (d * xh).abs() * unsure)
            s, q = terms[0].sum(0), terms[1].sum(0)
            sa, qa = terms[0].abs().sum(0), terms[1].abs().sum(0)
            if want_bnr:
                sa, qa = sa + 2 * sl[0].sum(0), qa + 2 * sl[1].sum(0)
            st_s, st_q = (s, q) if st_s is None else (st_s + s, st_q + q)
            st_sa, st_qa = (sa, qa) if st_sa is None else (st_sa + sa, st_qa + qa)
    if integer and not c.atomic:
        # nothing outside the written elements of D's storage may change -- except, for a bf16 output whose N is not a
        # multiple of 8, the rest of the last 16-byte chunk of each row (the TMA store's granularity, documented in
        # include/virtex_b200.h)
        changed = Dflat != Dflat0
        changed[torch.cat(written)] = False
        if bf and N % 8:
            pad = torch.cat(written).view(-1, N)[:, -1:] + torch.arange(1, 8 - N % 8 + 1, device=changed.device)
            changed[pad.reshape(-1)] = False
        if bool(changed.any()):
            pos = changed.nonzero()[:8, 0] - (after.D.storage_offset() + c.d_off)
            raise AssertionError(f"{int(changed.sum())} elements of D's storage outside the output changed, first at "
                                 f"(row, col) {[(int(i) // c.ldd, int(i) % c.ldd) for i in pos]} (ldd {c.ldd})")
    if want_stats or want_bnr:
        t = c.stats if want_stats else c.bnr_sums
        ta, tb = (after.stats, before.stats) if want_stats else (after.bnr_sums, before.bnr_sums)
        o = t.storage_offset()
        got = _flat(ta)[o:o + 2 * N].double().view(2, N)
        b0 = _flat(tb)[o:o + 2 * N].double().view(2, N)
        if st_s is None:
            st_s = st_q = st_sa = st_qa = torch.zeros(N, dtype=F64, device=got.device)
        want = b0 + torch.stack([st_s, st_q])
        bound = _sums_bound(c, p, R, torch.stack([st_sa, st_qa]), b0, integer)
        err = (got - want).abs()
        assert bool((err <= bound).all()), (("stats" if want_stats else "bnr sums"),
                                            float((err - bound).max()), float(err.max()))
    return rep.worst


# ------------------------------------------------------------------------------------------------ integer data
def integer_fill(c, gen):
    """Fills the tensors of call c (already substitutes) with integer-regime data, in place; `gen` is a generator on
    the device of the call's tensors."""
    dev = c.D.device

    def ints(shape, lo, hi):
        return torch.randint(lo, hi + 1, shape, generator=gen, device=dev)

    def pick(values, n):
        return torch.tensor(values, dtype=F64, device=dev)[torch.randint(0, len(values), (n,), generator=gen, device=dev)]

    def sparse(shape, density):
        return ints(shape, -1, 1) * (torch.rand(shape, generator=gen, device=dev) < density)

    def fill_flat(t, vals):
        f = _flat(t)
        o = t.storage_offset()
        f[o:o + vals.numel()] = vals.to(t.dtype)

    # expected sum_k |a b| per output element: 12 for bf16 outputs, 256 for fp32 ones (exact below 2^24)
    target = 256.0 if c.out_f32 else 12.0
    dens = min(1.0, math.sqrt(target / max(1, c.K)))
    # the outputs and accumulated buffers first, so that aliased residuals get their own values afterwards
    for t, lo, hi in ((c.D, -64, 64), (c.stats, -8, 8), (c.bnr_sums, -8, 8)):
        if t is not None:
            f = _flat(t)
            f.copy_(ints(f.shape, lo, hi).to(t.dtype))
    for t in (c.A, c.B):
        f = _flat(t)
        if f.data_ptr() == _flat(c.D).data_ptr():
            continue
        f.copy_(sparse(f.shape, dens).to(t.dtype))
    if c.residual is not None:
        # only the residual's own footprint: it may share D's storage (in-place accumulation)
        if c.out_view is None:
            rows = torch.arange(c.M, device=dev)
            idx = c.residual.storage_offset() + rows[:, None] * c.ldr + torch.arange(c.N, device=dev)[None, :]
        else:
            idx, ok = _row_index(c, 0, c.M, c.residual.storage_offset(), c.ldr, c.out_view)
            idx = idx[ok]
        _flat(c.residual)[idx.reshape(-1)] = ints((idx.numel(),), -4, 4).to(BF16)
    if c.bias is not None:
        fill_flat(c.bias, ints((c.N,), -4, 4))
    if c.col_scale is not None:
        fill_flat(c.col_scale, pick([-2.0, -1.0, 1.0, 2.0], c.N))
        fill_flat(c.col_shift, ints((c.N,), -4, 4))
    for t in (c.residual_mask, c.bnr_mask):
        if t is not None:
            f = _flat(t)
            f.copy_(ints(f.shape, 0, 255).to(torch.uint8))
    if c.bnr_y is not None:
        f = _flat(c.bnr_y)
        f.copy_(ints(f.shape, -8, 8).to(BF16))
        N = c.N
        mean = ints((N,), -2, 2).double()
        invstd = pick([0.5, 1.0, 2.0], N)
        scale = pick([-2.0, -1.0, -0.5, 0.5, 1.0, 2.0], N)
        # shifts are odd multiples of 1/4: y * scale (a multiple of 1/2) + shift is never zero
        shift = (ints((N,), -6, 5) * 2 + 1).double() / 4
        fill_flat(c.bnr_bnp, torch.stack([mean, invstd, scale, shift]).reshape(-1))


# ------------------------------------------------------------------------------------------------ workloads
# Every GEMM-issuing path of the shipped models, at the batch sizes the GPU test runs them: the bicaptioning configs
# (virtex_b200/configs: R-50 / R-101 / R-50W2X backbones, 1-4 layers, widths 512-2048), the token / multilabel
# classification and masked-LM pretexts, the downstream eval-mode ResNet with an fc, beam search, and a 200 x 200 image
# (im2col stem).  The batch-256 step of the base config is BATCH_256; it alone launches sched_chunk = 4 tiles per fetch
# and the bn3 reductions fused into conv1 dgrads (Engine.fuse_bn3_min_rows).
def _to(batch, device):
    return {k: v.to(device) for k, v in batch.items()}


def _live_bn(model):
    """BatchNorm weights drawn in [0.5, 1.5]: the zero-initialised last BN of every bottleneck would make the inner
    gradients of the backbone backward exactly zero, and their real-data checks vacuous."""
    g = torch.Generator().manual_seed(13)
    for n, p in model.named_parameters():
        if n.startswith("visual.") and p.dim() == 1 and n.endswith("weight"):
            p.data.copy_(torch.rand(p.shape, generator=g) + 0.5)
    return model


def _captioning(device, backbone="resnet50", hidden=1024, layers=1, B=2, image_size=224, ragged=True, seed=0):
    from oracle import virtex_oracle as O
    from virtex_b200.models import BidirectionalCaptioningModel
    from virtex_b200.modules import TorchvisionVisualBackbone, TransformerDecoderTextualHead
    torch.manual_seed(seed)
    visual = TorchvisionVisualBackbone(backbone, visual_feature_size=2048)
    textual = TransformerDecoderTextualHead(2048, 10000, hidden, layers, hidden // 64, 4 * hidden, dropout=0.1)
    model = _live_bn(BidirectionalCaptioningModel(visual, textual)).to(device).train()
    b = _to(O.synth_batch(B, seed=seed, ragged=ragged, image_size=image_size), device)
    eng = model.engine
    eng.forward(b["image"], b["caption_tokens"], b["noitpac_tokens"], b["caption_lengths"], training=True,
                with_grad=True)
    eng.backward(zero_grads=True)


def _masked_lm(device, B=3):
    from oracle import virtex_oracle as O
    from virtex_b200.models import MaskedLMModel
    from virtex_b200.modules import TorchvisionVisualBackbone, TransformerDecoderTextualHead
    torch.manual_seed(1)
    textual = TransformerDecoderTextualHead(2048, 10000, 1024, 1, 16, 4096, dropout=0.1, mask_future_positions=False)
    model = _live_bn(MaskedLMModel(TorchvisionVisualBackbone("resnet50", visual_feature_size=2048), textual))
    model = model.to(device).train()
    b = _to(O.synth_masked_batch(B, seed=5), device)
    eng = model.engine
    eng.forward(b["image"], b["caption_tokens"], b["caption_tokens"], b["caption_lengths"], training=True,
                with_grad=True, labels=b["masked_labels"])
    eng.backward(zero_grads=True)


def _classification(device, vocab, ignore, B):
    from tests import classification_oracle as CO
    from virtex_b200.models import MultiLabelClassificationModel, TokenClassificationModel
    from virtex_b200.modules import LinearTextualHead, TorchvisionVisualBackbone
    torch.manual_seed(2)
    cls = TokenClassificationModel if vocab == 10000 else MultiLabelClassificationModel
    model = _live_bn(cls(TorchvisionVisualBackbone("resnet50"), LinearTextualHead(2048, vocab), ignore)).to(device).train()
    b = _to(CO.synth_label_batch(B, seed=1, vocab=vocab, ignore=ignore, image_size=224), device)
    eng = model.engine
    eng.forward(b["image"], None, None, None, training=True, with_grad=True, labels=b["labels"])
    eng.backward(zero_grads=True)


def _downstream(device, B=2):
    from virtex_b200.modules import ResNetParams
    torch.manual_seed(3)
    cnn = ResNetParams("resnet50")
    cnn.fc = torch.nn.Linear(2048, 10)
    cnn = cnn.to(device).eval()
    image = torch.randn(B, 3, 224, 224, generator=torch.Generator().manual_seed(3)).to(device)
    with torch.no_grad():
        cnn(image)


def _beam_search(device, B=2, steps=4):
    from virtex_b200.factories import CaptionDecoderFactory
    from virtex_b200.models import ForwardCaptioningModel
    from virtex_b200.modules import TorchvisionVisualBackbone, TransformerDecoderTextualHead
    torch.manual_seed(4)
    textual = TransformerDecoderTextualHead(2048, 10000, 1024, 1, 16, 4096, dropout=0.1)
    decoder = CaptionDecoderFactory.create("beam_search", eos_index=2, max_steps=steps, beam_size=5)
    model = ForwardCaptioningModel(TorchvisionVisualBackbone("resnet50", visual_feature_size=2048), textual,
                                   decoder=decoder).to(device).eval()
    eng = model.engine
    image = torch.randn(B, 3, 224, 224, generator=torch.Generator().manual_seed(4)).to(device)
    st = eng.beam_start(image, 5, 2, steps, 1, 2)
    for _ in range(steps - 1):
        eng.beam_step(st)


WORKLOADS = {
    "r50_l1_h1024_b3": lambda d: _captioning(d, B=3),
    "r50_l1_h1024_b1": lambda d: _captioning(d, B=1, ragged=False, seed=1),
    "r50_l1_h1024_b32": lambda d: _captioning(d, B=32, seed=2),
    "r101_l1_h1024_b2": lambda d: _captioning(d, backbone="resnet101", seed=3),
    "r50w2x_l1_h1024_b2": lambda d: _captioning(d, backbone="wide_resnet50_2", seed=4),
    "r50_l2_h1024_b2": lambda d: _captioning(d, layers=2, seed=5),
    "r50_l3_h1024_b2": lambda d: _captioning(d, layers=3, seed=6),
    "r50_l4_h1024_b5": lambda d: _captioning(d, layers=4, B=5, seed=7),
    "r50_l1_h512_b5": lambda d: _captioning(d, hidden=512, B=5, seed=8),
    "r50_l1_h768_b2": lambda d: _captioning(d, hidden=768, seed=9),
    "r50_l1_h2048_b2": lambda d: _captioning(d, hidden=2048, seed=10),
    "image200_b2": lambda d: _captioning(d, image_size=200, seed=11),
    "token_classification_b3": lambda d: _classification(d, 10000, [0, 1, 2, 3], 3),
    "multilabel_classification_b5": lambda d: _classification(d, 81, [0], 5),
    "masked_lm_b3": _masked_lm,
    "downstream_eval_b2": _downstream,
    "beam_search_b2": _beam_search,
}
BATCH_256 = ("r50_l1_h1024_b256", lambda d: _captioning(d, B=256, seed=12))


# ------------------------------------------------------------------------------------------------ replay helpers
def snapshot(c):
    """A Call over copies, taken now, of the storages the call writes (D, stats, bnr sums) -- and so of any operand
    that shares them (an in-place residual) -- and over the live tensors otherwise."""
    snaps = {}
    for t in c.written():
        if _skey(t) not in snaps:
            snaps[_skey(t)] = _flat(t).clone()
    return c.replace(lambda t: torch.as_strided(snaps[_skey(t)], t.shape, t.stride(), t.storage_offset())
                     if _skey(t) in snaps else t)


def substitute(c):
    """The same call over fresh storages: every group of tensors that shares a storage gets one new buffer covering
    the bytes they span, with the same address alignment modulo 256, so that sizes, strides, relative offsets,
    aliasing and every alignment the kernel's path selection looks at are those of the original call."""
    spans = {}
    for t in c.tensors().values():
        extent = 1 + sum((s - 1) * st for s, st in zip(t.shape, t.stride()))
        lo, hi = t.data_ptr(), t.data_ptr() + extent * t.element_size()
        k = _skey(t)
        a, b = spans.get(k, (lo, hi))
        spans[k] = (min(a, lo), max(b, hi))
    bufs = {}
    for k, (lo, hi) in spans.items():
        n = (hi - lo + 512 + 7) // 8 * 8
        buf = torch.empty(n, dtype=torch.uint8, device=c.D.device)
        base = (lo - buf.data_ptr()) % 256
        bufs[k] = (buf, base, lo)

    def sub(t):
        buf, base, lo = bufs[_skey(t)]
        off = base + t.data_ptr() - lo
        assert off % t.element_size() == 0
        return torch.as_strided(buf.view(t.dtype), t.shape, t.stride(), off // t.element_size())
    return c.replace(sub)
