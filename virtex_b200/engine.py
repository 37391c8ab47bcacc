"""Execution engine of the bicaptioning step: schedules the C-ABI kernels over pre-allocated HBM buffers.

This replaces, for the hot path, what autograd + cuDNN + cuBLASLt + ATen do for the reference
(`virtex/models/captioning.py:99-143` forward; its autograd backward).  One `Engine` owns

  * a flat fp32 parameter arena (the modules' nn.Parameters are re-pointed to views of it), a flat fp32 gradient arena
    of identical layout (what the data-parallel all-reduce and the fused optimiser consume), and a flat bf16 mirror of
    the parameters (the GEMM B operands) plus packed bf16 layouts for the 3x3 / 7x7 convolution weights;
  * every activation / workspace buffer, allocated once per (batch, caption length) shape -- no allocation, no host
    synchronisation and no Python-side tensor math inside a step (the step is launch-ahead of the GPU by design; it is
    NOT captured in a CUDA graph today -- the GPU is 99 % busy without one, and the tensor maps are re-encoded per launch).

Data layout in HBM: backbone activations NHWC bf16 (a conv output is a row-major [N*H*W, C] matrix: 1x1 convs are
GEMMs as-is, 3x3/stride-1 convs are implicit GEMMs through 4-D TMA boxes), BN statistics / affine parameters fp32,
decoder residual stream fp32 with bf16 shadows feeding the GEMMs, logits bf16 (fp32 only for eval argmax).
"""
from __future__ import annotations

import math
import struct
from collections import namedtuple
from typing import Dict, List, Optional, Tuple

import torch
from torch import nn

from . import ops
from .modules import BasicBlock, LinearTextualHead
from .ops import call, gemm, _p, _stream

BF16, F32 = torch.bfloat16, torch.float32
_ALIGN = 64  # arena alignment in elements (256 B for fp32, 128 B for bf16: TMA base pointers need 16 B)
DECODE_MAX_KEYS = 64  # VTX_DECODE_MAX_KEYS of include/virtex_b200.h
ATTN_MAX_T = 1024  # VTX_ATTN_MAX_T: queries and keys per (image, head) of vtx_attn_fwd / _bwd


def _feature_grid(h, w):
    """(h, w) of the backbone's output for an h x w image: the stem conv, max-pool and layer2..4 each map x to
    (x - 1) // 2 + 1 (8 x 8 for 256 x 256, 10 x 10 for 320 x 320)."""
    for _ in range(5):
        h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    return h, w


def _check_attention(T, hw):
    """Raises before any launch when a caption of T tokens or h * w = hw feature positions exceed the attention
    kernels (self-attention: T queries and keys; cross-attention: T queries, hw keys)."""
    if T > ATTN_MAX_T or hw > ATTN_MAX_T:
        raise ValueError(f"attention takes at most {ATTN_MAX_T} queries and keys per image and head: got captions of "
                         f"{T} tokens and {hw} feature positions")


def _lse_rows(B, A, T):
    """fp32 log-sum-exp rows vtx_attn_fwd writes for T queries: B * A * (T rounded up to 32)."""
    return B * A * _round_up(T, 32)


def _round_up(x, m):
    return (x + m - 1) // m * m


class Arena:
    """Flat fp32 parameter / gradient storage with a bf16 mirror; parameters become views into it."""

    def __init__(self, named_params: List[Tuple[str, nn.Parameter]], device):
        self.device = device
        self.names: List[str] = []
        self.offsets: Dict[str, int] = {}
        self.numels: Dict[str, int] = {}
        self.shapes: Dict[str, torch.Size] = {}
        off = 0
        seen = {}
        for name, p in named_params:
            if id(p) in seen:
                continue
            seen[id(p)] = name
            self.names.append(name)
            self.offsets[name] = off
            self.numels[name] = p.numel()
            self.shapes[name] = p.shape
            off = _round_up(off + p.numel(), _ALIGN)
        self.total = off
        self.params = torch.zeros(off, dtype=F32, device=device)
        self.grads = torch.zeros(off, dtype=F32, device=device)
        self.mirror = torch.zeros(off, dtype=BF16, device=device)
        self._param_objs = {seen[id(p)]: p for _, p in named_params}
        with torch.no_grad():
            for name in self.names:
                p = self._param_objs[name]
                v = self.view(self.params, name)
                v.copy_(p.data.to(device=device, dtype=F32))
                p.data = v
                p.grad = None

    def view(self, flat, name):
        o = self.offsets[name]
        return flat[o:o + self.numels[name]].view(self.shapes[name])

    def p(self, name):
        return self.view(self.params, name)

    def g(self, name):
        return self.view(self.grads, name)

    def w(self, name):
        return self.view(self.mirror, name)

    def intact(self):
        """True while every parameter still aliases the arena (a `.to()` / `.half()` on the module breaks it)."""
        base, end = self.params.data_ptr(), self.params.data_ptr() + self.total * 4
        for name in (self.names[0], self.names[-1]):
            ptr = self._param_objs[name].data_ptr()
            if not (base <= ptr < end):
                return False
        return True

    def refresh_mirror(self):
        call("vtx_cast_bf16", self.params.data_ptr(), self.mirror.data_ptr(), self.total, _stream())


class _Workspace:
    """Named device buffers that only ever grow: after the first step of a given shape nothing is allocated."""

    def __init__(self, device):
        self.device = device
        self.flat: Dict[str, torch.Tensor] = {}

    def get(self, name, shape, dtype):
        shape = tuple(int(s) for s in shape)
        n = 1
        for s in shape:
            n *= s
        t = self.flat.get(name)
        if t is None or t.dtype != dtype or t.numel() < n:
            t = torch.empty(max(n, 1), dtype=dtype, device=self.device)
            self.flat[name] = t
        return t[:n].view(shape)

    def nbytes(self):
        return sum(t.numel() * t.element_size() for t in self.flat.values())


def _require_cuda(dev):
    if dev is None or dev.type != "cuda":
        raise RuntimeError("virtex_b200 has no CPU path: move the model to a CUDA device first (model.cuda())")


_Conv = namedtuple("_Conv", "w k stride cin cout")


def _block_convs(name, blk):
    """The main-branch convolutions of residual block `name`, in order, as _Conv(weight prefix, kernel size, stride,
    Cin, Cout); BN i follows conv i, and the last BN is the block output's.  A bottleneck is 1x1, 3x3 (the block's
    stride), 1x1, its widths read from the weights (4x apart for ResNet-50/101/152, 2x for the wide models); a basic
    block is two 3x3 convs, the first strided."""
    kinds = [(3, blk.stride), (3, 1)] if isinstance(blk, BasicBlock) else [(1, 1), (3, blk.stride), (1, 1)]
    convs = []
    for i, (k, stride) in enumerate(kinds, 1):
        cout, cin = getattr(blk, f"conv{i}").weight.shape[:2]
        convs.append(_Conv(f"{name}.conv{i}", k, stride, cin, cout))
    return convs


def _dgrad_route(conv, cols):
    """How the input gradient of main-branch conv `conv` runs: 'gemm' (1x1), 'implicit' (3x3, stride 1), 'parity'
    (3x3, stride 2: one implicit GEMM per parity class of the input position) or 'col2im' (per-tap gradients by a plain
    GEMM, scattered back: after an im2col forward, whose matrix is `cols`, and at other strides).  Only the GEMMs that
    write dx itself carry an epilogue over it; 'parity' carries only the BN-backward sums."""
    if conv.k == 1:
        return "gemm"
    if cols is not None or conv.stride not in (1, 2):
        return "col2im"
    return "implicit" if conv.stride == 1 else "parity"


def _transposed_wgrad(Cin, C, stride):
    """True when a 3x3 conv's weight gradient runs as conv_mode 4 (64 -> 64, stride 1), whose [(tap, cin), cout]
    layout the unpack job of kind 3 reads; every other 3x3 wgrad is the split-K conv_mode 2 into [C, 9 * Cin]."""
    return Cin == 64 and C == 64 and stride == 1


class Engine:
    """Forward/backward of (backbone) + (forward head) + (backward head) on one GPU.  Any part may be absent."""

    # BN-backward reductions (sum dz, sum dz * xhat) are accumulated by the epilogue of the GEMM that produces the
    # gradient (bn1 / bn2 of every block, bn3 of blocks followed by an identity block) instead of a separate pass.
    # bn3's for layer1-3 at batch 256 (the streaming masked-residual dgrad kernel of csrc/gemm_resid.cu reads y and the
    # mask beside dOut at HBM rate); layer4 and small batches keep the stand-alone pass, which costs about what the
    # persistent kernel's longer epilogue does.
    fuse_bn3_min_rows = 40000

    def __init__(self, visual=None, textual=None, backward_textual=None, prefix_map=None, ignore_indices=None):
        self.visual, self.textual, self.backward_textual = visual, textual, backward_textual
        named: List[Tuple[str, nn.Parameter]] = []
        if visual is not None:
            named += [("visual." + n, p) for n, p in visual.named_parameters()]
        if textual is not None:
            named += [("textual." + n, p) for n, p in textual.named_parameters()]
        if backward_textual is not None:
            named += [("backward_textual." + n, p) for n, p in backward_textual.named_parameters()]
        dev = None
        for _, p in named:
            dev = p.device
            break
        _require_cuda(dev)
        self.device = dev
        self.arena = Arena(named, dev)
        self.ws = _Workspace(dev)
        self.buffers: Dict[str, torch.Tensor] = {}
        if visual is not None:
            self.buffers.update({"visual." + n: b for n, b in visual.named_buffers()})
        head = textual if textual is not None else backward_textual
        self.pad = getattr(head, "padding_idx", 0) if head is not None else 0
        # a LinearTextualHead makes this the engine of a classification pretext model: pool + linear + K-hot loss instead
        # of a decoder (virtex/models/classification.py:43-108)
        self.classify = isinstance(textual, LinearTextualHead)
        # label ids the K-hot loss ignores, on the device once per engine (read by every loss launch)
        self.ignore = torch.tensor([int(i) for i in (ignore_indices or [])], dtype=torch.int64, device=dev)
        self._cls = None
        self.seed = torch.zeros(1, dtype=torch.int64, device=dev)
        self.loss = torch.zeros(2, dtype=F32, device=dev)       # per-direction mean NLL
        self.count = torch.zeros(2, dtype=F32, device=dev)      # per-direction number of valid targets
        self._packed: Dict[str, torch.Tensor] = {}
        self._tape = None
        self.generation = 0  # bumped by every forward(): a backward must match the forward that filled the tape
        self._weights_fresh = False
        self._eval_bn_fresh = False  # the running-statistics scale / shift of every BN (backbone_infer's epilogues)
        self._build_backbone_plan()

    # ------------------------------------------------------------------------------------------------ parameters
    def P(self, name):
        return self.arena.p(name)

    def W(self, name):
        return self.arena.w(name)

    def G(self, name):
        return self.arena.g(name)

    def mark_weights_dirty(self):
        self._weights_fresh = False
        self._eval_bn_fresh = False

    def _build_backbone_plan(self):
        self.blocks = []
        self._jobs: Dict[str, tuple] = {}
        if self.visual is None:
            return
        cnn = self.visual.cnn
        for li in range(1, 5):
            layer = getattr(cnn, f"layer{li}")
            for bi, blk in enumerate(layer):
                self.blocks.append((f"visual.cnn.layer{li}.{bi}", blk))
        self._convs = {name: _block_convs(name, blk) for name, blk in self.blocks}
        # fp32 weight-gradient scratch of every k > 1 convolution (GEMM output layout), one flat buffer zeroed once per
        # backward; the batched unpack jobs fold it into the OIHW gradient arena per all-reduce bucket
        sizes = [("visual.cnn.conv1", 64 * 256)]
        sizes += [(c.w, c.cout * 9 * c.cin) for convs in self._convs.values() for c in convs if c.k == 3]
        total = sum(_round_up(n, _ALIGN) for _, n in sizes)
        self._dwp_flat = torch.zeros(total, dtype=F32, device=self.device)
        self._dwp, off = {}, 0
        for key, n in sizes:
            self._dwp[key] = self._dwp_flat[off:off + n]
            off += _round_up(n, _ALIGN)

    # ------------------------------------------------------------------------------------ batched weight-layout jobs
    def _job_table(self, key, make):
        """Device-resident VtxWeightJob table, built once per key: (src, dst, total, O, I, KH, KW, ldk, kind) rows."""
        tab = self._jobs.get(key)
        if tab is None:
            rows = make()
            blk = ops.L.load().vtx_weight_job_block_elems()
            blob, b0 = b"", 0
            for src, dst, total, O, I, KH, KW, ldk, kind in rows:
                blob += struct.pack("<QQq8i", src.data_ptr(), dst.data_ptr(), total, O, I, KH, KW, ldk, kind, b0, 0)
                b0 += (total + blk - 1) // blk
            dev = torch.frombuffer(bytearray(blob), dtype=torch.uint8).to(self.device) if rows else None
            tab = self._jobs[key] = (dev, len(rows), b0)
        return tab

    def _run_jobs(self, key, make):
        dev, n, blocks = self._job_table(key, make)
        if n:
            call("vtx_conv_w_jobs", dev.data_ptr(), n, blocks, _stream())

    def _pack_rows(self):
        w = self.P("visual.cnn.conv1.weight")
        rows = [(w, self._pack_buf("visual.cnn.conv1.weight", (64, 160)), 64 * 160, 64, 3, 7, 7, 160, 0),
                (w, self._pack_buf("visual.cnn.conv1.weight#s2d", (64, 256)), 64 * 256, 64, 3, 7, 7, 256, 4)]
        for name, blk in self.blocks:
            parity = []
            for wname, k, stride, I, O in self._convs[name]:
                if k == 1:
                    continue
                w = self.P(wname + ".weight")
                rows.append((w, self._pack_buf(wname + ".weight", (O, 9 * I)), 9 * O * I, O, I, 3, 3, 9 * I, 0))
                if stride == 1:
                    rows.append((w, self._pack_buf(wname + ".weight#dgrad", (I, 9 * O)), 9 * O * I, O, I, 3, 3, 9 * O,
                                 1))
                else:  # stride-2 dgrad: one weight slice per parity class (ph, pw) of the input gradient
                    for ph in (0, 1):
                        for pw in (0, 1):
                            nt = (1 + ph) * (1 + pw)
                            parity.append((w, self._pack_buf(f"{wname}.weight#dgrad_s2_{ph}{pw}", (I, nt * O)),
                                           nt * O * I, O, I, ph, pw, nt * O, 6))
            if blk.stride == 2 and blk.downsample is not None:
                wdn = self.P(name + ".downsample.0.weight")
                C4, Cin = wdn.shape[0], wdn.shape[1]
                if Cin % 64 == 0:  # transposed copy: K-major B operand of the downsample's (implicit, strided-store) dgrad
                    rows.append((wdn, self._pack_buf(name + ".downsample.0.weight#t", (Cin, C4)), C4 * Cin, C4, Cin, 1, 1,
                                 C4, 7))
            rows += parity
        return rows

    def _unpack_rows(self, layer, stem_s2d):
        """Unpack-accumulate jobs of one gradient bucket: 'layer4' / 'layer3' / 'layer2' / 'rest' (layer1 + stem)."""
        rows = []
        want = "layer1" if layer == "rest" else layer
        for name, _ in self.blocks:
            if name.split(".")[2] != want:
                continue
            for wname, k, stride, I, O in self._convs[name]:
                if k == 3:
                    rows.append((self._dwp[wname], self.G(wname + ".weight"), 9 * O * I, O, I, 3, 3, 9 * I,
                                 3 if _transposed_wgrad(I, O, stride) else 2))
        if layer == "rest":
            g = self.G("visual.cnn.conv1.weight")
            if stem_s2d:
                rows.append((self._dwp["visual.cnn.conv1"], g, 64 * 147, 64, 3, 7, 7, 256, 5))
            else:
                rows.append((self._dwp["visual.cnn.conv1"], g, 64 * 147, 64, 3, 7, 7, 160, 2))
        return rows

    def prepare_weights(self, mirror=True, eval_bn=False):
        """bf16 mirror of all parameters + packed GEMM layouts of the k>1 convolution weights.  `eval_bn`: also the
        eval-mode bnp [4, C] = mean, invstd, scale, shift of every BN from its running statistics (backbone_infer)."""
        if mirror:
            self.arena.refresh_mirror()
        if self.visual is not None:
            self._run_jobs("pack", self._pack_rows)  # every packed conv-weight layout in one launch
            if eval_bn:
                for bn_name, C in self._bn_names():
                    self._bn_fwd(None, bn_name, 1, C, False, None, key="bnp_eval:")
                self._eval_bn_fresh = True
        self._weights_fresh = True

    def _bn_names(self):
        """(name, channels) of every BatchNorm of the backbone."""
        out = [("visual.cnn.bn1", 64)]
        for name, blk in self.blocks:
            convs = self._convs[name]
            out += [(f"{name}.bn{i}", c.cout) for i, c in enumerate(convs, 1)]
            if blk.downsample is not None:
                out.append((name + ".downsample.1", convs[-1].cout))
        return out

    def _pack_buf(self, key, shape):
        t = self._packed.get(key)
        if t is None:
            t = torch.empty(shape, dtype=BF16, device=self.device)
            self._packed[key] = t
        return t

    # ------------------------------------------------------------------------------------------------ backbone fwd
    def _bn_fwd(self, y, bn_name, M, C, training, stats, key="bnp:"):
        bnp = self.ws.get(key + bn_name, (4, C), F32)
        nbt = self.buffers[bn_name + ".num_batches_tracked"]
        call("vtx_bn_finalize", _p(stats), float(M), self.P(bn_name + ".weight").data_ptr(),
             self.P(bn_name + ".bias").data_ptr(), self.buffers[bn_name + ".running_mean"].data_ptr(),
             self.buffers[bn_name + ".running_var"].data_ptr(), nbt.data_ptr(), 0.1, 1e-5, int(training),
             bnp.data_ptr(), C, _stream())
        return bnp

    def _bn_act_fwd(self, y, bn_name, M, C, training, stats, out, res=None, bnp_res=None, relu=1, mask=None):
        """BN finalize (batch or running statistics -> bnp, running-stat update) + apply + ReLU (+ residual), one launch.
        `mask`: uint8 [M, C/8] ReLU sign bits for backward (block outputs, whose pre-activation includes the shortcut)."""
        bnp = self.ws.get("bnp:" + bn_name, (4, C), F32)
        call("vtx_bn_finalize_act", _p(stats), float(M), self.P(bn_name + ".weight").data_ptr(),
             self.P(bn_name + ".bias").data_ptr(), self.buffers[bn_name + ".running_mean"].data_ptr(),
             self.buffers[bn_name + ".running_var"].data_ptr(),
             self.buffers[bn_name + ".num_batches_tracked"].data_ptr(), 0.1, 1e-5, int(training), bnp.data_ptr(),
             y.data_ptr(), _p(res), _p(bnp_res), out.data_ptr(), _p(mask), M, C, relu, _stream())
        return bnp

    def _stats_slab(self, training):
        """One zeroed fp32 slab per step holding every BN's [2,C] sum/sumsq (fwd) and [2,C] dz sums (bwd)."""
        total = 4 * sum(C for _, C in self._bn_names())
        slab = self.ws.get("bn_slab", (total,), F32)
        slab.zero_()
        self._slab, self._slab_off = slab, 0
        return slab

    def _slab_take(self, n):
        t = self._slab[self._slab_off:self._slab_off + n]
        self._slab_off += n
        return t

    # Route choice + launch of the convolutions that have more than one route.  backbone_forward and backbone_infer
    # share them, so the training and eval forwards always run the same conv; `key` names the scratch buffer of the
    # route that needs one, and `epi` is passed through to the GEMM's epilogue.
    def _stem_conv(self, image, y0, Ho, Wo, key, **epi):
        """conv1 (7x7, stride 2) of the fp32 NCHW image into y0 [B*Ho*Wo, 64]; returns (s2d, cols): the GEMM operand
        the route built, and None for the other route."""
        B, _, H, W = image.shape
        M0 = B * Ho * Wo
        if H % 2 == 0 and W % 4 == 0 and Ho % 8 == 0 and Wo % 16 == 0:  # the 16 x 8 TMA boxes tile the output exactly
            # 4-tap implicit GEMM over the space-to-depth view of the image (csrc/stem_s2d.cu)
            s2d = self.ws.get(key + "stem.s2d", (B, H // 2 + 3, W // 2 + 3, 16), BF16)
            call("vtx_stem_s2d", image.data_ptr(), s2d.data_ptr(), B, H, W, _stream())
            gemm(s2d, self._packed["visual.cnn.conv1.weight#s2d"], y0, M0, 64, 256, lda=64, ldb=256,
                 conv=(B, Ho, Wo, 64), conv_mode=5, **epi)
            return s2d, None
        # other image sizes: im2col + plain GEMM
        cols = self.ws.get(key + "stem.cols", (M0, 160), BF16)
        call("vtx_stem_im2col", image.data_ptr(), cols.data_ptr(), B, H, W, 160, _stream())
        gemm(cols, self._packed["visual.cnn.conv1.weight"], y0, M0, 64, 160, **epi)
        return None, cols

    def _conv(self, conv, x, y, B, Hc, Wc, key, **epi):
        """Main-branch conv `conv` (a _Conv) of a residual block: x [B*Hc*Wc, Cin] -> y [Mout, C]; a 1x1 conv is a plain
        GEMM, a 3x3 conv (stride 1 or 2, pad 1) an implicit GEMM or im2col + GEMM.  Returns the im2col matrix when that
        route ran, else None."""
        wname, k, stride, Cin, C = conv
        Mout = y.shape[0]
        if k == 1:
            gemm(x, self.W(wname + ".weight").view(C, Cin), y, Mout, C, Cin, **epi)
            return None
        w = self._packed[wname + ".weight"]
        if Cin % 64 == 0:
            # implicit GEMM: 4-D TMA boxes gather the taps (zero fill = padding); stride 2 through TMA traversal strides
            gemm(x, w, y, Mout, C, 9 * Cin, lda=Cin, conv=(B, Hc, Wc, Cin), conv_mode=1, conv_stride=stride, **epi)
            return None
        cols = self.ws.get(key, (Mout, 9 * Cin), BF16)
        call("vtx_im2col3x3", x.data_ptr(), cols.data_ptr(), B, Hc, Wc, Cin, stride, _stream())
        gemm(cols, w, y, Mout, C, 9 * Cin, **epi)
        return cols

    def _downsample(self, name, x, y, B, Hc, Wc, stride, key, **epi):
        """1x1 shortcut conv (stride) of block `name`: x [B*Hc*Wc, Cin] -> y [Mout, C4]; returns the matrix the
        GEMM read (x itself at stride 1, otherwise its subsampled copy), or None when the strided implicit GEMM read x
        in place."""
        Mout, C4 = y.shape
        Cin = x.shape[1]
        wd = self.W(name + ".downsample.0.weight").view(C4, Cin)
        if stride == 1:
            gemm(x, wd, y, Mout, C4, Cin, **epi)
            return x
        if Cin % 64 == 0:  # strided 1x1 conv = one-tap implicit GEMM over x (no subsampled copy)
            gemm(x, wd, y, Mout, C4, Cin, lda=Cin, conv=(B, Hc, Wc, Cin), conv_mode=1, conv_stride=stride, conv_taps=1,
                 **epi)
            return None
        xs = self.ws.get(key, (Mout, Cin), BF16)
        call("vtx_subsample", x.data_ptr(), xs.data_ptr(), B, Hc, Wc, Cin, stride, _stream())
        gemm(xs, wd, y, Mout, C4, Cin, **epi)
        return xs

    def _block_output_fwd(self, rec, x, y, st, bn_name, out, mask, B, training):
        """The last BN of block rec["name"] (input y, statistics st) + shortcut (x itself, or the downsample conv and
        its BN) + ReLU into out, the ReLU sign bits into mask; returns the BN's bnp."""
        name, Mout, C = rec["name"], rec["Mout"], rec["Cout"]
        if rec["has_ds"]:
            yd = self.ws.get(name + ".yd", (Mout, C), BF16)
            std = self._slab_take(2 * C) if training else None
            xs = self._downsample(name, x, yd, B, rec["Hin"], rec["Win"], rec["stride"], name + ".xs", stats=std)
            bnpd = self._bn_fwd(yd, name + ".downsample.1", Mout, C, training, std)
            rec.update(xs=xs, yd=yd, bnpd=bnpd)
            return self._bn_act_fwd(y, bn_name, Mout, C, training, st, out, res=yd, bnp_res=bnpd, mask=mask)
        return self._bn_act_fwd(y, bn_name, Mout, C, training, st, out, res=x, mask=mask)

    def backbone_forward(self, image: torch.Tensor, training: bool):
        """image fp32 NCHW [B,3,H,W] -> NHWC bf16 feature matrix [B*h*w, C] (C = 2048 for the bottleneck ResNets, 512
        for ResNet-18/34); fills the tape used by backward."""
        if not self._weights_fresh:
            self.prepare_weights()
        if training:
            self._eval_bn_fresh = False  # the running statistics move
        B, _, H, W = image.shape
        s = _stream()
        ws = self.ws
        self._stats_slab(training)
        tape = {"B": B, "blocks": [], "training": training}
        # ---- stem: im2col -> GEMM(+stats) -> BN finalize -> BN+ReLU+maxpool
        Ho, Wo = (H + 6 - 7) // 2 + 1, (W + 6 - 7) // 2 + 1
        M0 = B * Ho * Wo
        y0 = ws.get("stem.y", (M0, 64), BF16)
        st = self._slab_take(128) if training else None
        s2d, cols = self._stem_conv(image, y0, Ho, Wo, "", stats=st)
        bnp0 = self._bn_fwd(y0, "visual.cnn.bn1", M0, 64, training, st)
        Hp, Wp = (Ho - 1) // 2 + 1, (Wo - 1) // 2 + 1
        x = ws.get("stem.pool", (B * Hp * Wp, 64), BF16)
        idx = ws.get("stem.idx", (B * Hp * Wp, 64), torch.uint8)
        call("vtx_bn_relu_maxpool", y0.data_ptr(), bnp0.data_ptr(), x.data_ptr(), idx.data_ptr(), B, Ho, Wo, 64, s)
        tape["stem"] = dict(cols=cols, s2d=s2d, y=y0, bnp=bnp0, idx=idx, Ho=Ho, Wo=Wo, Hp=Hp, Wp=Wp, M=M0)
        Hc, Wc, Cin = Hp, Wp, 64
        # ---- residual blocks (torchvision's basic and bottleneck blocks): every conv but the last with statistics ->
        # its BN + ReLU; the last with statistics -> the block output's BN + shortcut + ReLU
        for name, blk in self.blocks:
            convs = self._convs[name]
            n, C = len(convs), convs[-1].cout
            stride = blk.stride
            Hn, Wn = (Hc - 1) // stride + 1, (Wc - 1) // stride + 1
            Min, Mout = B * Hc * Wc, B * Hn * Wn
            rec = dict(name=name, x=x, Hin=Hc, Win=Wc, Hout=Hn, Wout=Wn, Cin=Cin, width=convs[0].cout, Cout=C,
                       stride=stride, Min=Min, Mout=Mout, has_ds=blk.downsample is not None, basic=n == 2)
            a, h, w = x, Hc, Wc
            for i, conv in enumerate(convs, 1):
                ho, wo = (h - 1) // conv.stride + 1, (w - 1) // conv.stride + 1
                y = ws.get(f"{name}.y{i}", (B * ho * wo, conv.cout), BF16)
                st = self._slab_take(2 * conv.cout) if training else None
                rec[f"cols{i}"] = self._conv(conv, a, y, B, h, w, f"{name}.cols{i}", stats=st)
                rec[f"y{i}"], rec[f"hw{i}"] = y, (h, w)  # hw: the conv's input grid
                if i < n:
                    a = ws.get(f"{name}.a{i}", y.shape, BF16)
                    rec[f"a{i}"] = a
                    rec[f"bnp{i}"] = self._bn_act_fwd(y, f"{name}.bn{i}", y.shape[0], conv.cout, training, st, a)
                h, w = ho, wo
            out = ws.get(name + ".out", (Mout, C), BF16)
            # backward needs only the SIGN of the block output's pre-activation: one bit per element instead of re-reading
            # the bf16 output twice (bn_bwd_reduce and bn_bwd_apply)
            m = ws.get(f"{name}.m{n}", (Mout, C // 8), torch.uint8) if training else None
            rec[f"bnp{n}"] = self._block_output_fwd(rec, x, y, st, f"{name}.bn{n}", out, m, B, training)
            rec.update({f"m{n}": m, "out": out})
            tape["blocks"].append(rec)
            x, Hc, Wc, Cin = out, Hn, Wn, C
        tape["feat"] = x
        tape["hw"] = (Hc, Wc)
        tape["C"] = Cin
        self._tape = tape
        return x, Hc, Wc

    def backbone_infer(self, image: torch.Tensor):
        """Eval-mode backbone forward: image fp32 NCHW [B,3,H,W] -> NHWC bf16 feature matrix [B*h*w, C].
        Every BN is the fixed per-channel affine map of its running statistics, applied by the epilogue of the GEMM
        that produces its input (VtxGemm.col_scale / col_shift), together with the shortcut and the ReLU: no raw conv
        output is stored and read back.  Writes no tape and no statistics; its buffers are its own, so a training
        tape stays intact.  The result is overwritten by the next call."""
        if not self._weights_fresh or not self._eval_bn_fresh:
            self.prepare_weights(eval_bn=True)
        B, _, H, W = image.shape
        s = _stream()
        ws = self.ws

        def ss(bn_name):  # scale and shift rows of the eval bnp
            bnp = ws.flat["bnp_eval:" + bn_name]
            C = bnp.numel() // 4
            return dict(col_scale=bnp[2 * C:3 * C], col_shift=bnp[3 * C:4 * C])

        # ---- stem: GEMM -> BN + ReLU + maxpool, as in backbone_forward
        Ho, Wo = (H + 6 - 7) // 2 + 1, (W + 6 - 7) // 2 + 1
        M0 = B * Ho * Wo
        y0 = ws.get("inf.stem.y", (M0, 64), BF16)
        self._stem_conv(image, y0, Ho, Wo, "inf.")
        Hp, Wp = (Ho - 1) // 2 + 1, (Wo - 1) // 2 + 1
        x = ws.get("inf.x1", (B * Hp * Wp, 64), BF16)
        idx = ws.get("inf.stem.idx", (B * Hp * Wp, 64), torch.uint8)
        call("vtx_bn_relu_maxpool", y0.data_ptr(), ws.flat["bnp_eval:visual.cnn.bn1"].data_ptr(), x.data_ptr(),
             idx.data_ptr(), B, Ho, Wo, 64, s)
        Hc, Wc = Hp, Wp
        # ---- residual blocks: each GEMM ends in its BN (+ shortcut) (+ ReLU): every conv but the last, the downsample,
        # then the last conv with the shortcut; block outputs alternate between two buffers
        for bi, (name, blk) in enumerate(self.blocks):
            convs = self._convs[name]
            n, C = len(convs), convs[-1].cout
            stride = blk.stride
            Hn, Wn = (Hc - 1) // stride + 1, (Wc - 1) // stride + 1
            Mout = B * Hn * Wn
            a, h, w = x, Hc, Wc
            for i, conv in enumerate(convs[:-1], 1):
                ho, wo = (h - 1) // conv.stride + 1, (w - 1) // conv.stride + 1
                y = ws.get(f"inf.a{i}", (B * ho * wo, conv.cout), BF16)
                self._conv(conv, a, y, B, h, w, f"inf.cols{i}", act=1, **ss(f"{name}.bn{i}"))
                a, h, w = y, ho, wo
            shortcut = x
            if blk.downsample is not None:
                shortcut = ws.get("inf.shortcut", (Mout, C), BF16)
                self._downsample(name, x, shortcut, B, Hc, Wc, stride, "inf.xs", **ss(name + ".downsample.1"))
            out = ws.get(f"inf.x{bi & 1}", (Mout, C), BF16)
            self._conv(convs[-1], a, out, B, h, w, f"inf.cols{n}", residual=shortcut, act=1, **ss(f"{name}.bn{n}"))
            x, Hc, Wc = out, Hn, Wn
        return x, Hc, Wc

    # ------------------------------------------------------------------------------------------------ backbone bwd
    def _wgrad(self, dY, X, dW, n_out, k_in, m_rows):
        """dW[n_out, k_in] (fp32, += ) = dY[m_rows, n_out]^T . X[m_rows, k_in]   (both operands MN-major, split-K)."""
        tiles = ((n_out + 127) // 128) * ((k_in + 255) // 256)
        sk = ops.split_k_for(tiles, (m_rows + 63) // 64)
        gemm(dY, X, dW, n_out, k_in, m_rows, a_mn=1, b_mn=1, atomic=True, split_k=sk, ldd=k_in, out_f32=True)

    def _bn_bwd(self, dA, a, y, bnp, bn_name, M, C, dy, two=None, dz_out=None, mask_from_y=0, sums=None):
        """dA -> dy through (ReLU from the bit mask `a`, or recomputed from y when mask_from_y) + train-mode BN;
        two = (y2, bnp2, bn2_name, dy2) shares dz.  `sums`: the [2, C] reduction already accumulated by the epilogue of
        the GEMM that produced dA (VtxGemm.bnr_*), so only the apply pass is left."""
        s = _stream()
        fused = sums is not None
        if not fused:
            sums = self._slab_take(2 * C)
        if two is None:
            if not fused:
                call("vtx_bn_bwd_reduce", dA.data_ptr(), _p(a), y.data_ptr(), bnp.data_ptr(), 0, 0, sums.data_ptr(), 0,
                     M, C, mask_from_y, s)
            call("vtx_bn_bwd_finalize_apply", sums.data_ptr(), 0, float(M), self.G(bn_name + ".weight").data_ptr(),
                 self.G(bn_name + ".bias").data_ptr(), 0, 0, dA.data_ptr(), _p(a), y.data_ptr(), bnp.data_ptr(),
                 dy.data_ptr(), 0, 0, 0, _p(dz_out), M, C, mask_from_y, s)
        else:
            y2, bnp2, bn2_name, dy2 = two
            sums2 = self._slab_take(2 * C)
            call("vtx_bn_bwd_reduce", dA.data_ptr(), _p(a), y.data_ptr(), bnp.data_ptr(), y2.data_ptr(),
                 bnp2.data_ptr(), sums.data_ptr(), sums2.data_ptr(), M, C, mask_from_y, s)
            call("vtx_bn_bwd_finalize_apply", sums.data_ptr(), sums2.data_ptr(), float(M),
                 self.G(bn_name + ".weight").data_ptr(), self.G(bn_name + ".bias").data_ptr(),
                 self.G(bn2_name + ".weight").data_ptr(), self.G(bn2_name + ".bias").data_ptr(), dA.data_ptr(), _p(a),
                 y.data_ptr(), bnp.data_ptr(), dy.data_ptr(), y2.data_ptr(), bnp2.data_ptr(), dy2.data_ptr(),
                 _p(dz_out), M, C, mask_from_y, s)

    def _conv_wgrad(self, conv, dy, x, cols, B, Hc, Wc):
        """Weight gradient of main-branch conv `conv` from dy [Mout, C] and its input x [B*Hc*Wc, Cin]: a 1x1 conv's
        straight into the gradient arena; a 3x3 conv's into its fp32 scratch _dwp [C, 9 * Cin] (fp32 atomics), from
        the forward's im2col matrix `cols` when that route ran, else by an implicit GEMM over x."""
        wname, k, stride, Cin, C = conv
        Mout = dy.shape[0]
        if k == 1:
            self._wgrad(dy, x, self.G(wname + ".weight"), C, Cin, Mout)
            return
        dwp = self._dwp[wname].view(C, 9 * Cin)
        if cols is not None:
            self._wgrad(dy, cols, dwp, C, 9 * Cin, Mout)
        elif _transposed_wgrad(Cin, C, stride):
            # wgrad in the [(tap, cin), cout] layout (vtx_conv_w_unpack_add_t folds it into OIHW)
            gemm(dy, x, dwp, 9 * Cin, C, Mout, atomic=True, lda=C, ldb=Cin, ldd=C, conv=(B, Hc, Wc, Cin), conv_mode=4,
                 out_f32=True)
        else:
            tiles = ((C + 127) // 128) * ((9 * Cin + 255) // 256)
            sk = ops.split_k_for(tiles, (Mout + 63) // 64)
            gemm(dy, x, dwp, C, 9 * Cin, Mout, atomic=True, split_k=sk, lda=C, ldb=Cin, conv=(B, Hc, Wc, Cin),
                 conv_mode=2, out_f32=True, conv_stride=stride)

    def _conv_dgrad(self, conv, dy, dx, cols, B, Hc, Wc, **epi):
        """Input gradient dx [B*Hc*Wc, Cin] of main-branch conv `conv` from dy [Mout, C], by the route _dgrad_route
        picks.  `epi` (bnr, residual, residual_mask; None entries are dropped) goes to the epilogue of the GEMM that
        writes dx; a route that cannot carry it raises."""
        wname, k, stride, Cin, C = conv
        epi = {key: v for key, v in epi.items() if v is not None}
        route = _dgrad_route(conv, cols)
        if route == "col2im" and epi or route == "parity" and set(epi) - {"bnr"}:
            raise ValueError(f"the {route} dgrad of {wname} has no epilogue for {sorted(epi)}")
        Mout, Min = dy.shape[0], dx.shape[0]
        if route == "gemm":
            gemm(dy, self.W(wname + ".weight").view(C, Cin), dx, Min, Cin, C, b_mn=1, **epi)
        elif route == "implicit":
            gemm(dy, self._packed[wname + ".weight#dgrad"], dx, Min, Cin, 9 * C, lda=C, conv=(B, Hc, Wc, C),
                 conv_mode=1, **epi)
        elif route == "parity":
            self._dgrad3x3_s2(dy, wname, dx, B, Hc, Wc, **epi)
        else:
            dcols = self.ws.get("bwd.dcols", (Mout, 9 * Cin), BF16)
            gemm(dy, self._packed[wname + ".weight"], dcols, Mout, 9 * Cin, C, b_mn=1)
            call("vtx_col2im3x3", dcols.data_ptr(), dx.data_ptr(), B, Hc, Wc, Cin, stride, _stream())

    def _dgrad3x3_s2(self, dy, wname, dx, B, Hc, Wc, bnr=None):
        """Input gradient dx [B*Hc*Wc, Cin] of a stride-2 3x3 conv from dy [Mout, C] as four implicit GEMMs, one per
        parity class (ph, pw) of the input position: row 2i+ph of dx gathers dy rows i+a, a < 1+ph, through kernel rows
        ph+1-2a (same along w); each class writes its own strided sub-grid of dx, so every element is written exactly
        once -- no per-tap gradient matrix, no col2im scatter.  bnr = (y, bnp, sums, None): the BN-backward sums of the
        BN whose output gradient dx is, accumulated by the epilogues (ReLU mask recomputed from y)."""
        Mout, C = dy.shape
        Cin = dx.shape[1]
        Hn, Wn = (Hc - 1) // 2 + 1, (Wc - 1) // 2 + 1
        for ph in (0, 1):
            for pw in (0, 1):
                th, tw = 1 + ph, 1 + pw
                Hs, Ws = (Hc - ph + 1) // 2, (Wc - pw + 1) // 2
                if Hs <= 0 or Ws <= 0:
                    continue
                voff = (ph * Wc + pw) * Cin * 2
                epi = {} if bnr is None else dict(bnr=(*bnr, bnr[0].data_ptr() + voff))
                gemm(dy, self._packed[f"{wname}.weight#dgrad_s2_{ph}{pw}"], dx, Mout, Cin, th * tw * C, lda=C,
                     conv=(B, Hn, Wn, C), conv_mode=1, tap_grid=(th, tw, 0), d_ptr=dx.data_ptr() + voff,
                     out_view=(Hs, Ws, 2 * Cin, 2 * Wc * Cin, Hc * Wc * Cin), **epi)

    def _downsample_wgrad(self, rec, dyd, B):
        """Weight gradient of block rec's 1x1 shortcut conv from its output gradient dyd [Mout, C4]."""
        name, Mout, C4, Cin = rec["name"], rec["Mout"], rec["Cout"], rec["Cin"]
        if rec["xs"] is not None:
            self._wgrad(dyd, rec["xs"], self.G(name + ".downsample.0.weight"), C4, Cin, Mout)
        else:  # one-tap implicit wgrad over the strided view of x, straight into the [C4, Cin, 1, 1] gradient
            tiles = ((C4 + 127) // 128) * ((Cin + 255) // 256)
            gemm(dyd, rec["x"], self.G(name + ".downsample.0.weight").view(C4, Cin), C4, Cin, Mout, atomic=True,
                 split_k=ops.split_k_for(tiles, (Mout + 63) // 64), lda=C4, ldb=Cin, conv=(B, rec["Hin"], rec["Win"], Cin),
                 conv_mode=2, conv_stride=rec["stride"], conv_taps=1, out_f32=True)

    def _downsample_dgrad_add(self, rec, dyd, dx, B):
        """dx [Min, Cin] += the input gradient of block rec's 1x1 shortcut conv, from dyd [Mout, C4]."""
        name, Min, Mout, C4, Cin, stride = rec["name"], rec["Min"], rec["Mout"], rec["Cout"], rec["Cin"], rec["stride"]
        Hc, Wc = rec["Hin"], rec["Win"]
        if stride == 1:
            gemm(dyd, self.W(name + ".downsample.0.weight").view(C4, Cin), dx, Min, Cin, C4, b_mn=1, residual=dx)
        elif stride == 2 and rec["xs"] is None:
            # dx[:, ::2, ::2] += dyd . Wd: one-tap implicit GEMM over the dyd grid whose output (and residual) is
            # the even-position sub-grid of dx -- in-place accumulation, no dxs buffer, no upsample_add pass
            gemm(dyd, self._packed[name + ".downsample.0.weight#t"], dx, Mout, Cin, C4, lda=C4,
                 conv=(B, rec["Hout"], rec["Wout"], C4), conv_mode=1, conv_taps=1, residual=dx, d_ptr=dx.data_ptr(),
                 out_view=((Hc + 1) // 2, (Wc + 1) // 2, 2 * Cin, 2 * Wc * Cin, Hc * Wc * Cin))
        else:
            dxs = self.ws.get("bwd.dxs", (Mout, Cin), BF16)
            gemm(dyd, self.W(name + ".downsample.0.weight").view(C4, Cin), dxs, Mout, Cin, C4, b_mn=1)
            call("vtx_upsample_add", dxs.data_ptr(), dx.data_ptr(), B, Hc, Wc, Cin, stride, _stream())

    def backbone_backward(self, dfeat: torch.Tensor, bucket_cb=None):
        """dfeat bf16 [B*h*w, C]: gradient w.r.t. the backbone output.  Accumulates into the gradient arena.
        `bucket_cb(tag)` is called when every gradient of 'layer4' / 'layer3' / 'layer2' has been enqueued."""
        tape = self._tape
        if getattr(self.visual, "frozen", False):
            return  # frozen backbone: no parameter gradients, nothing below the visual projection
        if not tape["training"]:
            raise RuntimeError("backward through eval-mode BatchNorm (running statistics) is not implemented")
        B = tape["B"]
        s = _stream()
        ws = self.ws
        dOut = dfeat
        scratch_i = 0
        prev_layer = None
        self._dwp_flat.zero_()
        stem_s2d = tape["stem"]["s2d"] is not None
        blocks = tape["blocks"]
        sums_out = None  # the current block's last-BN sums when the GEMM that produced dOut already accumulated them
        for bi in range(len(blocks) - 1, -1, -1):
            rec = blocks[bi]
            name, Cin = rec["name"], rec["Cin"]
            layer = name.split(".")[2]
            if prev_layer is not None and layer != prev_layer:
                self._run_jobs("unpack:" + prev_layer, lambda: self._unpack_rows(prev_layer, stem_s2d))
                if bucket_cb is not None:
                    bucket_cb(prev_layer)
            prev_layer = layer
            convs = self._convs[name]
            n, Min, Mout, C = len(convs), rec["Min"], rec["Mout"], rec["Cout"]
            # ---- block output: ReLU mask + the last BN (+ downsample BN) backward
            dy = ws.get(f"bwd.dy{n}", (Mout, C), BF16)
            m, y, bnp, bn_name = rec[f"m{n}"], rec[f"y{n}"], rec[f"bnp{n}"], f"{name}.bn{n}"
            if rec["has_ds"]:
                dyd = ws.get("bwd.dyd", (Mout, C), BF16)
                self._bn_bwd(dOut, m, y, bnp, bn_name, Mout, C, dy,
                             two=(rec["yd"], rec["bnpd"], name + ".downsample.1", dyd))
            else:
                # the shortcut gradient dz = dOut * [block output > 0] is never written: conv1's dgrad epilogue adds
                # dOut under the same bit mask (VtxGemm.residual_mask)
                self._bn_bwd(dOut, m, y, bnp, bn_name, Mout, C, dy, sums=sums_out)
            sums_out = None
            # ---- conv n .. conv2: wgrad + dgrad, whose epilogue accumulates the backward sums of the BN before it
            # (ReLU mask recomputed from its y) wherever the route allows; then that BN's backward
            for i in range(n, 1, -1):
                conv, cols, (h, w) = convs[i - 1], rec[f"cols{i}"], rec[f"hw{i}"]
                y, bnp = rec[f"y{i - 1}"], rec[f"bnp{i - 1}"]
                self._conv_wgrad(conv, dy, rec[f"a{i - 1}"], cols, B, h, w)
                da = ws.get(f"bwd.da{i - 1}", y.shape, BF16)
                sums = self._slab_take(2 * conv.cin) if _dgrad_route(conv, cols) != "col2im" else None
                self._conv_dgrad(conv, dy, da, cols, B, h, w, bnr=None if sums is None else (y, bnp, sums, None))
                dy = ws.get(f"bwd.dy{i - 1}", y.shape, BF16)
                self._bn_bwd(da, None, y, bnp, f"{name}.bn{i - 1}", y.shape[0], conv.cin, dy, mask_from_y=1, sums=sums)
            # ---- conv1: wgrad + dgrad (+ shortcut gradient)
            conv, cols, (h, w) = convs[0], rec["cols1"], rec["hw1"]
            self._conv_wgrad(conv, dy, rec["x"], cols, B, h, w)
            dx = ws.get(f"bwd.dx{scratch_i & 1}", (Min, Cin), BF16)
            scratch_i += 1
            if rec["has_ds"]:
                self._downsample_wgrad(rec, dyd, B)
                self._conv_dgrad(conv, dy, dx, cols, B, h, w)
                self._downsample_dgrad_add(rec, dyd, dx, B)
            else:
                # dx is the output gradient of the previous block: when that block has a single-branch last BN, its
                # backward sums (ReLU bit mask of THAT block) are accumulated here, over the staged dx tiles
                prev = blocks[bi - 1] if bi > 0 else None
                bnr = None
                if prev is not None and not prev["has_ds"] and Cin % 32 == 0 and Min >= self.fuse_bn3_min_rows:
                    p = len(self._convs[prev["name"]])
                    sums_out = self._slab_take(2 * Cin)
                    bnr = (prev[f"y{p}"], prev[f"bnp{p}"], sums_out, prev[f"m{p}"])
                self._conv_dgrad(conv, dy, dx, cols, B, h, w, residual=dOut, residual_mask=rec[f"m{n}"], bnr=bnr)
            dOut = dx
        # ---- stem: maxpool bwd -> ReLU/BN bwd -> wgrad
        st = tape["stem"]
        M0 = st["M"]
        da0 = ws.get("bwd.da0", (M0, 64), BF16)
        call("vtx_maxpool_bwd", dOut.data_ptr(), st["idx"].data_ptr(), da0.data_ptr(), B, st["Ho"], st["Wo"], 64, s)
        dy0 = ws.get("bwd.dy0", (M0, 64), BF16)
        self._bn_bwd(da0, None, st["y"], st["bnp"], "visual.cnn.bn1", M0, 64, dy0, mask_from_y=1)
        if stem_s2d:  # implicit wgrad over the space-to-depth view
            dwx = self._dwp["visual.cnn.conv1"].view(64, 256)
            gemm(dy0, st["s2d"], dwx, 64, 256, M0, lda=64, ldb=64, atomic=True, out_f32=True,
                 split_k=ops.split_k_for(1, M0 // 64), conv=(B, st["Ho"], st["Wo"], 64), conv_mode=6)
        else:
            dwp0 = self._dwp["visual.cnn.conv1"][:64 * 160].view(64, 160)
            self._wgrad(dy0, st["cols"], dwp0, 64, 160, M0)
        # layer1's 3x3 weight gradients + the stem's, in one launch (the 'rest' all-reduce bucket follows)
        self._run_jobs("unpack:rest:" + ("s2d" if stem_s2d else "cols"), lambda: self._unpack_rows("rest", stem_s2d))

    # ------------------------------------------------------------------------------------------------ head
    def _head_modules(self, direction):
        return self.textual if direction == "textual" else self.backward_textual

    def visual_projection_forward(self, feat, S):
        """mem[S,H] = feat[S,Cv] . Wvp^T + b   (computed once, shared by both directions)."""
        H = self.textual.hidden_size
        mem = self.ws.get("head.mem", (S, H), BF16)
        gemm(feat, self.W("textual.visual_projection.weight"), mem, S, H, feat.shape[1],
             bias=self.P("textual.visual_projection.bias"))
        return mem

    def head_forward(self, direction, mem, tokens, lengths, training, want_logits_f32=False):
        """tokens int64 [B,T] -> bf16 logits [B*T, V] (and the tape for backward)."""
        mod = self._head_modules(direction)
        B, T = tokens.shape
        M, H, Fd, V, A = B * T, mod.hidden_size, mod.feedforward_size, mod.vocab_size, mod.attention_heads
        S = mem.shape[0]
        p = float(mod.dropout) if training else 0.0
        d = direction
        di = 0 if d == "textual" else 1
        # self-attention mask: 1 = future + key padding (captioning), 2 = key padding only (masked language modelling)
        mm = 1 if mod.mask_future_positions else 2
        s = _stream()
        ws = self.ws
        seed = self.seed.data_ptr()
        site = di * 1000
        rec = dict(direction=d, B=B, T=T, M=M, S=S, Sk=S // B, H=H, A=A, Fd=Fd, p=p, layers=[], tokens=tokens,
                   lengths=lengths, mem=mem, mask_mode=mm)
        emb = "textual.embedding."
        z0 = ws.get(d + ".z0", (M, H), F32)
        st0 = ws.get(d + ".st0", (M, 2), F32)
        x = ws.get(d + ".x0", (M, H), F32)
        xb = ws.get(d + ".x0b", (M, H), BF16)
        call("vtx_embed_fwd", tokens.data_ptr(), self.P(emb + "words.weight").data_ptr(),
             self.P(emb + "positions.weight").data_ptr(), self.P(emb + "layer_norm.weight").data_ptr(),
             self.P(emb + "layer_norm.bias").data_ptr(), z0.data_ptr(), st0.data_ptr(), x.data_ptr(), xb.data_ptr(),
             M, T, H, self.pad, 1e-8, p, seed, site, s)
        rec.update(z0=z0, st0=st0)
        for l in range(mod.num_layers):
            k = f"{d}.L{l}."
            lr = dict(q=f"{d}.transformer.layers.{l}.", k=k, sb=site + 10 * (l + 1))
            pr = ws.get(k + "proj", (M, H), BF16)
            for i, sublayer in enumerate((self._self_attn_fwd, self._cross_attn_fwd, self._ffn_fwd), 1):
                z, st = ws.get(f"{k}z{i}", (M, H), F32), ws.get(f"{k}st{i}", (M, 2), F32)
                xo = ws.get(f"{k}x{i}", (M, H), F32)
                xb_out = ws.get(f"{k}n{i}b" if mod.norm_first else f"{k}x{i}b", (M, H), BF16)
                site_i = lr["sb"] + 2 * i - 1  # the branch's dropout before the residual add
                xb = self._residual_sublayer(mod.norm_first, f"{lr['q']}norm{i}.",
                                             lambda inp, out: sublayer(rec, lr, inp, out), x, xb, xo, xb_out, pr, z, st,
                                             M, H, p, site_i)
                x = xo
                lr.update({f"z{i}": z, f"st{i}": st})
            rec["layers"].append(lr)
        if mod.norm_first:  # final LayerNorm of pre-norm decoders (textual_heads.py:192-193)
            qn = f"{d}.transformer.norm."
            zf, stf = ws.get(d + ".zf", (M, H), F32), ws.get(d + ".stf", (M, 2), F32)
            xb = ws.get(d + ".xfb", (M, H), BF16)
            call("vtx_add_ln_fwd", x.data_ptr(), 0, self.P(qn + "weight").data_ptr(), self.P(qn + "bias").data_ptr(),
                 zf.data_ptr(), stf.data_ptr(), 0, xb.data_ptr(), M, H, 1e-5, 0.0, seed, 0, 1, s)
            rec.update(zf=zf, stf=stf)
        rec["x_out_b"] = xb
        # tied output projection
        wv = self.W("textual.embedding.words.weight")
        bo = self.P("textual.output.bias")
        if want_logits_f32:
            lf = ws.get(d + ".logits_f32", (M, V), F32)
            gemm(xb, wv, lf, M, V, H, bias=bo)
            rec["logits_f32"] = lf
        logits = ws.get(d + ".logits", (M, V), BF16)
        gemm(xb, wv, logits, M, V, H, bias=bo)
        rec["logits"] = logits
        return rec

    def _residual_sublayer(self, norm_first, norm, run, x, xb, xo, xb_out, pr, z, st, M, H, p, site):
        """One residual sublayer of a decoder layer, fp32 residual stream x [M, H] (bf16 shadow xb) -> xo, where
        `run(inp, pr)` writes the branch f(inp) of the bf16 input to pr and `norm` names the sublayer's LayerNorm.
        Pre-norm: xo = x + dropout(f(LN(x))), LN(x) in xb_out.  Post-norm: xo = LN(x + dropout(f(x))), its bf16 shadow
        in xb_out (the next sublayer's input).  z / st receive the LayerNorm's input and statistics; returns xb_out."""
        s, seed = _stream(), self.seed.data_ptr()
        w, b = self.P(norm + "weight").data_ptr(), self.P(norm + "bias").data_ptr()
        if norm_first:  # torch/nn/modules/transformer.py:1131-1143
            call("vtx_add_ln_fwd", x.data_ptr(), 0, w, b, z.data_ptr(), st.data_ptr(), 0, xb_out.data_ptr(), M, H, 1e-5,
                 0.0, seed, 0, 1, s)
            run(xb_out, pr)
            call("vtx_add_ln_fwd", x.data_ptr(), pr.data_ptr(), 0, 0, xo.data_ptr(), 0, 0, 0, M, H, 0.0, p, seed, site, 0,
                 s)
        else:
            run(xb, pr)
            call("vtx_add_ln_fwd", x.data_ptr(), pr.data_ptr(), w, b, z.data_ptr(), st.data_ptr(), xo.data_ptr(),
                 xb_out.data_ptr(), M, H, 1e-5, p, seed, site, 1, s)
        return xb_out

    def _attn_fwd(self, rec, q, k, v, o, lse, Tk, lengths, mask_mode, site):
        """Multi-head attention of the T query rows of each caption over its Tk key rows.  q, k, v, o: row-major views
        (column slices of a fused projection are fine) whose leading dimensions are their row strides."""
        call("vtx_attn_fwd", q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
             o.data_ptr(), o.stride(0), lse.data_ptr(), rec["B"], rec["A"], rec["T"], Tk, _p(lengths), mask_mode,
             rec["p"], self.seed.data_ptr(), site, _stream())

    def _attn_bwd(self, rec, q, k, v, do, lse, dq, dk, dv, Tk, lengths, mask_mode, site):
        """Backward of _attn_fwd: dq, dk, dv (views as q, k, v) from do and the forward's log-sum-exp rows."""
        call("vtx_attn_bwd", q.data_ptr(), q.stride(0), k.data_ptr(), k.stride(0), v.data_ptr(), v.stride(0),
             do.data_ptr(), do.stride(0), lse.data_ptr(), dq.data_ptr(), dq.stride(0), dk.data_ptr(), dk.stride(0),
             dv.data_ptr(), dv.stride(0), rec["B"], rec["A"], rec["T"], Tk, _p(lengths), mask_mode, rec["p"],
             self.seed.data_ptr(), site, _stream())

    # The three sublayers of a decoder layer.  Each forward reads the bf16 [M, H] input `x` (post-norm: the previous
    # LayerNorm's bf16 shadow; pre-norm: the sublayer's own LayerNorm output), writes its branch output to `out` and
    # keeps what its backward needs in the layer tape `lr`.  Each backward goes from the bf16 branch gradient `dy` to
    # the gradient `dx` of that input and accumulates the parameter gradients.
    def _self_attn_fwd(self, rec, lr, x, out):
        M, H, q, k = rec["M"], rec["H"], lr["q"] + "self_attn.", lr["k"]
        qkv = self.ws.get(k + "qkv", (M, 3 * H), BF16)
        gemm(x, self.W(q + "in_proj_weight"), qkv, M, 3 * H, H, bias=self.P(q + "in_proj_bias"))
        o = self.ws.get(k + "o_s", (M, H), BF16)
        lse = self.ws.get(k + "lse_s", (_lse_rows(rec["B"], rec["A"], rec["T"]),), F32)
        self._attn_fwd(rec, *qkv.split(H, 1), o, lse, rec["T"], rec["lengths"], rec["mask_mode"], lr["sb"])
        gemm(o, self.W(q + "out_proj.weight"), out, M, H, H, bias=self.P(q + "out_proj.bias"))
        lr.update(x_s=x, qkv=qkv, o_s=o, lse_s=lse)

    def _self_attn_bwd(self, rec, lr, dy, dx):
        M, H, q = rec["M"], rec["H"], lr["q"] + "self_attn."
        do = self.ws.get("hb.do", (M, H), BF16)
        self._linear_bwd(dy, lr["o_s"], q + "out_proj.weight", q + "out_proj.bias", do, M, H, H)
        dqkv = self.ws.get("hb.dqkv", (M, 3 * H), BF16)
        self._attn_bwd(rec, *lr["qkv"].split(H, 1), do, lr["lse_s"], *dqkv.split(H, 1), rec["T"], rec["lengths"],
                       rec["mask_mode"], lr["sb"])
        self._linear_bwd(dqkv, lr["x_s"], q + "in_proj_weight", q + "in_proj_bias", dx, M, 3 * H, H)

    def _cross_attn_fwd(self, rec, lr, x, out):
        M, H, S, q, k = rec["M"], rec["H"], rec["S"], lr["q"] + "multihead_attn.", lr["k"]
        w, b = self.W(q + "in_proj_weight"), self.P(q + "in_proj_bias")
        qc = self.ws.get(k + "qc", (M, H), BF16)
        gemm(x, w[:H], qc, M, H, H, bias=b[:H])
        kv = self.ws.get(k + "kv", (S, 2 * H), BF16)
        gemm(rec["mem"], w[H:], kv, S, 2 * H, H, bias=b[H:])
        o = self.ws.get(k + "o_c", (M, H), BF16)
        lse = self.ws.get(k + "lse_c", (_lse_rows(rec["B"], rec["A"], rec["T"]),), F32)
        self._attn_fwd(rec, qc, *kv.split(H, 1), o, lse, rec["Sk"], None, 0, lr["sb"] + 2)
        gemm(o, self.W(q + "out_proj.weight"), out, M, H, H, bias=self.P(q + "out_proj.bias"))
        lr.update(x_c=x, qc=qc, kv=kv, o_c=o, lse_c=lse)

    def _cross_attn_bwd(self, rec, lr, dy, dx, dmem, dmem_started):
        """Also adds the gradient of the visual memory to dmem [S, H] (overwrites it while not dmem_started)."""
        M, H, S, q = rec["M"], rec["H"], rec["S"], lr["q"] + "multihead_attn."
        do = self.ws.get("hb.do", (M, H), BF16)
        self._linear_bwd(dy, lr["o_c"], q + "out_proj.weight", q + "out_proj.bias", do, M, H, H)
        dqc = self.ws.get("hb.dqc", (M, H), BF16)
        dkv = self.ws.get("hb.dkv", (S, 2 * H), BF16)
        self._attn_bwd(rec, lr["qc"], *lr["kv"].split(H, 1), do, lr["lse_c"], dqc, *dkv.split(H, 1), rec["Sk"], None, 0,
                       lr["sb"] + 2)
        wn, bn = q + "in_proj_weight", q + "in_proj_bias"
        self._linear_bwd(dqc, lr["x_c"], wn, bn, dx, M, H, H, w_rows=slice(0, H))
        self._linear_bwd(dkv, rec["mem"], wn, bn, dmem, S, 2 * H, H, w_rows=slice(H, 3 * H),
                         residual=dmem if dmem_started else None)

    def _ffn_fwd(self, rec, lr, x, out):
        M, H, Fd, q, k = rec["M"], rec["H"], rec["Fd"], lr["q"], lr["k"]
        u = self.ws.get(k + "u", (M, Fd), BF16)
        gemm(x, self.W(q + "linear1.weight"), u, M, Fd, H, bias=self.P(q + "linear1.bias"))
        h = self.ws.get(k + "h", (M, Fd), BF16)
        call("vtx_gelu_dropout_fwd", u.data_ptr(), h.data_ptr(), M * Fd, rec["p"], self.seed.data_ptr(), lr["sb"] + 4,
             _stream())
        gemm(h, self.W(q + "linear2.weight"), out, M, H, Fd, bias=self.P(q + "linear2.bias"))
        lr.update(x_f=x, u=u, h=h)

    def _ffn_bwd(self, rec, lr, dy, dx):
        M, H, Fd, q = rec["M"], rec["H"], rec["Fd"], lr["q"]
        dh = self.ws.get("hb.dh", (M, Fd), BF16)
        self._linear_bwd(dy, lr["h"], q + "linear2.weight", q + "linear2.bias", dh, M, H, Fd)
        call("vtx_gelu_dropout_bwd", dh.data_ptr(), lr["u"].data_ptr(), dh.data_ptr(), M * Fd, rec["p"],
             self.seed.data_ptr(), lr["sb"] + 4, _stream())
        self._linear_bwd(dh, lr["x_f"], q + "linear1.weight", q + "linear1.bias", dx, M, Fd, H)

    def head_loss(self, rec, write_grad, labels=None):
        """Token-mean cross entropy (ignore_index = pad).  labels None: next-token targets tokens[:, 1:] against
        logits[:, :-1] (captioning.py:111-114); labels [B,T]: one label per position (masked_lm.py:68-72)."""
        di = 0 if rec["direction"] == "textual" else 1
        s = _stream()
        V = rec["logits"].shape[1]
        tgt, shift = (rec["tokens"], 1) if labels is None else (labels, 0)
        call("vtx_count_valid", tgt.data_ptr(), rec["B"], rec["T"], self.pad, shift, self.count[di:].data_ptr(), s)
        call("vtx_cross_entropy", rec["logits"].data_ptr(), V, tgt.data_ptr(), rec["B"], rec["T"], V, self.pad, shift,
             self.count[di:].data_ptr(), self.loss[di:].data_ptr(), int(write_grad), s)

    def _linear_bwd(self, dY, X, wname, bname, dX, M, n_out, k_in, w_rows=None, residual=None):
        """Backward of Y = X W^T + b for W [n_out, k_in] (optionally the row slice `w_rows` of a packed weight)."""
        W, dW, db = self.W(wname), self.G(wname), self.G(bname)
        if w_rows is not None:
            W, dW, db = W[w_rows], dW[w_rows], db[w_rows]
        self._linear_bwd_t(dY, X, W, dW, db, dX, M, n_out, k_in, residual)

    def _linear_bwd_t(self, dY, X, W, dW, db, dX, M, n_out, k_in, residual=None):
        """The same for explicit tensors: bf16 W [n_out, k_in]; fp32 dW, db accumulated into."""
        call("vtx_colsum", dY.data_ptr(), dY.stride(0), M, n_out, db.data_ptr(), _stream())
        self._wgrad(dY, X, dW, n_out, k_in, M)
        if dX is not None:
            gemm(dY, W, dX, M, k_in, n_out, b_mn=1, residual=residual)

    def head_backward(self, rec, dmem, dmem_started):
        """Backward of one direction from the dlogits already written in place of rec['logits'].
        Accumulates parameter gradients; adds this direction's contribution to dmem [S,H]."""
        d = rec["direction"]
        mod = self._head_modules(d)
        T, M, H, p = rec["T"], rec["M"], rec["H"], rec["p"]
        V = mod.vocab_size
        s = _stream()
        ws = self.ws
        seed = self.seed.data_ptr()
        dlog = rec["logits"]
        # tied output projection: d_bias, d_words (vocab-projection part), dx
        call("vtx_colsum", dlog.data_ptr(), V, M, V, self.G("textual.output.bias").data_ptr(), s)
        self._wgrad(dlog, rec["x_out_b"], self.G("textual.embedding.words.weight"), V, H, M)
        dxb = ws.get("hb.dxb", (M, H), BF16)
        gemm(dlog, self.W("textual.embedding.words.weight"), dxb, M, H, V, b_mn=1)
        dres_a = ws.get("hb.dres_a", (M, H), F32)
        dres_b = ws.get("hb.dres_b", (M, H), F32)
        dbr = ws.get("hb.dbr", (M, H), BF16)
        dy_a, dy_b = None, dxb  # gradient of the residual stream: fp32 part, bf16 part (of a bf16 shadow's reader)
        if mod.norm_first:
            qn = f"{d}.transformer.norm."
            call("vtx_ln_bwd", 0, dxb.data_ptr(), rec["zf"].data_ptr(), rec["stf"].data_ptr(),
                 self.P(qn + "weight").data_ptr(), 0, dres_a.data_ptr(), 0, self.G(qn + "weight").data_ptr(),
                 self.G(qn + "bias").data_ptr(), M, H, 0.0, seed, 0, 1, s)
            dy_a, dy_b = dres_a, None
        for l in reversed(range(mod.num_layers)):
            lr = rec["layers"][l]
            for i in (3, 2, 1):
                norm = f"{lr['q']}norm{i}."
                w, dw, db = (self.P(norm + "weight").data_ptr(), self.G(norm + "weight").data_ptr(),
                             self.G(norm + "bias").data_ptr())
                z, st = lr[f"z{i}"].data_ptr(), lr[f"st{i}"].data_ptr()
                site_i = lr["sb"] + 2 * i - 1
                if mod.norm_first:  # d(branch) = g * dropout mask (bf16); g itself keeps flowing through the skip path
                    call("vtx_ln_bwd", dres_a.data_ptr(), 0, 0, 0, 0, 0, 0, dbr.data_ptr(), 0, 0, M, H, p, seed, site_i,
                         0, s)
                else:  # through LN(x + dropout(branch)): fp32 gradient of x, bf16 gradient of the branch
                    dres = dres_b if i == 2 else dres_a
                    call("vtx_ln_bwd", _p(dy_a), _p(dy_b), z, st, w, 0, dres.data_ptr(), dbr.data_ptr(), dw, db, M, H,
                         p, seed, site_i, 1, s)
                    dy_a, dy_b = dres, dxb
                if i == 3:
                    self._ffn_bwd(rec, lr, dbr, dxb)
                elif i == 2:
                    self._cross_attn_bwd(rec, lr, dbr, dxb, dmem, dmem_started)
                    dmem_started = True
                else:
                    self._self_attn_bwd(rec, lr, dbr, dxb)
                if mod.norm_first:  # g += LN_backward(dxb)
                    call("vtx_ln_bwd", 0, dxb.data_ptr(), z, st, w, dres_a.data_ptr(), dres_a.data_ptr(), 0, dw, db, M,
                         H, 0.0, seed, 0, 1, s)
        emb = "textual.embedding."
        di = 0 if d == "textual" else 1
        call("vtx_embed_bwd", _p(dy_a), _p(dy_b), rec["tokens"].data_ptr(), rec["z0"].data_ptr(),
             rec["st0"].data_ptr(), self.P(emb + "layer_norm.weight").data_ptr(),
             self.G(emb + "words.weight").data_ptr(), self.G(emb + "positions.weight").data_ptr(),
             self.G(emb + "layer_norm.weight").data_ptr(), self.G(emb + "layer_norm.bias").data_ptr(), M, T, H,
             self.pad, p, seed, di * 1000, s)
        return dmem_started

    # ------------------------------------------------------------------------------------------------ classification
    def _pooled_logits(self, feat, B, hw, bf16=True, f32=False):
        """LinearTextualHead: pooled [B, C] = mean of the hw feature rows of each image; logits = pooled . W^T + b.
        bf16 logits (the loss's input) and / or fp32 logits (top-k), both with a leading dimension of V rounded up to
        8 -- the GEMM's bf16 row alignment -- so V = 81 (multilabel) runs with ld 88."""
        C, V = feat.shape[1], self.textual.vocab_size
        ld = _round_up(V, 8)
        pooled = self.ws.get("cls.pooled", (B, C), BF16)
        call("vtx_group_mean_fwd", feat.data_ptr(), pooled.data_ptr(), B, hw, C, _stream())
        w, b = self.W("textual.output.weight"), self.P("textual.output.bias")
        lf = logits = None
        if f32:
            lf = self.ws.get("cls.logits_f32", (B, ld), F32)
            gemm(pooled, w, lf, B, V, C, bias=b)
        if bf16:
            logits = self.ws.get("cls.logits", (B, ld), BF16)
            gemm(pooled, w, logits, B, V, C, bias=b)
        return pooled, logits, lf

    def classification_forward(self, feat, hw, labels, training, with_grad):
        """K-hot cross entropy of int64 labels [B, L] (classification.py:74-96) into self.loss[0]; leaves dlogits in
        the bf16 logits buffer when `with_grad`, fp32 logits for top-k when not `training`."""
        B = feat.shape[0] // hw
        V = self.textual.vocab_size
        pooled, logits, lf = self._pooled_logits(feat, B, hw, f32=not training)
        call("vtx_khot_xent", logits.data_ptr(), logits.stride(0), labels.data_ptr(), labels.stride(0), B,
             labels.shape[1], V, self.ignore.data_ptr(), self.ignore.numel(), self.loss.data_ptr(), int(with_grad),
             _stream())
        self._cls = dict(B=B, hw=hw, pooled=pooled, logits=logits, logits_f32=lf, with_grad=with_grad)
        self._feat = feat

    def classification_backward(self, bucket_cb=None):
        """Linear layer backward from the dlogits written by the loss, then the pool's adjoint into the backbone."""
        c = self._cls
        if c is None or not c["with_grad"]:
            raise RuntimeError("backward needs a preceding forward with with_grad=True (it leaves dlogits behind)")
        B, hw = c["B"], c["hw"]
        C, V = self._feat.shape[1], self.textual.vocab_size
        frozen = getattr(self.visual, "frozen", False)
        dpooled = None if frozen else self.ws.get("cls.dpooled", (B, C), BF16)
        # dgrad with K = V over the padded ld: the TMA zero-fills the K tail of both operands
        self._linear_bwd(c["logits"], c["pooled"], "textual.output.weight", "textual.output.bias", dpooled, B, V, C)
        if bucket_cb is not None:
            bucket_cb("head")
        if not frozen:
            dfeat = self.ws.get("hb.dfeat", (B * hw, C), BF16)
            call("vtx_group_mean_bwd", dpooled.data_ptr(), dfeat.data_ptr(), B, hw, C, _stream())
            self.backbone_backward(dfeat, bucket_cb)
        if bucket_cb is not None:
            bucket_cb("rest")

    def classification_topk(self, k):
        """Indices of the k largest fp32 logits of each image of the last eval-mode forward -> int64 [B, k]."""
        c = self._cls
        if c is None or c["logits_f32"] is None:
            raise RuntimeError("predictions need an eval-mode forward (model.eval()) first")
        lf = c["logits_f32"]
        out = self.ws.get("cls.topk", (c["B"], k), torch.int64)
        call("vtx_topk_rows", lf.data_ptr(), lf.stride(0), c["B"], self.textual.vocab_size, k, out.data_ptr(), _stream())
        return out

    # ------------------------------------------------------------------------------------------------ full model
    def forward(self, image, tokens, noitpac, lengths, training=True, with_grad=True, labels=None):
        """Loss of the bicaptioning model (labels None) or of the masked-LM sibling (labels = masked_labels [B,T], single
        direction).  Leaves dlogits in the logits buffers when `with_grad`."""
        if not self.arena.intact():
            raise RuntimeError("model parameters were moved after the engine adopted them; rebuild the engine")
        self.generation += 1
        self.loss.zero_()
        self.count.zero_()
        if not self.classify:  # an NCHW image fixes the backbone's h x w grid: check the attention shapes up front
            _check_attention(tokens.shape[1], math.prod(_feature_grid(*image.shape[2:])) if image.dim() == 4 else 0)
        # BatchNorm follows the backbone's OWN mode flag, like the reference's nn.BatchNorm2d: `model.train()` puts a
        # frozen backbone's BN back into batch-statistics mode (visual_backbones.py:48-52 only calls .eval() once)
        bn_training = bool(self.visual.cnn.training) if self.visual is not None else training
        feat, h, w = self.backbone_forward(image, bn_training)
        if self.classify:
            self.classification_forward(feat, h * w, labels, training, with_grad)
            return self.loss
        B = image.shape[0]
        S = B * h * w
        mem = self.visual_projection_forward(feat, S)
        recs = [self.head_forward("textual", mem, tokens, lengths, training, want_logits_f32=not training)]
        self.head_loss(recs[0], with_grad, labels)
        if self.backward_textual is not None:
            recs.append(self.head_forward("backward_textual", mem, noitpac, lengths, training))
            self.head_loss(recs[1], with_grad)
        self._recs, self._mem, self._feat = recs, mem, feat
        return self.loss

    def backward(self, zero_grads=True, bucket_cb=None):
        """Gradients of (loss_fwd + loss_bwd) w.r.t. every parameter into the flat gradient arena.
        `bucket_cb(tag)`, tag in {'head_b','head','layer4','layer3','layer2','rest'}, fires as gradient ranges complete (in
        backward order) so a data-parallel all-reduce can overlap the remaining backward."""
        if zero_grads:
            self.arena.grads.zero_()
        if self.classify:
            self.classification_backward(bucket_cb)
            return
        feat, mem = self._feat, self._mem
        S, H = mem.shape
        dmem = self.ws.get("hb.dmem", (S, H), BF16)
        started = False
        for rec in reversed(self._recs):
            started = self.head_backward(rec, dmem, started)
            if bucket_cb is not None and rec["direction"] == "backward_textual":
                bucket_cb("head_b")  # only this direction writes the backward_textual.* gradients
        Cv = feat.shape[1]
        dfeat = self.ws.get("hb.dfeat", (S, Cv), BF16)
        frozen = getattr(self.visual, "frozen", False)
        self._linear_bwd(dmem, feat, "textual.visual_projection.weight", "textual.visual_projection.bias",
                         None if frozen else dfeat, S, H, Cv)
        if bucket_cb is not None:
            bucket_cb("head")
        if not frozen:
            self.backbone_backward(dfeat, bucket_cb)
        if bucket_cb is not None:
            bucket_cb("rest")

    def predictions(self):
        """argmax over the fp32 forward-direction logits of the last eval-mode forward -> int64 [B,T]; for a
        classification head the top-10 classes of each image -> int64 [B, 10] (classification.py:104-106)."""
        if self.classify:
            return self.classification_topk(10)
        rec = self._recs[0]
        lf = rec["logits_f32"]
        out = self.ws.get("pred", (rec["M"],), torch.int64)
        call("vtx_argmax_rows", lf.data_ptr(), lf.stride(0), rec["M"], lf.shape[1], out.data_ptr(), _stream())
        return out.view(rec["B"], rec["T"])

    # ------------------------------------------------------------------------------------------------ beam search
    # AutoRegressiveBeamSearch (virtex/utils/beam_search.py:52-238) over CaptioningModel.decoding_step
    # (virtex/models/captioning.py:144-213), eval mode, forward-direction head only.  The reference recomputes the whole
    # prefix every step; here each step runs the decoder on one new position per beam row:
    #   * step 0 decodes [SOS] once per image (B rows, position 0, a one-slot self-attention cache of its own);
    #   * step t >= 1 decodes the beam's token t-1 at position t-1 (the reference's input drops SOS, so step 0's state
    #     is not a prefix of step 1's); its self-attention K|V go straight from the in-projection GEMM into slot t-1 of
    #     the row's cache, and attention reads slots 0..t-1 through the step-major index table, in which the beam
    #     selection gathers each surviving beam's ancestry -- the caches themselves are never moved;
    #   * cross-attention K|V of the image features are projected once per image and layer, shared by its beams.
    # Every buffer is a workspace key of the search's own ("bs."): a pending backward's tape is left alone.
    def beam_search(self, image, beam_size, per_node, max_steps, sos, eos):
        """image fp32 NCHW [B,3,H,W] -> int64 (B, L) on the device: the best beam of each image, EOS repeated after
        its first EOS; L <= max_steps is the number of steps run before every beam of every image ended in EOS."""
        st = self.beam_start(image, beam_size, per_node, max_steps, sos, eos)
        while st.L < max_steps and st.alive[st.L - 1].item():  # one device-to-host read per step
            self.beam_step(st)
        return st.best()

    def beam_start(self, image, beam_size, per_node, max_steps, sos, eos):
        """Backbone (folded BN), visual projection, cross-attention K|V of every layer, and step 0 -> the search
        state (_BeamState) after its first step."""
        mod = self.textual
        Sk, ckv = self._decode_prologue(image, max_steps - 1, "beam search", "bs.")
        B, ws = image.shape[0], self.ws
        H, V, R = mod.hidden_size, mod.vocab_size, B * beam_size
        st = _BeamState(B=B, beam=beam_size, per_node=per_node, max_steps=max_steps, eos=eos, R=R, Sk=Sk, ckv=ckv, L=1,
                        cur=0, pre="bs.")
        st.cache = [ws.get(f"bs.cache{l}", (R, max_steps - 1, 2 * H), BF16) for l in range(mod.num_layers)]
        st.cache0 = [ws.get(f"bs.cache0.{l}", (B, 1, 2 * H), BF16) for l in range(mod.num_layers)]
        st.pred = [ws.get(f"bs.pred{i}", (max_steps, R), torch.int64) for i in (0, 1)]
        st.index = [ws.get(f"bs.index{i}", (max_steps, R), torch.int32) for i in (0, 1)]
        st.scores = ws.get("bs.scores", (R,), F32)
        st.parent = ws.get("bs.parent", (R,), torch.int32)
        st.alive = ws.get("bs.alive", (max_steps,), torch.int32)
        st.alive.zero_()
        st.logits = ws.get("bs.logits", (R, V), F32)
        sos_t = ws.get("bs.sos", (B,), torch.int64)
        sos_t.fill_(sos)
        self._decode_position(st, B, sos_t, 0, 1, st.cache0, None)
        self._beam_select(st, B, None, beam_size, 1, 0)
        return st

    def _decode_prologue(self, image, positions, what, pre):
        """Checks that a decoder of `positions` self-attention positions fits the head and the attention kernel (before
        any launch), then runs the backbone (folded BN), the visual projection and the cross-attention K|V of every
        layer into workspace keys under `pre` -> (Sk feature positions per image, [bf16 (B * Sk, 2H)] per layer)."""
        mod = self.textual
        if positions > mod.max_caption_length:
            raise ValueError(f"{what} needs {positions} positions; the head has {mod.max_caption_length}")
        # vtx_attn_decode attends over at most DECODE_MAX_KEYS keys: the self-attention cache slots and the h * w
        # feature positions of cross-attention (h = w = 8 for a 256 x 256 image)
        h, w = _feature_grid(image.shape[2], image.shape[3])
        if positions > DECODE_MAX_KEYS or h * w > DECODE_MAX_KEYS:
            raise ValueError(f"{what} attends over at most {DECODE_MAX_KEYS} keys: it needs {positions} positions, a "
                             f"{image.shape[2]} x {image.shape[3]} image {h * w} feature positions")
        self.mark_weights_dirty()  # parameters may have been updated by any optimiser since the last call
        feat, h, w = self.backbone_infer(image)
        B, Sk, H = image.shape[0], h * w, mod.hidden_size
        mem = self.ws.get(pre + "mem", (B * Sk, H), BF16)
        gemm(feat, self.W("textual.visual_projection.weight"), mem, B * Sk, H, feat.shape[1],
             bias=self.P("textual.visual_projection.bias"))
        ckv = []
        for l in range(mod.num_layers):
            q = f"textual.transformer.layers.{l}.multihead_attn."
            kv = self.ws.get(f"{pre}ckv{l}", (B * Sk, 2 * H), BF16)
            gemm(mem, self.W(q + "in_proj_weight")[H:], kv, B * Sk, 2 * H, H, bias=self.P(q + "in_proj_bias")[H:])
            ckv.append(kv)
        return Sk, ckv

    def beam_step(self, st):
        """Step t = st.L: decode token t-1 of every beam at position t-1, score, select; st.L becomes t + 1."""
        t, R, cur = st.L, st.R, st.cur
        tokens = st.pred[cur][t - 1]
        self._decode_position(st, R, tokens, t - 1, st.beam, st.cache, st.index[cur])
        self._beam_select(st, R, tokens, st.per_node, st.beam, t)
        st.cur, st.L = 1 - cur, t + 1

    def _beam_select(self, st, rows, last, k, parents, s):
        """Both halves of a beam step over st.logits [rows, V]: per-row top-k, then per-image selection into the other
        ping-pong tables (step 0 writes table 0 directly)."""
        V = self.textual.vocab_size
        cv = self.ws.get("bs.cand_val", (rows, k), F32)
        ci = self.ws.get("bs.cand_idx", (rows, k), torch.int32)
        call("vtx_beam_rows", st.logits.data_ptr(), V, rows, V, _p(last), st.eos, k, cv.data_ptr(), ci.data_ptr(),
             _stream())
        src, dst = (st.cur, 1 - st.cur) if s > 0 else (None, 0)
        call("vtx_beam_select", cv.data_ptr(), ci.data_ptr(), parents, k, st.beam, st.scores.data_ptr() if s > 0 else 0,
             st.scores.data_ptr(), st.parent.data_ptr(), 0 if src is None else st.pred[src].data_ptr(),
             st.pred[dst].data_ptr(), 0 if src is None else st.index[src].data_ptr(), st.index[dst].data_ptr(), st.B, s,
             st.eos, st.alive.data_ptr(), _stream())

    # ------------------------------------------------------------------------------------------------ nucleus sampling
    # AutoRegressiveNucleusSampling (virtex/utils/nucleus_sampling.py:47-123) over CaptioningModel.decoding_step, eval
    # mode, forward-direction head only.  The reference's step t decodes [SOS, tok_1 .. tok_t] (SOS included), so each
    # step's state is a prefix of the next: step t decodes token t (SOS at t = 0) of every image at position t into
    # slot t of the image's own cache -- one row per image, no index table, no reordering.  Cross-attention K|V are
    # projected once per image and layer.  Workspace keys "ns.": a pending backward's tape is left alone, and the
    # dropout seed of the training step is not touched (the sampler's seed is a buffer of its own).
    def nucleus_sample(self, image, p, max_steps, sos, eos, seed):
        """image fp32 NCHW [B,3,H,W] -> int64 (B, L) on the device: one sampled caption per image, EOS repeated after
        its first EOS; L <= max_steps is the number of steps run before every caption ended in EOS.  `seed`: a Python
        int or an int64 device tensor of one element (read on the device)."""
        st = self.nucleus_start(image, p, max_steps, sos, eos, seed)
        while st.L < max_steps and st.alive[st.L - 1].item():  # one device-to-host read per step
            self.nucleus_step(st)
        return st.tokens().contiguous()

    def nucleus_start(self, image, p, max_steps, sos, eos, seed):
        """Backbone (folded BN), visual projection, cross-attention K|V of every layer, and step 0 (SOS at position 0)
        -> the sampler state (_NucleusState) after its first step."""
        if not 0.0 <= p <= 1.0:
            raise ValueError(f"nucleus size {p} is not in [0, 1]")
        mod = self.textual
        Sk, ckv = self._decode_prologue(image, max_steps, "nucleus sampling", "ns.")
        B, ws = image.shape[0], self.ws
        H, V = mod.hidden_size, mod.vocab_size
        st = _NucleusState(B=B, p=float(p), max_steps=max_steps, eos=eos, Sk=Sk, ckv=ckv, L=0, pre="ns.")
        st.seed = ws.get("ns.seed", (1,), torch.int64)
        if isinstance(seed, torch.Tensor):
            st.seed.copy_(seed.reshape(1))
        else:
            st.seed.fill_(struct.unpack("<q", struct.pack("<Q", int(seed) & (2 ** 64 - 1)))[0])
        st.cache = [ws.get(f"ns.cache{l}", (B, max_steps, 2 * H), BF16) for l in range(mod.num_layers)]
        st.pred = ws.get("ns.pred", (max_steps, B), torch.int64)
        st.alive = ws.get("ns.alive", (max_steps,), torch.int32)
        st.alive.zero_()
        st.logits = ws.get("ns.logits", (B, V), F32)
        sos_t = ws.get("ns.sos", (B,), torch.int64)
        sos_t.fill_(sos)
        self._nucleus_position(st, sos_t)
        return st

    def nucleus_step(self, st):
        """Step t = st.L: decode token t of every image at position t, sample token t + 1; st.L becomes t + 1."""
        self._nucleus_position(st, st.pred[st.L - 1])

    def _nucleus_position(self, st, tokens):
        t = st.L
        self._decode_position(st, st.B, tokens, t, 1, st.cache, None)
        call("vtx_nucleus_sample", st.logits.data_ptr(), st.logits.stride(0), st.B, st.logits.shape[1],
             tokens.data_ptr(), st.eos, st.p, st.seed.data_ptr(), t, st.pred.data_ptr(), st.alive.data_ptr(), _stream())
        st.L = t + 1

    def _decode_position(self, st, rows, tokens, pos, group, cache, index):
        """Forward head on one new position: tokens int64 [rows] at position `pos`, self-attention over cache slots
        0..pos (slot pos written here; through `index` when given), cross-attention of row m over image m // group
        -> fp32 logits st.logits[:rows].  Workspace keys under st.pre."""
        mod = self.textual
        H, A, Fd, V = mod.hidden_size, mod.attention_heads, mod.feedforward_size, mod.vocab_size
        ws, s, seed, k = self.ws, _stream(), self.seed.data_ptr(), st.pre
        emb = "textual.embedding."
        xs = [ws.get(f"{k}x{i}", (rows, H), F32) for i in (0, 1)]
        z, zst = ws.get(k + "z", (rows, H), F32), ws.get(k + "st", (rows, 2), F32)
        xb = ws.get(k + "xb", (rows, H), BF16)
        # the embedding kernel with T = 1 over position row `pos` is the one-position embedding
        call("vtx_embed_fwd", tokens.data_ptr(), self.P(emb + "words.weight").data_ptr(),
             self.P(emb + "positions.weight")[pos].data_ptr(), self.P(emb + "layer_norm.weight").data_ptr(),
             self.P(emb + "layer_norm.bias").data_ptr(), z.data_ptr(), zst.data_ptr(), xs[0].data_ptr(), xb.data_ptr(),
             rows, 1, H, self.pad, 1e-8, 0.0, seed, 0, s)
        qb, o = ws.get(k + "q", (rows, H), BF16), ws.get(k + "o", (rows, H), BF16)
        pr = ws.get(k + "proj", (rows, H), BF16)
        xbs = [ws.get(f"{k}xb{i}", (rows, H), BF16) for i in (0, 1)]
        n = 0
        for l in range(mod.num_layers):
            q = f"textual.transformer.layers.{l}."
            c = cache[l]

            def self_attn(inp, out):
                w, b = self.W(q + "self_attn.in_proj_weight"), self.P(q + "self_attn.in_proj_bias")
                gemm(inp, w[:H], qb, rows, H, H, bias=b[:H])
                gemm(inp, w[H:], c, rows, 2 * H, H, bias=b[H:], ldd=c.stride(0),
                     d_ptr=c.data_ptr() + pos * c.stride(1) * c.element_size())
                call("vtx_attn_decode", qb.data_ptr(), H, c.data_ptr(), c.data_ptr() + H * c.element_size(), c.stride(1),
                     c.stride(0), _p(index), rows, o.data_ptr(), H, rows, A, 1, pos + 1, s)
                gemm(o, self.W(q + "self_attn.out_proj.weight"), out, rows, H, H, bias=self.P(q + "self_attn.out_proj.bias"))

            def cross_attn(inp, out):
                w, b = self.W(q + "multihead_attn.in_proj_weight"), self.P(q + "multihead_attn.in_proj_bias")
                gemm(inp, w[:H], qb, rows, H, H, bias=b[:H])
                kv = st.ckv[l]
                call("vtx_attn_decode", qb.data_ptr(), H, kv.data_ptr(), kv.data_ptr() + H * kv.element_size(), 2 * H,
                     st.Sk * 2 * H, 0, 0, o.data_ptr(), H, rows // group, A, group, st.Sk, s)
                gemm(o, self.W(q + "multihead_attn.out_proj.weight"), out, rows, H, H,
                     bias=self.P(q + "multihead_attn.out_proj.bias"))

            def ffn(inp, out):
                self._ffn_fwd(dict(M=rows, H=H, Fd=Fd, p=0.0), dict(q=q, k=k, sb=0), inp, out)

            for i, run in enumerate((self_attn, cross_attn, ffn), 1):
                xb = self._residual_sublayer(mod.norm_first, f"{q}norm{i}.", run, xs[n & 1], xb, xs[1 - (n & 1)],
                                             xbs[n & 1], pr, z, zst, rows, H, 0.0, 0)
                n += 1
        if mod.norm_first:  # final LayerNorm of pre-norm decoders
            qn = "textual.transformer.norm."
            xb = xbs[n & 1]
            call("vtx_add_ln_fwd", xs[n & 1].data_ptr(), 0, self.P(qn + "weight").data_ptr(),
                 self.P(qn + "bias").data_ptr(), z.data_ptr(), zst.data_ptr(), 0, xb.data_ptr(), rows, H, 1e-5, 0.0, seed,
                 0, 1, s)
        gemm(xb, self.W("textual.embedding.words.weight"), st.logits, rows, V, H, bias=self.P("textual.output.bias"))


class _BeamState:
    """Buffers and progress of one running beam search (Engine.beam_start / beam_step): L steps have run; the current
    step-major tables are pred[cur] (int64 [max_steps, B * beam]) and index[cur]; scores holds each beam's sum of
    log-probabilities, st.logits the fp32 logits of the last step."""

    def __init__(self, **kw):
        self.__dict__.update(kw)

    def tokens(self):
        """int64 (B * beam, L): every beam's tokens so far."""
        return self.pred[self.cur][:self.L].t()

    def best(self):
        """int64 (B, L): beam 0 of every image (the best, beams are kept in descending score order)."""
        return self.tokens()[::self.beam].contiguous()


class _NucleusState:
    """Buffers and progress of one running nucleus sampler (Engine.nucleus_start / nucleus_step): L steps have run;
    pred is the step-major int64 table [max_steps, B] of sampled tokens (row t: token t + 1, SOS is token 0), st.logits
    the fp32 logits of the last step."""

    def __init__(self, **kw):
        self.__dict__.update(kw)

    def tokens(self):
        """int64 (B, L): every caption's tokens so far."""
        return self.pred[:self.L].t()


# ---------------------------------------------------------------------------------------------------- module-level API
def _module_engine(mod, **kw):
    eng = getattr(mod, "_vtx_engine", None)
    if eng is None or not eng.arena.intact():
        eng = Engine(**kw)
        object.__setattr__(mod, "_vtx_engine", eng)
    return eng


@torch.no_grad()
def backbone_features(backbone, image: torch.Tensor) -> torch.Tensor:
    """`TorchvisionVisualBackbone.forward`: (B,3,H,W) fp32 -> (B,C,H/32,W/32) fp32, NCHW-shaped like the reference.
    Module-level calls are inference-style (no autograd); training goes through the model-level engine."""
    eng = _module_engine(backbone, visual=backbone)
    eng.mark_weights_dirty()
    feat, h, w = eng.backbone_forward(image.contiguous().float(), training=backbone.cnn.training)
    B, C = image.shape[0], feat.shape[1]
    out = torch.empty(B, C, h, w, dtype=F32, device=image.device)
    call("vtx_nhwc_to_nchw_f32", feat.data_ptr(), out.data_ptr(), B, h * w, C, _stream())
    return out


class _CnnView:
    """A stand-alone ResNetParams as an engine's `visual`: its backbone parameters under the names the engine uses
    ('visual.cnn.*'), without `fc`, which its forward may replace at any time and reads afresh on every call."""

    frozen = False

    def __init__(self, cnn):
        self.cnn = cnn

    def named_parameters(self):
        return [("cnn." + n, p) for n, p in self.cnn.named_parameters() if not n.startswith("fc.")]

    def named_buffers(self):
        return [("cnn." + n, b) for n, b in self.cnn.named_buffers() if not n.startswith("fc.")]


def _cnn_engine(cnn):
    eng = cnn.__dict__.get("_vtx_engine")
    if eng is None or not eng.arena.intact():
        eng = Engine(visual=_CnnView(cnn))
        object.__setattr__(cnn, "_vtx_engine", eng)
    return eng


def _fc_of(cnn):
    fc = cnn.fc
    if isinstance(fc, nn.Identity):
        return None
    if not isinstance(fc, nn.Linear) or fc.bias is None:
        raise TypeError(f"ResNetParams.fc must be nn.Identity or nn.Linear with a bias, not {type(fc).__name__}")
    if fc.weight.device != cnn.conv1.weight.device:
        raise RuntimeError("ResNetParams.fc is not on the backbone's device: move it with .to(device)")
    return fc


def _resnet_pool_fc(eng, feat, B, hw, fc_w, fc_b):
    """Global average pool of the NHWC features (vtx_group_mean_fwd) and the fc GEMM -> (fp32 output, bf16 pooled,
    bf16 fc weight).  fc_w None: the output is the pooled features."""
    C = feat.shape[1]
    pooled = eng.ws.get("fc.pooled", (B, C), BF16)
    call("vtx_group_mean_fwd", feat.data_ptr(), pooled.data_ptr(), B, hw, C, _stream())
    if fc_w is None:
        return pooled.float(), pooled, None
    N = fc_w.shape[0]
    w = eng.ws.get("fc.weight_bf16", (N, C), BF16)  # cast on every call: the optimiser updates fc in place
    call("vtx_cast_bf16", fc_w.data_ptr(), w.data_ptr(), N * C, _stream())
    out = torch.empty(B, _round_up(N, 4), dtype=F32, device=feat.device)  # fp32 rows stay 16-byte aligned
    gemm(pooled, w, out, B, N, C, bias=fc_b)
    return out[:, :N], pooled, w


def _resnet_run(cnn, image, fc_w, fc_b):
    """Backbone (train mode: the training backbone_forward with batch statistics and the running-statistics update;
    eval mode: backbone_infer), pool and fc -> (fp32 output, engine, bf16 pooled, bf16 fc weight, h * w)."""
    eng = _cnn_engine(cnn)
    if cnn.training:
        eng.mark_weights_dirty()  # parameters may have been updated by any optimiser since the last call
        feat, h, w = eng.backbone_forward(image, training=True)
        eng.mark_weights_dirty()  # the running statistics moved
    else:
        feat, h, w = eng.backbone_infer(image)
    out, pooled, wb = _resnet_pool_fc(eng, feat, image.shape[0], h * w, fc_w, fc_b)
    return out, eng, pooled, wb, h * w


class _ResNetFunction(torch.autograd.Function):
    """ResNetParams.forward as one autograd node: gradients for fc (pool + linear backward) and, in train mode, for
    the backbone parameters passed in `params` (backbone_backward)."""

    @staticmethod
    def forward(ctx, cnn, image, fc_w, fc_b, *params):
        out, eng, pooled, wb, hw = _resnet_run(cnn, image, fc_w, fc_b)
        eng.generation += 1
        ctx.eng, ctx.generation, ctx.hw, ctx.n_params = eng, eng.generation, hw, len(params)
        ctx.pooled, ctx.wb, ctx.has_fc = pooled.clone(), wb, fc_w is not None
        return out

    @staticmethod
    def backward(ctx, g):
        eng = ctx.eng
        B, C = ctx.pooled.shape
        s = _stream()
        need_bb = ctx.n_params > 0
        if need_bb and eng.generation != ctx.generation:
            raise RuntimeError("the backbone ran another forward since this output was computed: its activation tape "
                               "was overwritten; call backward() before the next forward")
        dfc_w = dfc_b = None
        dpooled = eng.ws.get("fc.dpooled", (B, C), BF16) if need_bb else None
        if ctx.has_fc:
            N = ctx.wb.shape[0]
            ld = _round_up(N, 8)  # bf16 rows of the dlogits stay 16-byte aligned; the GEMMs' TMA zero-fills the K tail
            g32 = eng.ws.get("fc.dlogits_f32", (B, ld), F32)
            if ld != N:
                g32.zero_()
            g32[:, :N].copy_(g)
            dY = eng.ws.get("fc.dlogits", (B, ld), BF16)
            call("vtx_cast_bf16", g32.data_ptr(), dY.data_ptr(), B * ld, s)
            dfc_w = torch.zeros(N, C, dtype=F32, device=g.device)
            dfc_b = torch.zeros(N, dtype=F32, device=g.device)
            eng._linear_bwd_t(dY, ctx.pooled, ctx.wb, dfc_w, dfc_b, dpooled, B, N, C)
        elif need_bb:
            call("vtx_cast_bf16", g.contiguous().data_ptr(), dpooled.data_ptr(), B * C, s)
        grads = [None] * ctx.n_params
        if need_bb:
            dfeat = eng.ws.get("fc.dfeat", (B * ctx.hw, C), BF16)
            call("vtx_group_mean_bwd", dpooled.data_ptr(), dfeat.data_ptr(), B, ctx.hw, C, s)
            eng.arena.grads.zero_()
            eng.backbone_backward(dfeat)
            flat = eng.arena.grads.clone()  # the arena is reused by the next backward
            grads = [eng.arena.view(flat, n) if need else None
                     for n, need in zip(eng.arena.names, ctx.needs_input_grad[4:])]
        return (None, None, dfc_w, dfc_b, *grads)


def resnet_forward(cnn, image: torch.Tensor) -> torch.Tensor:
    """`ResNetParams.forward`, as torchvision's ResNet.forward: image fp32 NCHW (B,3,H,W) -> fc(flatten(avgpool(layer4)))
    in fp32, (B, num_classes) for an nn.Linear fc and the (B, 2048) pooled features for nn.Identity."""
    _require_cuda(image.device)
    image = image.contiguous().float()
    fc = _fc_of(cnn)
    fc_w = fc_b = None
    if fc is not None:
        fc_w, fc_b = fc.weight, fc.bias
        if fc_w.dtype != F32 or fc_b.dtype != F32 or not fc_w.is_contiguous():
            raise TypeError("ResNetParams.fc needs contiguous fp32 parameters")
    eng = _cnn_engine(cnn)
    params = [eng.arena._param_objs[n] for n in eng.arena.names]
    grad = torch.is_grad_enabled()
    if not cnn.training and grad and any(p.requires_grad for p in params):
        raise RuntimeError("backward through eval-mode BatchNorm is not implemented: freeze the backbone "
                           "(requires_grad = False) for an eval-mode forward with gradients, or run it under no_grad")
    bb = params if cnn.training and any(p.requires_grad for p in params) else []
    if grad and (bb or (fc is not None and (fc_w.requires_grad or fc_b.requires_grad))):
        return _ResNetFunction.apply(cnn, image, fc_w, fc_b, *bb)
    with torch.no_grad():
        return _resnet_run(cnn, image, fc_w, fc_b)[0].clone()


@torch.no_grad()
def head_logits(head, visual_features, caption_tokens, caption_lengths) -> torch.Tensor:
    """`TransformerDecoderTextualHead.forward`: (B,C,h,w), (B,T), (B,) -> fp32 logits (B,T,V)."""
    B, C, h, w = visual_features.shape
    _check_attention(caption_tokens.shape[1], h * w)
    eng = _module_engine(head, textual=head)
    eng.mark_weights_dirty()
    eng.prepare_weights()
    feat = visual_features.permute(0, 2, 3, 1).reshape(B * h * w, C).to(BF16).contiguous()
    mem = eng.visual_projection_forward(feat, B * h * w)
    rec = eng.head_forward("textual", mem, caption_tokens.contiguous(), caption_lengths.contiguous(),
                           training=head.training, want_logits_f32=True)
    return rec["logits_f32"].view(B, caption_tokens.shape[1], -1).clone()


@torch.no_grad()
def linear_head_logits(head, visual_features) -> torch.Tensor:
    """`LinearTextualHead.forward`: (B,C,h,w) -> fp32 logits (B,V)."""
    eng = _module_engine(head, textual=head)
    eng.mark_weights_dirty()
    eng.prepare_weights()
    B, C, h, w = visual_features.shape
    feat = visual_features.permute(0, 2, 3, 1).reshape(B * h * w, C).to(BF16).contiguous()
    _, _, lf = eng._pooled_logits(feat, B, h * w, bf16=False, f32=True)
    return lf[:, :head.vocab_size].clone()
