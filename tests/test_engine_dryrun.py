"""Host-logic dry run of the engine on the CPU box: every kernel launcher is replaced by a recorder that checks the
call against the C-ABI prototype (argument count) and the GEMM operands against the buffer sizes they imply.  No
arithmetic runs -- this is not a CPU path (the product refuses CPU tensors, tests/test_host_cpu.py::test_no_cpu_fallback);
it exercises the Python schedule (shapes, workspaces, tape, optional branches) for configurations and edge shapes that
the GPU suite also runs."""
import pytest
import torch

from oracle import virtex_oracle as O

BF16, F32 = torch.bfloat16, torch.float32


class Recorder:
    def __init__(self):
        self.calls = []
        self.drops = []   # (kernel, site, p) of every launch that applies a dropout mask


    def names(self):
        return [c if isinstance(c, str) else c[0] for c in self.calls]


# kernel -> (index of p, index of site, index of the pointer whose presence means the mask is applied or None), as
# negative offsets into the C-ABI argument list (virtex_b200/ops.py::_PROTOS)
_DROP_ARGS = {
    "vtx_embed_fwd": (-4, -2, None), "vtx_embed_bwd": (-4, -2, None),
    "vtx_add_ln_fwd": (-5, -3, 1),                    # the branch operand
    "vtx_ln_bwd": (-5, -3, 7),                        # d_branch
    "vtx_attn_fwd": (-4, -2, None), "vtx_attn_bwd": (-4, -2, None),
    "vtx_gelu_dropout_fwd": (-4, -2, None), "vtx_gelu_dropout_bwd": (-4, -2, None),
}


def _record_dropout(rec, name, args):
    if name in _DROP_ARGS:
        ip, isite, iptr = _DROP_ARGS[name]
        if iptr is None or args[iptr]:
            rec.drops.append((name, int(args[isite]), float(args[ip])))


def _check_gemm(A, B, D, M, N, K, lda=None, ldb=None, ldd=None, a_mn=0, b_mn=0, bias=None, act=0, residual=None, ldr=0,
                stats=None, atomic=False, split_k=1, tile_n=0, conv=None, conv_mode=0, out_f32=None, residual_mask=None,
                conv_stride=1, conv_taps=0, tap_grid=None, out_view=None, d_ptr=None, bnr=None):
    assert A.dtype == BF16 and B.dtype == BF16, (A.dtype, B.dtype)
    f32 = (D.dtype == F32) if out_f32 is None else bool(out_f32)
    assert D.dtype == (F32 if f32 else BF16)
    assert not atomic or f32
    assert split_k >= 1 and (split_k == 1 or atomic)
    ldd = D.stride(0) if ldd is None else ldd
    assert M > 0 and N > 0 and K > 0
    if conv_mode == 0:
        lda = A.stride(0) if lda is None else lda
        ldb = B.stride(0) if ldb is None else ldb
        assert A.numel() >= ((K - 1) * lda + M if a_mn else (M - 1) * lda + K), "A too small"
        assert B.numel() >= ((K - 1) * ldb + N if b_mn else (N - 1) * ldb + K), "B too small"
        assert D.numel() >= (M - 1) * ldd + N, "D too small"
    else:
        NI, H, W, C = conv
        assert C % 64 == 0
        taps = 1 if conv_taps == 1 else (tap_grid[0] * tap_grid[1] if tap_grid is not None else 9)
        if out_view is not None:
            assert conv_mode == 1 and d_ptr is not None and all(v % 8 == 0 for v in out_view[2:])
            assert residual is None or residual.data_ptr() == d_ptr  # a view GEMM accumulates in place or not at all
            assert D.data_ptr() <= d_ptr < D.data_ptr() + D.numel() * D.element_size()
        Ho, Wo = (H - 1) // conv_stride + 1, (W - 1) // conv_stride + 1   # conv = INPUT extent; outputs follow the stride
        if conv_mode == 1:
            assert M == NI * Ho * Wo and K == taps * C and A.numel() >= NI * H * W * C and B.numel() >= N * K
            assert out_view is not None or D.numel() >= (M - 1) * ldd + N
        elif conv_mode == 2:
            assert N == taps * C and K == NI * Ho * Wo and A.numel() >= K * M and B.numel() >= NI * H * W * C and f32 and atomic
            assert D.numel() >= (M - 1) * ldd + N
        elif conv_mode == 4:
            assert C == 64 and N == 64 and M == 9 * C and K == NI * H * W and f32 and atomic
            assert A.numel() >= K * N and B.numel() >= K * C and D.numel() >= M * N
        elif conv_mode == 5:   # stem fprop over the space-to-depth view
            assert C == 64 and N == 64 and K == 256 and M == NI * H * W
            assert A.numel() >= NI * (H + 3) * (W + 3) * 16 and B.numel() >= 64 * 256 and D.numel() >= M * N
        elif conv_mode == 6:   # stem wgrad
            assert C == 64 and M == 64 and N == 256 and K == NI * H * W and f32 and atomic
            assert A.numel() >= K * 64 and B.numel() >= NI * (H + 3) * (W + 3) * 16 and D.numel() >= M * N
        else:
            raise AssertionError(conv_mode)
    if stats is not None:
        assert stats.dtype == F32 and stats.numel() >= 2 * N and not f32 and bias is None and residual is None
    if bias is not None:
        assert bias.dtype == F32 and bias.numel() >= N
    if residual is not None:
        assert residual.dtype == BF16 and residual.numel() >= M * N
    if residual_mask is not None:
        assert residual is not None and residual_mask.dtype == torch.uint8 and residual_mask.numel() >= M * N // 8
        assert N % 32 == 0 and conv_mode == 0 and not f32
    if bnr is not None:   # BN-backward sums accumulated by the epilogue: (y, bnp, sums, bit mask or None[, y view pointer])
        y, bnp, sums, mbits = bnr[:4]
        assert not f32 and stats is None and bias is None and act == 0 and split_k == 1 and conv_mode in (0, 1) and N % 8 == 0
        assert y.dtype == BF16 and bnp.dtype == F32 and bnp.numel() == 4 * N and sums.dtype == F32 and sums.numel() == 2 * N
        if out_view is not None:   # y is addressed through the same strided view as D
            assert len(bnr) == 5 and bnr[4] - y.data_ptr() == d_ptr - D.data_ptr() and y.numel() == D.numel()
        else:
            assert len(bnr) == 4 and y.numel() >= M * N
        if mbits is not None:
            assert conv_mode == 0 and mbits.dtype == torch.uint8 and mbits.numel() >= M * N // 8


@pytest.fixture
def dry(monkeypatch):
    """Patch the launchers of virtex_b200.engine with checking recorders."""
    from virtex_b200 import engine as E, ops
    rec = Recorder()

    def fake_call(name, *args):
        assert len(args) == len(ops._PROTOS[name]), (name, len(args), len(ops._PROTOS[name]))
        rec.calls.append(name)
        _record_dropout(rec, name, args)

    def fake_gemm(A, B, D, M, N, K, **kw):
        _check_gemm(A, B, D, M, N, K, **kw)
        rec.calls.append(("gemm", M, N, K, kw.get("conv_mode", 0), kw.get("bnr") is not None))

    monkeypatch.setattr(E, "call", fake_call)
    monkeypatch.setattr(E, "gemm", fake_gemm)
    monkeypatch.setattr(E, "_stream", lambda: 0)
    monkeypatch.setattr(E, "_require_cuda", lambda dev: None)
    monkeypatch.setattr(ops, "num_sms", lambda: 148)
    return rec


def _model(spec, frozen=False, bidirectional=True):
    from virtex_b200.models import BidirectionalCaptioningModel, ForwardCaptioningModel
    from virtex_b200.modules import TorchvisionVisualBackbone, TransformerDecoderTextualHead
    visual = TorchvisionVisualBackbone(spec.backbone, visual_feature_size=spec.visual_feature_size, frozen=frozen)
    textual = TransformerDecoderTextualHead(
        visual_feature_size=spec.visual_feature_size, vocab_size=spec.vocab, hidden_size=spec.hidden,
        num_layers=spec.layers, attention_heads=spec.heads, feedforward_size=spec.ffn, dropout=0.1,
        norm_first=spec.norm_first, max_caption_length=spec.max_len, padding_idx=spec.pad)
    return (BidirectionalCaptioningModel if bidirectional else ForwardCaptioningModel)(visual, textual)


def _run(model, batch, training=True, backward=True):
    eng = model.engine
    loss = eng.forward(batch["image"], batch["caption_tokens"],
                       batch["noitpac_tokens"] if model.caption_backward else batch["caption_tokens"],
                       batch["caption_lengths"], training=training, with_grad=backward)
    assert tuple(loss.shape) == (2,)
    if backward:
        eng.backward(zero_grads=True)
    return eng


SMALL = dict(hidden=128, layers=1, heads=2, ffn=256)


@pytest.mark.parametrize("spec_kw,batch_kw", [
    (SMALL, dict(batch_size=2, seed=0)),
    (SMALL, dict(batch_size=1, seed=1)),                                   # batch of one
    (SMALL, dict(batch_size=3, seed=2, max_len=13, ragged=True)),          # captions shorter than the maximum
    (SMALL, dict(batch_size=5, seed=3, max_len=2)),                        # [SOS] [EOS] only
    (dict(hidden=256, layers=2, heads=4, ffn=512, norm_first=True), dict(batch_size=2, seed=4, ragged=True)),
    (dict(layers=4), dict(batch_size=2, seed=5)),                          # BASELINE config #4 architecture
    (dict(backbone="resnet101", hidden=2048, heads=32, ffn=8192), dict(batch_size=2, seed=6)),  # config #5
])
def test_training_step_schedule(dry, spec_kw, batch_kw):
    spec = O.Spec(**spec_kw)
    model = _model(spec)
    batch = O.synth_batch(**batch_kw)
    _run(model, batch)
    names = dry.names()
    n_blocks = sum(spec.blocks)
    gemms = [c for c in dry.calls if not isinstance(c, str)]
    # every conv has one fprop GEMM and one wgrad GEMM (stem: no dgrad); 3 convs (+ downsample in 4 blocks) per block
    assert len([g for g in gemms if g[0] == "gemm"]) >= 3 * (3 * n_blocks + 4 + 1) - 1
    assert names.count("vtx_cross_entropy") == 2 and names.count("vtx_embed_fwd") == 2
    assert names.count("vtx_attn_fwd") == 2 * 2 * spec.layers == names.count("vtx_attn_bwd")
    assert "vtx_stem_s2d" in names and "vtx_stem_im2col" not in names
    # layer1's three 64 -> 64 3x3 convs use the [(tap, cin), cout] wgrad (conv_mode 4)
    assert len([g for g in gemms if g[4] == 4]) == 3
    # BN-backward reductions: bn1 / bn2 of every block and bn3 of every block that is followed by an identity block and
    # has no downsample branch are accumulated by GEMM epilogues (a stride-2 conv2 dgrad is four GEMMs); stand-alone
    # reduce launches remain for the stem BN, the four two-branch blocks, the last block of every layer
    # ... and of those bn3 only at large tensor sizes (Engine.fuse_bn3_min_rows; none at the batch sizes of this test)
    fused_bn3 = 0
    assert len([g for g in gemms if g[5]]) == 2 * n_blocks + 3 * 3 + fused_bn3
    assert names.count("vtx_bn_bwd_reduce") == 1 + n_blocks - fused_bn3
    assert names.count("vtx_bn_bwd_finalize_apply") == 1 + 3 * n_blocks


def test_eval_forward_only_and_frozen_backbone(dry):
    spec = O.Spec(**SMALL)
    batch = O.synth_batch(3, seed=7, ragged=True)
    model = _model(spec)
    eng = _run(model, batch, training=False, backward=False)
    assert "vtx_argmax_rows" not in dry.names()  # predictions are computed on demand
    eng.predictions()
    assert "vtx_argmax_rows" in dry.names()
    assert not any(n.startswith("vtx_bn_bwd") for n in dry.names())
    dry.calls.clear()
    _run(_model(spec, frozen=True), batch)
    assert not any(n.startswith("vtx_bn_bwd") for n in dry.names())          # no backbone backward at all
    dry.calls.clear()
    _run(_model(spec, bidirectional=False), batch)
    assert dry.names().count("vtx_cross_entropy") == 1


def test_stem_branch_schedule(dry):
    """224-class image sizes run the space-to-depth implicit stem conv; sizes the TMA boxes do not tile exactly run
    the im2col route."""
    spec = O.Spec(**SMALL)
    _run(_model(spec), O.synth_batch(2, seed=8))
    names = dry.names()
    gemms = [c for c in dry.calls if not isinstance(c, str)]
    assert "vtx_stem_im2col" not in names and "vtx_stem_s2d" in names
    assert [g[4] for g in gemms if g[4] in (5, 6)] == [5, 6]
    # weight layouts: one batched pack launch + one batched unpack launch per gradient bucket (layer4/3/2, layer1+stem)
    assert names.count("vtx_conv_w_jobs") == 1 + 4 and "vtx_conv_w_pack" not in names
    dry.calls.clear()
    _run(_model(spec), O.synth_batch(2, seed=9, image_size=200))
    assert "vtx_stem_im2col" in dry.names() and "vtx_stem_s2d" not in dry.names()


def test_masked_lm_schedule(dry):
    """The masked-LM sibling: one direction, key-padding-only attention mask (mode 2), labels passed to the loss."""
    from virtex_b200.models import MaskedLMModel
    from virtex_b200.modules import TorchvisionVisualBackbone, TransformerDecoderTextualHead
    spec = O.Spec(**SMALL)
    visual = TorchvisionVisualBackbone(spec.backbone, visual_feature_size=spec.visual_feature_size)
    textual = TransformerDecoderTextualHead(spec.visual_feature_size, spec.vocab, spec.hidden, spec.layers, spec.heads,
                                            spec.ffn, dropout=0.1, mask_future_positions=False)
    model = MaskedLMModel(visual, textual)
    batch = O.synth_masked_batch(3, seed=5)
    eng = model.engine
    eng.forward(batch["image"], batch["caption_tokens"], batch["caption_tokens"], batch["caption_lengths"], training=True,
                with_grad=True, labels=batch["masked_labels"])
    eng.backward(zero_grads=True)
    assert dry.names().count("vtx_cross_entropy") == 1 and dry.names().count("vtx_attn_fwd") == 2
    assert eng._recs[0]["mask_mode"] == 2
    with pytest.raises(ValueError):
        MaskedLMModel(visual, TransformerDecoderTextualHead(spec.visual_feature_size, spec.vocab, spec.hidden, 1,
                                                            spec.heads, spec.ffn))


# forward kernel -> (its backward kernel, the element-index space its mask is hashed over)
_REPLAY = {"vtx_embed_fwd": ("vtx_embed_bwd", "rows"), "vtx_add_ln_fwd": ("vtx_ln_bwd", "rows"),
           "vtx_attn_fwd": ("vtx_attn_bwd", "attention"), "vtx_gelu_dropout_fwd": ("vtx_gelu_dropout_bwd", "ffn")}


@pytest.mark.parametrize("norm_first,bidirectional", [(False, False), (True, False), (False, True)])
def test_dropout_site_schedule(dry, norm_first, bidirectional):
    """Dropout masks are recomputed in backward from (seed, site, element index): every forward site must be replayed
    exactly once in backward by the matching kernel with the same p, no two forward sites may hash the same (site,
    index space), and eval passes p = 0 to every dropout-carrying kernel."""
    spec = O.Spec(hidden=128, layers=2, heads=2, ffn=256, norm_first=norm_first)
    model = _model(spec, bidirectional=bidirectional)
    _run(model, O.synth_batch(2, seed=3, ragged=True))
    fwd = [d for d in dry.drops if d[0] in _REPLAY]
    bwd = [d for d in dry.drops if d[0] not in _REPLAY]
    assert len(fwd) == (2 if bidirectional else 1) * (1 + 6 * spec.layers)
    assert all(p == pytest.approx(0.1) for _, _, p in fwd)
    keys = [(site, _REPLAY[name][1]) for name, site, _ in fwd]
    assert len(set(keys)) == len(keys), sorted(keys)
    want = sorted((_REPLAY[name][0], site, p) for name, site, p in fwd)
    assert sorted(bwd) == want
    # eval: the same launches, all with p = 0
    dry.drops.clear()
    _run(model, O.synth_batch(2, seed=3, ragged=True), training=False, backward=False)
    assert dry.drops and all(p == 0.0 for _, _, p in dry.drops), dry.drops
