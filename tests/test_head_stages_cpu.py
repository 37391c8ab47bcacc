"""The float64 stage references of tests/head_stages.py, chained in exact float64, against float64 autograd of torch's own
nn.TransformerDecoder (nn.TransformerDecoderLayer, activation gelu, batch_first, norm_first as given) fed the masks the
reference builds (a -inf future mask and a key-padding mask from caption_lengths), a restated WordAndPositionalEmbedding
(words with padding_idx, positions, LayerNorm eps 1e-8, pad rows zeroed), the tied output projection and token-mean
cross entropy.  Every intermediate, every parameter gradient and the feature gradient agree to 1e-12 of the largest
magnitude: the references the GPU replay holds the engine to are the head's mathematics, not a restatement of the
engine.  Dropout is off (p = 0): the references take masks as given scale tensors, which tests/test_head_kernels_gpu.py
and the replay pin to the kernels' masks.
"""
import pytest
import torch
from torch import nn

from tests import head_stages as S

F64 = torch.float64
PAD = 0


class _Embedding(nn.Module):
    """virtex/modules/embedding.py's WordAndPositionalEmbedding, restated."""

    def __init__(self, V, H, max_len):
        super().__init__()
        self.words = nn.Embedding(V, H, padding_idx=PAD)
        self.positions = nn.Embedding(max_len, H)
        self.layer_norm = nn.LayerNorm(H, eps=1e-8)

    def forward(self, tokens):
        T = tokens.shape[1]
        pos = torch.arange(T).unsqueeze(0).expand_as(tokens)
        y = self.layer_norm(self.words(tokens) + self.positions(pos))
        return y * (tokens != PAD).unsqueeze(-1).to(y.dtype)


def _rel_close(got, ref, what, tol=1e-12):
    got, ref = got.detach(), ref.detach()
    assert got.shape == ref.shape, (what, tuple(got.shape), tuple(ref.shape))
    scale = max(float(ref.abs().max()), 1e-300)
    err = float((got - ref).abs().max())
    assert err <= tol * scale, f"{what}: max error {err:.3g} > {tol:g} * {scale:.3g}"


def _case(norm_first, mask_mode, L=2, B=4, T=9, max_len=12, V=53, H=128, A=2, Fd=256, Sk=5, Cv=24, seed=0):
    g = torch.Generator().manual_seed(seed + 10 * L + 2 * int(norm_first) + mask_mode)
    emb = _Embedding(V, H, max_len)
    layer = nn.TransformerDecoderLayer(H, A, dim_feedforward=Fd, dropout=0.0, activation="gelu", batch_first=True,
                                       norm_first=norm_first)
    dec = nn.TransformerDecoder(layer, num_layers=L, norm=nn.LayerNorm(H) if norm_first else None)
    vp = nn.Linear(Cv, H)
    out_bias = nn.Parameter(torch.zeros(V))
    mods = dict(emb=emb, dec=dec, vp=vp)
    for m in mods.values():
        m.to(F64)
        for p in m.parameters():
            with torch.no_grad():
                p.copy_(torch.randn(p.shape, generator=g, dtype=F64) * (0.3 if p.dim() > 1 else 0.2))
    with torch.no_grad():
        for n, p in list(emb.named_parameters()) + list(dec.named_parameters()):
            if "norm" in n and n.endswith("weight"):
                p.copy_(1 + 0.3 * torch.randn(p.shape, generator=g, dtype=F64))
        emb.words.weight[PAD] = 0.7 * torch.randn(H, generator=g, dtype=F64)  # trained pad row: nonzero, tied output
        out_bias.copy_(0.5 * torch.randn(V, generator=g, dtype=F64))
    out_bias = out_bias.to(F64)
    # ragged captions: lengths T, 2 ([SOS] [EOS]) and two in between; one [PAD] id inside a caption's length
    lengths = torch.tensor([T, 2, 5, T - 2])[:B]
    tokens = torch.zeros(B, T, dtype=torch.int64)
    for b in range(B):
        n = int(lengths[b])
        row = torch.randint(4, V, (n,), generator=g)
        row[0], row[-1] = 1, 2
        tokens[b, :n] = row
    tokens[0, 3] = PAD
    tokens[2, 1] = tokens[0, 4]                      # one token in two captions: its word rows add
    labels = None
    if mask_mode == 2:
        labels = torch.zeros_like(tokens)
        labels[0, 2], labels[2, 3], labels[3, 1], labels[3, 4] = 7, 9, 11, 7
    feat = torch.randn(B * Sk, Cv, generator=g, dtype=F64).abs()
    # ---- autograd of torch's modules
    feat_a = feat.clone().requires_grad_(True)
    mem = vp(feat_a).view(B, Sk, H)
    mem.retain_grad()
    x0 = emb(tokens)
    caption_mask = lengths.unsqueeze(1) < torch.ones_like(tokens).cumsum(dim=1)
    future = torch.triu(torch.full((T, T), float("-inf"), dtype=F64), diagonal=1) if mask_mode == 1 else None
    hooks, seen = [], {}
    for l, lay in enumerate(dec.layers):
        for i, m in ((1, lay.self_attn), (2, lay.multihead_attn), (3, lay.linear2)):
            hooks.append(m.register_forward_hook(
                lambda mod, inp, out, key=f"L{l}.branch{i}": seen.__setitem__(key, out[0] if isinstance(out, tuple)
                                                                                  else out)))
        hooks.append(lay.register_forward_hook(lambda mod, inp, out, key=f"L{l}.x3": seen.__setitem__(key, out)))
    y = dec(x0, mem, tgt_mask=future, tgt_key_padding_mask=caption_mask)
    for h in hooks:
        h.remove()
    logits = nn.functional.linear(y, emb.words.weight, out_bias)
    if labels is None:
        loss = nn.functional.cross_entropy(logits[:, :-1].reshape(-1, V), tokens[:, 1:].reshape(-1), ignore_index=PAD)
    else:
        loss = nn.functional.cross_entropy(logits.reshape(-1, V), labels.reshape(-1), ignore_index=PAD)
    loss.backward()
    # ---- the chained stage references
    P = {"textual.embedding." + n: p.detach() for n, p in emb.named_parameters()}
    P.update({"textual.transformer." + n: p.detach() for n, p in dec.named_parameters()})
    P.update({"textual.visual_projection." + n: p.detach() for n, p in vp.named_parameters()})
    P["textual.output.bias"] = out_bias.detach()
    vals, grads, dfeat = S.head_forward_backward(P, "textual.", feat.view(B, Sk, Cv), tokens, lengths, PAD, A,
                                                 norm_first, mask_mode, labels=labels)
    return dict(vals=vals, grads=grads, dfeat=dfeat, seen=seen, mem=mem, x0=x0, logits=logits, loss=loss,
                feat=feat_a, mods=mods, L=L, T=T, max_len=max_len, tokens=tokens)


@pytest.mark.parametrize("norm_first", [False, True], ids=["post-norm", "pre-norm"])
@pytest.mark.parametrize("mask_mode", [1, 2], ids=["future+padding", "padding-only"])
def test_head_stages_match_transformer_decoder_autograd(norm_first, mask_mode):
    c = _case(norm_first, mask_mode)
    v = c["vals"]
    _rel_close(v["mem"], c["mem"], "visual projection")
    _rel_close(v["x0"], c["x0"], "embedding")
    for key, ref in c["seen"].items():
        _rel_close(v[key], ref, key)
    _rel_close(v["logits"], c["logits"], "logits")
    _rel_close(v["loss"], c["loss"], "loss")
    _rel_close(v["dmem"], c["mem"].grad, "dmem")
    _rel_close(c["dfeat"].reshape(c["feat"].shape), c["feat"].grad, "dfeat")
    m = c["mods"]
    named = [("textual.embedding." + n, p) for n, p in m["emb"].named_parameters()]
    named += [("textual.transformer." + n, p) for n, p in m["dec"].named_parameters()]
    named += [("textual.visual_projection." + n, p) for n, p in m["vp"].named_parameters()]
    for name, p in named:
        assert p.grad is not None, name
        _rel_close(c["grads"][name], p.grad, name)
    assert len(c["grads"]) == len(named) + 1, sorted(set(c["grads"]) - {n for n, _ in named})
    # the pad row gets only the output projection's share; positions rows >= T none at all
    assert not bool(c["grads"]["textual.embedding.positions.weight"][c["T"]:].any())


def test_head_stages_embedding_pad_and_repeats():
    """embed_bwd: the pad row receives nothing from the lookup, even for a [PAD] id inside a caption, and a repeated
    token's rows add."""
    g = torch.Generator().manual_seed(3)
    V, H, T = 11, 128, 6
    tokens = torch.tensor([[1, 5, 0, 5, 2, 0], [1, 5, 7, 2, 0, 0]])
    words = torch.randn(V, H, generator=g, dtype=F64).requires_grad_(True)
    pos = torch.randn(8, H, generator=g, dtype=F64).requires_grad_(True)
    gamma = (1 + 0.2 * torch.randn(H, generator=g, dtype=F64)).requires_grad_(True)
    beta = (0.1 * torch.randn(H, generator=g, dtype=F64)).requires_grad_(True)
    z, _, _, out = S.embed_fwd(tokens, words, pos, gamma, beta, PAD)
    up = torch.randn(out.shape, generator=g, dtype=F64)
    out.backward(up)
    dw, dp, dg, db = S.embed_bwd(up, tokens, z.detach(), gamma.detach(), PAD, V, 8)
    for name, got, ref in (("words", dw, words.grad), ("positions", dp, pos.grad), ("gamma", dg, gamma.grad),
                           ("beta", db, beta.grad)):
        _rel_close(got, ref, name)
    assert not bool(dw[PAD].any()) and not bool(dp[T:].any())
    assert bool(dw[5].any()) and not bool(dw[3].any())
