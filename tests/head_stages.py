"""Float64 references of the textual head's stages, one function per stage, each a pure function of tensors: the stage's
inputs and the parameters it reads (tests/test_head_stages_gpu.py feeds them the engine's own inputs of each stage and
the modules' parameters, rounded to bf16 by torch where the engine reads its bf16 mirror; tests/test_head_stages_cpu.py
chains them in exact float64 against autograd of torch's nn.TransformerDecoder).

Layouts: a caption batch is [B, T, H] (row b * T + t of the engine's [M, H] matrices); the visual memory is [B, Sk, H].
Dropout enters as given scale tensors (0 or 1 / (1 - p) per element, None for p = 0): the embedding's after its
LayerNorm and before the pad zeroing, each sublayer's on its branch before the residual add, the attention
probabilities' after the softmax, the FFN's after the GELU.  The engine's dropout sites are `site(...)`.

Where a stage is a linear layer, `linear` also returns sum_k |x_k w_k| + |b| (`mag`), from which the GPU replay builds
the VtxGemm bound of tests/gemm_reference.py.
"""
import math

import torch

F64 = torch.float64
EPS_EMBED, EPS_LN = 1e-8, 1e-5


def site(direction, layer=None, k=0):
    """Dropout site of the engine's head: direction * 1000 for the embedding; for layer l, direction * 1000 +
    10 (l + 1) + k with k = 0 self-attention probabilities, 1 / 3 / 5 the residual dropout of sublayer 1 / 2 / 3,
    2 cross-attention probabilities, 4 the FFN's GELU."""
    return direction * 1000 + (0 if layer is None else 10 * (layer + 1) + k)


# ------------------------------------------------------------------------------------------------ LayerNorm
def ln_fwd(z, gamma, beta, eps=EPS_LN):
    """LayerNorm over the last axis: (y, mean, rstd), biased variance."""
    mean = z.mean(-1, keepdim=True)
    rstd = (((z - mean) ** 2).mean(-1, keepdim=True) + eps).rsqrt()
    return (z - mean) * rstd * gamma + beta, mean[..., 0], rstd[..., 0]


def ln_bwd(g, z, gamma, eps=EPS_LN):
    """Backward of ln_fwd for upstream g: (dz, dgamma, dbeta), the parameter gradients summed over every row."""
    H = z.shape[-1]
    mean = z.mean(-1, keepdim=True)
    rstd = (((z - mean) ** 2).mean(-1, keepdim=True) + eps).rsqrt()
    xh = (z - mean) * rstd
    dxh = g * gamma
    s1 = dxh.sum(-1, keepdim=True) / H
    s2 = (dxh * xh).sum(-1, keepdim=True) / H
    dz = rstd * (dxh - s1 - xh * s2)
    rows = tuple(range(g.dim() - 1))
    return dz, (g * xh).sum(rows), g.sum(rows)


def _drop(x, scale):
    return x if scale is None else x * scale


# ------------------------------------------------------------------------------------------------ embedding
def embed_fwd(tokens, words, positions, gamma, beta, pad, scale=None):
    """WordAndPositionalEmbedding: z = words[tok] + positions[t], LayerNorm(eps 1e-8), dropout, zeroed where
    tok == pad.  (z, mean, rstd, out), [B, T, H] / [B, T]."""
    T = tokens.shape[1]
    z = words[tokens] + positions[:T][None]
    y, mean, rstd = ln_fwd(z, gamma, beta, EPS_EMBED)
    out = _drop(y, scale) * (tokens != pad).to(z.dtype)[..., None]
    return z, mean, rstd, out


def embed_bwd(g, tokens, z, gamma, pad, vocab, max_len, scale=None):
    """Backward of embed_fwd for upstream g [B, T, H]: (d_words [vocab, H], d_positions [max_len, H], dgamma, dbeta).
    Nothing reaches the pad row from the lookup (its rows are zeroed); repeated tokens add; positions rows >= T stay
    zero."""
    T, H = tokens.shape[1], z.shape[-1]
    keep = tokens != pad
    gk = _drop(g, scale) * keep.to(g.dtype)[..., None]
    dz, dgamma, dbeta = ln_bwd(gk, z, gamma, EPS_EMBED)
    d_words = g.new_zeros(vocab, H).index_add_(0, tokens[keep], dz[keep])
    d_pos = g.new_zeros(max_len, H)
    d_pos[:T] = dz.sum(0)
    return d_words, d_pos, dgamma, dbeta


# ------------------------------------------------------------------------------------------------ linear layers
def linear(x, w, b=None):
    """y = x w^T + b over the last axis, and mag = |x| |w|^T + |b|."""
    y = x @ w.t()
    mag = x.abs() @ w.abs().t()
    if b is not None:
        y, mag = y + b, mag + b.abs()
    return y, mag


def linear_bwd(dy, x, w):
    """Backward of linear: (dx, dW, db, mag of dx, mag of dW), the parameter gradients summed over every row."""
    d2, x2 = dy.reshape(-1, dy.shape[-1]), x.reshape(-1, x.shape[-1])
    dx = dy @ w
    dxm = dy.abs() @ w.abs()
    return dx, d2.t() @ x2, d2.sum(0), dxm, d2.abs().t() @ x2.abs()


# ------------------------------------------------------------------------------------------------ attention
def heads(x, A):
    """[B, T, A * 64] -> [B, A, T, 64]."""
    B, T, H = x.shape
    return x.reshape(B, T, A, H // A).transpose(1, 2)


def merge(x):
    """[B, A, T, 64] -> [B, T, A * 64]."""
    B, A, T, D = x.shape
    return x.transpose(1, 2).reshape(B, T, A * D)


def allowed(B, Tq, Tk, lengths, mask_mode, device=None):
    """[B, 1, Tq, Tk] keys each query may attend to: mask_mode 1 = j <= i and j < lengths[b] (future + key padding),
    2 = j < lengths[b] (key padding only), 0 = every key (cross-attention)."""
    i = torch.arange(Tq, device=device)[:, None]
    j = torch.arange(Tk, device=device)[None, :]
    if mask_mode == 0:
        return torch.ones(B, 1, Tq, Tk, dtype=torch.bool, device=device)
    ok = j[None] < lengths.view(B, 1, 1)
    if mask_mode == 1:
        ok = ok & (j <= i)[None]
    return ok[:, None]


def attention(q, k, v, A, lengths, mask_mode, scale=None):
    """Multi-head attention cores of [B, Tq, H] queries over [B, Tk, H] keys / values, head_dim 64, logits scaled by
    1/8: (o [B, Tq, H], softmax P [B, A, Tq, Tk])."""
    B, Tq, _ = q.shape
    Tk = k.shape[1]
    q4, k4, v4 = heads(q, A), heads(k, A), heads(v, A)
    s = (q4 @ k4.transpose(-1, -2)) / math.sqrt(q4.shape[-1])
    s = s.masked_fill(~allowed(B, Tq, Tk, lengths, mask_mode, q.device), float("-inf"))
    P = torch.softmax(s, -1)
    return merge(_drop(P, scale) @ v4), P


def attention_bwd(do, q, k, v, P, A, scale=None):
    """Backward of attention from the forward's softmax P: (dq, dk, dv), [B, T, H] each."""
    q4, k4, v4, do4 = heads(q, A), heads(k, A), heads(v, A), heads(do, A)
    Pd = _drop(P, scale)
    dv = Pd.transpose(-1, -2) @ do4
    dP = _drop(do4 @ v4.transpose(-1, -2), scale)
    dS = P * (dP - (P * dP).sum(-1, keepdim=True)) / math.sqrt(q4.shape[-1])
    return merge(dS @ k4), merge(dS.transpose(-1, -2) @ q4), merge(dv)


# ------------------------------------------------------------------------------------------------ GELU
def gelu(u):
    return 0.5 * u * (1.0 + torch.erf(u / math.sqrt(2.0)))


def gelu_grad(u):
    return 0.5 * (1.0 + torch.erf(u / math.sqrt(2.0))) + u * torch.exp(-0.5 * u * u) / math.sqrt(2.0 * math.pi)


# ------------------------------------------------------------------------------------------------ sublayers
def self_attn_fwd(x, w_in, b_in, w_out, b_out, A, lengths, mask_mode, scale=None):
    """nn.MultiheadAttention(x, x, x) of one decoder layer: (out, cache for self_attn_bwd)."""
    H = x.shape[-1]
    qkv, _ = linear(x, w_in, b_in)
    q, k, v = qkv[..., :H], qkv[..., H:2 * H], qkv[..., 2 * H:]
    o, P = attention(q, k, v, A, lengths, mask_mode, scale)
    out, _ = linear(o, w_out, b_out)
    return out, dict(x=x, qkv=qkv, o=o, P=P)


def self_attn_bwd(dy, c, w_in, w_out, A, scale=None):
    """(dx, {w_in, b_in, w_out, b_out: gradients}, do, dqkv)."""
    H = dy.shape[-1]
    qkv = c["qkv"]
    do, dwo, dbo, _, _ = linear_bwd(dy, c["o"], w_out)
    dq, dk, dv = attention_bwd(do, qkv[..., :H], qkv[..., H:2 * H], qkv[..., 2 * H:], c["P"], A, scale)
    dqkv = torch.cat([dq, dk, dv], -1)
    dx, dwi, dbi, _, _ = linear_bwd(dqkv, c["x"], w_in)
    return dx, dict(w_in=dwi, b_in=dbi, w_out=dwo, b_out=dbo), do, dqkv


def cross_attn_fwd(x, mem, w_in, b_in, w_out, b_out, A, scale=None):
    """nn.MultiheadAttention(x, mem, mem): Q from w_in[:H], K | V of the memory [B, Sk, H] from w_in[H:]."""
    H = x.shape[-1]
    qc, _ = linear(x, w_in[:H], b_in[:H])
    kv, _ = linear(mem, w_in[H:], b_in[H:])
    o, P = attention(qc, kv[..., :H], kv[..., H:], A, None, 0, scale)
    out, _ = linear(o, w_out, b_out)
    return out, dict(x=x, mem=mem, qc=qc, kv=kv, o=o, P=P)


def cross_attn_bwd(dy, c, w_in, w_out, A, scale=None):
    """(dx, dmem contribution, {w_in, b_in, w_out, b_out: gradients}, do, dqc, dkv)."""
    H = dy.shape[-1]
    kv = c["kv"]
    do, dwo, dbo, _, _ = linear_bwd(dy, c["o"], w_out)
    dqc, dk, dv = attention_bwd(do, c["qc"], kv[..., :H], kv[..., H:], c["P"], A, scale)
    dkv = torch.cat([dk, dv], -1)
    dx, dwq, dbq, _, _ = linear_bwd(dqc, c["x"], w_in[:H])
    dmem, dwkv, dbkv, _, _ = linear_bwd(dkv, c["mem"], w_in[H:])
    return dx, dmem, dict(w_in=torch.cat([dwq, dwkv]), b_in=torch.cat([dbq, dbkv]), w_out=dwo, b_out=dbo), do, dqc, dkv


def ffn_fwd(x, w1, b1, w2, b2, scale=None):
    u, _ = linear(x, w1, b1)
    h = _drop(gelu(u), scale)
    out, _ = linear(h, w2, b2)
    return out, dict(x=x, u=u, h=h)


def ffn_bwd(dy, c, w1, w2, scale=None):
    """(dx, {w1, b1, w2, b2: gradients}, dh after the GELU backward)."""
    dh, dw2, db2, _, _ = linear_bwd(dy, c["h"], w2)
    du = _drop(dh, scale) * gelu_grad(c["u"])
    dx, dw1, db1, _, _ = linear_bwd(du, c["x"], w1)
    return dx, dict(w1=dw1, b1=db1, w2=dw2, b2=db2), du


def post_norm_fwd(x, branch, gamma, beta, scale=None):
    """xo = LN(x + dropout(branch)): (xo, z)."""
    z = x + _drop(branch, scale)
    return ln_fwd(z, gamma, beta)[0], z


def post_norm_bwd(g, z, gamma, scale=None):
    """(gradient of x, gradient of the branch, dgamma, dbeta)."""
    dz, dg, db = ln_bwd(g, z, gamma)
    return dz, _drop(dz, scale), dg, db


def pre_norm_fwd(x, run, gamma, beta, scale=None):
    """xo = x + dropout(f(LN(x))) for the branch f = run: (xo, LN(x))."""
    n = ln_fwd(x, gamma, beta)[0]
    return x + _drop(run(n), scale), n


# ------------------------------------------------------------------------------------------------ output and loss
def targets(tokens, pad, labels=None):
    """Per-row targets [B, T]: next-token targets tokens[:, 1:] with the last position ignored (shift 1), or the
    masked-LM labels as given (shift 0)."""
    if labels is not None:
        return labels
    return torch.cat([tokens[:, 1:], torch.full_like(tokens[:, :1], pad)], 1)


def cross_entropy(logits, tgt, pad):
    """Token-mean cross entropy over targets != pad: (count, loss, dlogits of the loss)."""
    z = logits.reshape(-1, logits.shape[-1])
    t = tgt.reshape(-1)
    valid = t != pad
    n = int(valid.sum())
    lse = torch.logsumexp(z, -1)
    nll = lse - z.gather(1, t[:, None])[:, 0]
    d = (torch.softmax(z, -1) - torch.nn.functional.one_hot(t, z.shape[-1]).to(z.dtype)) * valid[:, None] / max(n, 1)
    return n, (nll * valid).sum() / max(n, 1), d.view(logits.shape)


# ------------------------------------------------------------------------------------------------ whole head
def layer_params(P, prefix):
    """The float64 parameters of decoder layer `prefix` (ending in '.') as the sublayer functions take them."""
    g = lambda n: P[prefix + n]  # noqa: E731
    return dict(sa=(g("self_attn.in_proj_weight"), g("self_attn.in_proj_bias"), g("self_attn.out_proj.weight"),
                    g("self_attn.out_proj.bias")),
                ca=(g("multihead_attn.in_proj_weight"), g("multihead_attn.in_proj_bias"),
                    g("multihead_attn.out_proj.weight"), g("multihead_attn.out_proj.bias")),
                ff=(g("linear1.weight"), g("linear1.bias"), g("linear2.weight"), g("linear2.bias")),
                norms=[(g(f"norm{i}.weight"), g(f"norm{i}.bias")) for i in (1, 2, 3)])


def head_forward_backward(P, head, feat, tokens, lengths, pad, A, norm_first, mask_mode, labels=None, dlogits=None):
    """One direction of the decoder head in float64, chained from the stage functions at p = 0: visual projection,
    embedding, layers, (final LayerNorm), tied output, cross entropy; then the backward of the loss (or of the given
    dlogits).  P: float64 parameters by name, `head` the prefix of the direction's decoder ('textual.' or
    'backward_textual.'); the embedding, output bias and visual projection are always 'textual.'.  Returns
    (values, grads, dfeat): the intermediates by name, the parameter gradients by name, the feature gradient."""
    B, T = tokens.shape
    V, H = P["textual.embedding.words.weight"].shape
    L = sum(1 for n in P if n.startswith(head + "transformer.layers.") and n.endswith(".norm1.weight"))
    vals, grads = {}, {}

    def add(name, g):
        grads[name] = grads[name] + g if name in grads else g

    mem, _ = linear(feat, P["textual.visual_projection.weight"], P["textual.visual_projection.bias"])
    emb = "textual.embedding."
    z0, _, _, x = embed_fwd(tokens, P[emb + "words.weight"], P[emb + "positions.weight"],
                            P[emb + "layer_norm.weight"], P[emb + "layer_norm.bias"], pad)
    vals.update(mem=mem, z0=z0, x0=x)
    caches = []
    for l in range(L):
        lp = layer_params(P, f"{head}transformer.layers.{l}.")
        fns = (lambda inp: self_attn_fwd(inp, *lp["sa"], A, lengths, mask_mode),
               lambda inp: cross_attn_fwd(inp, mem, *lp["ca"], A),
               lambda inp: ffn_fwd(inp, *lp["ff"]))
        lc = []
        for i, f in enumerate(fns, 1):
            gamma, beta = lp["norms"][i - 1]
            if norm_first:
                n = ln_fwd(x, gamma, beta)[0]
                br, c = f(n)
                xo = x + br
                lc.append((x, n, c))
            else:
                br, c = f(x)
                xo, z = post_norm_fwd(x, br, gamma, beta)
                lc.append((x, z, c))
            vals[f"L{l}.branch{i}"], vals[f"L{l}.x{i}"] = br, xo
            x = xo
        caches.append(lc)
    xf = x
    if norm_first:
        fn = head + "transformer.norm."
        x = ln_fwd(xf, P[fn + "weight"], P[fn + "bias"])[0]
    logits, _ = linear(x, P[emb + "words.weight"], P["textual.output.bias"])
    vals.update(x_out=x, logits=logits)
    n, loss, d = cross_entropy(logits, targets(tokens, pad, labels), pad)
    vals.update(count=n, loss=loss)
    if dlogits is None:
        dlogits = d
    # ---- backward
    dx, dw, db, _, _ = linear_bwd(dlogits, x, P[emb + "words.weight"])
    add(emb + "words.weight", dw)
    add("textual.output.bias", db)
    if norm_first:
        dx, dg, dbeta = ln_bwd(dx, xf, P[fn + "weight"])
        add(fn + "weight", dg)
        add(fn + "bias", dbeta)
    dmem = torch.zeros_like(mem)
    for l in reversed(range(L)):
        q = f"{head}transformer.layers.{l}."
        lp = layer_params(P, q)
        for i in (3, 2, 1):
            xin, zn, c = caches[l][i - 1]
            gamma = lp["norms"][i - 1][0]
            if norm_first:
                dbr = dx
            else:
                dx, dbr, dg, dbeta = post_norm_bwd(dx, zn, gamma)   # dx: the skip path's share
                add(q + f"norm{i}.weight", dg)
                add(q + f"norm{i}.bias", dbeta)
            if i == 3:
                din, gw, _ = ffn_bwd(dbr, c, lp["ff"][0], lp["ff"][2])
                names = dict(w1="linear1.weight", b1="linear1.bias", w2="linear2.weight", b2="linear2.bias")
            elif i == 2:
                din, dm, gw, _, _, _ = cross_attn_bwd(dbr, c, lp["ca"][0], lp["ca"][2], A)
                dmem = dmem + dm
                names = dict(w_in="multihead_attn.in_proj_weight", b_in="multihead_attn.in_proj_bias",
                             w_out="multihead_attn.out_proj.weight", b_out="multihead_attn.out_proj.bias")
            else:
                din, gw, _, _ = self_attn_bwd(dbr, c, lp["sa"][0], lp["sa"][2], A)
                names = dict(w_in="self_attn.in_proj_weight", b_in="self_attn.in_proj_bias",
                             w_out="self_attn.out_proj.weight", b_out="self_attn.out_proj.bias")
            for k, v in gw.items():
                add(q + names[k], v)
            if norm_first:
                dn, dg, dbeta = ln_bwd(din, xin, gamma)
                add(q + f"norm{i}.weight", dg)
                add(q + f"norm{i}.bias", dbeta)
                dx = dx + dn
            else:
                dx = dx + din
    dw, dp, dg, dbeta = embed_bwd(dx, tokens, z0, P[emb + "layer_norm.weight"], pad, V,
                                  P[emb + "positions.weight"].shape[0])
    add(emb + "words.weight", dw)
    add(emb + "positions.weight", dp)
    add(emb + "layer_norm.weight", dg)
    add(emb + "layer_norm.bias", dbeta)
    dfeat, dwv, dbv, _, _ = linear_bwd(dmem, feat, P["textual.visual_projection.weight"])
    add("textual.visual_projection.weight", dwv)
    add("textual.visual_projection.bias", dbv)
    vals["dmem"] = dmem
    return vals, grads, dfeat
