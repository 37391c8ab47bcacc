"""GPU tests of beam-search captioning (H100): the decoding kernels against float64 torch, the engine's incremental
logits against the full-recompute `decoding_step` at every step, captions against the fixtures written from the
reference's own search and against the float64 oracle at random initialisation, and the search's lack of side effects
on parameters, BatchNorm buffers and a pending backward."""
import os

import pytest
import torch

from oracle import virtex_oracle as O
from tests import captioning_oracle as C

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _call(name, *args):
    from virtex_b200.ops import call
    call(name, *args)


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


# ---------------------------------------------------------------------------------------------------------- kernels
def _attn_ref(q, K, V):
    """q (rows, heads, 64), K / V (rows, Tk, heads, 64) float64 -> (rows, heads, 64)."""
    s = torch.einsum("rhd,rjhd->rhj", q, K) / 8.0
    return torch.einsum("rhj,rjhd->rhd", torch.softmax(s, -1), V)


@pytest.mark.parametrize("heads", [2, 8, 16, 32])
def test_attn_decode_self_over_indexed_cache(heads):
    torch.manual_seed(heads)
    H, R, Tmax = 64 * heads, 10, 29
    cache = torch.randn(R, Tmax, 2 * H, device=DEV).bfloat16()
    q = torch.randn(R, H, device=DEV).bfloat16()
    index = torch.randint(0, R, (Tmax + 1, R), device=DEV, dtype=torch.int32)
    out = torch.empty(R, H, device=DEV, dtype=torch.bfloat16)
    for t in range(1, Tmax + 1):
        _call("vtx_attn_decode", q.data_ptr(), H, cache.data_ptr(), cache.data_ptr() + 2 * H, 2 * H, Tmax * 2 * H,
              index.data_ptr(), R, out.data_ptr(), H, R, heads, 1, t, _stream())
        rows = index[:t].t().long()                                   # (R, t): cache row of key j of row m
        kv = cache.double()[rows, torch.arange(t, device=DEV)[None, :]]  # (R, t, 2H)
        ref = _attn_ref(q.double().view(R, heads, 64), kv[..., :H].reshape(R, t, heads, 64),
                        kv[..., H:].reshape(R, t, heads, 64)).reshape(R, H)
        assert rel(out, ref) < 4e-3, (t, rel(out, ref))


@pytest.mark.parametrize("heads,beam", [(2, 5), (16, 5), (32, 3), (4, 1)])
def test_attn_decode_cross_shared_by_beams(heads, beam):
    torch.manual_seed(100 + heads)
    H, B, Sk = 64 * heads, 3, 49
    kv = torch.randn(B * Sk, 2 * H, device=DEV).bfloat16()
    q = torch.randn(B * beam, H, device=DEV).bfloat16()
    out = torch.empty(B * beam, H, device=DEV, dtype=torch.bfloat16)
    _call("vtx_attn_decode", q.data_ptr(), H, kv.data_ptr(), kv.data_ptr() + 2 * H, 2 * H, Sk * 2 * H, 0, 0,
          out.data_ptr(), H, B, heads, beam, Sk, _stream())
    kvr = kv.double().view(B, Sk, 2 * H).repeat_interleave(beam, 0)
    ref = _attn_ref(q.double().view(-1, heads, 64), kvr[..., :H].reshape(-1, Sk, heads, 64),
                    kvr[..., H:].reshape(-1, Sk, heads, 64)).reshape(-1, H)
    assert rel(out, ref) < 4e-3


@pytest.mark.parametrize("H", [128, 1024, 2048])
def test_one_position_embedding(H):
    """vtx_embed_fwd with T = 1 over one position row: word + position t, LayerNorm(1e-8), zero row for token 0."""
    torch.manual_seed(H)
    V, Tpos, M, pos = 1000, 30, 12, 17
    words, positions = torch.randn(V, H, device=DEV), torch.randn(Tpos, H, device=DEV)
    gamma, beta = torch.rand(H, device=DEV) + 0.5, torch.randn(H, device=DEV) * 0.1
    tokens = torch.randint(1, V, (M,), device=DEV)
    tokens[[0, 5]] = 0
    z, st = torch.empty(M, H, device=DEV), torch.empty(M, 2, device=DEV)
    out, out_b = torch.empty(M, H, device=DEV), torch.empty(M, H, device=DEV, dtype=torch.bfloat16)
    seed = torch.zeros(1, dtype=torch.int64, device=DEV)
    _call("vtx_embed_fwd", tokens.data_ptr(), words.data_ptr(), positions[pos].data_ptr(), gamma.data_ptr(),
          beta.data_ptr(), z.data_ptr(), st.data_ptr(), out.data_ptr(), out_b.data_ptr(), M, 1, H, 0, 1e-8, 0.0,
          seed.data_ptr(), 0, _stream())
    x = words.double()[tokens] + positions.double()[pos]
    ref = (x - x.mean(-1, keepdim=True)) / torch.sqrt(x.var(-1, unbiased=False, keepdim=True) + 1e-8)
    ref = (ref * gamma.double() + beta.double()) * (tokens != 0).double()[:, None]
    assert (out.double() - ref).abs().max() < 1e-4
    assert torch.equal(out[[0, 5]], torch.zeros(2, H, device=DEV))
    assert torch.equal(out_b, out.bfloat16())


def _rows_ref(logits, last, eos, k):
    """Rule 4 in float64 + top-k with ties in ascending index -> (values, indices)."""
    lp = torch.log_softmax(logits.double(), -1)
    if last is not None:
        lp[torch.arange(lp.shape[0], device=DEV), last] = -10000
        ended = last == eos
        lp[ended] = float("-inf")
        lp[ended, eos] = 0.0
    order = torch.argsort(-lp, dim=1, stable=True)[:, :k]  # descending value, ties in ascending index
    return lp.gather(1, order), order


@pytest.mark.parametrize("k,V", [(2, 10000), (5, 10000), (2, 64)])
def test_beam_rows_penalty_eos_and_ties(k, V):
    torch.manual_seed(k * V)
    R, eos = 40, 2
    logits = torch.randn(R, V, device=DEV) * 3
    last = torch.randint(0, V, (R,), device=DEV)
    last[::4] = eos                                       # rows that ended: 0 at EOS, -inf elsewhere
    top1 = logits.argmax(1)
    last[1::4] = top1[1::4]                               # the penalty removes the best token of these rows
    logits[3, :] = 1.0                                    # a row of exact ties
    cv = torch.empty(R, k, device=DEV)
    ci = torch.empty(R, k, device=DEV, dtype=torch.int32)
    for use_last in (False, True):
        lst = last if use_last else None
        _call("vtx_beam_rows", logits.data_ptr(), V, R, V, 0 if lst is None else lst.data_ptr(), eos, k, cv.data_ptr(),
              ci.data_ptr(), _stream())
        vals, idx = _rows_ref(logits, lst, eos, k)
        assert torch.equal(ci.long(), idx)
        finite = torch.isfinite(vals)
        assert torch.equal(finite, torch.isfinite(cv))
        assert (cv.double()[finite] - vals[finite]).abs().max() < 2e-5
        if use_last:
            assert (ci[1::4] != last[1::4, None].int()).all() and (cv[::4, 0] == 0).all() and (ci[::4, 0] == eos).all()
            assert torch.isinf(cv[::4, 1]).all()


@pytest.mark.parametrize("beam,s", [(5, 0), (5, 7), (3, 1), (1, 4)])
def test_beam_select_and_table_gather(beam, s):
    torch.manual_seed(beam * 10 + s)
    B, k, steps, eos = 7, (beam if s == 0 else 2), 30, 2
    parents = 1 if s == 0 else beam
    R = B * beam
    cv = (torch.randn(B * parents, k, device=DEV) * 2).sort(1, descending=True).values
    cv[0, -1] = float("-inf")
    cv[1] = cv[2]                                         # equal candidates: ties in ascending candidate index
    ci = torch.randint(0, 100, (B * parents, k), device=DEV, dtype=torch.int32)
    ci[4 * parents:5 * parents] = eos                      # image 4: every new token is EOS
    scores = torch.randn(R, device=DEV)
    scores[2] = scores[1]
    scores_in = scores.clone()
    pred_in = torch.randint(0, 10000, (steps, R), device=DEV)
    index_in = torch.randint(0, R, (steps, R), device=DEV, dtype=torch.int32)
    pred_out, index_out = torch.full_like(pred_in, -7), torch.full_like(index_in, -7)
    parent = torch.empty(R, device=DEV, dtype=torch.int32)
    alive = torch.zeros(steps, device=DEV, dtype=torch.int32)
    _call("vtx_beam_select", cv.data_ptr(), ci.data_ptr(), parents, k, beam, scores.data_ptr() if s else 0,
          scores.data_ptr(), parent.data_ptr(), pred_in.data_ptr() if s else 0, pred_out.data_ptr(),
          index_in.data_ptr() if s else 0, index_out.data_ptr(), B, s, eos, alive.data_ptr(), _stream())
    cand = (cv.view(B, parents, k) + (scores_in.view(B, parents, 1) if s else 0)).view(B, parents * k)
    order = torch.argsort(-cand, dim=1, stable=True)[:, :beam]
    want_par = (torch.arange(B, device=DEV)[:, None] * parents + order // k).reshape(-1)
    assert torch.equal(scores.view(B, beam), cand.gather(1, order))
    assert torch.equal(parent.long(), want_par)
    assert torch.equal(pred_out[s], ci.view(B, -1).gather(1, order).reshape(-1).long())
    assert torch.equal(index_out[s], torch.arange(R, device=DEV, dtype=torch.int32))
    if s:   # the gathered tables: bit-exact copies of the parents' rows
        assert torch.equal(pred_out[:s], pred_in[:s, want_par])
        assert torch.equal(index_out[:s], index_in[:s, want_par])
    assert (pred_out[s + 1:] == -7).all()
    new_tok = pred_out[s].view(B, beam)
    assert int(alive[s]) == int(bool((new_tok != eos).any()))


# ---------------------------------------------------------------------------------------------------------- models
def _model(spec, state, beam, max_steps, bidirectional):
    from virtex_b200.factories import CaptionDecoderFactory
    from virtex_b200.models import BidirectionalCaptioningModel, ForwardCaptioningModel
    from virtex_b200.modules import TorchvisionVisualBackbone, TransformerDecoderTextualHead
    visual = TorchvisionVisualBackbone(spec.backbone, visual_feature_size=2048)
    textual = TransformerDecoderTextualHead(2048, spec.vocab, spec.hidden, spec.layers, spec.heads, spec.ffn,
                                            dropout=0.1, norm_first=spec.norm_first, max_caption_length=spec.max_len)
    decoder = CaptionDecoderFactory.create("beam_search", eos_index=C.EOS, max_steps=max_steps, beam_size=beam)
    cls = BidirectionalCaptioningModel if bidirectional else ForwardCaptioningModel
    model = cls(visual, textual, sos_index=C.SOS, eos_index=C.EOS, decoder=decoder)
    model.load_state_dict(O.to_reference_state_dict(state, spec), strict=True)
    return model.to(DEV).eval()


def _spec(hidden, layers, norm_first, bidirectional):
    return O.Spec(hidden=hidden, layers=layers, heads=hidden // 64, ffn=4 * hidden, norm_first=norm_first,
                  caption_backward=bidirectional)


@pytest.mark.parametrize("hidden,layers,norm_first,bidirectional", [
    (128, 1, False, True), (256, 2, True, False), (1024, 4, False, False), (2048, 1, False, True), (512, 3, True, True)])
def test_incremental_logits_match_full_recompute(hidden, layers, norm_first, bidirectional):
    """At every step, the engine's fp32 logits of every row equal decoding_step's full recompute of the same prefix
    (relative L2 <= 3e-2, the decoder parity tolerance)."""
    spec = _spec(hidden, layers, norm_first, bidirectional)
    model = _model(spec, O.synth_state(spec, 40 + layers, bn3_gain=0.25), 5, 30, bidirectional)
    image = O.synth_batch(3, seed=11)["image"].to(DEV)
    eng = model.engine  # decoding_step runs on the head's own engine; this one keeps its copy of the same weights
    worst, worst_abs = 0.0, 0.0
    with torch.no_grad():
        st = eng.beam_start(image, 5, 2, 30, C.SOS, C.EOS)
        fmap, h, w = eng.backbone_infer(image)
        vf = fmap.view(3, h, w, -1).permute(0, 3, 1, 2).float()
        pairs = [(st.logits[:3].clone(), model.decoding_step(vf, torch.full((3,), C.SOS, device=DEV)))]
        for _ in range(1, 30):
            prefix = st.tokens().clone()
            eng.beam_step(st)
            pairs.append((st.logits.clone(), model.decoding_step(vf, prefix)))
    for got, ref in pairs:
        worst, worst_abs = max(worst, rel(got, ref)), max(worst_abs, float((got - ref).abs().max()))
    print(f"L{layers}_H{hidden} {'pre' if norm_first else 'post'}: worst rel L2 {worst:.2e}, max abs {worst_abs:.4f}")
    assert worst <= 3e-2


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(os.path.join(golden_dir, C.GOLDEN))


def _oracle(state, spec, image):
    vf, P = C.visual_features(state, image, spec)
    return C.head_step(P, spec, vf)


@pytest.mark.parametrize("case", list(C.CASES))
def test_captions_equal_reference_fixture_where_decisive(golden, case):
    """model({"image": x})["predictions"] equals the reference's captions for every image whose recorded gaps all
    exceed 0.1 nats; every caption scores, under the float64 oracle, within 0.05 nats of the reference's best."""
    c, spec, g = C.CASES[case], C.case_spec(case), golden[case]
    state = C.case_state(case)
    model = _model(spec, state, c["beam"], c["max_steps"], spec.caption_backward)
    image = C.case_image(case).to(DEV)
    with torch.no_grad():
        pred = model({"image": image})["predictions"]
    assert pred.dtype == torch.int64 and pred.device.type == "cuda"
    dec = C.decisive({k: g[k] for k in ("node_gaps", "image_gaps")} | {"predictions": g["beams"]}, c["beam"], 0.1)
    want = g["predictions"].to(DEV)
    assert bool(dec.any()), "the fixture state has no decisive image: the token comparison would be empty"
    if bool(dec.all()):
        assert pred.shape == want.shape
    L = min(pred.shape[1], want.shape[1])
    assert torch.equal(pred[dec.to(DEV), :L], want[dec.to(DEV), :L])
    step = _oracle(state, spec, image)
    with torch.no_grad():
        diff = (C.caption_score(step, pred) - g["scores"][:, 0].to(DEV)).abs().max()
    print(f"{case}: L {pred.shape[1]} (reference {want.shape[1]}), decisive {dec.tolist()}, score gap {float(diff):.2e}")
    assert pred.shape == want.shape
    assert diff <= 0.05


def _cleaned(logits, last, eos=C.EOS):
    """The search's per-row scores (rule 4 of the search) in float64."""
    lp = torch.log_softmax(logits.double(), -1)
    lp[torch.arange(lp.shape[0], device=lp.device), last] = -10000
    ended = last == eos
    lp[ended] = float("-inf")
    lp[ended, eos] = 0.0
    return lp


@pytest.mark.parametrize("hidden,layers,norm_first,bidirectional,B", [
    (128, 1, False, True, 3), (256, 2, True, False, 3), (1024, 4, False, False, 3), (2048, 1, False, True, 3),
    (1024, 1, False, True, 256)])
def test_random_init_every_selection_is_right_within_the_logit_error(hidden, layers, norm_first, bidirectional, B):
    """At random initialisation (near-uniform next-token distributions) bf16 reorders near-tied candidates, and once
    two searches take different candidates their later steps are not comparable.  So every step of the GPU search is
    replayed in float64 on the GPU's own beams.  Let eps be the step's largest absolute difference between the engine's
    fp32 logits and the float64 oracle's logits on the same prefixes; a log-probability then differs by at most 2 eps.
    Then, using the GPU's parent scores:
      * every new token is within 4 eps of its parent row's per-node cut (the second-best float64 score);
      * every kept candidate is within 4 eps of its image's beam-size cut over the float64 candidates;
      * every new score is the parent's score plus the token's float64 score within 2 eps;
    plus fp32 rounding of the scores (1e-4).  The caption length equals the float64 oracle's, and a caption equal to the
    oracle's best scores within 0.05 nats of it."""
    spec = _spec(hidden, layers, norm_first, bidirectional)
    state = O.synth_state(spec, 50 + layers, bn3_gain=0.25)
    model = _model(spec, state, 5, 30, bidirectional)
    image = O.synth_batch(B, seed=12)["image"].to(DEV)
    beam, steps, slack = 5, 30, 1e-4
    eng = model.engine
    step = _oracle(state, spec, image)
    worst_eps, worst_margin = 0.0, 0.0
    with torch.no_grad():
        st = eng.beam_start(image, beam, 2, steps, C.SOS, C.EOS)
        logits = step(torch.full((B,), C.SOS, device=DEV))
        eps = float((st.logits[:B].double() - logits).abs().max())
        lp = torch.log_softmax(logits, -1)
        chosen = lp.gather(1, st.tokens()[:, 0].view(B, beam))
        cut = lp.topk(beam).values[:, -1:]
        assert (chosen >= cut - 4 * eps - slack).all()
        assert ((st.scores.double().view(B, beam) - chosen).abs() <= 2 * eps + slack).all()
        worst_eps = eps
        while st.L < steps and st.alive[st.L - 1].item():
            prefix, S = st.tokens().clone(), st.scores.double().clone()
            eng.beam_step(st)
            logits = step(prefix)
            eps = float((st.logits.double() - logits).abs().max())
            lp = _cleaned(logits, prefix[:, -1])
            top = lp.topk(2).values                                          # (R, 2): the per-node cut is top[:, 1]
            cut = (top + S[:, None]).view(B, beam * 2).topk(beam).values[:, -1].repeat_interleave(beam)
            parent, tok = st.parent.long(), st.tokens()[:, -1]
            tok_lp = lp[parent, tok]
            assert (tok_lp >= top[parent, 1] - 4 * eps - slack).all()
            kept = tok_lp + S[parent]
            assert (kept >= cut - 4 * eps - slack).all()
            assert ((st.scores.double() - S[parent] - tok_lp).abs() <= 2 * eps + slack).all()
            worst_eps = max(worst_eps, eps)
            worst_margin = max(worst_margin, float((cut - kept).clamp_min(0).max()))
        pred = st.best()
        ref = C.beam_search(step, B, beam, steps, device=DEV)
        best = ref["predictions"][:, 0]
        diff = (C.caption_score(step, pred) - ref["scores"][:, 0]).abs()
    same = (pred == best).all(1) if pred.shape == best.shape else torch.zeros(B, dtype=torch.bool, device=DEV)
    print(f"L{layers}_H{hidden} B{B}: L {pred.shape[1]} oracle {best.shape[1]}, tokens equal for {int(same.sum())}/{B} "
          f"images; largest logit error {worst_eps:.4f}, largest kept-below-cut margin {worst_margin:.4f}")
    assert pred.shape[1] == best.shape[1]
    assert (diff[same] <= 0.05).all()


def test_search_has_no_side_effects():
    """Parameters and BatchNorm buffers stay bit-identical after a search, and forward -> search -> backward gives the
    gradients of forward -> backward."""
    spec = _spec(128, 1, False, True)
    model = _model(spec, O.synth_state(spec, 61, bn3_gain=0.25), 5, 30, True)
    batch = {k: v.to(DEV) for k, v in O.synth_batch(2, seed=13, ragged=True).items()}
    before = {k: v.clone() for k, v in model.state_dict().items()}
    model.eval()
    with torch.no_grad():
        model({"image": batch["image"]})
    for k, v in model.state_dict().items():
        assert torch.equal(v, before[k]), k

    def grads(search):
        model.train()
        for p in model.parameters():
            p.grad = None
        loss = model(batch)["loss"]
        if search:
            model.eval()
            with torch.no_grad():
                model({"image": batch["image"]})
            model.train()
        loss.backward()
        return {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}

    g0, g1, g2 = grads(False), grads(True), grads(False)
    assert g0.keys() == g1.keys()
    for n in g0:
        noise = rel(g2[n], g0[n])                   # run-to-run spread of the atomically accumulated gradients
        assert rel(g1[n], g0[n]) <= max(10 * noise, 1e-5), n
