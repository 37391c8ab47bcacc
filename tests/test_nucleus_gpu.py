"""GPU tests of nucleus-sampling captioning (H100): the sampling kernel against the float64 rule with the kernel's own
uniforms replayed on the host, its distribution (chi-square), determinism, the engine's incremental logits against the
full-recompute `decoding_step` at every step, captions against the fixture written from the reference's own sampler and
against the float64 nucleus on the GPU's own prefixes, and the sampler's lack of side effects."""
import os

import numpy as np
import pytest
import torch

from oracle import virtex_oracle as O
from tests import captioning_oracle as C
from tests import nucleus_oracle as N
from tests.dropout_replica import as_i64

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _sample(logits, last, p, seed, s, eos=N.EOS, steps=None):
    """One vtx_nucleus_sample launch at step s into a fresh table -> (tokens (R,), alive[s])."""
    from virtex_b200.ops import call
    R, V = logits.shape
    steps = steps or s + 1
    pred = torch.full((steps, R), -7, dtype=torch.int64, device=DEV)
    alive = torch.zeros(steps, dtype=torch.int32, device=DEV)
    seed_t = torch.tensor([as_i64(seed)], dtype=torch.int64, device=DEV)
    call("vtx_nucleus_sample", logits.data_ptr(), logits.stride(0), R, V, last.data_ptr(), eos, p, seed_t.data_ptr(), s,
         pred.data_ptr(), alive.data_ptr(), _stream())
    torch.cuda.synchronize()
    assert (pred[:s] == -7).all() and (pred[s + 1:] == -7).all()
    return pred[s], int(alive[s])


def _u24(seed, s, R):
    return torch.from_numpy(N.uniform24(seed, s, R, np.arange(R)).astype(np.int64)).to(DEV)


def _rows(V, seed):
    """64 rows of logits exercising the rules: varied spreads, the last token at the row's best, EOS rows, a row of
    exact ties spread over the vocabulary, and rows whose nucleus is the last token alone."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    R = 64
    scale = torch.logspace(-1, 1.3, R, device=DEV)[:, None]
    logits = torch.randn(R, V, device=DEV, generator=g) * scale
    last = torch.randint(0, V, (R,), device=DEV, generator=g)
    last[1::5] = logits.argmax(1)[1::5]                         # the ban removes the row's best token
    last[2::9] = N.EOS                                          # ended rows continue with EOS
    ties = torch.arange(3, V, max(1, V // 7), device=DEV)[:7]    # 7 exact ties over the vocabulary, nothing else
    logits[5] = -30.0
    logits[5, ties] = 20.0
    last[5] = 0
    logits[6, last[6]] = 60.0                                   # the nucleus is the banned token alone (p < 1)
    logits[7, 11] = 60.0
    last[7] = 11
    return logits.contiguous(), last, ties


@pytest.mark.parametrize("V", [64, 10000, 10001])
@pytest.mark.parametrize("p", [0.5, 0.9, 1.0])
def test_kernel_against_float64_rule_with_replayed_uniforms(V, p):
    logits, last, ties = _rows(V, V + int(10 * p))
    R = logits.shape[0]
    excluded, checked = 0, 0
    for seed, s in [(1, 0), (12345, 3), (2 ** 63 + 5, 29), (-77, 7)]:
        tok, alive = _sample(logits, last, p, seed, s)
        u24 = _u24(seed, s, R)
        ref = N.kernel_rule(logits, last, p, u24)
        assert alive == int(bool((tok != N.EOS).any()))
        ended = last == N.EOS
        assert (tok[ended] == N.EOS).all()
        # uniform fallback: floor(u * V), exactly
        assert torch.equal(tok[ref["alone"] & ~ended], ((u24 * V) >> 24)[ref["alone"] & ~ended])
        if p < 1.0:
            assert bool(ref["alone"][6]) and bool(ref["alone"][7])
        live = ~ended & ~ref["alone"]
        assert (tok[live] != last[live]).all()                  # the ban
        # rows whose cut lies within 1e-5 of p may keep a different crossing token in fp32; at p = 1 the disputed
        # tokens are the tail's, of mass below fp32 rounding, which the boundary exclusion covers
        sure = live & ((ref["margin"] > 1e-5) | (p >= 1.0))
        rows = torch.arange(R, device=DEV)
        assert ref["keep"][rows[sure], tok[sure]].all()          # the token lies in the float64 nucleus
        exact = sure & (ref["boundary"] > 1e-6)
        assert torch.equal(tok[exact], ref["token"][exact])      # ... and is the float64 inverse CDF at u
        excluded += int((live & ~exact).sum())
        checked += int(exact.sum())
        if p < 1.0:  # the exact-tie row: the nucleus is the first ties in ascending id
            n_keep = int(ref["keep"][5].sum())
            assert torch.equal(ref["keep"][5].nonzero().flatten(), ties[:n_keep])
            assert int(tok[5]) in ties[:n_keep].tolist()
    print(f"V {V} p {p}: {checked} rows compared token for token, {excluded} excluded within 1e-5 of the cut or 1e-6 "
          f"of a CDF boundary")
    assert checked >= R


def test_kernel_rejects_bad_arguments():
    from virtex_b200.lib import VtxError
    from virtex_b200.ops import call
    logits = torch.zeros(2, 40000, device=DEV)
    last = torch.zeros(2, dtype=torch.int64, device=DEV)
    pred = torch.zeros(1, 2, dtype=torch.int64, device=DEV)
    alive = torch.zeros(1, dtype=torch.int32, device=DEV)
    seed = torch.zeros(1, dtype=torch.int64, device=DEV)
    for V, p in ((40000, 0.9), (100, 1.5), (100, -0.1), (100, float("nan"))):
        with pytest.raises(VtxError):
            call("vtx_nucleus_sample", logits.data_ptr(), 40000, 2, V, last.data_ptr(), 2, p, seed.data_ptr(), 0,
                 pred.data_ptr(), alive.data_ptr(), _stream())


def test_kernel_distribution_chi_square():
    """65 536 draws from one fixed row (one row per draw, counters s * R + row) against the filtered distribution."""
    from scipy.stats import chisquare
    V, R, p = 64, 65536, 0.9
    g = torch.Generator(device=DEV).manual_seed(3)
    row = torch.randn(V, device=DEV, generator=g) * 1.5
    logits = row.expand(R, V).contiguous()
    last = torch.full((R,), int(row.argmax()), dtype=torch.int64, device=DEV)
    tok, _ = _sample(logits, last, p, 987654321, 0)
    ref = N.kernel_rule(logits[:1], last[:1], p, torch.zeros(1, dtype=torch.int64, device=DEV))
    cand = ref["keep"][0].clone()
    cand[last[0]] = False
    w = torch.where(cand, torch.exp(row.double() - row.double()[cand].max()), 0.0)
    prob = (w / w.sum()).cpu().numpy()
    counts = torch.bincount(tok, minlength=V).cpu().numpy()
    assert counts[~cand.cpu().numpy()].sum() == 0
    keep = prob * R >= 5
    obs = np.append(counts[keep], counts[~keep].sum())
    exp = np.append(prob[keep] * R, prob[~keep].sum() * R)
    if exp[-1] == 0:
        obs, exp = obs[:-1], exp[:-1]
    stat, pval = chisquare(obs, exp)
    print(f"chi-square over {len(obs)} bins: {stat:.1f}, p-value {pval:.3f}")
    assert pval > 1e-3


# ---------------------------------------------------------------------------------------------------------- models
def _model(spec, state, p, max_steps, bidirectional):
    from virtex_b200.factories import CaptionDecoderFactory
    from virtex_b200.models import BidirectionalCaptioningModel, ForwardCaptioningModel
    from virtex_b200.modules import TorchvisionVisualBackbone, TransformerDecoderTextualHead
    visual = TorchvisionVisualBackbone(spec.backbone, visual_feature_size=2048)
    textual = TransformerDecoderTextualHead(2048, spec.vocab, spec.hidden, spec.layers, spec.heads, spec.ffn,
                                            dropout=0.1, norm_first=spec.norm_first, max_caption_length=spec.max_len)
    decoder = CaptionDecoderFactory.create("nucleus_sampling", eos_index=C.EOS, max_steps=max_steps, nucleus_size=p)
    cls = BidirectionalCaptioningModel if bidirectional else ForwardCaptioningModel
    model = cls(visual, textual, sos_index=C.SOS, eos_index=C.EOS, decoder=decoder)
    model.load_state_dict(O.to_reference_state_dict(state, spec), strict=True)
    return model.to(DEV).eval()


def _spec(hidden, layers, norm_first, bidirectional):
    return O.Spec(hidden=hidden, layers=layers, heads=hidden // 64, ffn=4 * hidden, norm_first=norm_first,
                  caption_backward=bidirectional)


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def test_same_seed_same_captions_and_successive_calls_differ():
    spec = _spec(128, 1, False, True)
    model = _model(spec, O.synth_state(spec, 70, bn3_gain=0.25), 0.9, 30, True)
    image = O.synth_batch(4, seed=14)["image"].to(DEV)
    with torch.no_grad():
        torch.manual_seed(5)
        a = model({"image": image})["predictions"]
        c = model({"image": image})["predictions"]
        torch.manual_seed(5)
        b = model({"image": image})["predictions"]
    assert a.dtype == torch.int64 and a.device.type == "cuda"
    assert torch.equal(a, b)
    assert a.shape != c.shape or not torch.equal(a, c)


@pytest.mark.parametrize("hidden,layers,norm_first,bidirectional", [
    (128, 1, False, True), (256, 2, True, False), (1024, 4, False, False), (2048, 1, False, True), (512, 3, True, True)])
def test_incremental_logits_match_full_recompute(hidden, layers, norm_first, bidirectional):
    """At every step, the engine's fp32 logits equal decoding_step's full recompute of the same SOS-prefixed prefix
    (relative L2 <= 3e-2, the decoder parity tolerance)."""
    spec = _spec(hidden, layers, norm_first, bidirectional)
    model = _model(spec, O.synth_state(spec, 40 + layers, bn3_gain=0.25), 0.9, 30, bidirectional)
    image = O.synth_batch(3, seed=11)["image"].to(DEV)
    eng = model.engine
    worst = 0.0
    with torch.no_grad():
        st = eng.nucleus_start(image, 0.9, 30, C.SOS, C.EOS, 17)
        fmap, h, w = eng.backbone_infer(image)
        vf = fmap.view(3, h, w, -1).permute(0, 3, 1, 2).float()
        sos = torch.full((3, 1), C.SOS, dtype=torch.int64, device=DEV)
        pairs = [(st.logits.clone(), model.decoding_step(vf, sos))]
        while st.L < 30:
            prefix = torch.cat([sos, st.tokens()], 1)
            eng.nucleus_step(st)
            pairs.append((st.logits.clone(), model.decoding_step(vf, prefix)))
    for got, ref in pairs:
        worst = max(worst, rel(got, ref))
    print(f"L{layers}_H{hidden} {'pre' if norm_first else 'post'}: worst rel L2 {worst:.2e} over {len(pairs)} steps")
    assert worst <= 3e-2


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(os.path.join(golden_dir, N.GOLDEN))


def _run_and_check(eng, image, step, p, max_steps, seed, what):
    """Runs the sampler step by step on the engine and replays it in float64 on the GPU's own prefixes.  Let eps be the
    step's largest absolute difference between the engine's fp32 logits and the float64 oracle's; a token whose float64
    logit lies below another's by more than 2 eps is surely behind it in the engine's order too.  Every new token must
    then lie in the float64 nucleus widened by that error: the float64 mass of the tokens surely ahead of it is at most
    p, up to the factor e^(2 eps) and 1e-5 of fp32 rounding.  A token never repeats the previous one outside the
    banned-alone case (widened by the same error), an ended caption continues with EOS, and L follows rule 1.  -> the
    captions (B, L)."""
    B = image.shape[0]
    rows = torch.arange(B, device=DEV)
    worst = 0.0
    st = eng.nucleus_start(image, p, max_steps, C.SOS, C.EOS, seed)
    sos = torch.full((B, 1), C.SOS, dtype=torch.int64, device=DEV)
    while True:
        t = st.L - 1
        prefix = torch.cat([sos, st.tokens()[:, :t]], 1)
        logits = step(prefix).double()
        eps = float((st.logits.double() - logits).abs().max())
        worst = max(worst, eps)
        last, tok = prefix[:, -1], st.tokens()[:, t]
        ended = last == C.EOS
        assert (tok[ended] == C.EOS).all(), (what, t)
        pr = torch.softmax(logits, -1)
        ahead = (pr * (logits > logits[rows, tok][:, None] + 2 * eps)).sum(1)
        # the engine's nucleus may be the banned last token alone when, within the error, last is the best token and
        # its mass exceeds p; it then draws uniformly over the vocabulary
        p_last = pr[rows, last]
        alone = (p_last >= p * np.exp(-2 * eps) - 1e-5) & ~(logits > logits[rows, last][:, None] + 2 * eps).any(1)
        ok = ended | alone | ((ahead <= p * np.exp(2 * eps) + 1e-5) & (tok != last))
        assert ok.all(), (what, t, eps, ahead[~ok], p_last[~ok], tok[~ok], last[~ok])
        if not (st.L < max_steps and st.alive[st.L - 1].item()):
            break
        eng.nucleus_step(st)
    pred = st.tokens()
    # rule 1: the run stops at the first step whose tokens are all EOS, or after max_steps
    all_ended = [bool((pred[:, t] == C.EOS).all()) for t in range(pred.shape[1])]
    assert not any(all_ended[:-1]) and (all_ended[-1] or pred.shape[1] == max_steps), what
    print(f"{what}: L {pred.shape[1]}, largest logit error {worst:.4f}")
    return pred


@pytest.mark.parametrize("case", list(N.CASES))
def test_captions_against_reference_fixture(golden, case):
    c, spec, g = N.CASES[case], N.case_spec(case), golden[case]
    state = N.case_state(case)
    model = _model(spec, state, c["p"], c["max_steps"], spec.caption_backward)
    image = N.case_image(case).to(DEV)
    torch.manual_seed(0)
    with torch.no_grad():
        pred = model({"image": image})["predictions"]
    assert pred.dtype == torch.int64 and pred.device.type == "cuda"
    if case in N.PEAKED:   # the caption does not depend on the draws: equal to the reference's
        assert torch.equal(pred.cpu(), g["predictions"])
    vf, P = C.visual_features(state, image, spec)
    with torch.no_grad():
        mine = _run_and_check(model.engine, image, C.head_step(P, spec, vf), c["p"], c["max_steps"], 99, case)
    if case in N.PEAKED:
        assert torch.equal(mine.cpu(), g["predictions"])
    print(f"{case}: L {pred.shape[1]} (reference {g['predictions'].shape[1]})")


def test_random_init_b256_tokens_lie_in_the_float64_nucleus():
    spec = _spec(1024, 1, False, True)
    state = O.synth_state(spec, 51, bn3_gain=0.25)
    model = _model(spec, state, 0.9, 30, True)
    image = O.synth_batch(256, seed=12)["image"].to(DEV)
    with torch.no_grad():
        vf, P = C.visual_features(state, image, spec)
        _run_and_check(model.engine, image, C.head_step(P, spec, vf), 0.9, 30, 7, "random init L1_H1024 B256")


def test_sampling_has_no_side_effects():
    """Parameters and BatchNorm buffers stay bit-identical after sampling, and forward -> sampling -> backward gives the
    gradients of forward -> backward."""
    spec = _spec(128, 1, False, True)
    model = _model(spec, O.synth_state(spec, 61, bn3_gain=0.25), 0.9, 30, True)
    batch = {k: v.to(DEV) for k, v in O.synth_batch(2, seed=13, ragged=True).items()}
    before = {k: v.clone() for k, v in model.state_dict().items()}
    model.eval()
    with torch.no_grad():
        model({"image": batch["image"]})
    for k, v in model.state_dict().items():
        assert torch.equal(v, before[k]), k

    def grads(sample):
        model.train()
        for p in model.parameters():
            p.grad = None
        loss = model(batch)["loss"]
        if sample:
            model.eval()
            with torch.no_grad():
                model({"image": batch["image"]})
            model.train()
        loss.backward()
        return {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}

    g0, g1, g2 = grads(False), grads(True), grads(False)
    assert g0.keys() == g1.keys()
    for n in g0:
        noise = rel(g2[n], g0[n])
        assert rel(g1[n], g0[n]) <= max(10 * noise, 1e-5), n
