"""Float64 restatement of the reference's beam search over the captioning model -- TEST INFRASTRUCTURE.

`beam_search` restates AutoRegressiveBeamSearch.search (virtex/utils/beam_search.py:52-238) with the same torch calls
in the same order, vectorising only the per-row repetition penalty (a scatter of the same -10000 values), and also
records, per step, how decisive each selection was:
  * node gap  -- per row, the score of the last kept minus the first dropped of its per-node candidates (step 0: of
                 the beam_size first tokens of each image);
  * image gap -- per image, the last kept minus the first dropped of its beam_size * per_node candidates.
The step function is `head_step`: the oracle's float64 textual head (oracle/virtex_oracle.py) over the whole prefix,
as CaptioningModel.decoding_step does (virtex/models/captioning.py:165-213).  The fixtures under tests/golden/ are
written by scripts/make_captioning_golden.py from the reference's own model and search; this module's cases and
states are what that script and the tests share.
"""
import torch
import torch.nn.functional as F

from oracle import virtex_oracle as O

GOLDEN = "captioning_beam_search.pt"
SOS, EOS = 1, 2

_POST = dict(hidden=128, layers=1, heads=2, ffn=256)
_PRE = dict(hidden=256, layers=2, heads=4, ffn=512, norm_first=True, caption_backward=False)

# name -> spec, state seed, batch seed, B, beam, max_steps, state edits (see case_state), image contrast (case_image).
# The states are chosen so that every case has images whose selections are all decisive (every recorded gap above 0.1
# nats): the word embedding (input and tied output) is scaled up so that logits lie far apart, and in some states the
# cross-attention output is scaled up so that the image weighs more in each step.  With an EOS bias strong enough to
# stop the search early, or a raised padding token, no beam-5 state tried had decisive images (EOS and padding
# candidates compete closely across beams), so those two cases run at beam 1 and 2.
CASES = {
    "post_h128_beam5": dict(spec=_POST, seed=34, batch_seed=5, B=3, beam=5, max_steps=12, contrast=0.0,
                            edits={"words": 40.0}),
    "post_h128_beam1": dict(spec=_POST, seed=31, batch_seed=5, B=3, beam=1, max_steps=30, contrast=0.0,
                            edits={"words": 20.0}),
    "post_h128_beam1_all_eos": dict(spec=_POST, seed=31, batch_seed=5, B=3, beam=1, max_steps=30, contrast=0.0,
                                    edits={"words": 20.0, "bias": {EOS: 100.0}}),
    "post_h128_early_stop": dict(spec=_POST, seed=36, batch_seed=5, B=3, beam=1, max_steps=30, contrast=0.0,
                                 edits={"words": 20.0, "cross": 30.0, "bias": {EOS: 22.0}}),
    "post_h128_token0": dict(spec=_POST, seed=31, batch_seed=5, B=3, beam=2, max_steps=12, contrast=0.0,
                             edits={"words": 20.0, "bias": {0: 20.0}}),
    "pre_h256_beam5": dict(spec=_PRE, seed=36, batch_seed=5, B=3, beam=5, max_steps=12, contrast=0.5,
                           edits={"words": 20.0, "cross": 30.0}),
}


def case_spec(case):
    return O.Spec(**CASES[case]["spec"])


def case_state(case):
    """Synthetic state of the case (oracle.virtex_oracle.synth_state, residual branch gain 0.25 as in the bf16 parity
    tests): word embedding scaled by `edits['words']`, cross-attention output projection by `edits['cross']`, output
    bias entries raised by `edits['bias']`."""
    c = CASES[case]
    spec = case_spec(case)
    state = O.synth_state(spec, c["seed"], bn3_gain=0.25)
    state["textual.embedding.words.weight"] = state["textual.embedding.words.weight"] * c["edits"]["words"]
    for l in range(spec.layers):
        k = f"textual.transformer.layers.{l}.multihead_attn.out_proj.weight"
        state[k] = state[k] * c["edits"].get("cross", 1.0)
    bias = state["textual.output.bias"].clone()
    for tok, add in c["edits"].get("bias", {}).items():
        bias[tok] += add
    state["textual.output.bias"] = bias
    return state


def case_image(case):
    """Synthetic noise images; image b is scaled by 1 + contrast * b and shifted by contrast * b, so that the images'
    features differ beyond the noise."""
    c = CASES[case]
    image = O.synth_batch(c["B"], seed=c["batch_seed"])["image"]
    for b in range(c["B"]):
        image[b] = image[b] * (1 + c["contrast"] * b) + c["contrast"] * b
    return image


def visual_features(state, image, spec, dtype=torch.float64):
    """Eval-mode backbone features (B, 2048, h, w) in `dtype` on the image's device."""
    P = {k: (v.to(device=image.device, dtype=dtype) if v.is_floating_point() else v.to(image.device))
         for k, v in state.items()}
    with torch.no_grad():
        return O.backbone_forward(P, image.to(dtype), spec, training=False), P


def head_step(P, spec, features):
    """decoding_step of the forward-direction head in the dtype of P: (B*beam, T) or (B,) tokens -> (B*beam, V)."""

    def step(partial):
        B = features.shape[0]
        if partial.dim() == 1:
            partial = partial.unsqueeze(1)
        beam = partial.shape[0] // B
        vf = features.repeat_interleave(beam, 0) if beam > 1 else features
        lengths = torch.full((partial.shape[0],), partial.shape[1], dtype=torch.int64, device=partial.device)
        with torch.no_grad(), torch.device(features.device):  # the head builds its masks on the default device
            return O.head_forward(P, vf, partial, lengths, spec)[:, -1, :]

    return step


def _gap(values, kept):
    """Last kept minus first dropped along the last dim of descending `values` (inf when nothing is dropped)."""
    if values.shape[-1] <= kept:
        return torch.full(values.shape[:-1], float("inf"), dtype=values.dtype, device=values.device)
    return values[..., kept - 1] - values[..., kept]


def beam_search(step, B, beam, max_steps, eos=EOS, sos=SOS, per_node=2, device="cpu"):
    """-> dict(predictions (B, beam, L) int64, scores (B, beam), node_gaps [(rows,)] and image_gaps [(B,)] per step)."""
    start = torch.full((B,), sos, dtype=torch.int64, device=device)
    lp0 = F.log_softmax(step(start), dim=1)
    V = lp0.shape[1]
    top, cls = lp0.topk(beam)
    node_gaps = [_gap(lp0.topk(min(beam + 1, V))[0], beam)]
    image_gaps = [node_gaps[0].clone()]
    if beam == 1 and (cls == eos).all():
        return dict(predictions=cls.unsqueeze(-1), scores=top, node_gaps=node_gaps, image_gaps=image_gaps)
    predictions = cls.unsqueeze(-1)
    last_logprobs = top
    after_end = lp0.new_full((B * beam, V), float("-inf"))
    after_end[:, eos] = 0.0
    rows = torch.arange(B * beam, device=device)
    for _ in range(max_steps - 1):
        last = predictions[:, :, -1].reshape(B * beam)
        if (last == eos).all():
            break
        so_far = predictions.view(B * beam, -1)
        lp = F.log_softmax(step(so_far), dim=1)
        lp[rows, so_far[:, -1]] = -10000
        cleaned = torch.where(last.unsqueeze(-1).expand(B * beam, V) == eos, after_end, lp)
        top_lp, pred_cls = cleaned.topk(per_node)
        node_gaps.append(_gap(cleaned.topk(min(per_node + 1, V))[0], per_node))
        summed = (top_lp + last_logprobs.unsqueeze(2).expand(B, beam, per_node).reshape(B * beam, per_node))
        summed = summed.reshape(B, beam * per_node)
        cls = pred_cls.reshape(B, beam * per_node)
        reshaped = predictions.view(B * beam, 1, -1).repeat(1, per_node, 1).reshape(B, beam * per_node, -1)
        reshaped = torch.cat([reshaped, cls.unsqueeze(-1)], dim=-1)
        kept, idx = summed.topk(beam)
        image_gaps.append(_gap(summed.topk(min(beam + 1, beam * per_node))[0], beam))
        predictions = reshaped.gather(1, idx.unsqueeze(-1).repeat(1, 1, reshaped.shape[-1]))
        last_logprobs = kept
    return dict(predictions=predictions, scores=last_logprobs, node_gaps=node_gaps, image_gaps=image_gaps)


def decisive(result, beam, threshold):
    """(B,) bool: every recorded gap of the image exceeds `threshold` (its node gaps are those of its beam rows)."""
    B = result["predictions"].shape[0]
    ok = torch.ones(B, dtype=torch.bool, device=result["predictions"].device)
    for s, (ng, ig) in enumerate(zip(result["node_gaps"], result["image_gaps"])):
        ng = ng.view(B, -1)
        ok &= (ng > threshold).all(1) & (ig > threshold)
    return ok


def caption_score(step, captions, eos=EOS, sos=SOS):
    """Sum of the search's per-step scores along each caption (B, L): log_softmax of the first token, then at step t the
    cleaned score (repetition penalty, EOS continuation) of token t given tokens 0..t-1 -- the score beam search
    accumulates for that caption."""
    B, L = captions.shape
    start = torch.full((B,), sos, dtype=torch.int64, device=captions.device)
    lp = F.log_softmax(step(start), dim=1)
    score = lp.gather(1, captions[:, :1]).squeeze(1)
    for t in range(1, L):
        lp = F.log_softmax(step(captions[:, :t]), dim=1)
        lp[torch.arange(B, device=captions.device), captions[:, t - 1]] = -10000
        tok = captions[:, t]
        ended = captions[:, t - 1] == eos
        s_t = lp.gather(1, tok[:, None]).squeeze(1)
        s_t = torch.where(ended, torch.where(tok == eos, torch.zeros_like(s_t), torch.full_like(s_t, float("-inf"))), s_t)
        score = score + s_t
    return score
