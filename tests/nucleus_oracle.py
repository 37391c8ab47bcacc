"""Float64 restatement of the reference's nucleus sampling, and a host replica of the sampler kernel's uniforms -- TEST
INFRASTRUCTURE.

`nucleus_sampling` restates AutoRegressiveNucleusSampling.search (virtex/utils/nucleus_sampling.py:47-123) with the same
torch calls in the same order, vectorising only the per-row filtering loop (the same -1e12 values written at the same
positions), and records per step and row:
  * size   -- the number of tokens in the nucleus;
  * margin -- how far p lies from the cumulative probabilities that decide the cut: min |cumsum[i - 1] - p| over the
              sorted positions i = size - 1 (the crossing token) and i = size (the first token left out), where they
              exist (inf when neither does);
  * banned_alone -- the nucleus is the row's last token alone, so the reference samples uniformly over all V tokens.
The step function is captioning_oracle.head_step, whose prefix here includes SOS (decoding_step's input for the
sampler).  The fixture under tests/golden/ is written by scripts/make_nucleus_golden.py from the reference's own model
and sampler; this module's cases and states are what that script and the tests share.

`uniform24` restates the kernel's uniform (vtx_nucleus_sample, include/virtex_b200.h): the top 24 bits of
hash_u64(seed, 4000, s * R + row) (vtx_common.cuh, replicated in tests/dropout_replica.py); u = uniform24 / 2^24.
`kernel_rule` states the kernel's contract in float64 for one step: the nucleus, the ban and the inverse CDF.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import virtex_oracle as O
from tests import captioning_oracle as C
from tests.dropout_replica import hash_u64

GOLDEN = "captioning_nucleus_sampling.pt"
SOS, EOS = C.SOS, C.EOS
SITE = 4000  # kNucleusSite of csrc/decode.cu

# name -> spec, state seed, batch seed, B, nucleus size p, max_steps, state edits (see case_state), image contrast, and
# the CPU seed of torch.manual_seed before the reference's model({"image": x}).
#   * peaked: position t's embedding set to a multiple of token t's word embedding (edits["positions"]), so that every
#     step's nucleus is that one token, never the row's last one -- the caption does not depend on the random draws,
#     so the engine's must equal the reference's;
#   * spread: nuclei of hundreds to thousands of tokens;
#   * eos_stop: an EOS bias that ends every caption at a different step, so the batch stops before max_steps;
#   * banned_alone: SOS raised above everything, so the nucleus is SOS alone whenever SOS was the last token (every
#     other step), and the reference samples uniformly over the vocabulary.
CASES = {
    "post_h128_peaked": dict(spec=C._POST, seed=31, batch_seed=5, B=3, p=0.9, max_steps=12, contrast=0.0,
                             edits={"words": 20.0, "positions": (3.0, [100 + 37 * t for t in range(12)])}, rng=0),
    "post_h128_spread": dict(spec=C._POST, seed=34, batch_seed=5, B=3, p=0.9, max_steps=12, contrast=0.0,
                             edits={"words": 3.0}, rng=1),
    "pre_h256_spread": dict(spec=C._PRE, seed=36, batch_seed=5, B=3, p=0.5, max_steps=12, contrast=0.5,
                            edits={"words": 2.0}, rng=2),
    "post_h128_eos_stop": dict(spec=C._POST, seed=34, batch_seed=5, B=3, p=0.9, max_steps=30, contrast=0.0,
                               edits={"words": 2.0, "bias": {EOS: 8.0}}, rng=1),
    "post_h128_banned_alone": dict(spec=C._POST, seed=31, batch_seed=5, B=3, p=0.9, max_steps=8, contrast=0.0,
                                   edits={"words": 20.0, "bias": {SOS: 100.0}}, rng=4),
}
PEAKED = ("post_h128_peaked",)


def case_spec(case):
    return O.Spec(**CASES[case]["spec"])


def case_state(case):
    """Synthetic state of the case, edited as in captioning_oracle.case_state; edits["positions"] = (scale, tokens) sets
    position t's embedding to scale times the (scaled) word embedding of tokens[t]."""
    c, spec = CASES[case], case_spec(case)
    state = O.synth_state(spec, c["seed"], bn3_gain=0.25)
    state["textual.embedding.words.weight"] = state["textual.embedding.words.weight"] * c["edits"]["words"]
    for l in range(spec.layers):
        k = f"textual.transformer.layers.{l}.multihead_attn.out_proj.weight"
        state[k] = state[k] * c["edits"].get("cross", 1.0)
    if "positions" in c["edits"]:
        scale, tokens = c["edits"]["positions"]
        pos = state["textual.embedding.positions.weight"].clone()
        pos[:len(tokens)] = scale * state["textual.embedding.words.weight"][tokens]
        state["textual.embedding.positions.weight"] = pos
    bias = state["textual.output.bias"].clone()
    for tok, add in c["edits"].get("bias", {}).items():
        bias[tok] += add
    state["textual.output.bias"] = bias
    return state


def case_image(case):
    """Synthetic noise images, image b scaled by 1 + contrast * b and shifted by contrast * b."""
    c = CASES[case]
    image = O.synth_batch(c["B"], seed=c["batch_seed"])["image"]
    for b in range(c["B"]):
        image[b] = image[b] * (1 + c["contrast"] * b) + c["contrast"] * b
    return image


def cut_stats(logits, p, last):
    """Nucleus size, cut margin and banned-alone flag of every row (see the module docstring); float64 on the logits'
    device, ties in torch.sort's order."""
    sorted_logits, sorted_idx = torch.sort(logits.double(), descending=True)
    cum = torch.cumsum(F.softmax(sorted_logits, dim=-1), dim=-1)
    V = cum.shape[1]
    size = (torch.cat([torch.zeros_like(cum[:, :1], dtype=torch.bool), cum[:, :-1] > p], 1) == 0).sum(1)
    margin = torch.full((cum.shape[0],), float("inf"), dtype=torch.float64, device=cum.device)
    for i in (size - 1, size):
        ok = (i >= 1) & (i <= V - 1)
        j = (i - 1).clamp(0, V - 1)
        d = (cum.gather(1, j[:, None]).squeeze(1) - p).abs()
        margin = torch.where(ok, torch.minimum(margin, d), margin)
    alone = (size == 1) & (sorted_idx[:, 0] == last)
    return size, margin, alone


def nucleus_sampling(step, B, p, max_steps, generator=None, eos=EOS, sos=SOS, device="cpu"):
    """-> dict(predictions (B, L) int64, and per step: sizes, margins, banned_alone (B,) each)."""
    start = torch.full((B,), sos, dtype=torch.int64, device=device)
    predictions = [start]
    sizes, margins, alone = [], [], []
    rows = torch.arange(B, device=device)
    for _ in range(max_steps):
        last = predictions[-1]
        if (last == eos).all():
            break
        so_far = torch.stack(predictions).permute(1, 0)
        logits = step(so_far)
        size, margin, banned_alone = cut_stats(logits, p, last)
        sizes.append(size)
        margins.append(margin)
        alone.append(banned_alone)
        sorted_logits, sorted_idx = torch.sort(logits, descending=True)
        cumulative = torch.cumsum(F.softmax(sorted_logits, dim=-1), dim=-1)
        remove = cumulative > p
        remove[..., 1:] = remove[..., :-1].clone()
        remove[..., 0] = 0
        logits[remove.new_zeros(remove.shape).scatter(1, sorted_idx, remove)] = -1e12
        logits[rows, last] = -1e12
        probs = F.softmax(logits, dim=-1)
        pred = torch.multinomial(probs, 1, generator=generator).view(B)
        pred[last == eos] = eos
        predictions.append(pred)
    return dict(predictions=torch.stack(predictions[1:]).permute(1, 0), sizes=sizes, margins=margins,
                banned_alone=alone)


# ------------------------------------------------------------------------------------------------ the kernel's contract
def uniform24(seed, s, R, rows):
    """uint64 array: the kernel's 24-bit uniform of rows `rows` at step s of a table of R rows."""
    ctr = np.uint64(s) * np.uint64(R) + np.asarray(rows, dtype=np.uint64)
    return hash_u64(seed, SITE, ctr) >> np.uint64(40)


def kernel_rule(logits, last, p, u24, eos=EOS):
    """One sampling step in float64, ties in ascending id: logits (R, V), last (R,), u24 (R,) int64 -> dict(keep (R, V)
    bool nucleus, margin (R,), token (R,), boundary (R,) = distance of the target from the nearest CDF boundary, as a
    fraction of the total weight, alone (R,) the uniform fallback)."""
    x = logits.double()
    R, V = x.shape
    order = torch.argsort(-x, dim=1, stable=True)
    sp = torch.softmax(x, -1).gather(1, order)
    cum = sp.cumsum(1)
    before = torch.cat([torch.zeros_like(cum[:, :1]), cum[:, :-1]], 1)
    keep_sorted = before <= p
    keep_sorted[:, 0] = True
    keep = torch.zeros_like(keep_sorted).scatter(1, order, keep_sorted)
    _, margin, _ = cut_stats(x, p, last)
    rows = torch.arange(R, device=x.device)
    cand = keep.clone()
    cand[rows, last] = False
    alone = ~cand.any(1)
    m = torch.where(cand, x, -torch.inf).amax(1, keepdim=True)
    w = torch.where(cand, torch.exp(x - torch.where(torch.isfinite(m), m, 0)), 0)
    W = w.sum(1)
    cdf = w.cumsum(1) / W[:, None]
    u = u24.double() / 2 ** 24
    token = (cdf <= u[:, None]).sum(1).clamp_max(V - 1)
    prev = torch.where(token > 0, cdf.gather(1, (token - 1).clamp_min(0)[:, None]).squeeze(1), 0.0)
    boundary = torch.minimum((u - prev).abs(), (cdf.gather(1, token[:, None]).squeeze(1) - u).abs())
    token = torch.where(alone, (u24 * V) >> 24, token)
    boundary = torch.where(alone, torch.full_like(boundary, float("inf")), boundary)
    token = torch.where(last == eos, torch.full_like(token, eos), token)
    return dict(keep=keep, margin=margin, token=token, boundary=boundary, alone=alone)
