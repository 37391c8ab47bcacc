"""The reference's masked-LM token masking restated on the host, and a host replay of the masking kernel -- TEST
INFRASTRUCTURE ONLY.

`reference_item` restates MaskedLmDataset.__getitem__'s caption side (virtex/data/datasets/masked_lm.py:64-91) and
consumes a `random.Random` in the reference's order: random.choice of the caption, random.sample of the positions,
then per picked position (in sample order) random.random and, for a replacement, random.randint.  The fixture under
tests/golden/ is written by scripts/make_masked_lm_golden.py from the reference's own __getitem__ with a stub caption
source and tokenizer (`stub_ids`) and the global `random` seeded as `CASES` say; the restatement reproduces it bit for
bit (tests/test_task_ablations_cpu.py).

`device_masking` replays vtx_collate_masked_lm (include/virtex_b200.h) in numpy: the same hash_u64 draws, the same
selection of the k smallest (key, position) pairs, the same comparisons.  The GPU tests compare the kernel with it bit
for bit; the CPU tests check that its distribution is the reference's.
"""
import math
import random

import numpy as np

UNK, SOS, EOS, MASK = 0, 1, 2, 3
VOCAB = 10000
MAX_LEN = 30
GOLDEN = "masked_lm_masking.pt"
# tag -> (mask proportion, mask probability, replace probability, seed of the global random, repeats per length)
CASES = {"config": (0.15, 0.85, 0.10, 1234, 6),      # DATA.MASKED_LM of the config (what the reference trains with)
         "dataset": (0.15, 0.80, 0.10, 4321, 6)}     # MaskedLmDataset's own defaults
LENGTHS = range(0, 41)  # caption tokens between [SOS] and [EOS]; trimmed to MAX_LEN with them
TASK_CONFIGS = ("bicaptioning_R_50_L1_H2048", "captioning_R_50_L1_H2048", "masked_lm_R_50_L1_H2048",
                "token_classification_R_50", "multilabel_classification_R_50")

# hash sites of the kernel's draws (virtex_b200/csrc/input_pipe.cu)
KEY_SITE, FLAG_SITE, TOKEN_SITE = 5000, 5001, 5002
_M64 = (1 << 64) - 1


def stub_ids(L, vocab=VOCAB):
    """The stub tokenizer's ids of a caption of L tokens: fixed, never a special token."""
    return [4 + (7 * i + 13 * L) % (vocab - 4) for i in range(L)]


def reference_item(ids, rng: random.Random, max_len=MAX_LEN, proportion=0.15, mask_prob=0.85, replace_prob=0.10,
                   vocab=VOCAB, mask_id=MASK, pad=UNK):
    """(input ids, masked tokens, labels) of one __getitem__ whose tokenizer returns `ids`."""
    rng.choice([None])  # random.choice(captions) of a one-caption image still draws
    tokens = [SOS, *ids, EOS][:max_len]
    source = list(tokens)
    labels = [pad] * len(tokens)
    picked = rng.sample(list(range(1, len(tokens) - 1)), math.ceil((len(tokens) - 2) * proportion))
    for i in picked:
        if len(picked) == 1:
            labels[i] = tokens[i]
            tokens[i] = mask_id
        else:
            flag = rng.random()
            if flag <= mask_prob + replace_prob:
                if flag <= mask_prob:
                    labels[i] = tokens[i]
                    tokens[i] = mask_id
                else:
                    tokens[i] = rng.randint(0, vocab - 1)
    return source, tokens, labels


# ------------------------------------------------------------------------------------------------- device replay
def hash_u64(seed, site, ctr):
    """vtx_common.cuh's hash_u64 over uint64 arrays (wrapping arithmetic)."""
    with np.errstate(over="ignore"):
        ctr = np.asarray(ctr, np.uint64)
        x = (np.uint64(seed & _M64) ^ np.uint64((0x9E3779B97F4A7C15 * (site + 1)) & _M64)
             ^ (ctr * np.uint64(0xD6E8FEB86659FD93)))
        for _ in range(2):
            x = x ^ (x >> np.uint64(32))
            x = x * np.uint64(0xD6E8FEB86659FD93)
        return x ^ (x >> np.uint64(32))


def mulhi(h, n):
    """floor(h * n / 2^64) for uint64 h and 0 < n < 2^32 (the kernel's __umul64hi)."""
    n = np.uint64(n)
    hi, lo = h >> np.uint64(32), h & np.uint64(0xFFFFFFFF)
    return (hi * n + ((lo * n) >> np.uint64(32))) >> np.uint64(32)


def device_masking(token_lists, seed, max_len=MAX_LEN, pad=UNK, mask_id=MASK, vocab=VOCAB, proportion=0.15,
                   mask_prob=0.85, replace_prob=0.10, T=None):
    """(caption_tokens, masked_labels, caption_lengths) int64 numpy arrays, as vtx_collate_masked_lm writes them."""
    B = len(token_lists)
    lens = np.array([min(max_len, len(t)) for t in token_lists], np.int64)
    T = int(min(max_len, max(len(t) for t in token_lists))) if T is None else T
    cap = np.full((B, T), pad, np.int64)
    for b, t in enumerate(token_lists):
        cap[b, :lens[b]] = t[:lens[b]]
    pos = np.broadcast_to(np.arange(T, dtype=np.int64), (B, T))
    ctr = (np.arange(B, dtype=np.uint64)[:, None] << np.uint64(32)) | pos.astype(np.uint64)
    n = lens[:, None]
    cand = (pos >= 1) & (pos < n - 1)
    keys = hash_u64(seed, KEY_SITE, ctr)
    order = np.lexsort((pos, keys, ~cand), axis=1)  # candidates first, by (key, position)
    rank = np.empty_like(order)
    np.put_along_axis(rank, order, np.broadcast_to(np.arange(T), (B, T)), axis=1)
    k = np.where(lens > 2, np.ceil((lens - 2).astype(np.float64) * proportion), 0).astype(np.int64)[:, None]
    chosen = cand & (rank < k)
    u = (hash_u64(seed, FLAG_SITE, ctr) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
    mask = chosen & ((k == 1) | (u <= mask_prob))
    repl = chosen & ~mask & (u <= mask_prob + replace_prob)
    labels = np.where(mask, cap, pad)
    out = np.where(mask, mask_id, cap)
    out = np.where(repl, mulhi(hash_u64(seed, TOKEN_SITE, ctr), vocab).astype(np.int64), out)
    return out, labels, lens
