"""Write tests/golden/masked_lm_masking.pt by driving the UNMODIFIED reference's MaskedLmDataset.__getitem__ (a
checkout named by $VIRTEX_REFERENCE_ROOT) on the CPU:

    VIRTEX_REFERENCE_ROOT=/path/to/virtex python scripts/make_masked_lm_golden.py

The dataset runs with a stub caption source (one caption per image), a stub tokenizer returning the fixed ids of
tests/masked_lm_oracle.py::stub_ids, an identity image transform and the global `random` seeded per case; for every
caption length of masked_lm_oracle.LENGTHS it records the input ids, the masked tokens and the labels, under the
config's mask probability (0.85) and the dataset's default (0.80).  It also resolves the reference's five
configs/task_ablations/*.yaml into plain dicts."""
import os
import random
import sys
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_shim  # noqa: E402
from tests import masked_lm_oracle as MO  # noqa: E402

GOLDEN_DIR = os.path.join(ROOT, "tests", "golden")


class _Captions:
    """Stands in for CocoCaptionsDataset: image idx has one caption, "L" = the length of its token ids."""

    def __init__(self, data_root, split):
        self.lengths = []

    def __len__(self):
        return len(self.lengths)

    def __getitem__(self, idx):
        return {"image_id": idx, "image": np.zeros((2, 2, 3), np.uint8), "captions": [str(self.lengths[idx])]}


class _Tokenizer:
    def __init__(self, vocab):
        self.vocab = vocab

    def token_to_id(self, token):
        return {"<unk>": MO.UNK, "[SOS]": MO.SOS, "[EOS]": MO.EOS, "[MASK]": MO.MASK}[token]

    def get_vocab_size(self):
        return self.vocab

    def encode(self, caption):
        return MO.stub_ids(int(caption), self.vocab)


def masking_case(tag):
    from virtex.data.datasets import masked_lm
    proportion, mask_prob, replace_prob, seed, repeats = MO.CASES[tag]
    masked_lm.CocoCaptionsDataset = _Captions
    ds = masked_lm.MaskedLmDataset("unused", "train", _Tokenizer(MO.VOCAB),
                                   image_transform=lambda image, caption: {"image": image, "caption": caption},
                                   max_caption_length=MO.MAX_LEN, mask_proportion=proportion,
                                   mask_probability=mask_prob, replace_probability=replace_prob)
    ds._dset.lengths = [L for _ in range(repeats) for L in MO.LENGTHS]
    random.seed(seed)
    N = len(ds)
    # int16 rows [N, MAX_LEN] padded with -1 (every id is below 2^15)
    rows = {k: torch.full((N, MO.MAX_LEN), -1, dtype=torch.int16) for k in ("input", "caption_tokens", "masked_labels")}
    lengths = torch.zeros(N, dtype=torch.int64)
    for idx in range(N):
        out = ds[idx]
        n = int(out["caption_lengths"])
        lengths[idx] = n
        rows["input"][idx, :n] = torch.tensor([MO.SOS, *MO.stub_ids(ds._dset.lengths[idx]), MO.EOS][:MO.MAX_LEN])
        rows["caption_tokens"][idx, :n] = out["caption_tokens"]
        rows["masked_labels"][idx, :n] = out["masked_labels"]
    return {"proportion": proportion, "mask_prob": mask_prob, "replace_prob": replace_prob, "seed": seed,
            "repeats": repeats, "L": torch.tensor(ds._dset.lengths), "caption_lengths": lengths, **rows}


def resolve_configs():
    from virtex.config import Config

    def plain(n):
        return {k: plain(v) if isinstance(v, dict) else v for k, v in n.items()}
    return {name: plain(Config(os.path.join(ref_shim.REFERENCE_ROOT, "configs", "task_ablations", name + ".yaml"))._C)
            for name in MO.TASK_CONFIGS}


def main():
    if not ref_shim.available():
        raise SystemExit("reference tree not found: set VIRTEX_REFERENCE_ROOT to a checkout of the reference")
    warnings.filterwarnings("ignore")
    ref_shim.install()
    out = {"vocab": MO.VOCAB, "max_len": MO.MAX_LEN, "cases": {t: masking_case(t) for t in MO.CASES},
           "configs": resolve_configs()}
    for t, c in out["cases"].items():
        masked = int(((c["masked_labels"] != MO.UNK) & (c["masked_labels"] >= 0)).sum())
        print(f"{t}: {len(c['L'])} captions, {masked} [MASK] labels", flush=True)
    torch.save(out, os.path.join(GOLDEN_DIR, MO.GOLDEN))


if __name__ == "__main__":
    main()
