"""CPU tests of the task ablations: the host restatement of the reference's masked-LM masking against the fixture
written from the reference's MaskedLmDataset (scripts/make_masked_lm_golden.py), the distribution of the masking
kernel's draws (replayed on the host) against the reference's exact probabilities, the shipped task-ablation configs
against the reference's, the factory products they build, and Trainer.step's refusal of a masked-LM batch without
labels."""
import math
import os
import random

import numpy as np
import pytest
import torch

from tests import masked_lm_oracle as MO
from tests.test_engine_dryrun import dry  # noqa: F401  (fixture)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", MO.GOLDEN)


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN, weights_only=False)


def _rows(t, lengths):
    return [t[i, :int(n)].tolist() for i, n in enumerate(lengths)]


# ------------------------------------------------------------------------------------------ the reference's masking
@pytest.mark.parametrize("tag", list(MO.CASES))
def test_restatement_reproduces_the_reference(golden, tag):
    c = golden["cases"][tag]
    assert (c["proportion"], c["mask_prob"], c["replace_prob"], c["seed"], c["repeats"]) == MO.CASES[tag]
    rng = random.Random(c["seed"])
    lengths = c["caption_lengths"].tolist()
    inputs = _rows(c["input"], lengths)
    tokens = _rows(c["caption_tokens"], lengths)
    labels = _rows(c["masked_labels"], lengths)
    replaced = 0
    for i, L in enumerate(c["L"].tolist()):
        src, tok, lab = MO.reference_item(MO.stub_ids(L), rng, proportion=c["proportion"], mask_prob=c["mask_prob"],
                                          replace_prob=c["replace_prob"])
        assert src == inputs[i] and tok == tokens[i] and lab == labels[i], (tag, i, L)
        replaced += sum(a != b and b != MO.MASK for a, b in zip(src, tok))
    assert replaced > 0  # the fixture covers the random-token branch
    assert min(lengths) == 2 and max(lengths) == MO.MAX_LEN


# ----------------------------------------------------------------------------------------------- the device scheme
def _ragged(B, seed, lo=0, hi=45, vocab=MO.VOCAB):
    g = np.random.default_rng(seed)
    out = []
    for b in range(B):
        n = int(g.integers(lo, hi + 1))
        row = [int(x) for x in g.integers(4, vocab, n)]
        if n:
            row[0] = MO.SOS
        if n > 1:
            row[-1] = MO.EOS
        out.append(row)
    return out


@pytest.mark.parametrize("proportion,mask_prob,replace_prob", [(0.15, 0.85, 0.10), (0.15, 0.80, 0.10),
                                                               (0.5, 0.3, 0.3), (1.0, 1.0, 0.0), (0.0, 0.85, 0.1)])
def test_device_scheme_invariants(proportion, mask_prob, replace_prob):
    """Exact k for every n, boundary and padding positions untouched, labels only where [MASK] was written, and a
    single pick is always masked."""
    lists = _ragged(512, 3) + [[1], [1, 2], [1, 5, 2], [], list(range(4, 50))]
    cap, lab, lens = MO.device_masking(lists, seed=0xC0FFEE, proportion=proportion, mask_prob=mask_prob,
                                      replace_prob=replace_prob)
    T = cap.shape[1]
    for b, row in enumerate(lists):
        n = min(MO.MAX_LEN, len(row))
        assert lens[b] == n
        src = np.full(T, MO.UNK, np.int64)
        src[:n] = row[:n]
        k = math.ceil((n - 2) * proportion) if n > 2 else 0
        touched = np.nonzero((cap[b] != src) | (lab[b] != MO.UNK))[0]
        assert all(1 <= t <= n - 2 for t in touched), (b, touched)
        assert (cap[b, n:] == MO.UNK).all() and (lab[b, n:] == MO.UNK).all()
        labelled = lab[b] != MO.UNK
        assert (cap[b][labelled] == MO.MASK).all() and (lab[b][labelled] == src[labelled]).all()
        assert labelled.sum() <= k and len(touched) <= k
        if k == 1:
            assert labelled.sum() == 1
        if mask_prob == 1.0:
            assert labelled.sum() == k


def test_device_scheme_distribution():
    """About 10^6 fixed-seed draws per hash site: every candidate is picked with probability k / (n - 2), a pick of k >= 2 is [MASK] /
    random id / kept with 0.85 / 0.10 / 0.05, random ids are uniform over [0, V).  Deterministic: the bounds are 5
    standard deviations of the exact probabilities, evaluated once."""
    V = 81
    lens_pattern = np.arange(3, MO.MAX_LEN + 1)
    B = 60000
    lists = [[MO.SOS] + [7] * (int(lens_pattern[b % len(lens_pattern)]) - 2) + [MO.EOS] for b in range(B)]
    cap, lab, lens = MO.device_masking(lists, seed=20240607, vocab=V)
    src = np.where(np.arange(cap.shape[1])[None, :] < lens[:, None], 7, MO.UNK)
    src[:, 0] = MO.SOS
    src[np.arange(B), lens - 1] = MO.EOS
    # a picked position: labelled ([MASK]), or replaced (a different token), or kept -- kept picks are invisible, so the
    # selection is checked through the kernel's own (key, position) rank below and the split through the flags
    picked = lab != MO.UNK
    for n in lens_pattern:
        rows = lens == n
        k = math.ceil((n - 2) * 0.15)
        keys = MO.hash_u64(20240607, MO.KEY_SITE,
                           (np.nonzero(rows)[0].astype(np.uint64)[:, None] << np.uint64(32))
                           | np.arange(1, n - 1, dtype=np.uint64)[None, :])
        rank = np.argsort(np.argsort(keys, axis=1, kind="stable"), axis=1)
        freq = (rank < k).mean(axis=0)  # per candidate position
        p = k / (n - 2)
        sd = math.sqrt(p * (1 - p) / rows.sum()) + 1e-12
        assert np.abs(freq - p).max() < 5 * sd, (n, freq, p)
        assert ((rank < k).sum(axis=1) == k).all()
        if k == 1:
            assert picked[rows].sum(axis=1).tolist() == [1] * int(rows.sum())
    # the split of picks with k >= 2 (n >= 9)
    big = lens >= 9
    ctr = (np.arange(B, dtype=np.uint64)[:, None] << np.uint64(32)) | np.arange(cap.shape[1], dtype=np.uint64)[None]
    u = (MO.hash_u64(20240607, MO.FLAG_SITE, ctr) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
    inner = (np.arange(cap.shape[1])[None, :] >= 1) & (np.arange(cap.shape[1])[None, :] < lens[:, None] - 1)
    n_masked = (picked & big[:, None]).sum()
    n_repl = ((cap != src) & ~picked & big[:, None]).sum()  # a replacement by 7 itself stays invisible: expected 1/V
    n_picks = sum(math.ceil((int(n) - 2) * 0.15) for n in lens[big])
    for got, p in ((n_masked, 0.85), (n_repl, 0.10 * (1 - 1 / V))):
        sd = math.sqrt(p * (1 - p) / n_picks)
        assert abs(got / n_picks - p) < 5 * sd, (got / n_picks, p)
    assert n_picks > 100000
    # the flags themselves, over every inner position: uniform on [0, 1)
    uu = u[inner]
    for q in (0.1, 0.5, 0.85, 0.95):
        assert abs((uu <= q).mean() - q) < 5 * math.sqrt(q * (1 - q) / uu.size)
    # replacement ids: every id of [0, V) (specials included, like random.randint(0, V - 1)), chi-square at 5 sigma
    ids = MO.mulhi(MO.hash_u64(20240607, MO.TOKEN_SITE, ctr[inner]), V).astype(np.int64)
    counts = np.bincount(ids, minlength=V)
    assert counts.size == V and ids.min() == 0 and ids.max() == V - 1
    e = ids.size / V
    chi2 = ((counts - e) ** 2 / e).sum()
    assert abs(chi2 - (V - 1)) < 5 * math.sqrt(2 * (V - 1)), chi2
    assert uu.size + ids.size > 10 ** 6


def test_device_scheme_replacement_ids_cover_the_vocabulary():
    h = MO.hash_u64(5, MO.TOKEN_SITE, np.arange(200000, dtype=np.uint64))
    ids = MO.mulhi(h, MO.VOCAB).astype(np.int64)
    assert ids.min() == 0 and ids.max() == MO.VOCAB - 1
    # mulhi is floor(h * V / 2^64): exact against Python integers
    for x in h[:100].tolist():
        assert int(MO.mulhi(np.array([x], np.uint64), MO.VOCAB)[0]) == (x * MO.VOCAB) >> 64


# ------------------------------------------------------------------------------------------------------- configs
def _leaves(d, prefix=""):
    for k, v in d.items():
        if isinstance(v, dict):
            yield from _leaves(v, prefix + k + ".")
        else:
            yield prefix + k, v


@pytest.mark.parametrize("name", MO.TASK_CONFIGS)
def test_shipped_configs_resolve_to_the_reference(golden, name):
    from virtex_b200.config import Config
    mine = dict(_leaves(Config(f"task_ablations/{name}.yaml")._C.to_dict()))
    ref = dict(_leaves(golden["configs"][name]))
    assert set(ref) <= set(mine), set(ref) - set(mine)
    diff = {k: (mine[k], v) for k, v in ref.items() if mine[k] != v and not (isinstance(v, (list, tuple)) and
                                                                          list(v) == list(mine[k]))}
    assert not diff, diff


def test_factory_products_of_the_task_configs():
    from virtex_b200.config import Config
    from virtex_b200.data_gpu import _TASK_OF_MODEL
    from virtex_b200.factories import PretrainingModelFactory
    from virtex_b200.models import (BidirectionalCaptioningModel, ForwardCaptioningModel, MaskedLMModel,
                                    MultiLabelClassificationModel, TokenClassificationModel)
    want = {"bicaptioning_R_50_L1_H2048": (BidirectionalCaptioningModel, True),
            "captioning_R_50_L1_H2048": (ForwardCaptioningModel, True),
            "masked_lm_R_50_L1_H2048": (MaskedLMModel, False)}
    for name, (cls, future) in want.items():
        cfg = Config(f"task_ablations/{name}.yaml")
        m = PretrainingModelFactory.from_config(cfg)
        assert type(m) is cls and m.textual.mask_future_positions is future
        t = m.textual
        assert (t.hidden_size, t.num_layers, t.attention_heads, t.feedforward_size) == (2048, 1, 32, 8192)
        assert t.vocab_size == 10000 and t.padding_idx == 0
        assert _TASK_OF_MODEL[cfg.MODEL.NAME] == ("masked_lm" if cls is MaskedLMModel else "captioning")
    cfg = Config("task_ablations/masked_lm_R_50_L1_H2048.yaml")
    assert (cfg.DATA.MASKED_LM.MASK_PROPORTION, cfg.DATA.MASKED_LM.MASK_PROBABILITY,
            cfg.DATA.MASKED_LM.REPLACE_PROBABILITY) == (0.15, 0.85, 0.10)
    tok = PretrainingModelFactory.from_config(Config("task_ablations/token_classification_R_50.yaml"))
    assert type(tok) is TokenClassificationModel and tok.ignore_indices == [0, 1, 2, 3]
    assert tok.textual.output.out_features == 10000
    cfg = Config("task_ablations/multilabel_classification_R_50.yaml")
    ml = PretrainingModelFactory.from_config(cfg)
    assert type(ml) is MultiLabelClassificationModel and ml.ignore_indices == [0]
    assert ml.textual.output.out_features == 81 and cfg.OPTIM.NO_DECAY == "none"


def test_pipeline_needs_a_device_and_a_known_task():
    from virtex_b200.data_gpu import GpuInputPipeline
    with pytest.raises(RuntimeError, match="CUDA"):
        GpuInputPipeline("cpu", task="masked_lm")


# ------------------------------------------------------------------------------------------------------- trainer
def _masked_lm_model():
    from oracle import virtex_oracle as O
    from virtex_b200.models import MaskedLMModel
    from virtex_b200.modules import TorchvisionVisualBackbone, TransformerDecoderTextualHead
    spec = O.Spec(hidden=128, layers=1, heads=2, ffn=256)
    visual = TorchvisionVisualBackbone(spec.backbone, visual_feature_size=spec.visual_feature_size)
    textual = TransformerDecoderTextualHead(spec.visual_feature_size, spec.vocab, spec.hidden, spec.layers, spec.heads,
                                            spec.ffn, dropout=0.1, mask_future_positions=False)
    return MaskedLMModel(visual, textual), O.synth_masked_batch(3, seed=5)


def _bare_trainer(model):
    """A Trainer around `model` without its device-side optimiser state (Trainer.__init__ needs a GPU)."""
    from virtex_b200.trainer import Trainer
    t = object.__new__(Trainer)
    t.model, t.engine, t.world, t._pending = model, model.engine, 1, []
    t.optimizer_step = lambda: None
    return t


def test_trainer_step_trains_masked_lm_on_its_labels(dry):  # noqa: F811
    """On the engine dry run: a masked-LM batch without masked_labels raises before anything runs; with them, the
    loss is the labelled cross entropy (shift 0) of one direction."""
    from virtex_b200 import engine as E
    model, batch = _masked_lm_model()
    trainer = _bare_trainer(model)
    seed0 = model.engine.seed.clone()
    bad = {k: v for k, v in batch.items() if k != "masked_labels"}
    with pytest.raises(KeyError, match="masked_labels"):
        trainer.step(bad)
    assert dry.calls == [] and torch.equal(model.engine.seed, seed0)
    seen = []
    real = E.Engine.head_loss

    def spy(self, rec, write_grad, labels=None):
        seen.append(labels)
        return real(self, rec, write_grad, labels)

    E.Engine.head_loss = spy
    try:
        trainer.step(batch)
    finally:
        E.Engine.head_loss = real
    assert len(seen) == 1 and seen[0] is batch["masked_labels"]
    assert dry.names().count("vtx_cross_entropy") == 1 and "vtx_attn_bwd" in dry.names()
