"""CPU checks of the CIDEr metric: the float64 restatement against the reference's scores in tests/golden/cider.pt,
the fixture's corpus hashes, host packing and input validation of virtex_b200/metrics.py, the evaluator's id
handling, and TopkAccuracy."""
import json
import os

import numpy as np
import pytest
import torch

from tests import cider_oracle as C
from virtex_b200 import metrics as M


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(os.path.join(golden_dir, C.GOLDEN))


def test_seeded_corpora_match_the_fixture_hashes(golden):
    for name, seed, images in C.CORPORA:
        g = golden["seeded"][name]
        assert (g["seed"], g["images"]) == (seed, images)
        pred, gt = C.synthetic_corpus(seed, images)
        assert C.corpus_digest(pred, gt) == g["sha256"], name


def test_coco_shaped_corpus_has_the_shape_of_val2017():
    pred, gt = C.synthetic_corpus(2017, 5000)
    refs = [len(v) for v in gt.values()]
    words = [len(s.split()) for v in gt.values() for s in v]
    assert len(gt) == 5000 and set(refs) <= {5, 6, 7} and 26_000 < sum(refs) < 28_500
    assert 9.5 < np.mean(words) < 11.5 and max(words) <= M.MAX_WORDS
    assert list(pred) == list(gt)


@pytest.mark.parametrize("name", ["small", "medium"])
def test_oracle_equals_reference_on_seeded_corpora(golden, name):
    g = golden["seeded"][name]
    pred, gt = C.synthetic_corpus(g["seed"], g["images"])
    for run in g["runs"]:
        d = C.cider_details(pred, gt, sigma=run["sigma"])
        assert np.abs(d["img_scores"] - run["ref_img_scores"].numpy()).max() <= 1e-12
        assert abs(d["score"] - run["ref_score"]) <= 1e-12


def test_oracle_equals_reference_on_edge_cases(golden):
    names = set()
    for case in golden["edge"]:
        d = C.cider_details(case["predictions"], case["ground_truth"], sigma=case["sigma"])
        assert np.abs(d["img_scores"] - case["ref_img_scores"].numpy()).max() <= 1e-12, case["name"]
        assert abs(d["score"] - case["ref_score"]) <= 1e-12, case["name"]
        names.add(case["name"])
    assert names == {"mixed", "in_every_image", "single_image"}


def test_edge_cases_cover_the_quirks():
    (_, pred, gt, _), *_ = C.edge_cases()
    d = C.cider_details(pred, gt)
    assert {len(v) for v in gt.values()} >= {1, 7}
    assert d["hyp_norms"][2].sum() == 0.0                               # the empty prediction
    assert d["df"][("a",)] == len(gt) and ("zebra",) not in d["df"]     # weight 0; an n-gram only in predictions
    every = next(c for c in C.edge_cases() if c[0] == "in_every_image")
    e = C.cider_details(every[1], every[2])
    assert e["df"][("a",)] == 3 and e["hyp_norms"][0, 0] == 0.0         # weight 0: the "or 1" division


def test_packing_is_csr_over_one_vocabulary():
    gt = {5: ["a b  c", "b"], 3: ["c d"]}
    pred = {3: ["d e e"], 5: ["", "ignored"], 9: ["x"]}
    pg = M.PackedGroundTruth(gt)
    assert pg.image_ids == [5, 3]
    assert pg.vocab == {"a": 0, "b": 1, "c": 2, "d": 3}
    assert pg.words.tolist() == [0, 1, 2, 1, 2, 3]
    assert pg.sent_off.tolist() == [0, 3, 4, 6] and pg.img_off.tolist() == [0, 2, 3]
    assert pg.capacity == 1024 and pg.capacity >= 2 * M._occurrences(pg.lengths)
    pp = M.PackedPredictions(pred, pg)
    assert pp.words.tolist() == [3, 4, 4] and pp.sent_off.tolist() == [0, 0, 3]


def test_limits_and_n_raise_value_error():
    ok = {0: ["a b"]}
    with pytest.raises(ValueError, match="n=3"):
        M.cider(ok, ok, n=3)
    with pytest.raises(ValueError, match="n=5"):
        M.cider(ok, ok, n=5)
    with pytest.raises(ValueError, match="empty"):
        M.PackedGroundTruth({})
    with pytest.raises(ValueError, match="0 references"):
        M.PackedGroundTruth({0: []})
    with pytest.raises(ValueError, match="33 references"):
        M.PackedGroundTruth({0: ["a"] * (M.MAX_REFS + 1)})
    M.PackedGroundTruth({0: ["a"] * M.MAX_REFS})
    long = " ".join(["w"] * (M.MAX_WORDS + 1))
    with pytest.raises(ValueError, match="257 words"):
        M.PackedGroundTruth({0: [long]})
    with pytest.raises(ValueError, match="257 words"):
        M.PackedPredictions({0: [long]}, M.PackedGroundTruth(ok))
    with pytest.raises(ValueError, match="1025 words"):
        M.PackedGroundTruth({0: [" ".join(["w"] * 256)] * 4 + ["w"]})
    M.PackedGroundTruth({0: [" ".join(["w"] * 256)] * 4})


def test_total_word_limit(monkeypatch):
    monkeypatch.setattr(M, "MAX_TOTAL_WORDS", 5)
    with pytest.raises(ValueError, match="references have more than 5 words"):
        M.PackedGroundTruth({0: ["a b c"], 1: ["d e f"]})
    gt = M.PackedGroundTruth({0: ["a"], 1: ["b"]})
    with pytest.raises(ValueError, match="predictions have more than 5 words"):
        M.PackedPredictions({0: ["a b c"], 1: ["d e f"]}, gt)


def test_missing_prediction_raises_key_error():
    with pytest.raises(KeyError):
        M.cider({0: ["a"]}, {0: ["a"], 1: ["b"]})


def test_evaluator_id_handling_fills_and_scales(tmp_path, monkeypatch):
    ann = {"annotations": [{"image_id": 1, "caption": "A Dog."}, {"image_id": 2, "caption": "a cat"},
                           {"image_id": 1, "caption": "a dog runs"}, {"image_id": 3, "caption": "a bird"}]}
    path = tmp_path / "captions.json"
    path.write_text(json.dumps(ann))
    calls = []

    def tokenize(d):     # stands in for the PTB tokenizer: lower-case, drop the full stop
        calls.append(d)
        return {k: [c.lower().replace(".", "") for c in v] for k, v in d.items()}

    seen = {}

    class Tables:
        def __init__(self, gt):
            self.gt = gt

        def score(self, pred, sigma):
            seen["pred"], seen["sigma"] = pred, sigma
            return torch.tensor([0.25], dtype=torch.float64), None, None

    monkeypatch.setattr(M, "CiderTables", Tables)
    spice_args = []
    ev = M.CocoCaptionsEvaluator(str(path), tokenize, spice=lambda res, gt: spice_args.append((res, gt)) or 0.5)
    assert ev.ground_truth == {1: ["a dog", "a dog runs"], 2: ["a cat"], 3: ["a bird"]}
    preds = [{"image_id": 2, "caption": "first"}, {"image_id": 7, "caption": "not in gt"},
             {"image_id": 2, "caption": "A CAT"}, {"image_id": 1, "caption": "dog."}]
    pred_path = tmp_path / "preds.json"
    pred_path.write_text(json.dumps(preds))
    for p in (preds, str(pred_path)):
        out = ev.evaluate(p)
        assert out == {"CIDEr": 25.0, "SPICE": 50.0}
        assert calls[-1] == {2: ["A CAT"], 7: ["not in gt"], 1: ["dog."]}     # a repeated id keeps its last caption
        res, gt = spice_args[-1]
        assert res == {1: ["dog"], 2: ["a cat"], 3: [""]} and gt is ev.ground_truth
        vocab = seen["pred"]
        assert seen["sigma"] == 6.0 and vocab.sent_off.tolist() == [0, 1, 3, 3]
    assert set(M.CocoCaptionsEvaluator(str(path), tokenize).evaluate(preds)) == {"CIDEr"}


def test_alias_module_exports_the_reference_names():
    from virtex.utils import metrics as alias
    assert alias.cider is M.cider and alias.CocoCaptionsEvaluator is M.CocoCaptionsEvaluator
    assert alias.TopkAccuracy is M.TopkAccuracy


@pytest.mark.parametrize("k", [1, 3, 20])
def test_topk_accuracy_matches_the_formula(k):
    g = torch.Generator().manual_seed(k)
    acc = M.TopkAccuracy(k)
    correct = total = 0
    for b in (7, 1, 12):
        logits = torch.randn(b, 10, generator=g)
        labels = torch.randint(0, 10, (b,), generator=g)
        ranks = (logits > logits.gather(1, labels[:, None])).sum(1)
        correct += int((ranks < k).sum())
        total += b
        got = acc(logits, labels)
    assert abs(float(got) - correct / (total + 1e-12) * 100) < 1e-4
    single = M.TopkAccuracy(k)
    single(torch.tensor([0.1, 0.7, 0.2]), torch.tensor(1))
    assert abs(float(single.get_result()) - 100.0) < 1e-6
    acc.reset()
    assert acc.num_total == 0.0 and acc.num_correct == 0.0
