"""GPU tests of the CIDEr metric (virtex_b200/metrics.py, csrc/cider.cu) against the float64 restatement of
tests/cider_oracle.py and the reference's scores recorded in tests/golden/cider.pt."""
import json
import os

import numpy as np
import pytest
import torch

from tests import cider_oracle as C

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(os.path.join(golden_dir, C.GOLDEN))


@pytest.fixture(scope="module")
def M():
    torch.cuda.set_device(0)
    from virtex_b200 import metrics
    return metrics


def _device_scores(M, pred, gt, sigma=6.0):
    tables = M.CiderTables(M.PackedGroundTruth(gt))
    mean, img, h = tables.score(M.PackedPredictions(pred, tables.gt), sigma)
    return tables, float(mean.item()), img.cpu().numpy(), {k: v.cpu().numpy() for k, v in h.items()}


def _long_corpus():
    """Sentences longer than a warp, images with up to 32 references, a 12-word vocabulary (many repeats)."""
    rng = np.random.default_rng(3)
    vocab = [f"t{i}" for i in range(12)]

    def sent(n):
        return " ".join(vocab[i] for i in rng.integers(0, len(vocab), n))

    gt, pred = {}, {}
    for i in range(40):
        if i % 3 == 0:
            gt[i] = [sent(int(rng.integers(20, 32))) for _ in range(32)]
        elif i % 3 == 1:
            gt[i] = [sent(int(rng.integers(200, 256))) for _ in range(4)]
        else:
            gt[i] = [sent(int(rng.integers(0, 6))) for _ in range(int(rng.integers(1, 9)))]
        pred[i] = [sent(int(rng.choice([0, 1, 3, 40, 256])))]
    return pred, gt


def _check_intermediates(tables, h, pred, gt, want):
    gid = tables.gid.cpu().numpy()
    tf = tables.tf.cpu().numpy()
    ent = tables.ent.cpu().numpy()
    df = tables.df.cpu().numpy()
    off = tables.gt.sent_off
    sentences = [s for image_id in gt for s in gt[image_id]]
    assert len(sentences) == len(want["ref_tf"])
    for s, (text, counts) in enumerate(zip(sentences, want["ref_tf"])):
        words = text.split()
        got = {}
        for p in range(len(words)):
            for k in range(1, 5):
                e = off[s] + p
                if p + k > len(words):
                    assert gid[e, k - 1] == -1 and tf[e, k - 1] == 0 and ent[e, k - 1] == -1.0
                    continue
                g = tuple(words[p:p + k])
                assert df[gid[e, k - 1]] == want["df"][g], g
                if tf[e, k - 1] > 0:
                    got[g] = int(tf[e, k - 1])
        assert got == counts
    lengths = np.maximum(np.diff(off) - 1, 0)
    assert np.array_equal(lengths, want["ref_lengths"])
    norm = tables.norm.cpu().numpy()
    assert np.all(np.abs(norm - want["ref_norms"]) <= 1e-12 * np.maximum(want["ref_norms"], 1e-300))
    # predictions: tf by words, norms, lengths
    hoff = np.concatenate([[0], np.cumsum([len(pred[i][0].split()) for i in gt])])
    for i, (image_id, counts) in enumerate(zip(gt, want["hyp_tf"])):
        words = pred[image_id][0].split()
        got = {tuple(words[p:p + k]): int(h["tf"][hoff[i] + p, k - 1])
               for p in range(len(words)) for k in range(1, 5) if p + k <= len(words) and h["tf"][hoff[i] + p, k - 1]}
        assert got == counts
    assert np.array_equal(np.maximum(np.diff(hoff) - 1, 0), want["hyp_lengths"])
    hn = want["hyp_norms"]
    assert np.all(np.abs(h["norm"] - hn) <= 1e-12 * np.maximum(hn, 1e-300))


@pytest.mark.parametrize("corpus", ["medium", "long", "edge"])
def test_intermediates_equal_oracle(M, golden, corpus):
    if corpus == "medium":
        g = golden["seeded"]["medium"]
        pred, gt = C.synthetic_corpus(g["seed"], g["images"])
    elif corpus == "long":
        pred, gt = _long_corpus()
    else:
        case = golden["edge"][0]
        pred, gt = case["predictions"], case["ground_truth"]
    tables, _, _, h = _device_scores(M, pred, gt)
    _check_intermediates(tables, h, pred, gt, C.cider_details(pred, gt))


@pytest.mark.parametrize("name", ["small", "medium"])
def test_seeded_scores_match_oracle_and_reference(M, golden, name):
    g = golden["seeded"][name]
    pred, gt = C.synthetic_corpus(g["seed"], g["images"])
    assert C.corpus_digest(pred, gt) == g["sha256"]
    for run in g["runs"]:
        want = C.cider_details(pred, gt, sigma=run["sigma"])
        _, score, img, _ = _device_scores(M, pred, gt, run["sigma"])
        assert np.abs(img - want["img_scores"]).max() <= 1e-12
        assert np.abs(img - run["ref_img_scores"].numpy()).max() <= 1e-12
        assert abs(score - want["score"]) <= 1e-12 and abs(score - run["ref_score"]) <= 1e-12
        assert M.cider(pred, gt, sigma=run["sigma"]) == score


def test_edge_cases_match_reference(M, golden):
    for case in golden["edge"]:
        _, score, img, _ = _device_scores(M, case["predictions"], case["ground_truth"], case["sigma"])
        assert np.abs(img - case["ref_img_scores"].numpy()).max() <= 1e-12, case["name"]
        assert abs(score - case["ref_score"]) <= 1e-12, case["name"]


def test_long_sentences_and_many_references_match_oracle(M):
    pred, gt = _long_corpus()
    for sigma in (6.0, 2.0):
        want = C.cider_details(pred, gt, sigma=sigma)
        _, score, img, _ = _device_scores(M, pred, gt, sigma)
        assert np.abs(img - want["img_scores"]).max() <= 1e-12
        assert abs(score - want["score"]) <= 1e-12


def test_coco_val2017_shaped_corpus(M, golden):
    g = golden["seeded"]["coco_val2017"]
    pred, gt = C.synthetic_corpus(g["seed"], g["images"])
    assert C.corpus_digest(pred, gt) == g["sha256"]
    run = g["runs"][0]
    want = C.cider_details(pred, gt, sigma=run["sigma"])
    tables, score, img, h = _device_scores(M, pred, gt, run["sigma"])
    assert np.abs(img - want["img_scores"]).max() <= 1e-12
    assert np.abs(img - run["ref_img_scores"].numpy()).max() <= 1e-12
    assert abs(score - want["score"]) <= 1e-12 and abs(score - run["ref_score"]) <= 1e-12
    df = tables.df.cpu().numpy()
    assert int((df > 0).sum()) == sum(1 for v in want["df"].values())
    assert sorted(df[df > 0].tolist()) == sorted(want["df"].values())


def test_two_calls_are_bit_identical(M, golden):
    g = golden["seeded"]["medium"]
    pred, gt = C.synthetic_corpus(g["seed"], g["images"])
    _, s1, img1, h1 = _device_scores(M, pred, gt)
    _, s2, img2, h2 = _device_scores(M, pred, gt)
    assert s1 == s2 and img1.tobytes() == img2.tobytes() and h1["norm"].tobytes() == h2["norm"].tobytes()
    assert M.cider(pred, gt) == M.cider(pred, gt) == s1


def test_evaluator_cached_path_is_bit_identical_to_cider(M, golden, tmp_path):
    g = golden["seeded"]["medium"]
    pred, gt = C.synthetic_corpus(g["seed"], g["images"])
    ann = [{"image_id": k, "caption": c} for k, v in gt.items() for c in v]
    path = tmp_path / "captions.json"
    path.write_text(json.dumps({"annotations": ann}))
    ev = M.CocoCaptionsEvaluator(str(path), lambda d: {k: list(v) for k, v in d.items()})
    dropped = list(gt)[:5]
    preds = [{"image_id": k, "caption": v[0]} for k, v in pred.items() if k not in dropped]
    preds.append({"image_id": -1, "caption": "not in the ground truth"})
    res = {k: ([""] if k in dropped else pred[k]) for k in gt}
    want = M.cider(res, gt)
    for _ in range(2):
        assert ev.evaluate(preds) == {"CIDEr": 100 * want}
    assert abs(want - C.cider(res, gt)) <= 1e-12


def test_input_validation(M):
    from virtex_b200 import ops
    from virtex_b200.lib import VtxError
    gt = {0: ["a b c"], 1: ["b c d"]}
    with pytest.raises(ValueError):
        M.cider(gt, gt, n=2)
    with pytest.raises(KeyError):
        M.cider({0: ["a"]}, gt)
    with pytest.raises(ZeroDivisionError):
        M.cider(gt, gt, sigma=0.0)
    with pytest.raises(ValueError, match="references"):
        M.cider({0: ["a"]}, {0: ["a"] * 33})
    with pytest.raises(ValueError, match="words"):
        M.cider({0: [" ".join(["a"] * 257)]}, {0: ["a"]})
    keys = torch.zeros(1000, dtype=torch.int64, device="cuda")
    w = torch.zeros(4, dtype=torch.int32, device="cuda")
    with pytest.raises(VtxError, match="power of two"):
        ops.call("vtx_cider_intern", w.data_ptr(), w.data_ptr(), 1, keys.data_ptr(), 1000, 1, w.data_ptr(),
                 ops._stream())
    d = torch.zeros(4, dtype=torch.float64, device="cuda")
    with pytest.raises(VtxError, match="sigma"):
        ops.call("vtx_cider_score", w.data_ptr(), d.data_ptr(), d.data_ptr(), w.data_ptr(), w.data_ptr(),
                 d.data_ptr(), d.data_ptr(), w.data_ptr(), w.data_ptr(), 1, 0.0, d.data_ptr(), ops._stream())


def test_launches_run_on_the_current_stream_and_do_not_grow_with_the_corpus(M, golden, monkeypatch):
    from virtex_b200 import ops
    g = golden["seeded"]["small"]
    pred, gt = C.synthetic_corpus(g["seed"], g["images"])
    want = M.cider(pred, gt)
    streams = []
    call = ops.call

    def spy(name, *args):
        streams.append((name, args[-1]))
        return call(name, *args)

    monkeypatch.setattr(ops, "call", spy)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        got = M.cider(pred, gt)
    assert got == want
    assert [n for n, _ in streams] == ["vtx_cider_intern", "vtx_cider_df", "vtx_cider_vectors", "vtx_cider_intern",
                                       "vtx_cider_vectors", "vtx_cider_score", "vtx_cider_mean"]
    assert {s for _, s in streams} == {side.cuda_stream}
    streams.clear()
    big = golden["seeded"]["medium"]
    M.cider(*C.synthetic_corpus(big["seed"], big["images"]))
    assert len(streams) == 7
