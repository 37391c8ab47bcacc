"""Float64 restatement of the CIDEr score of the reference's CocoCaptionsEvaluator, and seeded COCO-val-shaped corpora.

`cider_details` follows the contract virtex_b200/metrics.py documents: `str.split()` words; n-grams of orders 1..4
counted per sentence; df(g) = ground-truth images whose references contain g; entries tf * (log N - log max(1, df));
per-order norms summed in first-occurrence order; length = max(words - 1, 0); per (hypothesis, reference) and order,
sum over the hypothesis's n-grams of min(vh, vr) * vr, divided by (|h| |r|) or 1, times e^(-(len_h - len_r)^2 / (2
sigma^2)); image score = 10 * mean over orders of the sum over references / references; corpus = mean over images.
It returns every intermediate the kernels write, keyed by n-gram tuples.
"""
import hashlib
import json
import math

import numpy as np

ORDERS = 4
GOLDEN = "cider.pt"
# seeded corpora of the golden: (name, seed, images); "coco_val2017" has the shape of COCO Captions val2017
CORPORA = (("small", 7, 64), ("medium", 11, 600), ("coco_val2017", 2017, 5000))
SIGMAS = (6.0, 1.0, 0.5, 25.0)


def ngram_counts(sentence):
    """{n-gram tuple: count} in first-occurrence order, orders 1..4, and the word count."""
    words = sentence.split()
    counts = {}
    for k in range(1, ORDERS + 1):
        for i in range(len(words) - k + 1):
            g = tuple(words[i:i + k])
            counts[g] = counts.get(g, 0) + 1
    return counts, len(words)


def cider_details(predictions, ground_truth, n=4, sigma=6.0):
    if n != ORDERS:
        raise ValueError("only n = 4")
    ids = list(ground_truth)
    hyps = [ngram_counts(predictions[i][0]) for i in ids]
    refs = [[ngram_counts(s) for s in ground_truth[i]] for i in ids]
    df = {}
    for image_refs in refs:
        seen = set()
        for counts, _ in image_refs:
            seen.update(counts)
        for g in seen:
            df[g] = df.get(g, 0) + 1
    log_n = math.log(len(ids))

    def vectorise(counts):
        vec = [{} for _ in range(ORDERS)]
        sq = [0.0] * ORDERS
        for g, tf in counts.items():
            e = float(tf) * (log_n - math.log(max(1, df.get(g, 0))))
            vec[len(g) - 1][g] = e
            sq[len(g) - 1] += e * e
        return vec, [math.sqrt(s) for s in sq]

    gauss_den = 2 * sigma ** 2
    img_scores = []
    ref_norms, hyp_norms = [], []
    for (hc, hw), image_refs in zip(hyps, refs):
        hv, hn = vectorise(hc)
        hyp_norms.append(hn)
        hl = max(hw - 1, 0)
        score = [0.0] * ORDERS
        for rc, rw in image_refs:
            rv, rn = vectorise(rc)
            ref_norms.append(rn)
            delta = float(hl - max(rw - 1, 0))
            for k in range(ORDERS):
                val = 0.0
                for g, vh in hv[k].items():
                    vr = rv[k].get(g, 0.0)
                    val += min(vh, vr) * vr
                val /= (hn[k] * rn[k]) or 1
                val *= math.e ** (-(delta ** 2) / gauss_den)
                score[k] += val
        total = 0.0
        for s in score:
            total += s
        img_scores.append(total / ORDERS / len(image_refs) * 10.0)
    img_scores = np.asarray(img_scores, np.float64)
    return {
        "score": float(np.mean(img_scores)),
        "img_scores": img_scores,
        "df": df,
        "ref_tf": [c for image_refs in refs for c, _ in image_refs],
        "ref_lengths": np.asarray([max(w - 1, 0) for image_refs in refs for _, w in image_refs], np.int64),
        "ref_norms": np.asarray(ref_norms, np.float64).reshape(-1, ORDERS),
        "hyp_tf": [c for c, _ in hyps],
        "hyp_lengths": np.asarray([max(w - 1, 0) for _, w in hyps], np.int64),
        "hyp_norms": np.asarray(hyp_norms, np.float64).reshape(-1, ORDERS),
    }


def cider(predictions, ground_truth, n=4, sigma=6.0):
    return cider_details(predictions, ground_truth, n, sigma)["score"]


def synthetic_corpus(seed, n_images, vocab=10_000):
    """COCO-val-shaped captions: a Zipf(1.1) vocabulary, 5 references per image (6 or 7 for about one image in
    six), each a variant of a per-image base caption of 8 to 18 words (35 % of its words substituted, 5 % dropped, up
    to 2 appended), and one prediction per image that is a closer variant (25 % substituted).  Returns (predictions, ground_truth) with
    integer image ids in a shuffled order."""
    rng = np.random.default_rng(seed)
    p = 1.0 / np.arange(1, vocab + 1) ** 1.1
    cdf = np.cumsum(p / p.sum())
    words = [f"w{i}" for i in range(vocab)]

    def draw(size):
        return [words[i] for i in np.minimum(np.searchsorted(cdf, rng.random(size), side="right"), vocab - 1)]

    def variant(base, sub):
        out = []
        u = rng.random(len(base))
        fresh = draw(len(base))
        for w, r, f in zip(base, u, fresh):
            if r < sub:
                out.append(f)
            elif r >= sub + 0.05:
                out.append(w)
        out.extend(draw(int(rng.integers(0, 3))))
        return " ".join(out)

    ids = rng.permutation(np.arange(100_000, 100_000 + 7 * n_images, 7))[:n_images].tolist()
    gt, pred = {}, {}
    for image_id in ids:
        base = draw(int(np.clip(rng.normal(10.5, 2.0), 8, 18)))
        n_refs = int(rng.choice([5, 5, 5, 5, 5, 6, 7]))
        gt[image_id] = [variant(base, 0.35) for _ in range(n_refs)]
        pred[image_id] = [variant(base, 0.25)]
    return pred, gt


def corpus_digest(predictions, ground_truth):
    blob = json.dumps([[[k, v] for k, v in ground_truth.items()], [[k, v] for k, v in predictions.items()]])
    return hashlib.sha256(blob.encode()).hexdigest()


def edge_cases():
    """Small corpora, stored literally in the golden: (name, predictions, ground_truth, sigma)."""
    gt = {
        1: ["a man riding a horse on a beach", "a person rides a horse near the sea"],
        2: ["a dog dog dog runs in the park", "two dogs play on the grass", "a dog is running", "the dog runs",
            "dogs running in a park", "a brown dog in the park", "a dog plays outside"],
        3: ["a cat on a couch"],
        4: ["A Red bus on the road", "a red bus parked by a road"],
        5: ["un café près de la tour Eiffel", "a café with straße signs", "ünïcödé words ☕ in a café"],
        6: ["a kite flying in a blue sky", "a kite in the sky"],
    }
    pred = {
        1: ["a man riding a horse on a beach"],      # identical to a reference
        2: ["dog dog dog dog dog"],                  # repeated words: the min(vh, vr) clip
        3: [""],                                     # empty prediction
        4: ["a RED bus"],                            # shorter than four words, case differs
        5: ["un café près de ☕"],                    # non-ASCII words
        6: ["zebra quokka flying"],                  # n-grams found only in predictions
    }
    cases = [("mixed", pred, gt, s) for s in (6.0, 0.5, 3.0, 100.0)]
    # "a" appears in every image's references: weight 0; image 2's references hold only "a" at order 1 -> norm 0
    every = {10: ["a", "a b c d"], 11: ["a a", "x a y"], 12: ["a q"]}
    cases.append(("in_every_image", {10: ["a"], 11: ["a"], 12: ["a q"]}, every, 6.0))
    # one image only: every reference n-gram has df = N, so all reference entries are 0
    cases.append(("single_image", {0: ["a b c d e"]}, {0: ["a b c d e", "a b c"]}, 6.0))
    return cases
