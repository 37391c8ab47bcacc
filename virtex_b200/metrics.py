"""Caption metrics on the sm_90a kernels: the CIDEr score of the reference's CocoCaptionsEvaluator.

`cider(predictions, ground_truth, n=4, sigma=6.0)` restates `cider` of virtex/utils/metrics.py:177-264, quirks
included: words are `str.split()` tokens, every sentence contributes its 1- to 4-grams, document frequencies count
the ground-truth images whose references contain an n-gram, a sentence's length is its number of bigrams
(max(words - 1, 0)), and a similarity whose norm product is exactly 0.0 is divided by 1.  Only `n == 4` is accepted:
the reference counts 4-grams whatever `n` is, so any other `n` either raises there or scores differently.

The host splits the captions and interns the words as int32 ids; everything else is one device pass (see
include/virtex_b200.h, Caption metrics (CIDEr)), and the score is the pass's one device-to-host read.
`CocoCaptionsEvaluator` keeps the ground truth's tables -- word ids, n-gram table, df, reference vectors and norms --
on the device, so `evaluate` interns and scores the predictions only.  The document frequencies depend on the ground
truth alone, so the cached path is the very computation `cider` runs: the two return bit-identical scores.
"""
import json
import math
from collections import defaultdict
from typing import Any, Callable, Dict, List, Optional

import numpy as np
import torch

from . import ops

ORDERS = 4
# Size limits of csrc/cider.cu (include/virtex_b200.h); COCO Captions has at most 7 references per image and 50 words
# per tokenized caption.
MAX_REFS = 32                  # references per image
MAX_WORDS = 256                # words per sentence (reference or prediction)
MAX_IMAGE_WORDS = 1024         # reference words of one image
MAX_TOTAL_WORDS = 1 << 24      # reference words, and prediction words, of one corpus


def _occurrences(lengths):
    """n-gram occurrences of orders 1..4 in sentences of these lengths."""
    lengths = np.asarray(lengths, np.int64)
    return int(sum(np.maximum(lengths - k + 1, 0).sum() for k in range(1, ORDERS + 1)))


class PackedGroundTruth:
    """Ground truth in CSR form: words int32 [W] (ids from `vocab`), sent_off int32 [S + 1], img_off int32 [N + 1],
    with the images in the order of `ground_truth`'s keys.  Raises ValueError beyond the kernels' size limits."""

    def __init__(self, ground_truth: Dict[Any, List[str]]):
        self.image_ids = list(ground_truth)
        if not self.image_ids:
            raise ValueError("cider: ground_truth is empty")
        vocab: Dict[str, int] = {}
        setdefault = vocab.setdefault
        words: List[int] = []
        lengths: List[int] = []
        img_off = [0]
        for image_id in self.image_ids:
            refs = ground_truth[image_id]
            if not 1 <= len(refs) <= MAX_REFS:
                raise ValueError(f"cider: image {image_id!r} has {len(refs)} references; 1 .. {MAX_REFS} are supported")
            n_words = 0
            for ref in refs:
                toks = ref.split()
                if len(toks) > MAX_WORDS:
                    raise ValueError(f"cider: a reference of image {image_id!r} has {len(toks)} words; at most "
                                     f"{MAX_WORDS} are supported")
                words.extend([setdefault(w, len(vocab)) for w in toks])
                lengths.append(len(toks))
                n_words += len(toks)
            if n_words > MAX_IMAGE_WORDS:
                raise ValueError(f"cider: the references of image {image_id!r} have {n_words} words; at most "
                                 f"{MAX_IMAGE_WORDS} are supported")
            img_off.append(len(lengths))
            if len(words) > MAX_TOTAL_WORDS:
                raise ValueError(f"cider: the references have more than {MAX_TOTAL_WORDS} words")
        self.vocab = vocab
        self.words = np.asarray(words, np.int32)
        self.lengths = np.asarray(lengths, np.int32)
        self.sent_off = np.concatenate([[0], np.cumsum(self.lengths)]).astype(np.int32)
        self.img_off = np.asarray(img_off, np.int32)
        # the n-gram table holds at most one key per occurrence; twice that keeps linear probing short
        cap = 1024
        while cap < 2 * _occurrences(self.lengths):
            cap *= 2
        self.capacity = cap


class PackedPredictions:
    """`predictions[image_id][0]` for every ground-truth image, in CSR form over the ground truth's vocabulary; words
    the ground truth lacks get fresh ids (distinct per word).  A missing image raises KeyError, as in the reference."""

    def __init__(self, predictions: Dict[Any, List[str]], gt: PackedGroundTruth):
        get = gt.vocab.get
        extra: Dict[str, int] = {}
        base = len(gt.vocab)
        words: List[int] = []
        lengths: List[int] = []
        for image_id in gt.image_ids:
            toks = predictions[image_id][0].split()
            if len(toks) > MAX_WORDS:
                raise ValueError(f"cider: the prediction of image {image_id!r} has {len(toks)} words; at most "
                                 f"{MAX_WORDS} are supported")
            for w in toks:
                i = get(w)
                if i is None:
                    i = extra.setdefault(w, base + len(extra))
                words.append(i)
            lengths.append(len(toks))
        if len(words) > MAX_TOTAL_WORDS:
            raise ValueError(f"cider: the predictions have more than {MAX_TOTAL_WORDS} words")
        self.words = np.asarray(words, np.int32)
        self.lengths = np.asarray(lengths, np.int32)
        self.sent_off = np.concatenate([[0], np.cumsum(self.lengths)]).astype(np.int32)


def _device_words(words, device):
    # an empty corpus side still needs a valid pointer
    return torch.from_numpy(words if words.size else np.zeros(1, np.int32)).to(device)


class CiderTables:
    """The ground truth's tables on the device: word ids, the n-gram table, df, and every reference's tf, tf-idf
    entries and norms ([words, 4] and [sentences, 4], include/virtex_b200.h).  Built by three launches."""

    def __init__(self, gt: PackedGroundTruth, device=None):
        self.gt = gt
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        dev, st = self.device, ops._stream()
        W, S, N = gt.words.size, gt.lengths.size, len(gt.image_ids)
        self.n_img = N
        self.words = _device_words(gt.words, dev)
        self.sent_off = torch.from_numpy(gt.sent_off).to(dev)
        self.img_off = torch.from_numpy(gt.img_off).to(dev)
        self.keys = torch.zeros(gt.capacity, dtype=torch.int64, device=dev)
        self.df = torch.zeros(gt.capacity, dtype=torch.int32, device=dev)
        rows = max(W, 1)
        self.gid = torch.empty(rows, ORDERS, dtype=torch.int32, device=dev)
        self.tf = torch.empty(rows, ORDERS, dtype=torch.int32, device=dev)
        self.ent = torch.empty(rows, ORDERS, dtype=torch.float64, device=dev)
        self.norm = torch.empty(S, ORDERS, dtype=torch.float64, device=dev)
        ops.call("vtx_cider_intern", self.words.data_ptr(), self.sent_off.data_ptr(), S, self.keys.data_ptr(),
                 gt.capacity, 1, self.gid.data_ptr(), st)
        ops.call("vtx_cider_df", self.gid.data_ptr(), self.sent_off.data_ptr(), self.img_off.data_ptr(), N,
                 self.df.data_ptr(), st)
        ops.call("vtx_cider_vectors", self.words.data_ptr(), self.gid.data_ptr(), self.sent_off.data_ptr(), S,
                 self.df.data_ptr(), N, self.tf.data_ptr(), self.ent.data_ptr(), self.norm.data_ptr(), st)
        self._ready = torch.cuda.Event()
        self._ready.record()

    def score(self, pred: PackedPredictions, sigma: float):
        """Launch the predictions' pass on the current stream.  Returns (corpus mean [1], per-image scores [N], the
        predictions' device arrays {gid, tf, ent, norm}); nothing is read back."""
        if float(sigma) == 0.0:
            raise ZeroDivisionError("float division by zero")   # the reference's -(delta ** 2) / (2 * sigma ** 2)
        torch.cuda.current_stream(self.device).wait_event(self._ready)
        dev, st, N = self.device, ops._stream(), self.n_img
        words = _device_words(pred.words, dev)
        off = torch.from_numpy(pred.sent_off).to(dev)
        rows = max(pred.words.size, 1)
        h = {"gid": torch.empty(rows, ORDERS, dtype=torch.int32, device=dev),
             "tf": torch.empty(rows, ORDERS, dtype=torch.int32, device=dev),
             "ent": torch.empty(rows, ORDERS, dtype=torch.float64, device=dev),
             "norm": torch.empty(N, ORDERS, dtype=torch.float64, device=dev)}
        img_score = torch.empty(N, dtype=torch.float64, device=dev)
        mean = torch.empty(1, dtype=torch.float64, device=dev)
        ops.call("vtx_cider_intern", words.data_ptr(), off.data_ptr(), N, self.keys.data_ptr(), self.gt.capacity, 0,
                 h["gid"].data_ptr(), st)
        ops.call("vtx_cider_vectors", words.data_ptr(), h["gid"].data_ptr(), off.data_ptr(), N, self.df.data_ptr(), N,
                 h["tf"].data_ptr(), h["ent"].data_ptr(), h["norm"].data_ptr(), st)
        ops.call("vtx_cider_score", h["gid"].data_ptr(), h["ent"].data_ptr(), h["norm"].data_ptr(), off.data_ptr(),
                 self.gid.data_ptr(), self.ent.data_ptr(), self.norm.data_ptr(), self.sent_off.data_ptr(),
                 self.img_off.data_ptr(), N, float(sigma), img_score.data_ptr(), st)
        ops.call("vtx_cider_mean", img_score.data_ptr(), N, mean.data_ptr(), st)
        return mean, img_score, h


def _check_n(n):
    if n != ORDERS:
        raise ValueError(f"cider: n={n} is not supported; the reference counts n-grams of orders 1..4 whatever n is, "
                         "so only n=4 scores as documented")


def cider(predictions: Dict[Any, List[str]], ground_truth: Dict[Any, List[str]], n: int = 4,
          sigma: float = 6.0) -> float:
    """CIDEr of `predictions[image_id][0]` against `ground_truth[image_id]` over the ground truth's images (the
    reference's `cider`, virtex/utils/metrics.py:177-264), on the current CUDA device."""
    _check_n(n)
    gt = PackedGroundTruth(ground_truth)
    pred = PackedPredictions(predictions, gt)
    mean, _, _ = CiderTables(gt).score(pred, sigma)
    return float(mean.item())


class CocoCaptionsEvaluator:
    """CIDEr (and SPICE, when a scorer is given) of caption predictions in COCO format: the reference's
    CocoCaptionsEvaluator (virtex/utils/metrics.py:75-122) with the ground truth's CIDEr tables built once on the
    device.

    Args:
        gt_annotations_path: COCO Captions annotations (typically ``captions_val2017.json``).
        tokenize: ``{image_id: [caption, ...]} -> {image_id: [tokenized caption, ...]}``, the signature of the
            reference's PTB ``tokenize`` (Stanford CoreNLP, Java), which this project does not ship.
        spice: optional ``spice(res, gt) -> float`` with the signature of the reference's ``spice``.
    """

    def __init__(self, gt_annotations_path: str, tokenize: Callable, spice: Optional[Callable] = None):
        with open(gt_annotations_path) as f:
            gt_annotations = json.load(f)["annotations"]
        ground_truth: Dict[int, List[str]] = defaultdict(list)
        for ann in gt_annotations:
            ground_truth[ann["image_id"]].append(ann["caption"])
        self._tokenize = tokenize
        self._spice = spice
        self.ground_truth = tokenize(ground_truth)
        self._tables = CiderTables(PackedGroundTruth(self.ground_truth))

    def evaluate(self, preds) -> Dict[str, float]:
        """``preds``: ``[{"image_id": int, "caption": str}, ...]`` or the path of such a JSON file.  Returns
        ``{"CIDEr": 100 * cider}``, plus ``"SPICE": 100 * spice`` when a SPICE scorer was given."""
        if isinstance(preds, str):
            with open(preds) as f:
                preds = json.load(f)
        # a repeated image id keeps its last caption; ids outside the ground truth are dropped, missing ones score ""
        tokenized = self._tokenize({ann["image_id"]: [ann["caption"]] for ann in preds})
        res = {k: tokenized[k] if k in tokenized else [""] for k in self.ground_truth}
        mean, _, _ = self._tables.score(PackedPredictions(res, self._tables.gt), 6.0)
        out = {"CIDEr": 100 * float(mean.item())}
        if self._spice is not None:
            out["SPICE"] = 100 * float(self._spice(res, self.ground_truth))
        return out


class TopkAccuracy:
    """Top-k classification accuracy accumulated over batches (virtex/utils/metrics.py:22-72): the percentage of
    samples whose label is among the k highest predictions, ``num_correct / (num_total + 1e-12) * 100``."""

    def __init__(self, k: int = 1):
        self._k = k
        self.reset()

    def reset(self):
        self.num_total = 0.0
        self.num_correct = 0.0

    def __call__(self, predictions: torch.Tensor, ground_truth: torch.Tensor):
        """predictions (C,) or (B, C) scores, ground_truth () or (B,) labels; returns the accuracy so far."""
        if self._k == 1:
            top = predictions.argmax(dim=-1, keepdim=True)
        else:
            top = predictions.topk(min(self._k, predictions.shape[-1]), dim=-1).indices
        hits = (top == ground_truth.unsqueeze(-1)).float().sum()
        self.num_total += ground_truth.numel()
        self.num_correct += hits
        return self.get_result()

    def get_result(self):
        return self.num_correct / (self.num_total + 1e-12) * 100
