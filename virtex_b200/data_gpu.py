"""GPU input pipeline: the reference's per-sample CPU transforms + collate as four kernels per batch.

Drop-in for what `CaptioningDataset.__getitem__` + `collate_fn` (virtex/data/datasets/captioning.py:51-100) produce with
the transform lists of the base config (virtex/factories.py:131-155, `DATA.IMAGE_TRANSFORM_TRAIN/VAL`): the same batch
dict {"image" fp32 [B,3,224,224], "caption_tokens", "noitpac_tokens", "caption_lengths"}, built on the device from
token-id lists and images of any size, each given either decoded (uint8 HWC RGB array) or encoded (the JPEG file's
bytes: `bytes`, `bytearray`, `memoryview` or a 1-D uint8 array), mixed freely within a batch.  Encoded images are
decoded on the device by virtex_b200.jpeg, bit-exact with the reference's cv2.imread + cvtColor(BGR2RGB).
Tokenisation and the caption-side left<->right swap of the paired horizontal flip (virtex/data/transforms.py:29-36, a
string operation) stay on the host; the host also draws the random parameters, so the kernels are deterministic and
testable:

    pipe = GpuInputPipeline(device)
    sizes = [jpeg.image_size(buf) for buf in buffers]                              # or img.shape[:2]
    params = [pipe.sample_train_params(rng, *hw) for hw in sizes]                  # or pipe.val_params(H, W)
    batch = pipe(buffers, params, token_lists)

One pinned staging buffer and one H2D copy per batch carry the compressed bytes or raw pixels (uint8: 4x fewer PCIe
bytes than the fp32 tensors the reference's DataLoader ships) plus a ~100 B/image parameter table.  JPEGs the device
path does not reproduce (progressive, CMYK, truncated, corrupt entropy data, ...) are decoded by cv2 on the host and
take the decoded-array path; batch["_jpeg_fallbacks"] (a CPU int64 scalar, present when the batch had encoded images)
counts them.  No CPU fallback otherwise: CUDA tensors out.

The same call builds the batches of the other pretext tasks (`task`, below): masked language modelling, with the
reference's token masking drawn on the device, and token / multilabel classification.
"""
import math
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

from . import jpeg
from .ops import _stream, call

IMAGENET_MEAN = (0.485, 0.456, 0.406)
IMAGENET_STD = (0.229, 0.224, 0.225)


class ImageParams:
    """Sampled parameters of one image: source region, resized size, output-window offset, flip, colour jitter."""
    __slots__ = ("region", "resized", "offset", "flip", "jitter")

    def __init__(self, region, resized, offset=(0, 0), flip=False, jitter=None):
        self.region, self.resized, self.offset, self.flip, self.jitter = region, resized, offset, flip, jitter


TASKS = ("captioning", "masked_lm", "token_classification", "multilabel_classification")
# MODEL.NAME -> the batch a model of that name trains on
_TASK_OF_MODEL = {"virtex": "captioning", "bicaptioning": "captioning", "captioning": "captioning",
                  "masked_lm": "masked_lm", "token_classification": "token_classification",
                  "multilabel_classification": "multilabel_classification"}


class GpuInputPipeline:
    """`task` chooses the batch built from `token_lists` (captioning by default, as above):

      masked_lm                  "caption_tokens" (masked), "masked_labels", "caption_lengths": MaskedLmDataset's
                                 masking and collate (virtex/data/datasets/masked_lm.py:64-119), padded with
                                 `padding_idx`, drawn on the device (vtx_collate_masked_lm)
      token_classification       "labels": the trimmed token lists padded with `padding_idx` (TokenClassificationDataset)
      multilabel_classification  "labels": `token_lists` are the per-image category lists, padded with 0 and never
                                 trimmed (MultiLabelClassificationDataset)

    `GpuInputPipeline.from_config(config, device)` takes every setting from a Config."""

    def __init__(self, device, crop_size: int = 224, max_caption_length: int = 30, padding_idx: int = 0,
                 mean=IMAGENET_MEAN, std=IMAGENET_STD, task: str = "captioning", vocab_size: int = 10000,
                 mask_index: int = 3, mask_proportion: float = 0.15, mask_probability: float = 0.85,
                 replace_probability: float = 0.10):
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("GpuInputPipeline runs on a CUDA device (there is no CPU path)")
        if task not in TASKS:
            raise ValueError(f"task {task!r} is not one of {TASKS}")
        self.S, self.max_len, self.pad = crop_size, max_caption_length, padding_idx
        self.task, self.vocab_size, self.mask_index = task, vocab_size, mask_index
        self.mask_proportion, self.mask_probability = mask_proportion, mask_probability
        self.replace_probability = replace_probability
        m = np.array(mean, np.float32) * np.float32(255.0)
        inv = np.float32(1) / (np.array(std, np.float32) * np.float32(255.0))
        self.norm = torch.from_numpy(np.concatenate([m, inv])).to(self.device)
        self._pinned: Optional[torch.Tensor] = None
        self._dev: Optional[torch.Tensor] = None
        self._copied: Optional[torch.cuda.Event] = None  # the last H2D copy out of the pinned staging buffer

    @classmethod
    def from_config(cls, config, device) -> "GpuInputPipeline":
        """The pipeline of `config`'s MODEL.NAME with DATA.IMAGE_CROP_SIZE, MAX_CAPTION_LENGTH, UNK_INDEX (padding),
        VOCAB_SIZE, MASK_INDEX and MASKED_LM.* (virtex/factories.py:230-243)."""
        D = config.DATA
        return cls(device, crop_size=D.IMAGE_CROP_SIZE, max_caption_length=D.MAX_CAPTION_LENGTH,
                   padding_idx=D.UNK_INDEX, task=_TASK_OF_MODEL[config.MODEL.NAME], vocab_size=D.VOCAB_SIZE,
                   mask_index=D.MASK_INDEX, mask_proportion=D.MASKED_LM.MASK_PROPORTION,
                   mask_probability=D.MASKED_LM.MASK_PROBABILITY, replace_probability=D.MASKED_LM.REPLACE_PROBABILITY)

    # ------------------------------------------------------------------------------------------- host-side sampling
    def sample_train_params(self, rng: np.random.Generator, H: int, W: int, scale=(0.2, 1.0), ratio=(0.75, 1.333),
                            flip_p=0.5, jitter=(0.4, 0.4, 0.4, 0.1), jitter_p=0.8) -> ImageParams:
        """random_resized_crop -> horizontal_flip -> color_jitter of the base config (factories.py:136-152)."""
        area = H * W
        box = None
        for _ in range(10):
            target = rng.uniform(*scale) * area
            aspect = math.exp(rng.uniform(math.log(ratio[0]), math.log(ratio[1])))
            w, h = int(round(math.sqrt(target * aspect))), int(round(math.sqrt(target / aspect)))
            if 0 < w <= W and 0 < h <= H:
                box = (int(rng.integers(0, H - h + 1)), int(rng.integers(0, W - w + 1)), h, w)
                break
        if box is None:
            in_ratio = W / H
            if in_ratio < ratio[0]:
                w, h = W, int(round(W / ratio[0]))
            elif in_ratio > ratio[1]:
                h, w = H, int(round(H * ratio[1]))
            else:
                w, h = W, H
            box = ((H - h) // 2, (W - w) // 2, h, w)
        jit = None
        if rng.uniform() < jitter_p:
            b, c, s, hh = jitter
            jit = (rng.uniform(max(0, 1 - b), 1 + b), rng.uniform(max(0, 1 - c), 1 + c),
                   rng.uniform(max(0, 1 - s), 1 + s), rng.uniform(-hh, hh), tuple(int(i) for i in rng.permutation(4)))
        return ImageParams(box, (self.S, self.S), (0, 0), bool(rng.uniform() < flip_p), jit)

    def val_params(self, H: int, W: int, resize: int = 256) -> ImageParams:
        """smallest_resize(256) -> center_crop(224) (DATA.IMAGE_TRANSFORM_VAL)."""
        scale = resize / min(H, W)
        nh, nw = int(round(H * scale)), int(round(W * scale))
        if nh < self.S or nw < self.S:
            raise ValueError("image too small for the centre crop")
        return ImageParams((0, 0, H, W), (nh, nw), ((nh - self.S) // 2, (nw - self.S) // 2))

    # ------------------------------------------------------------------------------------------------------- batch
    def __call__(self, images: Sequence, params: Sequence[ImageParams],
                 token_lists: Optional[Sequence[Sequence[int]]] = None,
                 seed: Optional[int] = None) -> Dict[str, torch.Tensor]:
        """The batch of `images` (with `params`) and `token_lists` for the pipeline's task.  masked_lm draws its 64-bit
        seed on the device from torch's default CUDA generator (no host synchronisation: torch.manual_seed reproduces
        a batch, successive batches differ), or takes `seed` when given."""
        B, S = len(images), self.S
        assert B == len(params) and B > 0
        # encoded images: parsed here and decoded on the device, or decoded by cv2 when the device path cannot
        arrs, heads, blobs = [], {}, {}
        for n, im in enumerate(images):
            if jpeg.is_encoded(im):
                h, b = jpeg.parse_or_none(im)
                if h is None:
                    arrs.append(jpeg.host_decode(b, f"image {n}"))
                else:
                    arrs.append(None)
                    heads[n], blobs[n] = h, b
            else:
                arrs.append(np.ascontiguousarray(im.cpu().numpy() if torch.is_tensor(im) else im))
        n_host = sum(jpeg.is_encoded(im) for im in images) - len(heads)
        geom_i = np.zeros((B, 8), np.int32)
        geom_d = np.zeros((B, 2), np.float64)
        jit_i = np.zeros((B, 6), np.int32)
        jit_d = np.zeros((B, 4), np.float64)
        offs = np.zeros(B, np.int64)
        total = 0
        for n, (a, p) in enumerate(zip(arrs, params)):
            if a is None:
                H, W = heads[n].height, heads[n].width
            elif a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3:
                raise ValueError("images must be uint8 HWC RGB arrays or encoded JPEG bytes")
            else:
                H, W = a.shape[:2]
            y0, x0, h, w = p.region
            if not (0 <= y0 and 0 <= x0 and y0 + h <= H and x0 + w <= W and h > 0 and w > 0):
                raise ValueError(f"crop box {p.region} outside the {H}x{W} image")
            geom_i[n] = (H, W, y0, x0, h, w, p.offset[0], p.offset[1])
            geom_d[n] = (h / p.resized[0], w / p.resized[1])
            jit_i[n, 0] = int(p.flip)
            jit_i[n, 2:] = (0, 1, 2, 3)
            jit_d[n] = (1.0, 1.0, 1.0, 0.0)
            if p.jitter is not None:
                jit_i[n, 1] = 1
                jit_d[n] = p.jitter[:4]
                jit_i[n, 2:] = p.jitter[4]
            if a is not None:
                offs[n] = total
                total += (a.size + 15) // 16 * 16
        # compressed bytes follow the pixels; the device decodes them into a region after the staged bytes
        jidx = sorted(heads)
        src_off = np.zeros(len(jidx), np.int64)
        for k, n in enumerate(jidx):
            src_off[k] = total
            total += (len(blobs[n]) + 15) // 16 * 16
        dec_off = np.zeros(len(jidx), np.int64)
        dec_total = 0
        for k, n in enumerate(jidx):
            dec_off[k] = dec_total
            dec_total += (heads[n].height * heads[n].width * 3 + 15) // 16 * 16
        plan = jpeg.Plan([heads[n] for n in jidx], src_off, dec_off) if jidx else None
        tok_flat = tok_offs = None
        if token_lists is not None:
            assert len(token_lists) == B
            tok_offs = np.zeros(B + 1, np.int64)
            tok_offs[1:] = np.cumsum([len(t) for t in token_lists])
            tok_flat = np.fromiter((x for t in token_lists for x in t), np.int64, int(tok_offs[-1]))
        tok_tabs = [tok_flat, tok_offs] if tok_flat is not None else []
        seed_tab = None
        if tok_flat is not None and self.task == "masked_lm" and seed is not None:
            seed_tab = np.array([int(seed) & (2 ** 64 - 1)], np.uint64)  # travels with the batch's one copy
            tok_tabs.append(seed_tab)
        # decoded JPEG pixels land after the staged bytes (need_al); their offsets are known from the headers
        tab_bytes0 = sum((t.nbytes + 15) // 16 * 16 for t in [geom_d, jit_d, offs, geom_i, jit_i] + tok_tabs +
                         (plan.tables() if plan else []))
        need_al = (total + tab_bytes0 + 15) // 16 * 16
        for k, n in enumerate(jidx):
            offs[n] = need_al + dec_off[k]
        # ---- one pinned staging buffer: [pixels | compressed bytes | tables], one H2D copy
        tables = [geom_d, jit_d, offs] + tok_tabs + [geom_i, jit_i]
        if plan is not None:
            tables += plan.tables()
        tab_bytes = sum((t.nbytes + 15) // 16 * 16 for t in tables)
        need = total + tab_bytes
        if self._pinned is None or self._pinned.numel() < need:
            self._pinned = torch.empty(int(need * 1.25) + 1024, dtype=torch.uint8).pin_memory()
        if self._dev is None or self._dev.numel() < need_al + dec_total:
            self._dev = torch.empty(max(self._pinned.numel(), int((need_al + dec_total) * 1.25)), dtype=torch.uint8,
                                    device=self.device)
        if self._copied is not None:
            self._copied.synchronize()  # the previous batch's copy must have left the staging buffer
        host = self._pinned.numpy()
        for a, o in zip(arrs, offs):
            if a is not None:
                host[o:o + a.size] = a.reshape(-1)
        for k, n in enumerate(jidx):
            host[src_off[k]:src_off[k] + len(blobs[n])] = np.frombuffer(blobs[n], np.uint8)
        views, cur = [], total
        for t in tables:
            host[cur:cur + t.nbytes] = np.frombuffer(t.tobytes(), np.uint8)
            views.append((cur, t))
            cur += (t.nbytes + 15) // 16 * 16
        self._dev[:need].copy_(self._pinned[:need], non_blocking=True)
        self._copied = torch.cuda.Event()
        self._copied.record()
        base = self._dev.data_ptr()
        ptr = {id(t): base + o for o, t in views}
        s = _stream()
        if plan is not None:
            status = jpeg.decoder_for(self.device).run(plan, base, [ptr[id(t)] for t in plan.tables()], base + need_al)
            for k, n in enumerate(jidx):
                if status[k]:  # the device found the entropy data corrupt: cv2 decodes it (what the reference reads)
                    a = jpeg.host_decode(blobs[n], f"image {n}")
                    if a.shape[:2] != (heads[n].height, heads[n].width):
                        raise ValueError(f"image {n}: cv2 decoded {a.shape[:2]}, the headers say "
                                         f"{(heads[n].height, heads[n].width)}")
                    self._dev[offs[n]:offs[n] + a.size].copy_(torch.from_numpy(a.reshape(-1)))
                    n_host += 1
        img_u8 = torch.empty(B, S, S, 3, dtype=torch.uint8, device=self.device)
        gray = torch.zeros(B, dtype=torch.int64, device=self.device)
        out = torch.empty(B, 3, S, S, dtype=torch.float32, device=self.device)
        call("vtx_image_resample", base, ptr[id(offs)], ptr[id(geom_i)], ptr[id(geom_d)], ptr[id(jit_i)],
             img_u8.data_ptr(), B, S, s)
        call("vtx_image_gray_sum", img_u8.data_ptr(), ptr[id(jit_i)], ptr[id(jit_d)], gray.data_ptr(), B, S, s)
        call("vtx_image_jitter_normalize", img_u8.data_ptr(), ptr[id(jit_i)], ptr[id(jit_d)], gray.data_ptr(),
             self.norm.data_ptr(), out.data_ptr(), B, S, s)
        batch = {"image": out, "_image_u8": img_u8}
        if any(jpeg.is_encoded(im) for im in images):
            batch["_jpeg_fallbacks"] = torch.tensor(n_host, dtype=torch.int64)
        if tok_flat is not None:
            batch.update(self._collate(B, token_lists, ptr[id(tok_flat)], ptr[id(tok_offs)],
                                       ptr[id(seed_tab)] if seed_tab is not None else None, s))
        return batch

    def _collate(self, B, token_lists, flat, offs, seed_ptr, s) -> Dict[str, torch.Tensor]:
        """The task's token / label tensors from the staged flat lists (device pointers)."""
        longest = max(len(t) for t in token_lists)
        # category lists are not captions: no trimming, padding with 0 (MultiLabelClassificationDataset.collate_fn)
        max_len, pad = (longest, 0) if self.task == "multilabel_classification" else (self.max_len, self.pad)
        T = int(min(max_len, longest))
        new = lambda *shape: torch.empty(*shape, dtype=torch.int64, device=self.device)
        cap, lens = new(B, T), new(B)
        if self.task == "masked_lm":
            labels = new(B, T)
            if seed_ptr is None:
                seed_t = new(1).random_(-2 ** 63, None)  # all 64 bits, from torch's default CUDA generator
                seed_ptr = seed_t.data_ptr()
            call("vtx_collate_masked_lm", flat, offs, cap.data_ptr(), labels.data_ptr(), lens.data_ptr(), B, T, max_len,
                 pad, self.mask_index, self.vocab_size, self.mask_proportion, self.mask_probability,
                 self.replace_probability, seed_ptr, s)
            return {"caption_tokens": cap, "masked_labels": labels, "caption_lengths": lens}
        rev = new(B, T)
        call("vtx_collate_tokens", flat, offs, cap.data_ptr(), rev.data_ptr(), lens.data_ptr(), B, T, max_len, pad, s)
        if self.task == "captioning":
            return {"caption_tokens": cap, "noitpac_tokens": rev, "caption_lengths": lens}
        return {"labels": cap}
