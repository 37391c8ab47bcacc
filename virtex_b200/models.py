"""`CaptioningModel` family: drop-in for virtex/models/captioning.py:12-283 on the H100 engine.

Same constructor arguments, attribute names, weight sharing between the two directions
(captioning.py:57-63) and the same `forward(batch) -> {"loss", "loss_components", ["predictions"]}` contract.
`output["loss"]` carries a grad_fn: `loss.backward()` runs the engine's hand-written backward and delivers gradients
for every parameter (so torch optimisers, GradScaler-free AMP loops and DistributedDataParallel hooks keep working).
The throughput path (`virtex_b200.trainer.Trainer`) drives the same engine without autograd in between.
"""
import copy
import functools
from typing import Any, Dict, List

import torch
from torch import nn

from .engine import Engine
from .modules import LinearTextualHead, TextualHead, VisualBackbone


class _StepFunction(torch.autograd.Function):
    """Whole-model forward/backward as one autograd node; the kernels are scheduled by `Engine`."""

    @staticmethod
    def forward(ctx, model, image, tokens, noitpac, lengths, labels, *params):
        eng = model.engine
        eng.seed.add_(1)  # fresh dropout masks every training forward (nn.Dropout draws from an advancing RNG stream)
        loss = eng.forward(image, tokens, noitpac, lengths, training=model.training, with_grad=True, labels=labels)
        ctx.model = model
        ctx.generation = eng.generation
        ctx.n_params = len(params)
        out = loss.clone()
        return out[0], out[1]

    @staticmethod
    def backward(ctx, g_fwd, g_bwd):
        model = ctx.model
        eng = model.engine
        if eng.generation != ctx.generation:
            raise RuntimeError(
                "the engine ran another forward since this loss was computed (a validation forward, or a second "
                "micro-batch): its single activation tape was overwritten; call backward() before the next forward")
        # d(loss_f + loss_b): both components enter the total with weight 1 (captioning.py:133).  A common factor (a loss
        # scaler) is applied to every gradient; DIFFERENT weights per direction are not representable after the fused
        # cross-entropy has written dlogits, so they are rejected instead of being silently ignored.
        if g_bwd is not g_fwd and getattr(model, "caption_backward", False) and not torch.equal(g_fwd, g_bwd):
            raise NotImplementedError("the two captioning directions must enter the loss with the same weight")
        eng.backward(zero_grads=True)
        arena = eng.arena
        scaled = arena.grads * g_fwd  # ONE fused scale over the flat arena; parameter gradients are views of the result
        by_id = model._engine_param_names
        grads = []
        for p in model._engine_params:
            name = by_id.get(id(p))
            if name is None or not p.requires_grad:
                grads.append(None)
            else:
                grads.append(arena.view(scaled, name))
        return (None, None, None, None, None, None, *grads)


class _EngineModel(nn.Module):
    """A model whose arithmetic runs on an `Engine` over its own parameters, built lazily and rebuilt after the module
    is moved or cast (which re-points the parameters away from the engine's arena)."""

    def _new_engine(self) -> Engine:
        raise NotImplementedError

    @property
    def engine(self) -> Engine:
        eng = self._engine
        if eng is None or not eng.arena.intact():
            eng = self._new_engine()
            object.__setattr__(self, "_engine", eng)
            names = {}
            for n in eng.arena.names:
                names[id(eng.arena._param_objs[n])] = n
            object.__setattr__(self, "_engine_param_names", names)
            object.__setattr__(self, "_engine_params", [eng.arena._param_objs[n] for n in eng.arena.names])
        return eng

    def _apply(self, fn, *a, **k):
        # moving / casting the module invalidates the arena views; rebuild lazily afterwards
        object.__setattr__(self, "_engine", None)
        return super()._apply(fn, *a, **k)

    def load_state_dict(self, *a, **k):
        out = super().load_state_dict(*a, **k)
        if self._engine is not None:
            self._engine.mark_weights_dirty()
        return out


class CaptioningModel(_EngineModel):
    def __init__(self, visual: VisualBackbone, textual: TextualHead, caption_backward: bool = False,
                 sos_index: int = 1, eos_index: int = 2, decoder: Any = None):
        super().__init__()
        self.visual = visual
        self.textual = textual
        self.padding_idx = self.textual.padding_idx
        self.caption_backward = caption_backward
        if self.caption_backward:
            self.backward_textual = copy.deepcopy(self.textual)
            # share visual projection and input/output embeddings between directions (captioning.py:60-63)
            self.backward_textual.visual_projection = self.textual.visual_projection
            self.backward_textual.embedding = self.textual.embedding
            self.backward_textual.output = self.textual.output
        self.sos_index = sos_index
        self.eos_index = eos_index
        self.decoder = decoder
        self._engine = None

    def _new_engine(self) -> Engine:
        return Engine(self.visual, self.textual, self.backward_textual if self.caption_backward else None)

    # ---------------------------------------------------------------------------------------------------- forward
    def forward(self, batch: Dict[str, torch.Tensor]) -> Dict[str, Any]:
        if "caption_tokens" not in batch:
            if self.decoder is None:
                raise ValueError("Decoder for predicting captions is missing!")
            if self.decoder.name == "nucleus_sampling":
                return {"predictions": self._nucleus_sampling(batch["image"])}
            return {"predictions": self._beam_search(batch["image"])}
        image = batch["image"]
        if image.device.type != "cuda":
            raise RuntimeError("virtex_b200 has no CPU path: the batch must live on the model's CUDA device")
        image = image.contiguous().float()
        tokens = batch["caption_tokens"].contiguous()
        lengths = batch["caption_lengths"].contiguous()
        noitpac = batch["noitpac_tokens"].contiguous() if self.caption_backward else tokens
        eng = self.engine
        eng.mark_weights_dirty()  # parameters may have been updated by any optimiser since the last call
        if self.training and torch.is_grad_enabled():
            loss_f, loss_b = _StepFunction.apply(self, image, tokens, noitpac, lengths, None, *self._engine_params)
        else:
            loss = eng.forward(image, tokens, noitpac, lengths, training=self.training, with_grad=False).clone()
            loss_f, loss_b = loss[0], loss[1]
        output: Dict[str, Any] = {"loss": loss_f, "loss_components": {"captioning_forward": loss_f.detach().clone()}}
        if self.caption_backward:
            output["loss"] = loss_f + loss_b
            output["loss_components"]["captioning_backward"] = loss_b.detach().clone()
        if not self.training:
            output["predictions"] = eng.predictions().clone()
        return output

    def _beam_search(self, image):
        """Captions of the forward-direction head by the reference's beam search (captioning.py:144-163), decoded
        incrementally by the engine: int64 (B, L) on the device."""
        dec = self.decoder
        if dec.name != "beam_search":
            raise NotImplementedError(f"{dec.name} decoding is not implemented; beam_search is")
        if self.training:
            raise RuntimeError("beam search runs in eval mode (running BatchNorm statistics, no dropout): call "
                               "model.eval() first")
        if image.device.type != "cuda":
            raise RuntimeError("virtex_b200 has no CPU path: the batch must live on the model's CUDA device")
        with torch.no_grad():
            return self.engine.beam_search(image.contiguous().float(), dec.beam_size, dec.per_node_beam_size,
                                           dec.max_steps, self.sos_index, dec.eos_index)

    def _nucleus_sampling(self, image):
        """Captions of the forward-direction head by the reference's nucleus sampling (nucleus_sampling.py:47-123),
        decoded incrementally by the engine: int64 (B, L) on the device.  Each call draws a fresh 64-bit seed on the
        device from torch's default CUDA generator (no host synchronisation), so torch.manual_seed makes a call
        reproducible and successive calls sample different captions, as the reference's torch.multinomial does."""
        dec = self.decoder
        if self.training:
            raise RuntimeError("nucleus sampling runs in eval mode (running BatchNorm statistics, no dropout): call "
                               "model.eval() first")
        if image.device.type != "cuda":
            raise NotImplementedError("nucleus sampling runs on the model's CUDA device only; it has no CPU path")
        with torch.no_grad():
            seed = torch.empty(1, dtype=torch.int64, device=image.device).random_(-2 ** 63, None)  # all 64 bits
            return self.engine.nucleus_sample(image.contiguous().float(), dec.nucleus_size, dec.max_steps,
                                              self.sos_index, dec.eos_index, seed)

    def decoding_step(self, visual_features, partial_captions):
        """Logits of the next token of every partial caption (captioning.py:165-213): (B, C, h, w) fp32 features and
        (B * beam, T) tokens, or (B * beam,) for the first step -> fp32 (B * beam, V).  The whole prefix is recomputed by
        the textual head; the reference's own decoders can drive this model through it."""
        tokens = partial_captions if partial_captions.dim() == 2 else partial_captions[:, None]
        rows, prefix = tokens.shape
        per_image = rows // visual_features.shape[0]  # the beams of image b are rows b * per_image ...
        features = visual_features.repeat_interleave(per_image, 0) if per_image > 1 else visual_features
        lengths = torch.full((rows,), prefix, dtype=torch.int64, device=tokens.device)  # no padding in a prefix
        return self.textual(features, tokens, lengths)[:, -1]


class ForwardCaptioningModel(CaptioningModel):
    def __init__(self, visual, textual, sos_index: int = 1, eos_index: int = 2, decoder: Any = None):
        super().__init__(visual, textual, sos_index=sos_index, eos_index=eos_index, caption_backward=False,
                         decoder=decoder)


class BidirectionalCaptioningModel(CaptioningModel):
    def __init__(self, visual, textual, sos_index: int = 1, eos_index: int = 2, decoder: Any = None):
        super().__init__(visual, textual, sos_index=sos_index, eos_index=eos_index, caption_backward=True,
                         decoder=decoder)


VirTexModel = BidirectionalCaptioningModel


class MaskedLMModel(CaptioningModel):
    """Drop-in for virtex/models/masked_lm.py:11-86 on the same engine: one textual head whose self-attention masks
    padded keys only (`mask_future_positions=False`, textual_heads.py:255-262), cross entropy between the logits of
    EVERY position and `batch["masked_labels"]` (ignore_index = padding), and in eval mode the argmax predictions with
    the positions that carry no label set to the padding index (masked_lm.py:78-84)."""

    def __init__(self, visual: VisualBackbone, textual: TextualHead):
        super().__init__(visual, textual, caption_backward=False)
        if getattr(textual, "mask_future_positions", False):
            raise ValueError("masked language modelling needs a textual head built with mask_future_positions=False")

    def forward(self, batch: Dict[str, torch.Tensor]) -> Dict[str, Any]:
        image = batch["image"]
        if image.device.type != "cuda":
            raise RuntimeError("virtex_b200 has no CPU path: the batch must live on the model's CUDA device")
        image = image.contiguous().float()
        tokens = batch["caption_tokens"].contiguous()
        lengths = batch["caption_lengths"].contiguous()
        labels = batch["masked_labels"].contiguous()
        eng = self.engine
        eng.mark_weights_dirty()
        if self.training and torch.is_grad_enabled():
            loss, _ = _StepFunction.apply(self, image, tokens, tokens, lengths, labels, *self._engine_params)
        else:
            loss = eng.forward(image, tokens, tokens, lengths, training=self.training, with_grad=False,
                               labels=labels).clone()[0]
        output: Dict[str, Any] = {"loss": loss, "loss_components": {"masked_lm": loss.detach().clone()}}
        if not self.training:
            predictions = eng.predictions().clone()
            predictions[labels == self.padding_idx] = self.padding_idx
            output["predictions"] = predictions
        return output


class ClassificationModel(_EngineModel):
    """Drop-in for virtex/models/classification.py:12-108 on the same engine: a `LinearTextualHead` (global average pool
    + one linear layer) over the backbone and the K-hot cross entropy

        loss = mean_b( -mean_{u in U_b} log_softmax(logits_b)[u] ),   U_b = unique ids of batch["labels"][b] minus
                                                                              ignore_indices,

    NaN for a row whose U_b is empty (that row contributes no gradient).  In eval mode `predictions` holds the top-10
    class ids of each image, int64 (B, 10).  Labels outside [0, vocab_size) are skipped; the reference would raise."""

    def __init__(self, visual: VisualBackbone, textual: TextualHead, ignore_indices: List[int]):
        super().__init__()
        if not isinstance(textual, LinearTextualHead):
            raise ValueError("the classification models run on a LinearTextualHead (MODEL.TEXTUAL.NAME 'none')")
        self.visual = visual
        self.textual = textual
        self.ignore_indices = ignore_indices
        self._engine = None

    def _new_engine(self) -> Engine:
        return Engine(self.visual, self.textual, ignore_indices=self.ignore_indices)

    def forward(self, batch: Dict[str, torch.Tensor]) -> Dict[str, Any]:
        image = batch["image"]
        if image.device.type != "cuda":
            raise RuntimeError("virtex_b200 has no CPU path: the batch must live on the model's CUDA device")
        image = image.contiguous().float()
        labels = batch["labels"]
        labels = (labels if labels.dtype == torch.int64 else labels.long()).contiguous()
        eng = self.engine
        eng.mark_weights_dirty()
        if self.training and torch.is_grad_enabled():
            loss, _ = _StepFunction.apply(self, image, None, None, None, labels, *self._engine_params)
        else:
            loss = eng.forward(image, None, None, None, training=self.training, with_grad=False,
                               labels=labels).clone()[0]
        output: Dict[str, Any] = {"loss": loss, "loss_components": {"classification": loss.detach().clone()}}
        if not self.training:
            output["predictions"] = eng.predictions().clone()
        return output

    def _eval_predictions(self, batch):
        self.eval()
        with torch.no_grad():
            predictions = self.forward(batch)["predictions"]
        self.train()
        return predictions


class TokenClassificationModel(ClassificationModel):
    """Targets: the unique caption tokens of each image, special tokens ignored."""

    def log_predictions(self, batch: Dict[str, torch.Tensor], tokenizer) -> str:
        """Caption and top-10 predicted tokens per image; `tokenizer` needs only `decode` and `id_to_token`."""
        text = ""
        for tokens, preds in zip(batch["caption_tokens"], self._eval_predictions(batch)):
            names = " ".join(tokenizer.id_to_token(p) for p in preds.tolist())
            text += (f"\n                Caption tokens : {tokenizer.decode(tokens.tolist())}"
                     f"\n                Predictions (f): {names}\n\n                ")
        return text


class MultiLabelClassificationModel(ClassificationModel):
    """Targets: the unique instance categories of each image, background (id 0) ignored."""

    def log_predictions(self, batch: Dict[str, torch.Tensor], tokenizer=None) -> str:
        """Sorted ground-truth category ids (background dropped) beside as many sorted top predictions."""
        text = ""
        for tokens, preds in zip(batch["caption_tokens"], self._eval_predictions(batch)):
            gt = sorted(t for t in tokens.tolist() if t != 0)
            pred = sorted(preds.tolist()[:len(gt)])
            text += (f"\n                COCO Instance IDs (GT)   : {gt}"
                     f"\n                COCO Instance IDs (Pred) : {pred}\n\n                ")
        return text
