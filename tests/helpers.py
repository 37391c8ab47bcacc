"""The product's model of an oracle spec, for the tests."""
from oracle import virtex_oracle as O


def virtex_model(spec: O.Spec, dropout=0.0):
    """The product's VirTexModel for `spec`, freshly initialised, on the CPU."""
    from virtex_b200.models import VirTexModel
    from virtex_b200.modules import TorchvisionVisualBackbone, TransformerDecoderTextualHead
    visual = TorchvisionVisualBackbone(spec.backbone, visual_feature_size=spec.visual_feature_size)
    textual = TransformerDecoderTextualHead(
        visual_feature_size=spec.visual_feature_size, vocab_size=spec.vocab, hidden_size=spec.hidden,
        num_layers=spec.layers, attention_heads=spec.heads, feedforward_size=spec.ffn, dropout=dropout,
        norm_first=spec.norm_first, max_caption_length=spec.max_len, padding_idx=spec.pad,
        mask_future_positions=spec.mask_future)
    return VirTexModel(visual, textual)


def build_model(spec: O.Spec, state, dropout=0.0):
    """virtex_model(spec) on the GPU with the oracle's weights `state` loaded strictly."""
    model = virtex_model(spec, dropout)
    model.load_state_dict(O.to_reference_state_dict(state, spec), strict=True)
    return model.cuda()


def to_cuda(batch):
    return {k: v.cuda() for k, v in batch.items()}
