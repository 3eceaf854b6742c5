"""Training model -- drop-in for `olmoasr.model` of the reference (olmoasr/model.py).

Same classes, constructor arguments, parameter names and shapes (token embedding has n_vocab + 1 rows with
padding_idx 51864), same call signature `model(mel, tokens, padding_mask, verbose)` returning fp32 logits, plus
`model.loss(mel, tokens, targets, padding_mask)` which fuses the tied-logits GEMM with the token cross-entropy of
scripts/training/train_timestamps.py:1444-1448.  All compute runs in liboasr_b200.so (see _core.py).
"""
from ._core import (AudioEncoder, Conv1d, LayerNorm, Linear, MultiHeadAttention, OLMoASRBase, ResidualAttentionBlock,
                    TextDecoder, sinusoids)
from .config.model_dims import ModelDimensions


class OLMoASR(OLMoASRBase):
    _train_vocab_pad = True

    def decode(self, mel, options=None, **kwargs):
        from .decoding import decode as decode_function
        return decode_function(self, mel, options, **kwargs) if options is not None else decode_function(self, mel, **kwargs)

    def detect_language(self, mel, tokenizer=None):
        from .decoding import detect_language as detect_language_function
        return detect_language_function(self, mel, tokenizer)

    def transcribe(self, audio, **kwargs):
        from .transcribe import transcribe as transcribe_function
        return transcribe_function(self, audio, **kwargs)

    def transcribe_batch(self, audios, **kwargs):
        from .transcribe import transcribe_batch as transcribe_batch_function
        return transcribe_batch_function(self, audios, **kwargs)


__all__ = ["LayerNorm", "Linear", "Conv1d", "sinusoids", "MultiHeadAttention", "ResidualAttentionBlock", "AudioEncoder",
           "TextDecoder", "OLMoASR", "ModelDimensions"]
