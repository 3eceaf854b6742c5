"""Inference model -- drop-in for `olmoasr.inf_model` of the reference (olmoasr/inf_model.py): token embedding with
n_vocab rows (no pad row, scripts/eval/gen_inf_ckpt.py:4-11), single kaiming draw per projection, uninitialised
decoder positional embedding until a checkpoint is loaded, `forward(mel, tokens, padding_mask=None)`."""
from typing import Optional

from torch import Tensor

from ._core import (AudioEncoder, Conv1d, LayerNorm, Linear, MultiHeadAttention, OLMoASRBase, ResidualAttentionBlock,
                    TextDecoder, sinusoids)
from .config.model_dims import ModelDimensions


class OLMoASR(OLMoASRBase):
    _train_vocab_pad = False

    def forward(self, mel: Tensor, tokens: Tensor, padding_mask: Optional[Tensor] = None) -> Tensor:  # inf_model.py:403-406
        return self.decoder(tokens, self.encoder(mel), padding_mask=padding_mask)

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
