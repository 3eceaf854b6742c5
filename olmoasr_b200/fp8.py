"""FP8 training of the block projections.

    with olmoasr_b200.fp8.fp8_autocast():
        loss = model(mel, tokens, padding_mask)
    loss.backward()          # inside or outside the context

Inside the context the fused training blocks run the forward and dgrad GEMMs of every block projection (qkv, out,
cross q, cross kv, fc1, fc2) on Hopper's FP8 tensor cores (csrc/gemm_sm90.cu, `oasr_gemm_fp8`); the forward records the
mode for its backward, like torch.autocast.  The recipe is fixed:

- per-row dynamic scaling: each row r of a 16-bit operand becomes q = fp8(x * fmax / amax_r) with scale amax_r / fmax
  (csrc/fp8.cu), so results are deterministic and an activation-checkpoint recompute gives the same bits;
- forward y = x W^T: x e4m3 per token row, W e4m3 per output row; dgrad dx = dy W: dy e5m2 per row, W^T e4m3 per input
  feature (both wgmma operands must be K-major, so the dgrad reads a transposed weight copy);
- the fp8 weight copies are built from the block's 16-bit operands and rebuilt when a parameter changes (once per
  optimizer step); under FSDP on every call, like the 16-bit views;
- the encoder output, which feeds every decoder layer's cross K/V projection, is quantised once per decoder forward.

Everything else computes as before: the conv stem, LayerNorm, attention, the tied logits and loss head, every weight
gradient (they read the saved bf16 activations), and decode() / transcribe() / the kv-cache hook path, which run in
bf16 inside the context too.  The compute type is bf16: the context raises ValueError under
torch.autocast("cuda", torch.float16) and on blocks with LoRA adapters.  It keeps no state, adds no buffers and changes
no state_dict key.  `fp8_autocast(enabled=False)` turns FP8 off inside an outer region.

Activation checkpointing: the recompute of a checkpointed block must take the forward's route.  torch restores
torch.autocast's state for it but knows nothing of this context, so pass `context_fn=fp8_checkpoint_context_fn`:

    y = torch.utils.checkpoint.checkpoint(block, x, use_reentrant=False, context_fn=fp8_checkpoint_context_fn)

Then the backward may run inside or outside the context and the recompute quantises the same rows again (same bits).
Without it, run the backward inside the same context as the forward.
"""
from __future__ import annotations

from ._core import fp8_autocast, fp8_checkpoint_context_fn, fp8_enabled

__all__ = ["fp8_autocast", "fp8_checkpoint_context_fn", "fp8_enabled"]
