"""Host logic of FP8 training (olmoasr_b200/fp8.py and the FP8 route of the fused blocks) on the CPU: tests/cpu_backend.py
stands in for the dense kernels, and the per-row quantiser and the FP8 GEMM are stood in for below (the GEMM by the dense
GEMM over the dequantised operands).  The stand-ins record every call, so these tests pin which GEMMs run in FP8.  The
kernels themselves are checked on the GPU in tests/test_fp8_gpu.py."""
import pytest
import torch

from tests import cpu_backend
from oracle import logmel, synth

FMAX = {0: 448.0, 1: 57344.0}
FP8 = {0: torch.float8_e4m3fn, 1: torch.float8_e5m2}


def quantize_fp8_rows(x, fmt, *, transpose=False):
    xf = (x.t() if transpose else x).float()
    amax = xf.abs().amax(1)
    zero = amax == 0
    fmax = torch.full_like(amax, FMAX[fmt])      # tensor / tensor: IEEE division (a python scalar would make torch
    inv = torch.where(zero, torch.ones_like(amax), fmax / amax)   # multiply by its reciprocal instead)
    s = torch.where(zero, torch.ones_like(amax), amax / fmax)
    return (xf * inv[:, None]).to(FP8[fmt]), s


CALLS = []


def gemm_fp8(a, a_scale, b, b_scale, M, N, K, *, out=None, out2=None, bias=None, aux=None, epi=0, block_n=0):
    CALLS.append(("fp8", a.dtype, M, N, K, epi))
    assert b.dtype == torch.float8_e4m3fn and a.dtype in (torch.float8_e4m3fn, torch.float8_e5m2)
    assert epi in ((0, 1, 2) if a.dtype == torch.float8_e4m3fn else (0, 2, 3)), (a.dtype, epi)
    A = a.float() * a_scale[:M, None]
    B = b.float() * b_scale[:N, None]
    return cpu_backend.gemm(A, B, M, N, K, out=out, out2=out2, bias=bias, aux=aux, epi=epi)


def gemm(a, b, M, N, K, *, a_mn=False, b_mn=False, out=None, out2=None, bias=None, aux=None, epi=0, split_k=1, block_n=0):
    CALLS.append(("wgrad" if a_mn else "bf16", a.dtype, M, N, K, epi))
    return cpu_backend.gemm(a, b, M, N, K, a_mn=a_mn, b_mn=b_mn, out=out, out2=out2, bias=bias, aux=aux, epi=epi,
                            split_k=split_k, block_n=block_n)


def _dims():
    from olmoasr_b200.config.model_dims import ModelDimensions
    return ModelDimensions(80, 1500, 64, 1, 2, 51864, 448, 64, 1, 2)


@pytest.fixture()
def setup(monkeypatch):
    from olmoasr_b200 import kernels
    from olmoasr_b200.model import OLMoASR

    cpu_backend.install(monkeypatch)
    for fn in (quantize_fp8_rows, gemm_fp8, gemm):
        monkeypatch.setattr(kernels, fn.__name__, fn)
    CALLS.clear()
    torch.manual_seed(0)
    m = OLMoASR(_dims())
    mel = torch.from_numpy(logmel.log_mel_spectrogram(synth.waveforms(2).numpy()))
    ti, ty, pm, lens = synth.text_batch(2)
    return m, mel, ti, ty, pm, lens


def _kinds():
    out = {"fp8": 0, "bf16": 0, "wgrad": 0}
    for c in CALLS:
        out[c[0]] += 1
    return out


def test_context_nests_and_is_exception_safe():
    from olmoasr_b200 import fp8
    from olmoasr_b200._core import bf16_compute

    assert not fp8.fp8_enabled()
    with fp8.fp8_autocast():
        assert fp8.fp8_enabled()
        with fp8.fp8_autocast():
            assert fp8.fp8_enabled()
        assert fp8.fp8_enabled()
        with bf16_compute():          # decode() / transcribe() run in bf16 inside the context
            assert not fp8.fp8_enabled()
        assert fp8.fp8_enabled()
    assert not fp8.fp8_enabled()
    with fp8.fp8_autocast():
        with fp8.fp8_autocast(enabled=False):   # off inside an outer region, back on at its end
            assert not fp8.fp8_enabled()
        assert fp8.fp8_enabled()
    with pytest.raises(RuntimeError, match="boom"):
        with fp8.fp8_autocast():
            with fp8.fp8_autocast():
                raise RuntimeError("boom")
    assert not fp8.fp8_enabled()


# tiny: 2 encoder blocks x 4 projections, 2 decoder blocks x 7 (qkv, out, cross q, cross kv, cross out, fc1, fc2)
N_PROJ = 2 * 4 + 2 * 7


def test_projections_route_to_fp8_only_inside_the_context(setup):
    from olmoasr_b200.fp8 import fp8_autocast

    m, mel, ti, ty, pm, lens = setup

    def step():
        CALLS.clear()
        m.zero_grad(set_to_none=True)
        loss = m(mel, ti, pm, targets=ty)
        fwd = _kinds()
        loss.backward()
        return fwd, _kinds(), loss.item()

    fwd16, all16, loss16 = step()
    with fp8_autocast():
        fwd8, all8, loss8 = step()
    # without the context not one FP8 call; the forward GEMMs of the projections, the stem's two and the logits
    assert all16["fp8"] == 0 and fwd16["bf16"] == N_PROJ + 3
    # inside it every projection's forward and dgrad is FP8; the stem and the logits stay bf16, every wgrad too
    assert fwd8["fp8"] == N_PROJ and fwd8["bf16"] == 3
    assert all8["fp8"] == 2 * N_PROJ
    assert all8["bf16"] == all16["bf16"] - 2 * N_PROJ
    assert all8["wgrad"] == all16["wgrad"]
    dgrads = [c for c in CALLS if c[0] == "fp8" and c[1] == torch.float8_e5m2]
    assert len(dgrads) == N_PROJ      # every dgrad reads e5m2 gradients; every forward e4m3 activations
    assert abs(loss8 - loss16) <= 0.05 * abs(loss16)


def test_backward_outside_the_context_keeps_the_forward_route(setup):
    from olmoasr_b200.fp8 import fp8_autocast

    m, mel, ti, ty, pm, _ = setup
    with fp8_autocast():
        loss = m(mel, ti, pm, targets=ty)
    CALLS.clear()
    loss.backward()
    assert _kinds()["fp8"] == N_PROJ


def test_state_dict_and_buffers_unchanged(setup):
    from olmoasr_b200.fp8 import fp8_autocast

    m, mel, ti, ty, pm, _ = setup
    keys = list(m.state_dict())
    bufs = [n for n, _ in m.named_buffers()]
    with fp8_autocast():
        m(mel, ti, pm, targets=ty).backward()
    assert list(m.state_dict()) == keys
    assert [n for n, _ in m.named_buffers()] == bufs


def test_lora_raises(setup, monkeypatch):
    from olmoasr_b200 import kernels
    from olmoasr_b200.fp8 import fp8_autocast
    from olmoasr_b200.lora import add_lora

    m, mel, ti, ty, pm, _ = setup
    monkeypatch.setattr(kernels, "cast_scaled16", lambda src, s, dst: dst.copy_((s * src).to(dst.dtype)))
    add_lora(m, 8, 16, ["decoder.mlp.0"])
    with fp8_autocast(), pytest.raises(ValueError, match="LoRA"):
        m(mel, ti, pm, targets=ty)


def test_checkpoint_recompute_follows_the_forward_with_the_context_fn(setup):
    """torch.utils.checkpoint with fp8_checkpoint_context_fn: the backward runs outside the context, the recompute of
    every block still takes the FP8 route, and the gradients equal those of the same step without checkpointing."""
    from torch.utils.checkpoint import checkpoint
    from olmoasr_b200.fp8 import fp8_autocast, fp8_checkpoint_context_fn

    m, mel, ti, ty, pm, _ = setup
    with fp8_autocast():
        m(mel, ti, pm, targets=ty).backward()
    want = {n: p.grad.clone() for n, p in m.named_parameters()}
    m.zero_grad(set_to_none=True)
    blocks = list(m.encoder.blocks) + list(m.decoder.blocks)
    for blk in blocks:
        blk.forward = lambda *a, _f=blk.forward, **kw: checkpoint(_f, *a, use_reentrant=False,
                                                                  context_fn=fp8_checkpoint_context_fn, **kw)
    with fp8_autocast():
        loss = m(mel, ti, pm, targets=ty)
    CALLS.clear()
    loss.backward()                       # outside the context
    for blk in blocks:
        del blk.forward
    k = _kinds()
    assert k["fp8"] == 2 * N_PROJ       # each block's recomputed forward and its dgrads, all FP8
    for n, p in m.named_parameters():
        assert torch.equal(p.grad, want[n]), n
