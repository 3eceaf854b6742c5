"""Launch traces of the training backward in every gradient-destination mode, on the CPU with tests/cpu_backend.py
standing in for the kernels.  Each kernel call is recorded with its tensor arguments (shape, dtype, strides, storage
offset -- or the element offset into the gradient slab G), its scalar arguments and whether it was issued through the
side stream, for one forward + backward of the tiny model in five configurations.  The traces must equal
tests/golden/grad_routing_trace.json, which was recorded (`python -m tests.test_grad_routing_cpu`) from the backward as
it was before the per-Function gradient-destination code was replaced by `_core._GradDest`: the host code that decides
where gradients go may change, the launches it makes may not."""
import copy
import json
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

from tests import cpu_backend
from oracle import logmel, synth

GOLDEN = Path(__file__).resolve().parent / "golden" / "grad_routing_trace.json"
CONFIGS = ("no_slabs", "slab_direct", "slab_handover", "bf16_params", "fp32_logits_direct")


def _model():
    from olmoasr_b200.config.model_dims import ModelDimensions
    from olmoasr_b200.model import OLMoASR

    torch.manual_seed(0)
    m = OLMoASR(ModelDimensions(80, 1500, 64, 1, 2, 51864, 448, 64, 1, 2))
    with torch.no_grad():      # non-trivial LayerNorm affine parameters and biases, as in tests/test_host_model_cpu.py
        for k, p in m.named_parameters():
            if k.endswith("ln.weight") or "_ln.weight" in k or "ln_post.weight" in k:
                p.add_(0.1 * torch.randn_like(p))
            elif k.endswith(".bias"):
                p.add_(0.05 * torch.randn_like(p))
    return m


def _fmt(v, G):
    if isinstance(v, torch.Tensor):
        where = f"@{v.storage_offset()}"
        if G is not None and v.untyped_storage().data_ptr() == G.untyped_storage().data_ptr():
            where = f"@G{v.storage_offset() - G.storage_offset()}"
        return f"{str(v.dtype).removeprefix('torch.')}{list(v.shape)}{list(v.stride())}{where}"
    if isinstance(v, (list, tuple)):
        return "(" + ", ".join(_fmt(x, G) for x in v) + ")"
    return repr(v)


class _Recorder:
    """Wraps every stand-in that cpu_backend installed on olmoasr_b200.kernels, and _core._Side.run."""

    def __init__(self, mp):
        from olmoasr_b200 import _core, kernels

        self.entries, self.G, self.side = [], None, 0
        cpu_backend.install(mp)
        for name in dir(kernels):
            fn = getattr(kernels, name)
            if getattr(fn, "__module__", None) == cpu_backend.__name__:
                mp.setattr(kernels, name, self._wrap(name, fn))
        run = _core._Side.run

        def side_run(side, fn):
            self.side += 1
            try:
                return run(side, fn)
            finally:
                self.side -= 1

        mp.setattr(_core._Side, "run", side_run)

    def _wrap(self, name, fn):
        def call(*args, **kwargs):
            parts = [_fmt(a, self.G) for a in args] + [f"{k}={_fmt(v, self.G)}" for k, v in kwargs.items()]
            self.entries.append(f"{name}({', '.join(parts)})" + (" side" if self.side else ""))
            return fn(*args, **kwargs)
        return call

    def take(self):
        out, self.entries = self.entries, []
        return out


def _run(config, rec):
    """One forward + backward in `config`: (trace {"forward", "backward"}, {name: gradient})."""
    m = _model()
    mel = torch.from_numpy(logmel.log_mel_spectrogram(synth.waveforms(2).numpy()))
    ti, ty, pm, _ = synth.text_batch(2)
    rec.G = None
    if config == "bf16_params":      # FSDP MixedPrecision(param_dtype=bf16): bf16 parameter views, no slabs
        m = copy.deepcopy(m).to(torch.bfloat16)
        m.encoder.positional_embedding.data = m.encoder.positional_embedding.data.to(torch.bfloat16)
        mel, pm = mel.to(torch.bfloat16), pm.to(torch.bfloat16)
    elif config != "no_slabs":
        sl = m.use_slabs(direct_grads=config != "slab_handover")
        sl.sync_shadows()
        sl.zero_grad()
        rec.G = sl.G
    rec.take()
    if config == "fp32_logits_direct":
        lg = m(mel, ti, pm)
        fwd = rec.take()
        F.cross_entropy(lg.view(-1, lg.shape[-1]), ty.view(-1), ignore_index=51864).backward()
    else:
        loss = m(mel, ti, pm, targets=ty)
        fwd = rec.take()
        loss.backward()
    trace = {"forward": fwd, "backward": rec.take()}
    return trace, {k: p.grad.detach().clone() for k, p in m.named_parameters()}


def _record_all(mp):
    rec = _Recorder(mp)
    return {c: _run(c, rec) for c in CONFIGS}


@pytest.fixture(scope="module")
def runs():
    with pytest.MonkeyPatch.context() as mp:
        yield _record_all(mp)


@pytest.mark.parametrize("config", CONFIGS)
def test_backward_launches_match_the_golden_trace(runs, config):
    want = json.loads(GOLDEN.read_text())[config]
    got = runs[config][0]
    assert got["forward"] == want["forward"]
    assert got["backward"] == want["backward"]


def test_every_gradient_destination_mode_gives_the_same_gradients(runs):
    def rel(a, b):
        return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-30))

    plain = runs["no_slabs"][1]
    for config in ("slab_direct", "slab_handover"):
        grads = runs[config][1]
        assert grads.keys() == plain.keys()
        for k, g in grads.items():
            assert g.dtype == torch.float32 and rel(g, plain[k]) <= 2e-3, (config, k, rel(g, plain[k]))


if __name__ == "__main__":
    with pytest.MonkeyPatch.context() as mp:
        traces = {c: t for c, (t, _) in _record_all(mp).items()}
    GOLDEN.write_text(json.dumps(traces, indent=0) + "\n")
    print({c: (len(t["forward"]), len(t["backward"])) for c, t in traces.items()})
