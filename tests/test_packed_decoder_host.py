"""Host route of packed decoder training (`model(..., targets=, text_lens=)`) on the CPU: tests/cpu_backend.py stands in
for the dense kernels, and the packed kernels are stood in for below by running the dense stand-ins on one sample at a
time.  Checks that the packed route computes the dense route's loss and gradients (autograd and slab mode), that targets
past a sample's length count as ignored, and every argument error.  The kernels themselves are checked on the GPU in
tests/test_packed_decoder_gpu.py."""
import copy

import pytest
import torch

from tests import cpu_backend
from oracle import logmel, synth

BF = torch.bfloat16


# ---- packed stand-ins: each sample of the PackedBatch through the dense stand-in, as B = 1 ----------------------------
def _samples(pk, Tkv):
    cu = pk.cu.tolist()
    for b, n in enumerate(pk.lens):
        q_rows = slice(cu[b], cu[b + 1])
        kv_rows = q_rows if Tkv is None else slice(b * Tkv, (b + 1) * Tkv)
        yield n, q_rows, kv_rows, (n if Tkv is None else Tkv)


def attention_fwd_varlen(q, k, v, pk, H, Tkv=None, scale=None, want_lse=True, out=None):
    o = torch.empty((pk.N, H * 64), dtype=BF)
    lse = torch.empty((H, pk.N))
    for n, qr, kr, tkv in _samples(pk, Tkv):
        ob, lb = cpu_backend.attention_fwd(q[qr], k[kr], v[kr], 1, H, n, tkv, causal=Tkv is None, scale=scale)
        o[qr], lse[:, qr] = ob, lb.reshape(H, n)
    if out is not None:
        out.copy_(o)
        o = out
    return o, (lse if want_lse else None)


def attention_bwd_varlen(q, k, v, o, dout, lse, pk, H, Tkv=None, scale=None, dq=None, dk=None, dv=None):
    kv_rows = pk.N if Tkv is None else pk.B * Tkv
    dq = torch.empty((pk.N, H * 64), dtype=BF) if dq is None else dq
    dk = torch.empty((kv_rows, H * 64), dtype=BF) if dk is None else dk
    dv = torch.empty((kv_rows, H * 64), dtype=BF) if dv is None else dv
    for n, qr, kr, tkv in _samples(pk, Tkv):
        cpu_backend.attention_bwd(q[qr], k[kr], v[kr], o[qr], dout[qr], None, 1, H, n, tkv, causal=Tkv is None, scale=scale,
                                  dq=dq[qr], dk=dk[kr], dv=dv[kr])
    return dq, dk, dv


def embed_fwd_packed(ids, emb, pos, pk, dtype=BF):
    r = pk.rows.long()
    return (emb[ids.reshape(-1)[r]].float() + pos[r % pk.S].float()).to(BF)


def embed_bwd_packed(ids, dx, demb, dpos, pk, padding_idx):
    r = pk.rows.long()
    flat = ids.reshape(-1)[r]
    keep = flat != padding_idx
    demb.index_add_(0, flat[keep], dx.float()[keep])
    dpos.index_add_(0, r % pk.S, dx.float())


def _dims():
    from olmoasr_b200.config.model_dims import ModelDimensions
    return ModelDimensions(80, 1500, 64, 1, 2, 51864, 448, 64, 1, 2)


@pytest.fixture()
def setup(monkeypatch):
    from olmoasr_b200 import kernels
    from olmoasr_b200.model import OLMoASR

    cpu_backend.install(monkeypatch)
    for fn in (attention_fwd_varlen, attention_bwd_varlen, embed_fwd_packed, embed_bwd_packed):
        monkeypatch.setattr(kernels, fn.__name__, fn)
    torch.manual_seed(0)
    m = OLMoASR(_dims())
    with torch.no_grad():
        for k, p in m.named_parameters():
            if k.endswith(".bias"):
                p.add_(0.05 * torch.randn_like(p))
    mel = torch.from_numpy(logmel.log_mel_spectrogram(synth.waveforms(2).numpy()))
    ti, ty, pm, lens = synth.text_batch(2)
    return m, mel, ti, ty, pm, lens


def _rel(a, b):
    return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-30))


def _grads(m):
    return {k: p.grad.clone() for k, p in m.named_parameters()}


def _assert_same(loss_p, loss_d, gp, gd):
    assert abs(loss_p.item() - loss_d.item()) <= 1e-5 * abs(loss_d.item()), (loss_p.item(), loss_d.item())
    # the per-sample matmuls sum in another fp32 order, which now and then moves a bf16 rounding of an activation by an ulp
    for k in gd:
        assert _rel(gp[k], gd[k]) <= 5e-3, (k, _rel(gp[k], gd[k]))


def test_packed_matches_dense_in_autograd_mode(setup):
    m, mel, ti, ty, pm, lens = setup
    dense = copy.deepcopy(m)
    loss_d = dense(mel, ti, pm, targets=ty)
    loss_d.backward()
    loss_p = m(mel, ti, targets=ty, text_lens=lens)
    loss_p.backward()
    _assert_same(loss_p, loss_d, _grads(m), _grads(dense))


def test_packed_matches_dense_in_slab_mode(setup):
    m, mel, ti, ty, pm, lens = setup
    dense = copy.deepcopy(m)
    for mod in (m, dense):
        sl = mod.use_slabs()
        sl.sync_shadows()
        sl.zero_grad()
    loss_d = dense.loss(mel, ti, ty, pm)
    loss_d.backward()
    loss_p = m.loss(mel, ti, ty, text_lens=[int(n) for n in lens])
    loss_p.backward()
    _assert_same(loss_p, loss_d, _grads(m), _grads(dense))
    for k, p in m.named_parameters():
        assert p.grad.data_ptr() == m._slabs.grad(p).data_ptr(), k


def test_targets_past_the_length_count_as_ignored(setup):
    m, mel, ti, ty, pm, lens = setup
    lens = torch.tensor([50, 17])                  # shorter than the transcripts: the tails are real tokens, not padding
    pm_short = torch.zeros(2, 448, 448)
    ty_short = ty.clone()
    for b, n in enumerate(lens.tolist()):
        pm_short[b, :, n:] = float("-inf")
        ty_short[b, n:] = 51864
    with torch.no_grad():
        loss_d = m(mel, ti, pm_short, targets=ty_short)
        loss_p = m(mel, ti, targets=ty, text_lens=lens)
    assert abs(loss_p.item() - loss_d.item()) <= 1e-5 * abs(loss_d.item())


class _OnDevice(torch.Tensor):
    """A host tensor that reports itself as a CUDA tensor (this test runs without a GPU)."""

    @property
    def is_cuda(self):
        return True


@pytest.mark.parametrize("case", ["cuda", "no_targets", "with_mask", "too_few", "too_many", "zero", "past_ctx", "float",
                                  "bools", "floats_in_list"])
def test_bad_text_lens_raise_value_error(setup, case):
    m, mel, ti, ty, pm, lens = setup
    kw = {"targets": ty, "text_lens": lens}
    mask = None
    if case == "cuda":
        kw["text_lens"] = lens.as_subclass(_OnDevice)
    elif case == "no_targets":
        del kw["targets"]
    elif case == "with_mask":
        mask = pm
    elif case == "too_few":
        kw["text_lens"] = lens[:1]
    elif case == "too_many":
        kw["text_lens"] = [5, 6, 7]
    elif case == "zero":
        kw["text_lens"] = [0, 5]
    elif case == "past_ctx":
        kw["text_lens"] = [5, 449]
    elif case == "float":
        kw["text_lens"] = lens.float()
    elif case == "bools":
        kw["text_lens"] = [True, True]
    elif case == "floats_in_list":
        kw["text_lens"] = [5.0, 6.5]
    with pytest.raises(ValueError):
        m(mel, ti, mask, **kw)
    if "targets" in kw:
        with pytest.raises(ValueError):
            m.loss(mel, ti, ty, mask, text_lens=kw["text_lens"])
