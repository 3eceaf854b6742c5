"""The attention reference against autograd, and the power of its tolerance rule (no GPU needed).

tests/attention_reference.py is what the attention kernels are held to, so it is checked here on its own: its explicit
backward formulas against fp64 autograd through a dense masked softmax, and its tolerance rule against deliberately
wrong problems -- each one a plausible kernel bug -- which it must reject while it accepts a result with the yardstick's
own rounding error."""
import pytest
import torch

from tests import attention_reference as ar

HD = 64


def _inputs(B, H, Tq, Tkv, std, dtype, seed):
    """16-bit q, k, v, dout whose scaled scores have standard deviation ~std (q and k ~ N(0, std): q.k / 8 ~ N(0, std^2))."""
    g = torch.Generator().manual_seed(seed)
    a = std ** 0.5
    q = (torch.randn(B * Tq, H * HD, generator=g, dtype=torch.float64) * a).to(dtype)
    k = (torch.randn(B * Tkv, H * HD, generator=g, dtype=torch.float64) * a).to(dtype)
    v = torch.randn(B * Tkv, H * HD, generator=g, dtype=torch.float64).to(dtype)
    do = torch.randn(B * Tq, H * HD, generator=g, dtype=torch.float64).to(dtype)
    return q, k, v, do


def _autograd(q, k, v, do, B, H, Tq, Tkv, causal, kv_len, scale):
    qh, kh, vh = (t.double().view(B, -1, H, HD).transpose(1, 2).clone().requires_grad_(True) for t in (q, k, v))
    s = (qh @ kh.transpose(-1, -2)) * scale
    mask = torch.zeros(B, 1, Tq, Tkv, dtype=torch.bool)
    for b in range(B):
        mask[b, 0] = ~ar.visibility(Tq, Tkv, causal, ar.n_visible(kv_len, b, Tkv), "cpu")
    s = s.masked_fill(mask, float("-inf"))
    lse = torch.logsumexp(s, dim=-1)
    o = torch.softmax(s, dim=-1) @ vh
    o.backward(do.double().view(B, Tq, H, HD).transpose(1, 2))
    flat = lambda t: t.transpose(1, 2).reshape(-1, H * HD)   # noqa: E731
    return {"o": flat(o.detach()), "lse": lse.detach(), "dq": flat(qh.grad), "dk": flat(kh.grad), "dv": flat(vh.grad)}


@pytest.mark.parametrize("B,H,Tq,Tkv,causal,kv_len,scale", [
    (2, 2, 300, 300, True, [200, 300], None),     # decoder self: causal and per-sample key counts
    (2, 1, 130, 257, False, None, None),          # cross-attention
    (2, 2, 77, 150, False, [40, 151], 0.3),       # kv_len without causal, one past Tkv; a non-default scale
    (2, 1, 65, 65, True, [0, -3], None),          # kv_len <= 0: clamped to one visible key
])
def test_reference_matches_autograd(B, H, Tq, Tkv, causal, kv_len, scale):
    q, k, v, do = _inputs(B, H, Tq, Tkv, 1.0, torch.bfloat16, 3)
    lens = None if kv_len is None else torch.tensor(kv_len, dtype=torch.int32)
    ref = ar.reference(q, k, v, do, B, H, Tq, Tkv, causal=causal, kv_len=lens, scale=scale)
    want = _autograd(q, k, v, do, B, H, Tq, Tkv, causal, kv_len, ar.HD ** -0.5 if scale is None else scale)
    for key, w in want.items():
        err = (ref[key] - w).abs().max().item() / max(w.abs().max().item(), 1.0)   # one visible key: dS = 0
        assert err < 1e-12, f"{key}: {err}"


def _tile0_not_rescaled(q, k, v, B, H, T):
    """O of a forward that keeps key tile 0's weights relative to tile 0's own maximum on rows whose maximum is in
    key tile 1 (keys 128..255): the online-softmax rescale forgotten."""
    outs = []
    for b in range(B):
        qh, kh, vh = (ar._heads(t, b, T, H, torch.float64) for t in (q, k, v))
        s = (qh @ kh.transpose(1, 2)) * ar.HD ** -0.5
        m = s.amax(dim=-1, keepdim=True)
        m0 = s[..., :128].amax(dim=-1, keepdim=True)
        late = s.argmax(dim=-1, keepdim=True).div(128, rounding_mode="floor") == 1
        p = torch.exp(s - m)
        p[..., :128] = torch.where(late, torch.exp(s[..., :128] - m0), p[..., :128])
        outs.append(ar._rows((p @ vh) / p.sum(dim=-1, keepdim=True)))
    return torch.cat(outs)


WRONG = ["last visible key dropped", "first hidden key admitted", "causal diagonal excluded",
         "V rows 127 and 128 exchanged", "tile 0 not rescaled"]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("std", [1.0, 4.0])
@pytest.mark.parametrize("wrong", WRONG)
def test_check_rejects_wrong_attention(wrong, std, dtype):
    B, H, T = 2, 2, 300
    q, k, v, do = _inputs(B, H, T, T, std, dtype, 11)
    causal = wrong == "causal diagonal excluded"
    lens = None if causal or wrong == "tile 0 not rescaled" else torch.tensor([250, 181], dtype=torch.int32)
    kw = dict(causal=causal, kv_len=lens)
    ref = ar.reference(q, k, v, do, B, H, T, T, **kw)
    emu = ar.reference(q, k, v, do, B, H, T, T, emulate=dtype, **kw)
    # the rule accepts a result carrying exactly the yardstick's rounding error
    for key in ("o", "dq", "dk", "dv"):
        ar.check(emu[key], ref[key], emu[key], dtype=dtype, name=key)

    bad_v = v
    vis_fn = None
    if wrong == "last visible key dropped":
        vis_fn = lambda b, vis: vis & (torch.arange(T) != int(lens[b]) - 1)   # noqa: E731
    elif wrong == "first hidden key admitted":
        vis_fn = lambda b, vis: vis | (torch.arange(T) == int(lens[b]))        # noqa: E731
    elif wrong == "causal diagonal excluded":   # row 0 keeps its only key
        vis_fn = lambda b, vis: vis & ~torch.eye(T, dtype=torch.bool) | (vis & (torch.arange(T) == 0)[:, None])  # noqa: E731
    elif wrong == "V rows 127 and 128 exchanged":
        bad_v = v.clone()
        for b in range(B):
            bad_v[[b * T + 127, b * T + 128]] = v[[b * T + 128, b * T + 127]]
    if wrong == "tile 0 not rescaled":
        got = {"o": _tile0_not_rescaled(q, k, v, B, H, T)}
    else:
        got = ar.reference(q, k, bad_v, do, B, H, T, T, vis_fn=vis_fn, **kw)
    for key in got:
        if key in ("lse", "smax") or (key == "dv" and bad_v is not v):   # dV = P^T dO does not read V
            continue
        with pytest.raises(AssertionError):
            ar.check(got[key], ref[key], emu[key], dtype=dtype, name=key)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_check_keeps_its_power_when_most_reference_rows_are_zero(dtype):
    """kv_len <= 0 leaves each query of a sample one key, so the dQ of those samples is exactly zero in fp64 and
    more than half of the tensor's rows are zero.  A dQ 50% wrong on every row of the other samples must still fail,
    and a zero reference is compared exactly."""
    B, H, T = 4, 2, 300
    q, k, v, do = _inputs(B, H, T, T, 1.0, dtype, 7)
    kw = dict(causal=True, kv_len=torch.tensor([0, -5, T + 1, 10 ** 6], dtype=torch.int32))
    ref = ar.reference(q, k, v, do, B, H, T, T, **kw)
    emu = ar.reference(q, k, v, do, B, H, T, T, emulate=dtype, **kw)
    zero = ref["dq"].reshape(-1, HD).norm(dim=1) == 0
    assert zero.float().mean() > 0.5
    ar.check(emu["dq"], ref["dq"], emu["dq"], dtype=dtype, name="dq")
    wrong = emu["dq"].clone()
    wrong[2 * T:] *= 1.5
    with pytest.raises(AssertionError):
        ar.check(wrong, ref["dq"], emu["dq"], dtype=dtype, name="dq")
    rows = torch.arange(B * T) < 2 * T      # the one-key samples alone: an identically zero reference
    ar.check(torch.zeros_like(wrong), ref["dq"], emu["dq"], rows=rows, dtype=dtype, name="dq")
    with pytest.raises(AssertionError):
        ar.check(emu["dq"] + 2.0 ** -30, ref["dq"], emu["dq"], rows=rows, dtype=dtype, name="dq")
