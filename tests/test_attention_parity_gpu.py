"""Attention kernels against the fp64 reference of tests/attention_reference.py, in bf16 and fp16.

Training kernels (oasr_attention_fwd / _bwd and their fp16 twins): the benchmarked head counts and shapes, the mask
edges around the 64-query / 128-key tiles, peaked score regimes, the lse output, the model's strided call pattern with
sentinel-guarded outputs, and bit-exact isolation properties.  Every O / dQ / dK / dV comparison uses
attention_reference.check (per-row relative error against the rounding-point yardstick); every case also checks lse.

Decode attention (oasr_dec_attention / _grouped): an fp64 statement of decode.cu's rounding points over the engine's
self-attention cache and cross K | V layouts, at cache lengths, head counts and split counts the engine uses.
"""
import ctypes

import pytest
import torch

from tests import attention_reference as ar
from tests.decode_reference import dec_out_ref, dec_scores_ref, ulp

pytestmark = pytest.mark.gpu

HD = 64
DTYPES = [torch.bfloat16, torch.float16]
DT_ID = {torch.bfloat16: "bf16", torch.float16: "fp16"}


def _inputs(B, H, Tq, Tkv, dtype, std=1.0, seed=0, peak=None, q_zero=False):
    """16-bit q, k, v, dout on the GPU whose scaled scores have standard deviation ~std.  peak = key index that beats
    every other key's score by ~30 for every query (dimension 63 of each head carries it)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    a = std ** 0.5
    q = torch.randn(B * Tq, H * HD, device="cuda", generator=g) * a
    k = torch.randn(B * Tkv, H * HD, device="cuda", generator=g) * a
    v = torch.randn(B * Tkv, H * HD, device="cuda", generator=g)
    do = torch.randn(B * Tq, H * HD, device="cuda", generator=g)
    if peak is not None:
        q.view(B * Tq, H, HD)[:, :, 63] = 4.0
        kh = k.view(B, Tkv, H, HD)
        kh[:, :, :, 63] = 0.0
        kh[:, peak, :, 63] = 60.0     # 4 * 60 / 8 = 30 above the key's other terms
    if q_zero:
        q.zero_()
    return tuple(t.to(dtype) for t in (q, k, v, do))


def _valid_keys(B, Tkv, kv_len):
    """bool (B*Tkv,): keys the kernels attend to (kv_len clamped to [1, Tkv])."""
    lens = kv_len.tolist() if kv_len is not None else None
    return torch.cat([torch.arange(Tkv, device="cuda") < ar.n_visible(lens, b, Tkv) for b in range(B)])


def _lens(kv_len):
    return None if kv_len is None else torch.tensor(kv_len, device="cuda", dtype=torch.int32)


def _kernels(q, k, v, do, B, H, Tq, Tkv, causal=False, kv_len=None, scale=None):
    from olmoasr_b200 import kernels as K

    o, lse = K.attention_fwd(q, k, v, B, H, Tq, Tkv, causal=causal, kv_len=kv_len, scale=scale)
    dq, dk, dv = K.attention_bwd(q, k, v, o, do, lse, B, H, Tq, Tkv, causal=causal, kv_len=kv_len, scale=scale)
    torch.cuda.synchronize()
    return {"o": o, "lse": lse, "dq": dq, "dk": dk, "dv": dv}


def _single_key(B, Tq, Tkv, causal, kv_len):
    """Rows whose dS = P o (dP - D) is zero in exact arithmetic: queries that see exactly one key (P = 1, dP = D), and
    keys seen only by such queries.  bool (B*Tq,), (B*Tkv,)."""
    lens = kv_len.tolist() if kv_len is not None else None
    sq, sk = [], []
    for b in range(B):
        vis = ar.visibility(Tq, Tkv, causal, ar.n_visible(lens, b, Tkv), "cuda")
        one = vis.sum(dim=1) == 1
        sq.append(one)
        sk.append(vis.any(dim=0) & ~(vis & ~one[:, None]).any(dim=0))
    return torch.cat(sq), torch.cat(sk)


def _parity(B, H, Tq, Tkv, dtype, causal=False, kv_len=None, scale=None, **gen):
    """Kernels against the fp64 reference: O, dQ, dK, dV (visible keys) by the tolerance rule, lse, and exactly zero
    dK / dV on hidden keys.  dQ / dK rows whose dS is zero in exact arithmetic (see _single_key) are only bounded: the
    kernel's dP and D are fp32 sums of the same products in different orders, so there they are rounding noise."""
    q, k, v, do = _inputs(B, H, Tq, Tkv, dtype, **gen)
    lens = _lens(kv_len)
    got = _kernels(q, k, v, do, B, H, Tq, Tkv, causal, lens, scale)
    ref = ar.reference(q, k, v, do, B, H, Tq, Tkv, causal=causal, kv_len=lens, scale=scale)
    emu = ar.reference(q, k, v, do, B, H, Tq, Tkv, causal=causal, kv_len=lens, scale=scale, emulate=dtype)
    valid = _valid_keys(B, Tkv, lens)
    single_q, single_k = _single_key(B, Tq, Tkv, causal, lens)
    rows = {"o": None, "dq": ~single_q, "dk": valid & ~single_k, "dv": valid}
    for key in ("dq", "dk"):
        noise = got[key][single_q if key == "dq" else single_k]
        assert noise.numel() == 0 or float(noise.abs().max()) <= 1e-3, f"{key} where dS is exactly zero"
    for key in ("o", "dq", "dk", "dv"):
        if rows[key] is None or rows[key].any():
            ar.check(got[key], ref[key], emu[key], rows=rows[key], name=key)
    ar.check_lse(got["lse"], ref)
    for key in ("dk", "dv"):
        assert not got[key][~valid].any(), f"{key} of hidden keys is not zero"


# ---------------------------------------------------------------------------------------------------- production
def _text_lens(B):
    from olmoasr_b200 import synthetic

    return synthetic.text_batch(B)[3].tolist()


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("H", [6, 8, 12, 16, 20])
@pytest.mark.parametrize("use", ["encoder", "decoder", "cross"])
def test_production_shapes(use, H, dtype):
    if use == "encoder":
        _parity(2, H, 1500, 1500, dtype, seed=H)
    elif use == "decoder":
        _parity(4, H, 448, 448, dtype, causal=True, kv_len=_text_lens(4), seed=H)
    else:
        _parity(2, H, 448, 1500, dtype, seed=H)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("use", ["encoder", "decoder"])
def test_medium_bench_shape(use, dtype):
    """The medium training step's attention calls: B = 16, H = 16."""
    if use == "encoder":
        _parity(16, 16, 1500, 1500, dtype, seed=1)
    else:
        _parity(16, 16, 448, 448, dtype, causal=True, kv_len=_text_lens(16), seed=1)


# ---------------------------------------------------------------------------------------------------- mask edges
EDGE_LENS = [1, 2, 63, 64, 65, 127, 128, 129, 255, 256, 257, 447, 448, 1000]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_kv_len_on_tile_edges(dtype):
    """One causal call whose samples' key counts sit on and next to the 64-query and 128-key tile edges (where the
    backward's all-visible fast paths switch on and off); 1000 > T is clamped to T."""
    _parity(len(EDGE_LENS), 2, 448, 448, dtype, causal=True, kv_len=EDGE_LENS, seed=2)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("T", [1, 63, 65, 129, 191])
def test_ragged_lengths(T, dtype):
    _parity(2, 2, T, T, dtype, causal=True, kv_len=[T, T // 2 + 1], seed=T)
    _parity(2, 2, T, 2 * T + 1, dtype, seed=T)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_kv_len_without_causal(dtype):
    _parity(3, 2, 200, 1500, dtype, kv_len=[1500, 700, 129], seed=3)


# ---------------------------------------------------------------------------------------------------- score regimes
REGIMES = {"std1": dict(std=1.0), "std4": dict(std=4.0), "std12": dict(std=12.0),
           "late_max": dict(peak="late"), "early_max": dict(peak=3), "q_zero": dict(q_zero=True)}


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("regime", list(REGIMES))
@pytest.mark.parametrize("use", ["cross", "decoder"])
def test_score_regimes(use, regime, dtype):
    """Peaked rows: the online-softmax rescale (late maximum: earlier tiles' weights underflow), exp2 underflow and the
    P o (dP - D) cancellation; q = 0 gives a uniform softmax, O = mean of V."""
    gen = dict(REGIMES[regime], seed=4)
    if use == "cross":
        if gen.get("peak") == "late":
            gen["peak"] = 700
        _parity(1, 4, 256, 1500, dtype, **gen)
    else:
        if gen.get("peak") == "late":
            gen["peak"] = 200
        _parity(2, 4, 448, 448, dtype, causal=True, kv_len=[448, 300], **gen)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_uniform_softmax_is_the_mean_of_v(dtype):
    B, H, T = 1, 2, 1500
    q, k, v, do = _inputs(B, H, T, T, dtype, q_zero=True, seed=5)
    got = _kernels(q, k, v, do, B, H, T, T)
    mean = v.double().mean(dim=0, keepdim=True).expand(T, -1)
    ar.check(got["o"], mean, mean.to(dtype).float(), name="o")
    assert not got["dk"].any()   # dK = scale dS^T Q with Q = 0


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("use", ["cross", "decoder"])
def test_non_default_scale(use, dtype):
    """Both kernels fold scale into scale_log2 and multiply dQ / dK by it."""
    if use == "cross":
        _parity(2, 2, 200, 700, dtype, scale=0.37, seed=6)
    else:
        _parity(2, 2, 300, 300, dtype, causal=True, kv_len=[300, 150], scale=0.05, seed=6)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_check_catches_an_off_by_one_kv_len(dtype):
    """The rule's power on real kernel output: kv_len - 1 given to the kernels but not to the reference must fail."""
    B, H, T = 4, 8, 448
    lens = _text_lens(B)
    q, k, v, do = _inputs(B, H, T, T, dtype, seed=13)
    got = _kernels(q, k, v, do, B, H, T, T, True, _lens([n - 1 for n in lens]))
    ref = ar.reference(q, k, v, do, B, H, T, T, causal=True, kv_len=lens)
    emu = ar.reference(q, k, v, do, B, H, T, T, causal=True, kv_len=lens, emulate=dtype)
    for key in ("o", "dq", "dk", "dv"):
        with pytest.raises(AssertionError):
            ar.check(got[key], ref[key], emu[key], name=key)


# ---------------------------------------------------------------------------------------------------- kv_len clamps
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_kv_len_clamps(dtype):
    """kv_len = 0 (and below) is clamped to one visible key; kv_len > Tkv is Tkv.  Bits equal the clamped call's."""
    B, H, T = 4, 2, 300
    q, k, v, do = _inputs(B, H, T, T, dtype, seed=7)
    clamped = _kernels(q, k, v, do, B, H, T, T, causal=True, kv_len=_lens([1, 1, T, T]))
    raw = _kernels(q, k, v, do, B, H, T, T, causal=True, kv_len=_lens([0, -5, T + 1, 10 ** 6]))
    for key in clamped:
        assert torch.equal(raw[key], clamped[key]), key
    _parity(B, H, T, T, dtype, causal=True, kv_len=[0, -5, T + 1, 10 ** 6], seed=7)


# ---------------------------------------------------------------------------------------------------- layout
def _sentinel(rows, cols, dtype):
    """A buffer with 1 spare row above, 1 below and 64 spare columns either side of a (rows, cols) view."""
    buf = torch.full((rows + 2, cols + 128), -1032.0, device="cuda", dtype=dtype)   # exact in bf16 and fp16
    return buf, buf[1:rows + 1, 64:64 + cols]


def _outside_unchanged(buf, rows, cols):
    inside = torch.zeros_like(buf, dtype=torch.bool)
    inside[1:rows + 1, 64:64 + cols] = True
    return bool((buf[~inside] == -1032.0).all())


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("use", ["decoder", "cross"])
def test_model_call_pattern(use, dtype):
    """q / k / v as column views of qkv (row stride 3d) or cross K / V of kvc (row stride 2d), O written into a view
    of a wider buffer, dq / dk / dv into views of sentinel-filled buffers: bits equal the contiguous run and nothing
    outside the views changes."""
    from olmoasr_b200 import kernels as K

    B, H = 3, 4
    d = H * HD
    causal = use == "decoder"
    Tq, Tkv = (448, 448) if causal else (448, 1500)
    lens = _lens([448, 97, 257]) if causal else None
    q, k, v, do = _inputs(B, H, Tq, Tkv, dtype, seed=8)
    want = _kernels(q, k, v, do, B, H, Tq, Tkv, causal, lens)

    if causal:
        qkv = torch.cat([q, k, v], dim=1)
        qs, ks, vs = qkv[:, :d], qkv[:, d:2 * d], qkv[:, 2 * d:]
    else:
        kvc = torch.cat([k, v], dim=1)
        qs, ks, vs = q.clone(), kvc[:, :d], kvc[:, d:]
    obuf, o = _sentinel(B * Tq, d, dtype)
    _, lse = K.attention_fwd(qs, ks, vs, B, H, Tq, Tkv, causal=causal, kv_len=lens, out=o)
    if causal:
        gbuf, g = _sentinel(B * Tq, 3 * d, dtype)
        dq, dk, dv = g[:, :d], g[:, d:2 * d], g[:, 2 * d:]
    else:
        qbuf, dq = _sentinel(B * Tq, d, dtype)
        gbuf, g = _sentinel(B * Tkv, 2 * d, dtype)
        dk, dv = g[:, :d], g[:, d:]
    K.attention_bwd(qs, ks, vs, o, do, lse, B, H, Tq, Tkv, causal=causal, kv_len=lens, dq=dq, dk=dk, dv=dv)
    torch.cuda.synchronize()
    for key, t in (("o", o), ("lse", lse), ("dq", dq), ("dk", dk), ("dv", dv)):
        assert torch.equal(t, want[key]), key
    assert _outside_unchanged(obuf, B * Tq, d)
    assert _outside_unchanged(gbuf, B * Tq if causal else B * Tkv, 3 * d if causal else 2 * d)
    if not causal:
        assert _outside_unchanged(qbuf, B * Tq, d)


# ---------------------------------------------------------------------------------------------------- isolation
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("use", ["decoder", "cross"])
def test_hidden_keys_do_not_affect_results(use, dtype):
    """K / V rows past kv_len filled with 1e4 instead of zeros: O, lse, dQ and the valid keys' dK / dV keep their bits;
    hidden keys' dK / dV are exactly zero."""
    B, H = 3, 2
    causal = use == "decoder"
    Tq, Tkv = (448, 448) if causal else (200, 1500)
    lens = _lens([448, 63, 129] if causal else [1500, 700, 129])
    q, k, v, do = _inputs(B, H, Tq, Tkv, dtype, seed=9)
    valid = _valid_keys(B, Tkv, lens)
    k0, v0, k1, v1 = k.clone(), v.clone(), k.clone(), v.clone()
    for t, fill in ((k0, 0.0), (v0, 0.0), (k1, 1e4), (v1, -1e4)):
        t[~valid] = fill
    a = _kernels(q, k0, v0, do, B, H, Tq, Tkv, causal, lens)
    b = _kernels(q, k1, v1, do, B, H, Tq, Tkv, causal, lens)
    for key in ("o", "lse", "dq"):
        assert torch.equal(a[key], b[key]), key
    for key in ("dk", "dv"):
        assert torch.equal(a[key][valid], b[key][valid]), key
        assert not a[key][~valid].any() and not b[key][~valid].any(), key


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("use", ["decoder", "cross"])
def test_sample_alone_equals_sample_in_batch(use, dtype):
    B, H = 5, 2
    causal = use == "decoder"
    Tq, Tkv = (300, 300) if causal else (200, 700)
    lens = [300, 77, 129, 255, 1] if causal else None
    q, k, v, do = _inputs(B, H, Tq, Tkv, dtype, seed=10)
    full = _kernels(q, k, v, do, B, H, Tq, Tkv, causal, _lens(lens))
    i = 2
    qi, doi = (t[i * Tq:(i + 1) * Tq].clone() for t in (q, do))
    ki, vi = (t[i * Tkv:(i + 1) * Tkv].clone() for t in (k, v))
    one = _kernels(qi, ki, vi, doi, 1, H, Tq, Tkv, causal, _lens(lens[i:i + 1]) if lens else None)
    for key, n in (("o", Tq), ("dq", Tq), ("dk", Tkv), ("dv", Tkv)):
        assert torch.equal(one[key], full[key][i * n:(i + 1) * n]), key
    assert torch.equal(one["lse"][0], full["lse"][i])


def test_repeated_fp16_calls_are_bit_identical():
    B, H, T = 3, 4, 448
    q, k, v, do = _inputs(B, H, T, T, torch.float16, seed=11)
    lens = _lens([448, 200, 65])
    a = _kernels(q, k, v, do, B, H, T, T, True, lens)
    for _ in range(2):
        b = _kernels(q, k, v, do, B, H, T, T, True, lens)
        for key in a:
            assert torch.equal(a[key], b[key]), key


# ---------------------------------------------------------------------------------------------------- validation
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_backward_rejects_misaligned_o(dtype):
    """O is read with 16-byte loads: a view 8 bytes off a 16-byte boundary is refused before any launch."""
    from olmoasr_b200 import kernels as K
    from olmoasr_b200._lib import OasrError

    B, H, T = 1, 2, 128
    d = H * HD
    q, k, v, do = _inputs(B, H, T, T, dtype, seed=12)
    o, lse = K.attention_fwd(q, k, v, B, H, T, T)
    buf = torch.zeros(B * T, d + 8, device="cuda", dtype=dtype)
    o8 = buf[:, 4:4 + d]
    o8.copy_(o)
    assert o8.data_ptr() % 16 == 8 and o8.stride(0) % 8 == 0
    with pytest.raises(OasrError, match="16-byte aligned"):
        K.attention_bwd(q, k, v, o8, do, lse, B, H, T, T)


# ---------------------------------------------------------------------------------------------------- decode
def _dec_call(q, k, v, seq_stride, row_stride, n, H, splits, dtype, pos=None, n_keys=0, kv_group=1):
    from olmoasr_b200._lib import DTYPE_BF16, DTYPE_F16, DecAttnArgs, call, ptr, stream

    d = H * HD
    scores = torch.full((n, H, 1536), float("nan"), device="cuda")
    part = torch.full((splits, n, d), float("nan"), device="cuda")
    a = DecAttnArgs()
    a.q, a.ldq = ptr(q), q.stride(0)
    a.k, a.v, a.kv_seq_stride, a.kv_row_stride = ptr(k), ptr(v), seq_stride, row_stride
    a.scores, a.scores_ld = ptr(scores), scores.stride(1)
    a.out_partial, a.ld_out = ptr(part), d
    a.pos_ptr, a.n_keys = ptr(pos), n_keys
    a.n_seq, a.n_head, a.n_splits, a.scale = n, H, splits, 64 ** -0.25
    a.dtype = DTYPE_F16 if dtype == torch.float16 else DTYPE_BF16
    if kv_group == 1:
        call("oasr_dec_attention", ctypes.byref(a), stream())
    else:
        call("oasr_dec_attention_grouped", ctypes.byref(a), kv_group, stream())
    torch.cuda.synchronize()
    out = part[0].clone()
    for s in range(1, splits):     # the consumer adds the fp32 partials in split order
        out += part[s]
    return scores, out


def _check_scores(got, ref, dtype, what):
    """Kernel scores against the fp64 statement's: at most 1% of them (or 2) differ at all, each by at most one T ulp
    -- its fp32 sum and the exact one fall on either side of a rounding boundary -- plus the fp32 sum's own error
    (64 x 2^-24 of sum |terms|), which only matters where the terms cancel to near zero."""
    ref, mag = ref
    got = got.double()
    diff = (got - ref).abs()
    bound = ulp(torch.maximum(got.abs(), ref.abs()), dtype) + 2.0 ** -18 * mag
    assert bool((diff <= bound).all()), f"{what}: worst score error {float((diff / bound).max()):.3g} x the bound"
    n_off = int((diff > 0).sum())
    assert n_off <= max(2, 0.01 * diff.numel()), f"{what}: {n_off} of {diff.numel()} scores differ"


def _check_out(got, ref, dtype, what):
    """Per (n, h) relative L2 error of the attention output against the reference from the same scores."""
    u = ar.U[dtype]
    g = got.double().view(ref.shape)
    err = (g - ref).norm(dim=-1) / ref.norm(dim=-1).clamp_min(1e-30)
    assert float(err.max()) <= u, f"{what}: worst (n, h) error {float(err.max()):.3g} > u"
    assert float(err.mean()) <= u / 32, f"{what}: mean (n, h) error {float(err.mean()):.3g} > u/32"


SELF_KEYS = [1, 2, 16, 17, 128, 129, 256, 447, 448]


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("H", [6, 16, 20])
def test_decode_self_attention(H, dtype):
    """Self-attention over the engine's (n, 448, d) caches with the key count read from the device position.  The
    fused kernel (one split) hides its scores; the two-kernel form computes them with the same arithmetic, so its
    scores (checked against fp64) serve as the fused kernel's too."""
    d, cache = H * HD, 448
    for n in (1, 5, 64):
        for std in (1.0, 12.0):
            g = torch.Generator(device="cuda").manual_seed(100 * n + H)
            a = std ** 0.5                # q, k ~ N(0, std): (q hd^-1/4) . (k hd^-1/4) ~ N(0, std^2)
            q = (torch.randn(n, d, device="cuda", generator=g) * a).to(dtype)
            kc = (torch.randn(n, cache, d, device="cuda", generator=g) * a).to(dtype)
            vc = torch.randn(n, cache, d, device="cuda", generator=g).to(dtype)
            for keys in SELF_KEYS:
                what = f"n={n} std={std} keys={keys}"
                pos = torch.tensor([keys - 1], device="cuda", dtype=torch.int32)
                args = (q, kc, vc, cache * d, d, n, H)
                sc2, out2 = _dec_call(*args, 2, dtype, pos=pos)
                _, out1 = _dec_call(*args, 1, dtype, pos=pos)
                kh = kc[:, :keys].view(n, keys, H, HD)
                vh = vc[:, :keys].view(n, keys, H, HD)
                _check_scores(sc2[:, :, :keys], dec_scores_ref(q.view(n, H, HD), kh, dtype, 64 ** -0.25), dtype, what)
                ref = dec_out_ref(sc2[:, :, :keys], vh, dtype)
                _check_out(out2, ref, dtype, what + " split")
                _check_out(out1, ref, dtype, what + " fused")


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("kv_group", [1, 5])
def test_decode_cross_attention(kv_group, dtype):
    """Cross-attention over the (n * 1500, 2d) K | V layout, split into 1, 2, 3, 7 or 8 key ranges; with kv_group 5
    sequence r reads entry r // 5."""
    H, T, n_kv = 20, 1500, 2
    d, n = H * HD, n_kv * kv_group
    for std in (1.0, 12.0):
        g = torch.Generator(device="cuda").manual_seed(7 + kv_group)
        a = std ** 0.5
        q = (torch.randn(n, d, device="cuda", generator=g) * a).to(dtype)
        kv = torch.randn(n_kv, T, 2 * d, device="cuda", generator=g)
        kv[..., :d] *= a
        kv = kv.to(dtype)
        kh = kv[..., :d].reshape(n_kv, T, H, HD).repeat_interleave(kv_group, dim=0)
        vh = kv[..., d:].reshape(n_kv, T, H, HD).repeat_interleave(kv_group, dim=0)
        sref = dec_scores_ref(q.view(n, H, HD), kh, dtype, 64 ** -0.25)
        args = (q, kv, kv[..., d:], T * 2 * d, 2 * d, n, H)
        sc2, _ = _dec_call(*args, 2, dtype, n_keys=T, kv_group=kv_group)
        for splits in (1, 2, 3, 7, 8):
            what = f"std={std} splits={splits}"
            sc, out = _dec_call(*args, splits, dtype, n_keys=T, kv_group=kv_group)
            if splits > 1:
                _check_scores(sc[:, :, :T], sref, dtype, what)
                assert torch.equal(sc[:, :, :T], sc2[:, :, :T]), what   # split count does not change a score
            _check_out(out, dec_out_ref(sc2[:, :, :T], vh, dtype), dtype, what)
