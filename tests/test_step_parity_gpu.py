"""The training step's memory-bound kernels and the fused AdamW against the fp64 statements of tests/step_reference.py,
at every launch form the step makes, in bf16 and fp16, at the widths of config/model_dims.py (d = 384 .. 1280):

- the conv stem's glue at mel (B, 80, 3000) (B = 32 for the B x 3000-row col2im and conv1 column sum), a short T = 37
  (the im2col tail block, the last odd frame), add_pos over B x 1500 rows and fp16 sums that overflow;
- the decoder embedding over B x 448 rows with a hot id in more than 128 rows, padding and out-of-range ids, a
  positional offset, frozen tables, accumulation into a non-zero slab and packed batches (a zero-length sample, N < S);
- the bias column sums at every (M, N, ld, column offset) the step passes and on the scalar path;
- the optimizer over flat slabs (tiny's numel and 5 x 10^7 elements) and the pointer table (odd sizes, views off
  16-byte alignment), with the amp form, skipped steps, fp16 shadows and the bias corrections at t = 1, 2, 300, 10^6.

Every buffer a kernel writes carries guard cells that must keep their sentinel.
"""
import math

import pytest
import torch

from tests import step_reference as sr
from tests import training_reference as tr

pytestmark = pytest.mark.gpu

DTYPES = [torch.bfloat16, torch.float16]
DT_ID = {torch.bfloat16: "bf16", torch.float16: "fp16"}
WIDTHS = [384, 512, 768, 1024, 1280]
V, PAD, S_TEXT = 51865, 51864, 448
SENTINEL = 7.0
HYPER = dict(lr=1.5e-3, beta1=0.9, beta2=0.98, eps=1e-6, wd=0.1)


@pytest.fixture(scope="module")
def K():
    from olmoasr_b200 import kernels
    return kernels


@pytest.fixture(scope="module")
def n_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _dev_gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _rand(shape, g, scale=1.0, dtype=torch.float32):
    return (torch.randn(shape, device="cuda", generator=g) * scale).to(dtype)


def _wide(shape, g, dtype):
    """Values over 2^-10 .. 2^10: fp32 sums of a few 16-bit values are exact, a wide range makes them round."""
    e = torch.randint(-10, 11, shape, device="cuda", generator=g).float()
    return (torch.randn(shape, device="cuda", generator=g) * torch.exp2(e)).to(dtype)


def _guarded(n, dtype=torch.float32, pad=64):
    """(buffer, view): n elements at the buffer's start (16-byte aligned), followed by `pad` sentinel cells."""
    buf = torch.full((n + pad,), SENTINEL, device="cuda", dtype=dtype)
    return buf, buf[:n]


def _check_rounded(got, ref, emu, dtype, name, exact=True):
    """check16, and (for the fp32-add kernels) the kernel equals the fp32 restatement bit for bit."""
    tr.check16(tr.errors16(got, ref, emu, dtype), dtype, name=name)
    if exact:
        e = emu["out"].to(dtype)
        assert torch.equal(got.view(torch.int16), e.view(torch.int16)), f"{name}: not the fp32 restatement's bits"


# ================================================================================================ conv stem
def _stem(K, B, T, d, dtype, g, kpad=240, overflow=False):
    C = 80
    T2 = sr.conv2_out_len(T)
    mel = _rand((B, C, T), g, 2.0)
    A1 = K.im2col_conv1(mel, kpad, dtype)
    assert torch.equal(A1, sr.im2col_conv1(mel, kpad, dtype)), "im2col_conv1"
    w1 = _rand((d, C, 3), g)
    assert torch.equal(K.cast_conv_weight(w1, dtype=dtype), sr.cast_conv_weight(w1, dtype)), "cast_conv_weight"
    h1 = _rand((B * T, d), g, 1.0, dtype)
    assert torch.equal(K.im2col_conv2(h1, B, T, d), sr.im2col_conv2(h1, B, T, d)), "im2col_conv2"
    # add_pos over B x T2 rows
    x = _rand((B * T2, d), g, 2.0, dtype)
    pos = _rand((T2, d), g)
    if overflow:
        x[::3] = 60000.0 * torch.sign(x[::3].float()).to(dtype)
        pos[::2] = 10000.0 * torch.sign(pos[::2])
    got = K.add_pos(x, pos, T2)
    _check_rounded(got, sr.add_pos(x, pos, T2, dtype), sr.add_pos(x, pos, T2, dtype, work=torch.float32), dtype,
                   f"add_pos d={d} B={B}")
    if overflow:
        assert bool(torch.isinf(got).any())
    # gelu_bwd (conv2's GELU backward) and col2im + conv1's GELU backward
    dy = _rand((B * T2, d), g, 1.0, dtype)
    pre = _rand((B * T2, d), g, 2.0, dtype)
    dA = _rand((B * T2, 3 * d), g, 1.0, dtype)
    pre1 = _rand((B * T, d), g, 2.0, dtype)
    if overflow:
        dy[::5], pre[::5] = 65000.0, 2.0                             # 65000 gelu'(2) = 70 500: inf
        taps = dA.view(B * T2, 3, d)
        taps[:, 0, :8] = taps[:, 2, :8] = 40000.0                    # an odd row's two taps sum past 65 504
        pre1[:, :8] = 1.5
    got = K.gelu_bwd(dy, pre)
    tr.check16(tr.errors16(got, sr.gelu_bwd(dy, pre, dtype), sr.gelu_bwd(dy, pre, dtype, work=torch.float32), dtype),
               dtype, name=f"gelu_bwd d={d} B={B}")
    got = K.col2im_conv2_gelu_bwd(dA, pre1, B, T, T2, d)
    ref = sr.col2im_conv2_gelu_bwd(dA, pre1, B, T, T2, d, dtype)
    emu = sr.col2im_conv2_gelu_bwd(dA, pre1, B, T, T2, d, dtype, work=torch.float32)
    tr.check16(tr.errors16(got, ref, emu, dtype), dtype, name=f"col2im d={d} B={B} T={T}")
    if overflow:
        assert bool(torch.isinf(got).any())
    del ref, emu
    # conv weight gradients, fresh and accumulated into a slab view
    gw = _rand((d, 3 * C), g)
    assert torch.equal(K.unpermute_conv_wgrad(gw, d, C), sr.unpermute_conv_wgrad(gw, d, C)), "unpermute fresh"
    buf, out = _guarded(d * C * 3)
    out.copy_(_rand(d * C * 3, g))
    want = sr.unpermute_conv_wgrad(gw, d, C, out=out.view(d, C, 3))
    K.unpermute_conv_wgrad(gw, d, C, out=out.view(d, C, 3))
    assert torch.equal(out.view(d, C, 3), want) and bool((buf[out.numel():] == SENTINEL).all()), "unpermute accumulate"


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("d", WIDTHS)
def test_stem_forms(K, d, dtype):
    """mel (2, 80, 3000): im2col, the weight casts, add_pos over 2 x 1500 rows, gelu_bwd, col2im and the wgrad permutes."""
    _stem(K, 2, 3000, d, dtype, _dev_gen(d))


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_stem_short_odd_t(K, dtype):
    """T = 37: im2col_conv1's tail block of 5 frames, conv2's last output reading frame 37 (zero), padded Kpad."""
    _stem(K, 3, 37, 384, dtype, _dev_gen(37), kpad=248)


def test_stem_fp16_overflow(K):
    """fp16 sums past 65504: add_pos, gelu_bwd and col2im's tap sum give the infinities .to(half) gives."""
    _stem(K, 2, 3000, 512, torch.float16, _dev_gen(65), overflow=True)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_stem_full_batch(K, n_sms, dtype):
    """B = 32 at d = 1024: col2im over 96 000 rows, add_pos over 48 000 and conv1's bias column sum over 96 000."""
    B, T, d = 32, 3000, 1024
    g = _dev_gen(32)
    dA = _rand((B * 1500, 3 * d), g, 1.0, dtype)
    pre1 = _rand((B * T, d), g, 2.0, dtype)
    got = K.col2im_conv2_gelu_bwd(dA, pre1, B, T, 1500, d)
    parts = []
    for s in tr.rows_in_slabs(B, 8):                                 # 8 samples at a time: fp64 copies stay small
        rs, rt = slice(s.start * T, s.stop * T), slice(s.start * 1500, s.stop * 1500)
        nb = s.stop - s.start
        ref = sr.col2im_conv2_gelu_bwd(dA[rt], pre1[rs], nb, T, 1500, d, dtype)
        emu = sr.col2im_conv2_gelu_bwd(dA[rt], pre1[rs], nb, T, 1500, d, dtype, work=torch.float32)
        parts.append(tr.errors16(got[rs], ref, emu, dtype))
        del ref, emu
    tr.check16(parts, dtype, name="col2im B=32")
    x = _rand((B * 1500, d), g, 2.0, dtype)
    pos = _rand((1500, d), g)
    _check_rounded(K.add_pos(x, pos, 1500), sr.add_pos(x, pos, 1500, dtype), sr.add_pos(x, pos, 1500, dtype, work=torch.float32),
                   dtype, "add_pos B=32")
    _colsum_case(K, got, d, dtype, "conv1 bias B=32", n_sms)


def test_cast_bf16_is_the_torch_cast(K):
    """The fp32 -> bf16 weight cast, whole 8-element groups and a tail."""
    x = _rand(1000 * 1024 + 5, _dev_gen(3), 3.0)
    assert torch.equal(K.cast_bf16(x).view(torch.int16), x.bfloat16().view(torch.int16))


# ================================================================================================ embedding
def _ids(B, S, g, hot=True):
    ids = torch.randint(0, V, (B, S), device="cuda", generator=g)
    if hot:
        ids.view(-1)[130::max(1, B * S // 300)] = 7                  # > 128 rows, the first after row 128
    ids[0, S - 20:] = PAD
    ids[-1, 3], ids[-1, 4] = V, -1                                  # outside [0, V): read row 0, no gradient
    return ids


def _check_embed_bwd(got_e, got_p, ids, dx, demb0, dpos0, name, rows=None):
    if rows is None:
        ref = sr.embed_bwd(ids, dx, demb0, dpos0, PAD)
        emu = sr.embed_bwd(ids, dx, demb0, dpos0, PAD, work=torch.float32)
    else:
        ref = sr.embed_bwd_packed(ids, dx, demb0, dpos0, PAD, rows)
        emu = sr.embed_bwd_packed(ids, dx, demb0, dpos0, PAD, rows, work=torch.float32)
    for got, k in ((got_e, "demb"), (got_p, "dpos")):
        if emu[k] is None:
            continue
        assert torch.equal(got, emu[k]), f"{name} {k}: not the kernel-order fp32 sum ({int((got != emu[k]).sum())} elements)"
        tr.check32(tr.errors32(got, ref[k], emu[k], ref["allow_" + k]), name=f"{name} {k}")
    return emu


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("d", WIDTHS)
def test_embedding_forms(K, d, dtype):
    """16 x 448 dense rows: forward bit for bit against the fp32 restatement and within the fp64 rule; backward into a
    non-zero token table (the tied logits' wgrad has already written) and a zero positional table."""
    g = _dev_gen(400 + d)
    B, S = 16, S_TEXT
    ids = _ids(B, S, g)
    emb, pos = _rand((V, d), g, 0.5), _rand((S_TEXT, d), g, 0.5)
    out = K.embed_fwd(ids, emb, pos, 0, dtype=dtype)
    _check_rounded(out, sr.embed_fwd(ids, emb, pos, 0, dtype), sr.embed_fwd(ids, emb, pos, 0, dtype, work=torch.float32),
                   dtype, f"embed_fwd d={d}")
    dx = _wide((B * S, d), g, dtype)
    ebuf = torch.full((V + 2, d), SENTINEL, device="cuda")
    demb = ebuf[1:V + 1]
    demb.copy_(_rand((V, d), g))
    demb0 = demb.clone()
    dpos = torch.zeros(S_TEXT, d, device="cuda")
    K.embed_bwd(ids, dx, demb, dpos, PAD)
    assert bool((ebuf[0] == SENTINEL).all() and (ebuf[-1] == SENTINEL).all()), "embed_bwd wrote outside the table"
    assert torch.equal(demb[PAD], demb0[PAD]), "the padding row moved"
    _check_embed_bwd(demb, dpos, ids, dx, demb0, torch.zeros_like(dpos), f"embed_bwd d={d}")
    # frozen tables: a null target skips its sum and leaves the other's bits unchanged
    e2, p2 = demb0.clone(), torch.zeros_like(dpos)
    K.embed_bwd(ids, dx, e2, None, PAD)
    K.embed_bwd(ids, dx, None, p2, PAD)
    assert torch.equal(e2, demb) and torch.equal(p2, dpos)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_embedding_position_offset(K, dtype):
    """pos_offset = 37, S = 200: the forward reads pos[s + 37]; the backward writes dpos[37:237] through a view and
    leaves every other positional row alone."""
    g = _dev_gen(41)
    B, S, off, d = 4, 200, 37, 768
    ids = _ids(B, S, g, hot=False)
    emb, pos = _rand((V, d), g, 0.5), _rand((S_TEXT, d), g, 0.5)
    out = K.embed_fwd(ids, emb, pos, off, dtype=dtype)
    _check_rounded(out, sr.embed_fwd(ids, emb, pos, off, dtype), sr.embed_fwd(ids, emb, pos, off, dtype, work=torch.float32),
                   dtype, "embed_fwd offset")
    dx = _wide((B * S, d), g, dtype)
    dpos = torch.full((S_TEXT, d), SENTINEL, device="cuda")
    dpos[off:off + S] = _rand((S, d), g)
    dpos0 = dpos[off:off + S].clone()
    demb = torch.zeros(V, d, device="cuda")
    K.embed_bwd(ids, dx, demb, dpos[off:], PAD)
    assert bool((dpos[:off] == SENTINEL).all() and (dpos[off + S:] == SENTINEL).all()), "dpos written outside [off, off + S)"
    _check_embed_bwd(demb, dpos[off:off + S], ids, dx, torch.zeros_like(demb), dpos0, "embed_bwd offset")


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("lens", [[448, 0, 131, 300, 1, 448, 77, 250], [3, 0, 5]], ids=["mixed", "N<S"])
def test_embedding_packed(K, lens, dtype):
    """Packed rows: the forward is the dense forward's rows; the backward equals the dense kernel run on the same rows
    with zeros in the padded rows, bit for bit, and the kernel-order restatement."""
    from olmoasr_b200._core import PackedBatch
    g = _dev_gen(sum(lens))
    B, S, d = len(lens), S_TEXT, 1024
    pk = PackedBatch(lens, S, "cuda")
    ids = _ids(B, S, g, hot=False)
    ids.view(-1)[pk.rows.long()[130::5]] = 7                         # a hot id among the packed rows
    emb, pos = _rand((V, d), g, 0.5), _rand((S, d), g, 0.5)
    dense = K.embed_fwd(ids, emb, pos, 0, dtype=dtype)
    assert torch.equal(K.embed_fwd_packed(ids, emb, pos, pk, dtype), dense[pk.rows.long()])
    dxp = _wide((pk.N, d), g, dtype)
    dxd = torch.zeros(B * S, d, device="cuda", dtype=dtype)
    dxd[pk.rows.long()] = dxp
    e0 = _rand((V, d), g)
    ep, pp = e0.clone(), torch.zeros(S, d, device="cuda")
    ed, pd = e0.clone(), torch.zeros(S, d, device="cuda")
    K.embed_bwd_packed(ids, dxp, ep, pp, pk, PAD)
    K.embed_bwd(ids, dxd, ed, pd, PAD)
    assert torch.equal(ep, ed) and torch.equal(pp, pd), "packed backward differs from the dense one"
    _check_embed_bwd(ep, pp, ids, dxp, e0, torch.zeros_like(pp), f"embed_bwd packed {lens}", rows=pk.rows)


# ================================================================================================ bias column sums
def _colsum_case(K, dy, N, dtype, name, n_sms):
    """db (in a guarded buffer, non-zero) += column sums of the (M, N) view dy: the fp64 rule, two runs' bits, the
    guard cells."""
    g = _dev_gen(N)
    buf = torch.full((N + 16,), SENTINEL, device="cuda")
    db = buf[8:8 + N]
    db.copy_(_rand(N, g))
    db0 = db.clone()
    K.colsum_(dy, db, N)
    first = db.clone()
    assert bool((buf[:8] == SENTINEL).all() and (buf[8 + N:] == SENTINEL).all()), f"{name}: wrote outside db"
    db.copy_(db0)
    K.colsum_(dy, db, N)
    assert torch.equal(db, first), f"{name}: two runs differ"
    ref = sr.colsum(dy, db0, n_sms=n_sms)
    emu = sr.colsum(dy, db0, work=torch.float32)
    tr.check32(tr.errors32(first, ref["out"], emu["out"], ref["allow"]), name=name)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("d", WIDTHS)
def test_colsum_forms(K, n_sms, d, dtype):
    """Every (M, N, ld, offset) of the step: the q and v members of the fused qkv gradient (ld 3d, offsets 0 and 2d),
    the cross k/v value member (ld 2d, offset d), the whole fused width (autograd mode), fc1 (4d), the conv biases
    (2 x 3000 and 2 x 1500 rows), decoder rows (16 x 448) and a packed M (2056)."""
    g = _dev_gen(700 + d)
    M = 3000
    qkv = _rand((M, 3 * d), g, 1.0, dtype)
    kv = _rand((M, 2 * d), g, 1.0, dtype)
    cases = [("q member", qkv[:, :d], d), ("v member", qkv[:, 2 * d:], d), ("cross v member", kv[:, d:], d),
             ("fused qkv", qkv, 3 * d), ("fc1", _rand((M, 4 * d), g, 0.3, dtype), 4 * d),
             ("conv1", _rand((6000, d), g, 0.3, dtype), d), ("conv2", _rand((3000, d), g, 0.3, dtype), d),
             ("decoder", _rand((16 * 448, d), g, 1.0, dtype), d), ("packed", _rand((2056, 3 * d), g, 1.0, dtype)[:, :d], d)]
    for name, dy, N in cases:
        _colsum_case(K, dy, N, dtype, f"colsum {name} d={d}", n_sms)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_colsum_scalar_path(K, n_sms, dtype):
    """N % 8 != 0 (the last tile's columns), ld % 8 != 0, and a view one or three elements off 16-byte alignment."""
    g = _dev_gen(9)
    base = _rand((3001, 1544), g, 1.0, dtype)
    for name, dy, N in (("N % 8 = 3", base[:, :523], 523), ("ld % 8 = 6 (ld 1158)", base.view(-1)[:3000 * 1158].view(3000, 1158)[:, :1024], 1024),
                        ("one element off", base[:, 1:385], 384), ("three elements off", base[1:, 3:1283], 1280)):
        _colsum_case(K, dy, N, dtype, f"colsum {name}", n_sms)


# ================================================================================================ optimizer
def _call(name, *args):
    from olmoasr_b200._lib import call, stream
    call(name, *args, stream())


def _ptr(t):
    return None if t is None else t.data_ptr()


def _flat_buffers(n, g, dtype, p_scale=0.02):
    bufs = {k: _guarded(n) for k in ("p", "g", "m", "v")}
    bufs["p"][1].copy_(_rand(n, g, p_scale))
    bufs["g"][1].copy_(_rand(n, g, 1e-3))
    bufs["m"][1].copy_(_rand(n, g, 1e-4))
    bufs["v"][1].copy_(_rand(n, g, 1e-4) ** 2)
    bufs["s"] = _guarded(n, dtype)
    return bufs


def _flat_step(bufs, n, dtype, t_before, max_norm=1.0, inv_scale=1.0, loss_scale=None, ext_found_inf=None):
    """oasr_grad_sqnorm_flat -> oasr_optim_prepare(_amp) -> oasr_adamw_flat16 with the device step counter at t_before.
    Returns (sqnorm, state) read back after the step."""
    from olmoasr_b200 import _lib
    nsq, fi = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda")
    st = torch.zeros(8, device="cuda")
    st[0] = t_before
    b1, b2 = HYPER["beta1"], HYPER["beta2"]
    P, G, M_, V_, S_ = (bufs[k][1] for k in ("p", "g", "m", "v", "s"))
    _call("oasr_grad_sqnorm_flat", _ptr(G), n, inv_scale, _ptr(nsq))
    if loss_scale is None and ext_found_inf is None:
        _call("oasr_optim_prepare", _ptr(nsq), _ptr(fi), _ptr(st), inv_scale, max_norm, b1, b2)
    else:
        ls = None if loss_scale is None else torch.tensor([loss_scale], device="cuda")
        ef = None if ext_found_inf is None else torch.tensor([ext_found_inf], device="cuda")
        _call("oasr_optim_prepare_amp", _ptr(nsq), _ptr(fi), _ptr(st), _ptr(ls), _ptr(ef), inv_scale, max_norm, b1, b2)
    _call("oasr_adamw_flat16", _ptr(P), _ptr(G), _ptr(M_), _ptr(V_), _ptr(S_), n, _ptr(st), HYPER["lr"], b1, b2, HYPER["eps"],
          HYPER["wd"], _lib.DTYPE_F16 if dtype == torch.float16 else _lib.DTYPE_BF16)
    torch.cuda.synchronize()
    return float(nsq), fi, st.cpu().tolist()


def _check_state(st_got, want, name):
    """The device state (step, coef, bc1, bc2s, skip, grad norm) against prepare()'s statement."""
    assert st_got[0] == want["step"] and st_got[4] == want["skip"], f"{name}: step / skip {st_got[:5]} vs {want}"
    sr.check_scalar(st_got[5], want["norm"], want["norm_rel"], f"{name} grad norm")
    if not want["skip"]:
        for i, k in ((1, "coef"), (2, "bc1"), (3, "bc2s")):
            sr.check_scalar(st_got[i], want[k], want[k + "_rel"], f"{name} {k}")


def _check_update(p0, g0, m0, v0, got, want_st, kernel_st, dtype, name, shadow=None):
    """p', m', v' (fp32) within adamw()'s allowance of the fp64 statement; the shadow T(p') bit for bit."""
    ref = sr.adamw(p0, g0, m0, v0, want_st, **HYPER)
    k32 = dict(zip(("coef", "bc1", "bc2s"), kernel_st[1:4]))
    emu = sr.adamw(p0, g0, m0, v0, k32, **HYPER, work=torch.float32)
    for k in ("p", "m", "v"):
        tr.check32(tr.errors32(got[k], ref[k], emu[k], ref["allow_" + k]), name=f"{name} {k}")
    del ref, emu
    if shadow is not None:
        assert torch.equal(shadow.view(torch.int16), got["p"].to(dtype).view(torch.int16)), f"{name}: shadow is not T(p')"


def _tiny_numel():
    import olmoasr_b200 as ob
    from olmoasr_b200.model import OLMoASR
    return sum(p.numel() for p in OLMoASR(ob.VARIANT_TO_DIMS["tiny"]).parameters())


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("t", [1, 2, 300, 10 ** 6])
def test_adamw_flat_tiny(t, dtype):
    """A slab of tiny's numel at step t (the device counter set to t - 1): the norm, the clip, the bias corrections,
    the update and the shadows; the guard cells after every slab."""
    n = _tiny_numel()
    g = _dev_gen(t)
    bufs = _flat_buffers(n, g, dtype)
    p0, g0, m0, v0 = (bufs[k][1].clone() for k in ("p", "g", "m", "v"))
    nsq, fi, st = _flat_step(bufs, n, dtype, t - 1, max_norm=1.0)
    sq = sr.grad_sqnorm([g0], 1.0)
    sr.check_scalar(nsq, sq["sqnorm"], sq["allow"] / sq["sqnorm"], "sqnorm tiny")
    want = sr.prepare(sq["sqnorm"], 1.0, 1.0, HYPER["beta1"], HYPER["beta2"], t - 1, sqnorm_allow=sq["allow"])
    assert want["coef"] < 1.0                                        # ||g|| = 1e-3 sqrt(numel) > 1: clipped
    _check_state(st, want, f"tiny t={t}")
    got = {k: bufs[k][1] for k in ("p", "m", "v")}
    _check_update(p0, g0, m0, v0, got, want, st, dtype, f"flat tiny t={t} {DT_ID[dtype]}", shadow=bufs["s"][1])
    for k, (buf, view) in bufs.items():
        assert bool((buf[n:] == SENTINEL).all()), f"guard after {k} written"
    assert float(fi) == 0.0


def test_adamw_flat_large_slab_fp16_shadows():
    """5 x 10^7 + 3 elements: 3052 partials for add_partials, a short last chunk (12 419, not a multiple of 4), fp16
    shadows of masters above 65504 are inf."""
    n = 5 * 10 ** 7 + 3
    dtype = torch.float16
    g = _dev_gen(50)
    bufs = _flat_buffers(n, g, dtype)
    bufs["p"][1][::1000003] = 70000.0
    bufs["p"][1][7::1000003] = -70000.0
    p0, g0, m0, v0 = (bufs[k][1].clone() for k in ("p", "g", "m", "v"))
    nsq, fi, st = _flat_step(bufs, n, dtype, 0, max_norm=1.0)
    sq = sr.grad_sqnorm([g0], 1.0)
    sr.check_scalar(nsq, sq["sqnorm"], sq["allow"] / sq["sqnorm"], "sqnorm 5e7")
    want = sr.prepare(sq["sqnorm"], 1.0, 1.0, HYPER["beta1"], HYPER["beta2"], 0, sqnorm_allow=sq["allow"])
    _check_state(st, want, "5e7")
    got = {k: bufs[k][1] for k in ("p", "m", "v")}
    _check_update(p0, g0, m0, v0, got, want, st, dtype, "flat 5e7 fp16", shadow=bufs["s"][1])
    assert bool(torch.isposinf(bufs["s"][1][::1000003].float()).all() and torch.isneginf(bufs["s"][1][7::1000003].float()).all())
    for k, (buf, view) in bufs.items():
        assert bool((buf[n:] == SENTINEL).all()), f"guard after {k} written"


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
def test_adamw_flat_amp_and_skips(dtype):
    """The amp form with a loss scale of 65536 and an external found_inf of 0 applies the step on g / S; an external
    found_inf of 1 with finite gradients, and a non-finite norm, skip it: no parameter, moment, shadow or counter moves.
    grad_norm() (st[5]) is ||g|| of the unscaled gradients on every path -- the skipped amp step included, which used to
    report ||g||^2."""
    n = 300007
    S = 65536.0
    g = _dev_gen(11)
    bufs = _flat_buffers(n, g, dtype)
    bufs["g"][1].mul_(S)
    p0, g0, m0, v0 = (bufs[k][1].clone() for k in ("p", "g", "m", "v"))
    bufs["s"][1].copy_(p0.to(dtype))
    sq = sr.grad_sqnorm([g0], 1.0)
    unscaled = math.sqrt(sq["sqnorm"]) / S
    # external found_inf set: skipped, the norm still ||g||
    _, fi, st = _flat_step(bufs, n, dtype, 5, loss_scale=S, ext_found_inf=1.0)
    want = sr.prepare(sq["sqnorm"], 1.0, 1.0, HYPER["beta1"], HYPER["beta2"], 5, loss_scale=S, found_inf=True, sqnorm_allow=sq["allow"])
    assert abs(want["norm"] - unscaled) <= 1e-12 * unscaled
    _check_state(st, want, "amp found_inf")
    assert float(fi) == 1.0
    for k, t0 in (("p", p0), ("g", g0), ("m", m0), ("v", v0)):
        assert torch.equal(bufs[k][1], t0), f"skipped step moved {k}"
    assert torch.equal(bufs["s"][1], p0.to(dtype))
    # external found_inf clear: applied on g / S
    _, fi, st = _flat_step(bufs, n, dtype, 5, loss_scale=S, ext_found_inf=0.0)
    want = sr.prepare(sq["sqnorm"], 1.0, 1.0, HYPER["beta1"], HYPER["beta2"], 5, loss_scale=S, sqnorm_allow=sq["allow"])
    _check_state(st, want, "amp")
    got = {k: bufs[k][1] for k in ("p", "m", "v")}
    _check_update(p0, g0, m0, v0, got, want, st, dtype, f"amp {DT_ID[dtype]}", shadow=bufs["s"][1])
    # a non-finite gradient: skipped, found_inf raised, grad_norm() inf
    p1, m1, v1, s1 = (bufs[k][1].clone() for k in ("p", "m", "v", "s"))
    bufs["g"][1][12345] = float("inf")
    _, fi, st = _flat_step(bufs, n, dtype, 6)
    assert float(fi) == 1.0 and st[0] == 6 and st[4] == 1.0 and st[5] == float("inf")
    for k, t0 in (("p", p1), ("m", m1), ("v", v1), ("s", s1)):
        assert torch.equal(bufs[k][1], t0), f"skipped step moved {k}"


def _table_params(g, sizes, offsets):
    """Parameters (and gradients, moments) as views `offset` elements into guarded buffers: odd sizes, and offsets
    that are not multiples of 4 put chunks on the scalar path."""
    out = []
    for n, off in zip(sizes, offsets):
        views = {}
        for k, scale in (("p", 0.02), ("g", 1e-3), ("m", 1e-4), ("v", 1e-4)):
            buf = torch.full((n + off + 64,), SENTINEL, device="cuda")
            v = buf[off:off + n]
            v.copy_(_rand(n, g, scale) ** (2 if k == "v" else 1))
            views[k] = (buf, v, off)
        out.append(views)
    return out


@pytest.mark.parametrize("amp", [False, True], ids=["plain", "amp"])
def test_adamw_pointer_table(amp):
    """FusedAdamW's pointer-table path (oasr_grad_sqnorm + optim_prepare(_amp) + oasr_adamw_step) over odd-sized tensors
    and views off 16-byte alignment, from step 299 (resumed): every tensor's update, the norm and the guards; then the
    amp form's skip with a finite norm, whose grad_norm() is ||g||."""
    from olmoasr_b200.optim import FusedAdamW
    g = _dev_gen(12 + amp)
    sizes = [1024 * 384, 384, 51865 * 8 + 1, 7, 45, 100003, 16384 * 3 + 5]
    offsets = [0, 1, 2, 3, 0, 5, 6]
    S = 1024.0 if amp else None
    views = _table_params(g, sizes, offsets)
    params = []
    for vw in views:
        p = vw["p"][1].requires_grad_(True)
        if amp:
            vw["g"][1].mul_(S)
        p.grad = vw["g"][1]
        params.append(p)
    opt = FusedAdamW(params, lr=HYPER["lr"], betas=(HYPER["beta1"], HYPER["beta2"]), eps=HYPER["eps"],
                     weight_decay=HYPER["wd"], max_grad_norm=1.0)
    for p, vw in zip(params, views):
        opt.state[p] = {"step": torch.tensor(299.0), "exp_avg": vw["m"][1], "exp_avg_sq": vw["v"][1]}
    before = [{k: vw[k][1].detach().clone() for k in ("p", "m", "v")} for vw in views]
    grads = [p.grad.detach().clone() for p in params]
    if amp:
        opt.grad_scale = torch.tensor(S, device="cuda")
        opt.found_inf = torch.tensor(0.0, device="cuda")
    opt.step()
    torch.cuda.synchronize()
    sq = sr.grad_sqnorm(grads, 1.0)
    want = sr.prepare(sq["sqnorm"], 1.0, 1.0, HYPER["beta1"], HYPER["beta2"], 299, loss_scale=S, sqnorm_allow=sq["allow"])
    st = opt._dev_state.cpu().tolist()
    _check_state(st, want, f"table amp={amp}")
    sr.check_scalar(float(opt.grad_norm()), want["norm"], want["norm_rel"], "table grad_norm()")
    for i, (vw, b0, gr) in enumerate(zip(views, before, grads)):
        got = {k: vw[k][1].detach() for k in ("p", "m", "v")}
        _check_update(b0["p"], gr, b0["m"], b0["v"], got, want, st, None, f"table tensor {i} amp={amp}")
        for k in ("p", "g", "m", "v"):
            buf, v, off = vw[k]
            assert bool((buf[:off] == SENTINEL).all() and (buf[off + v.numel():] == SENTINEL).all()), f"tensor {i}: guard of {k}"
    if amp:     # GradScaler's flag set with finite gradients: nothing moves, grad_norm() is still ||g||
        after = [{k: vw[k][1].detach().clone() for k in ("p", "m", "v")} for vw in views]
        opt.found_inf = torch.tensor(1.0, device="cuda")
        opt.step()
        torch.cuda.synchronize()
        skip = sr.prepare(sq["sqnorm"], 1.0, 1.0, HYPER["beta1"], HYPER["beta2"], 300, loss_scale=S, found_inf=True,
                          sqnorm_allow=sq["allow"])
        _check_state(opt._dev_state.cpu().tolist(), skip, "table amp skip")
        assert opt.applied_steps() == 300
        for vw, a in zip(views, after):
            assert all(torch.equal(vw[k][1], a[k]) for k in ("p", "m", "v")), "a skipped step moved a tensor"


# ================================================================================================ alignment checks
def test_misaligned_views_are_refused(K):
    """The vectorised kernels' wrappers refuse views that start inside a 16-byte word with ValueError, and the C entry
    points refuse them too (OasrError), before any launch."""
    from olmoasr_b200._lib import OasrError
    dt = torch.bfloat16
    g = _dev_gen(13)
    flat = _rand(3000 * 384 + 8, g, 1.0, dt)
    off = flat[1:1 + 3000 * 384].view(3000, 384)                     # 2 bytes past an aligned start
    ok = flat[:3000 * 384].view(3000, 384)
    pos = _rand((1500, 384), g)
    posf = _rand(1500 * 384 + 4, g)
    pos_off = posf[1:1 + 1500 * 384].view(1500, 384)
    with pytest.raises(ValueError):
        K.add_pos(off, pos, 1500)
    with pytest.raises(ValueError):
        K.add_pos(ok, pos_off, 1500)
    with pytest.raises(ValueError):
        K.gelu_bwd(off, ok)
    with pytest.raises(ValueError):
        K.gelu_bwd(ok, off)
    with pytest.raises(ValueError):
        K.im2col_conv2(off, 2, 1500, 384)
    emb = _rand((1000, 384), g)
    embf = _rand(1000 * 384 + 4, g)
    ids = torch.randint(0, 1000, (2, 16), device="cuda", generator=g)
    with pytest.raises(ValueError):
        K.embed_fwd(ids, embf[2:2 + 1000 * 384].view(1000, 384), pos, 0)
    with pytest.raises(ValueError):
        K.embed_fwd(ids, emb, pos_off, 0)
    from olmoasr_b200._lib import call, stream
    out = torch.empty_like(ok)
    with pytest.raises(OasrError):
        call("oasr_add_pos16", off.data_ptr(), pos.data_ptr(), out.data_ptr(), 3000, 1500, 384, 0, stream())
    with pytest.raises(OasrError):
        call("oasr_gelu_bwd16", ok.data_ptr(), off.data_ptr(), out.data_ptr(), 3000 * 384, 0, stream())
    with pytest.raises(OasrError):
        call("oasr_im2col_conv2", off.data_ptr(), out.data_ptr(), 2, 1500, 750, 384, stream())
    with pytest.raises(OasrError):
        call("oasr_embed_fwd16", ids.data_ptr(), emb.data_ptr(), pos.data_ptr(), off.data_ptr() + 4, 2, 16, 384, 0, 1000, 0, stream())
    torch.cuda.synchronize()
