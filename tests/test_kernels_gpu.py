"""Per-kernel parity on the GPU: every C-ABI entry point against a plain torch fp32 statement of the same
reference op (and the numpy oracle for the log-mel).  Tolerances are bf16 output rounding (2^-8 relative)
unless a comment says otherwise."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def K():
    from olmoasr_b200 import kernels
    return kernels


def _close(got, want, rtol=1.0 / 128, atol=None):
    scale = want.abs().max().item() + 1e-12
    atol = atol if atol is not None else rtol * scale
    err = (got.float() - want.float()).abs().max().item()
    assert err <= atol, f"max err {err} > {atol} (scale {scale})"


# ------------------------------------------------------------------------------------------------ GEMM
@pytest.mark.parametrize("M,N,Kd,bn", [(128, 64, 64, 64), (256, 256, 512, 256), (1000, 200, 240, 128), (300, 1865, 128, 256)])
@pytest.mark.parametrize("a_mn,b_mn", [(0, 0), (0, 1), (1, 1)])
def test_gemm_layouts(K, M, N, Kd, bn, a_mn, b_mn):
    torch.manual_seed(0)
    A = torch.randn(M, Kd, device="cuda").bfloat16()
    B = torch.randn(N, Kd, device="cuda").bfloat16()
    a = A.t().contiguous() if a_mn else A
    b = B.t().contiguous() if b_mn else B
    if (a_mn and M % 8) or (b_mn and N % 8):
        pytest.skip("MN-major operands need a 16-byte aligned row stride")
    out = K.gemm(a, b, M, N, Kd, a_mn=bool(a_mn), b_mn=bool(b_mn), epi=K.EPI_F32, block_n=bn)
    _close(out, A.float() @ B.float().t(), rtol=1e-4)


# Production shapes of the headline benchmark (medium model).  The unit shapes above never make a persistent CTA process a
# second tile: these do (many tiles per CTA), which exercises the stage ring wrapping across tiles, the epilogue of one
# tile overlapping the loads of the next, M-fastest rasterisation and split-K.
def _rel_l2(got, want):
    return float((got.float() - want.float()).norm() / want.float().norm())


def test_gemm_production_fc1_gelu_and_gelu_bwd(K):
    torch.manual_seed(11)
    M, N, Kd = 48000, 4096, 1024            # encoder fc1: 375 x 32 = 12000 tiles of 128 x 128
    A = torch.randn(M, Kd, device="cuda").bfloat16()
    B = (torch.randn(N, Kd, device="cuda") / math.sqrt(Kd)).bfloat16()
    bias = torch.randn(N, device="cuda")
    ref = A.float() @ B.float().t()
    rb = (ref + bias.bfloat16().float()).bfloat16().float()
    h, g = K.gemm(A, B, M, N, Kd, bias=bias, epi=K.EPI_BF16_GELU, block_n=256)
    assert _rel_l2(h, rb) < 3e-3 and (h.float() - rb).abs().max().item() <= 2.0 ** -6 * rb.abs().max().item()
    assert _rel_l2(g, F.gelu(h.float())) < 4e-3
    del ref, rb, g
    # fc2 dgrad with the GELU-backward epilogue: dh = bf16(bf16(dy W2) * gelu'(h)),  (48000 x 1024) @ (1024 x 4096)
    dy = torch.randn(M, Kd, device="cuda").bfloat16()
    W2 = (torch.randn(Kd, N, device="cuda") / math.sqrt(Kd)).bfloat16()      # stored (N_out=1024, K_in=4096): read MN-major
    got = K.gemm(dy, W2, M, N, Kd, b_mn=True, aux=h, epi=K.EPI_BF16_GELU_BWD, block_n=256)
    x = h.float().requires_grad_(True)
    F.gelu(x).backward((dy.float() @ W2.float()).bfloat16().float())
    assert _rel_l2(got, x.grad) < 4e-3


def test_gemm_production_tied_logits_raster_m(K):
    torch.manual_seed(12)
    M, V, d = 14336, 51865, 1024            # decoder logits: B (the embedding) is the larger operand -> M-fastest raster
    x = torch.randn(M, d, device="cuda").bfloat16()
    E = (torch.randn(V, d, device="cuda") / math.sqrt(d)).bfloat16()
    ld = (V + 255) // 256 * 256
    buf = torch.full((M, ld), 7.0, device="cuda", dtype=torch.bfloat16)
    K.gemm(x, E, M, V, d, out=buf, block_n=256)
    for r0 in (0, 4096, 14336 - 1024):      # compare in row slabs: the fp32 reference of the whole product is 3 GB
        ref = x[r0:r0 + 1024].float() @ E.float().t()
        assert _rel_l2(buf[r0:r0 + 1024, :V], ref) < 3e-3, r0
    pad = buf[:, V:]
    assert bool((pad == 7.0).all())                              # padding columns: untouched


def test_gemm_production_wgrad_split_k(K):
    torch.manual_seed(13)
    M, N, Kd = 48000, 1024, 1024            # dW = dy^T x: 32 output tiles, reduction over 48000 rows, split-K + fp32 red.add
    dy = (torch.randn(M, N, device="cuda") * 0.05).bfloat16()
    x = torch.randn(M, Kd, device="cuda").bfloat16()
    ref = dy.float().t() @ x.float()
    for split in (1, 4, 7):
        out = torch.full((N, Kd), 1.0, device="cuda")
        K.gemm(dy, x, N, Kd, M, a_mn=True, b_mn=True, out=out, epi=K.EPI_F32_ATOMIC_ADD, split_k=split, block_n=256)
        assert _rel_l2(out - 1.0, ref) < 2e-4, split     # 48000-term fp32 tensor-core accumulation vs cuBLAS fp32 (measured 5.6e-5)
    out = K.gemm(dy, x, N, Kd, M, a_mn=True, b_mn=True, epi=K.EPI_F32, block_n=256)
    assert _rel_l2(out, ref) < 2e-4


def test_gemm_decoder_shape_three_waves_and_residual(K):
    torch.manual_seed(14)
    M, N, Kd = 14336, 1024, 1024            # 112 x 8 = 896 tiles on 132 SMs: 6.8 waves
    A = torch.randn(M, Kd, device="cuda").bfloat16()
    B = (torch.randn(N, Kd, device="cuda") / math.sqrt(Kd)).bfloat16()
    bias = torch.randn(N, device="cuda")
    aux = torch.randn(M, N, device="cuda").bfloat16()
    ref = aux.float() + ((A.float() @ B.float().t()) + bias.bfloat16().float()).bfloat16().float()
    got = K.gemm(A, B, M, N, Kd, bias=bias, aux=aux, epi=K.EPI_BF16_RESIDUAL, block_n=256)
    assert _rel_l2(got, ref) < 3e-3
    got128 = K.gemm(A, B, M, N, Kd, bias=bias, aux=aux, epi=K.EPI_BF16_RESIDUAL, block_n=128)
    assert _rel_l2(got128, ref) < 3e-3


def test_gemm_sm_budget(K):
    """A reduced SM budget (the persistent grid shrinks, every CTA takes more tiles) gives the same numbers as the
    default."""
    torch.manual_seed(15)
    M, N, Kd = 6144, 3072, 1024
    A = torch.randn(M, Kd, device="cuda").bfloat16()
    B = (torch.randn(N, Kd, device="cuda") / math.sqrt(Kd)).bfloat16()
    bias = torch.randn(N, device="cuda")
    base = K.gemm(A, B, M, N, Kd, bias=bias, block_n=256)
    ref = ((A.float() @ B.float().t()) + bias.bfloat16().float())
    assert _rel_l2(base, ref) < 3e-3
    prev = K.set_gemm_sm_budget(132)
    try:
        b132 = K.gemm(A, B, M, N, Kd, bias=bias, block_n=256)
        K.set_gemm_sm_budget(20)
        b20 = K.gemm(A, B, M, N, Kd, bias=bias, block_n=256)       # 1152 tiles on 20 CTAs: ~58 tiles per CTA
    finally:
        K.set_gemm_sm_budget(prev)
    assert torch.equal(b132, base) and torch.equal(b20, base)


def test_gemm_rejects_bad_arguments(K):
    from olmoasr_b200._lib import OasrError
    A = torch.zeros(16, 12, device="cuda", dtype=torch.bfloat16)  # row stride 12 elements: not TMA-legal
    B = torch.zeros(16, 12, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(OasrError):
        K.gemm(A, B, 16, 16, 12)
    with pytest.raises(ValueError):
        K.gemm(A.float(), B, 16, 16, 12)


# ------------------------------------------------------------------------------------------------ LayerNorm
# ------------------------------------------------------------------------------------------------ attention
def _sdpa_ref(q, k, v, B, H, Tq, Tkv, causal, kv_len):
    qh = q.float().view(B, Tq, H, 64).permute(0, 2, 1, 3)
    kh = k.float().view(B, Tkv, H, 64).permute(0, 2, 1, 3)
    vh = v.float().view(B, Tkv, H, 64).permute(0, 2, 1, 3)
    mask = None
    if causal or kv_len is not None:
        mask = torch.zeros(B, 1, Tq, Tkv, device=q.device)
        if causal:
            mask = mask + torch.full((Tq, Tkv), -float("inf"), device=q.device).triu_(1)
        if kv_len is not None:
            for i in range(B):
                mask[i, :, :, int(kv_len[i]):] = -float("inf")
    o = F.scaled_dot_product_attention(qh, kh, vh, attn_mask=mask)
    return o.permute(0, 2, 1, 3).reshape(B * Tq, H * 64)


@pytest.mark.parametrize("B,H,Tq,Tkv,causal,use_len", [
    (2, 2, 128, 128, False, False),
    (1, 1, 300, 300, False, False),
    (2, 3, 1500, 1500, False, False),   # encoder self-attention shape
    (3, 2, 448, 448, True, True),       # decoder self-attention: causal + per-sample length
    (2, 2, 448, 1500, False, False),    # cross-attention
    (1, 2, 5, 7, False, False),         # tiny ragged
    (2, 3, 700, 700, False, True),      # ragged tiles + lengths
])
def test_attention_fwd_bwd(K, B, H, Tq, Tkv, causal, use_len):
    torch.manual_seed(3)
    d = H * 64
    # strided views into fused projection buffers, as the model uses them
    qkv = torch.randn(B * Tq, 3 * d, device="cuda").bfloat16()
    kvb = torch.randn(B * Tkv, 2 * d, device="cuda").bfloat16() if Tkv != Tq else None
    q = qkv[:, :d]
    k = qkv[:, d:2 * d] if kvb is None else kvb[:, :d]
    v = qkv[:, 2 * d:] if kvb is None else kvb[:, d:]
    kv_len = None
    if use_len:
        kv_len = torch.tensor([31 + 150 * i for i in range(B)], device="cuda", dtype=torch.int32).clamp(max=Tkv)
    o, lse = K.attention_fwd(q, k, v, B, H, Tq, Tkv, causal=causal, kv_len=kv_len)
    qr, kr, vr = (t.float().clone().requires_grad_(True) for t in (q, k, v))
    oref = _sdpa_ref(qr, kr, vr, B, H, Tq, Tkv, causal, kv_len)
    _close(o, oref.detach(), rtol=1.0 / 64)
    dout = torch.randn(B * Tq, d, device="cuda").bfloat16()
    oref.backward(dout.float())
    dq, dk, dv = K.attention_bwd(q, k, v, o, dout, lse, B, H, Tq, Tkv, causal=causal, kv_len=kv_len)
    _close(dq, qr.grad, rtol=1.0 / 48)
    _close(dk, kr.grad, rtol=1.0 / 48)
    _close(dv, vr.grad, rtol=1.0 / 48)


def test_cross_block_reductions_repeat_bit_for_bit(K):
    """Sums that span CTAs (split-K, attention dQ, LayerNorm / bias / embedding gradients, the CE loss sum) are added in a
    fixed order, never with floating-point atomics: the same call on the same inputs gives the same bits every time."""
    torch.manual_seed(21)
    twice = lambda f: (f(), f())
    dy = (torch.randn(12000, 1024, device="cuda") * 0.05).bfloat16()
    x = torch.randn(12000, 1024, device="cuda").bfloat16()

    def wgrad():
        out = torch.zeros(1024, 1024, device="cuda")
        K.gemm(dy, x, 1024, 1024, 12000, a_mn=True, b_mn=True, out=out, epi=K.EPI_F32_ATOMIC_ADD, split_k=6, block_n=128)
        return out
    a, b = twice(wgrad)
    assert torch.equal(a, b)
    B, H, T = 2, 4, 1500
    qkv = torch.randn(B * T, 3 * H * 64, device="cuda").bfloat16()
    q, k, v = qkv[:, :H * 64], qkv[:, H * 64:2 * H * 64], qkv[:, 2 * H * 64:]
    o, lse = K.attention_fwd(q, k, v, B, H, T, T)
    do = torch.randn(B * T, H * 64, device="cuda").bfloat16()
    a, b = twice(lambda: K.attention_bwd(q, k, v, o, do, lse, B, H, T, T))
    assert all(torch.equal(u, w) for u, w in zip(a, b))
    w, bias = torch.randn(1024, device="cuda"), torch.randn(1024, device="cuda")
    _, mean, rstd = K.layernorm_fwd(x, w, bias)

    def ln_params():
        dw, db = torch.zeros(1024, device="cuda"), torch.zeros(1024, device="cuda")
        K.layernorm_bwd(dy, x, w, mean, rstd, dw, db)
        return dw, db
    a, b = twice(ln_params)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])

    def colsum():
        db = torch.zeros(1024, device="cuda")
        K.colsum_(dy, db, 1024)
        return db
    a, b = twice(colsum)
    assert torch.equal(a, b)
    ids = torch.randint(0, 50, (16, 448), device="cuda")          # many repeated ids

    def emb():
        demb, dpos = torch.zeros(51865, 384, device="cuda"), torch.zeros(448, 384, device="cuda")
        K.embed_bwd(ids, dy[:16 * 448, :384].contiguous(), demb, dpos, 51864)
        return demb, dpos
    a, b = twice(emb)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    logits = (torch.randn(2048, 51968, device="cuda") * 3).bfloat16()
    y = torch.randint(0, 51865, (2048,), device="cuda")
    a, b = twice(lambda: K.ce_fwd(logits, y, 51865, 51864)[1])
    assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ misc
def test_padding_mask_to_key_counts_and_validation(monkeypatch):
    """The dense additive mask of train_timestamps.py:314-315 -> per-sample key counts on the device; any other additive
    mask is rejected (model.py:740-743 would accept it; this implementation does not support it and must say so)."""
    from olmoasr_b200 import _core
    from olmoasr_b200 import synthetic as synth

    monkeypatch.setattr(_core, "STRICT_MASK", True)
    ti, ty, pm, lens = synth.text_batch(5)
    kv = _core.kv_len_from_padding_mask(pm.cuda())
    want = (pm[:, 0, :] == 0).sum(-1)
    assert kv.dtype == torch.int32 and torch.equal(kv.cpu().long(), want)
    assert torch.equal(_core.kv_len_from_padding_mask(want.cuda()), want.cuda().int())       # lengths pass straight through
    big_neg = pm.clone(); big_neg[big_neg == -float("inf")] = torch.finfo(torch.float32).min
    assert torch.equal(_core.kv_len_from_padding_mask(big_neg.cuda()).cpu().long(), want)     # finfo.min masks are fine
    bad = pm.clone(); bad[2, 100, 3] = -1.0                                                   # an arbitrary additive bias
    with pytest.raises(ValueError, match="padding_mask"):
        _core.kv_len_from_padding_mask(bad.cuda())
    bad2 = pm.clone(); bad2[1, 7, 440] = 0.0                                                  # a hole behind the length
    with pytest.raises(ValueError, match="padding_mask"):
        _core.kv_len_from_padding_mask(bad2.cuda())
    # deferred mode: the error surfaces on the next call instead of stalling the stream
    monkeypatch.setattr(_core, "STRICT_MASK", False)
    _core.kv_len_from_padding_mask(bad.cuda())
    torch.cuda.synchronize()
    with pytest.raises(ValueError, match="padding_mask"):
        _core.kv_len_from_padding_mask(pm.clone().cuda())
    _core.kv_len_from_padding_mask(pm.clone().cuda())                                         # flag was cleared


# ------------------------------------------------------------------------------------------------ log-mel
def test_logmel_matches_oracle(golden_dir):
    from olmoasr_b200 import audio
    from oracle import logmel, synth

    wav = synth.waveforms(3)
    wav[1] *= 0.01                       # very different per-clip maxima: the floor must be per clip
    wav[2, 40000:] = 0.0                 # trailing silence hits the 1e-10 clamp and the max-8 floor
    got = audio.log_mel_spectrogram(wav.cuda()).cpu().numpy()
    want = logmel.log_mel_spectrogram(wav.numpy())
    assert got.shape == (3, 80, 3000)
    assert np.abs(got - want).max() < 1e-4      # SURVEY.md section 7: <= 1e-4 abs in fp32
    gold = np.load(golden_dir / "logmel_hf.npz")
    one = audio.log_mel_spectrogram(synth.waveforms(2)[0].cuda()).cpu().numpy()
    assert np.abs(one[:, ::7] - gold["noise"]).max() < 1e-4
    i16 = synth.waveforms(2, int16=True)
    a = audio.log_mel_spectrogram(i16.cuda()).cpu().numpy()
    b = logmel.log_mel_spectrogram(logmel.int16_to_float(i16.numpy()))
    assert np.abs(a - b).max() < 1e-4
    short = audio.log_mel_spectrogram(audio.pad_or_trim(wav[0, :51237].cuda()))
    assert short.shape == (80, 3000)
    # any length (ffmpeg output is arbitrary): n // 160 frames like upstream, end reflection at the true last sample
    odd = wav[0, :51237]
    a = audio.log_mel_spectrogram(odd.cuda(), padding=480000).cpu().numpy()
    b = logmel.log_mel_spectrogram(np.pad(odd.numpy(), (0, 480000)))
    assert a.shape == b.shape == (80, (51237 + 480000) // 160) and np.abs(a - b).max() < 1e-4
    for n in (51237, 51200, 640 * 7 + 1, 401):
        c = audio.log_mel_spectrogram(wav[0, :n].cuda()).cpu().numpy()
        e = logmel.log_mel_spectrogram(wav[0, :n].numpy())
        assert c.shape == e.shape == (80, n // 160) and np.abs(c - e).max() < 1e-4, n
    tone = (0.3 * np.sin(2 * np.pi * 440.0 * np.arange(480000) / 16000.0)).astype(np.float32)     # a spectral line: FFT leakage check
    t = audio.log_mel_spectrogram(torch.from_numpy(tone).cuda()).cpu().numpy()
    assert np.abs(t[:, ::7] - gold["tone"]).max() < 2e-4
