"""LoRA on the GPU: the GEMM's low-rank tail, adapters with B = 0 leaving the model's bits alone, adapter gradients
against the merged-weight model, and merge_lora."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

from olmoasr_b200 import kernels as K

DTYPES = [torch.bfloat16, torch.float16]


def _t(shape, dt, scale=1.0):
    return (torch.randn(shape, device="cuda") * scale).to(dt)


FWD = [K.EPI_BF16, K.EPI_BF16_GELU, K.EPI_BF16_RESIDUAL]
BWD = [K.EPI_BF16, K.EPI_BF16_RESIDUAL, K.EPI_BF16_GELU_BWD]
SHAPES = [(7168, 1024, 1024), (7168, 3072, 1024), (24000, 1024, 4096), (7168, 4096, 1024)]


@pytest.mark.parametrize("dt", DTYPES, ids=["bf16", "fp16"])
@pytest.mark.parametrize("K2", [8, 32, 64, 72, 192])
@pytest.mark.parametrize("block_n", [64, 128, 256])
@pytest.mark.parametrize("b_mn", [False, True], ids=["fwd", "dgrad"])
def test_tail_equals_the_gemm_over_the_concatenated_reduction(dt, K2, block_n, b_mn):
    """With K a multiple of 64 the tail's k-blocks are exactly the k-blocks the plain GEMM runs over [A | A2] [B | B2]^T
    (zero-filled past K2 in both), so the two must agree bit for bit for every epilogue; the plain GEMM is pinned to
    fp64 in tests/test_training_parity_gpu.py.  One fp64 check on top guards against both being wrong together."""
    torch.manual_seed(K2 + block_n)
    for si, (M, N, Kd) in enumerate(SHAPES[:2] if K2 not in (8, 192) else SHAPES):
        a, a2 = _t((M, Kd), dt), _t((M, K2), dt)
        b = _t((Kd, N) if b_mn else (N, Kd), dt, Kd ** -0.5)
        b2 = _t((K2, N) if b_mn else (N, K2), dt, K2 ** -0.5)
        bias = torch.randn(N, device="cuda") * 0.1
        aux = _t((M, N), dt)
        A = torch.cat([a, a2], 1).contiguous()
        B = torch.cat([b, b2], 0 if b_mn else 1).contiguous()
        for epi in (BWD if b_mn else FWD):
            kw = dict(epi=epi, block_n=block_n)
            if epi in (K.EPI_BF16_RESIDUAL, K.EPI_BF16_GELU_BWD):
                kw["aux"] = aux
            if epi != K.EPI_BF16_GELU_BWD:
                kw["bias"] = bias
            got = K.gemm_lowrank(a, b, a2, b2, M, N, Kd, K2, b_mn=b_mn, **kw)
            want = K.gemm(A, B, M, N, Kd + K2, b_mn=b_mn, **kw)
            for g, w in zip(got if isinstance(got, tuple) else (got,), want if isinstance(want, tuple) else (want,)):
                assert torch.equal(g, w), (M, N, Kd, epi)
            if epi == K.EPI_BF16 and si == 0:
                ref = A.double() @ (B.double() if b_mn else B.double().t()) + bias.to(dt).double()
                err = float((got.double() - ref).norm() / ref.norm())
                assert err <= (4e-3 if dt == torch.bfloat16 else 5e-4), err


def test_tail_rejects_bad_ranks_and_pairs():
    a, b = _t((128, 64), torch.bfloat16), _t((64, 64), torch.bfloat16)
    with pytest.raises(Exception):
        K.gemm_lowrank(a, b, _t((128, 200), torch.bfloat16), _t((64, 200), torch.bfloat16), 128, 64, 64, 200)
    with pytest.raises(ValueError):
        K.gemm_lowrank(a, b, _t((128, 8), torch.bfloat16), _t((8, 64), torch.bfloat16), 128, 64, 64, 8, b_mn=True,
                       epi=K.EPI_BF16_GELU)


def test_merge_kernel_matches_fp64():
    torch.manual_seed(1)
    w, b, a = torch.randn(1024, 4096, device="cuda"), torch.randn(1024, 32, device="cuda"), torch.randn(32, 4096, device="cuda")
    got = K.lora_merge(w, b, a, 0.5)
    ref = w.double() + 0.5 * b.double() @ a.double()
    assert float((got.double() - ref).abs().max()) <= 1e-4
    assert torch.equal(got, K.lora_merge(w, b, a, 0.5))          # deterministic
    w2 = w.clone()
    K.lora_merge(w2, b, a, 0.5, out=w2)                           # in place
    assert torch.equal(w2, got)


def _model(variant="tiny"):
    import olmoasr_b200 as ob
    from olmoasr_b200.model import OLMoASR

    torch.manual_seed(0)
    return OLMoASR(ob.VARIANT_TO_DIMS[variant]).cuda()


def _batch(B=2):
    import olmoasr_b200 as ob
    from oracle import synth

    wav = synth.waveforms(B)
    ti, ty, pm, lens = synth.text_batch(B)
    return ob.log_mel_spectrogram(wav.cuda()), ti.cuda(), ty.cuda(), pm.cuda(), lens


ALL = ("encoder.attn.query", "encoder.attn.key", "encoder.attn.value", "encoder.attn.out", "encoder.mlp.0", "encoder.mlp.2",
       "decoder.attn.query", "decoder.attn.value", "decoder.cross_attn.query", "decoder.cross_attn.key",
       "decoder.cross_attn.value", "decoder.cross_attn.out", "decoder.mlp.0", "decoder.mlp.2")


@pytest.mark.parametrize("route", ["dense", "packed", "fp16"])
def test_zero_b_adapters_leave_the_loss_bits_alone(route):
    from olmoasr_b200.lora import add_lora

    m = _model()
    mel, ti, ty, pm, lens = _batch()
    lm = add_lora(copy.deepcopy(m), 32, 64, targets=ALL)

    def loss(model):
        with torch.no_grad(), torch.autocast("cuda", torch.float16, enabled=route == "fp16"):
            if route == "packed":
                return model(mel, ti, targets=ty, text_lens=lens)
            return model(mel, ti, pm, targets=ty)

    assert torch.equal(loss(m), loss(lm))


def _randomize_b(m, scale=0.02):
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith("lora_B"):
                p.copy_(scale * torch.randn_like(p))


def _merged_copy(base, lm):
    from olmoasr_b200.lora import effective_weight

    ref = copy.deepcopy(base)
    sd = {k: v for k, v in lm.state_dict().items() if ".lora_" not in k}
    for name, mod in lm.named_modules():
        if getattr(mod, "has_lora", False):
            sd[name + ".weight"] = effective_weight(mod).clone()
    ref.load_state_dict(sd)
    return ref


@pytest.mark.parametrize("fp16", [False, True], ids=["bf16", "fp16"])
def test_adapter_gradients_match_the_merged_weight_model(fp16):
    """Adapter gradients against the chain rule through the plain model whose weights are W + s B A.  Both models round
    their activations to 16 bits independently, so the comparison is over all adapters at once (a wrong scale or sign
    is off by 50 % or more on every adapter); the loss is scaled like GradScaler does so fp16 gradients do not flush."""
    from olmoasr_b200.lora import add_lora

    base = _model("tiny")
    mel, ti, ty, pm, lens = _batch()
    lm = add_lora(copy.deepcopy(base), 32, 64, targets=ALL)
    _randomize_b(lm)
    frozen = {k: p.detach().clone() for k, p in lm.named_parameters() if ".lora_" not in k}
    ref = _merged_copy(base, lm)
    scale = 1024.0 if fp16 else 1.0
    with torch.autocast("cuda", torch.float16, enabled=fp16):
        loss = lm(mel, ti, pm, targets=ty)
        loss_ref = ref(mel, ti, pm, targets=ty)
    (loss * scale).backward()
    (loss_ref * scale).backward()
    assert abs(loss.item() - loss_ref.item()) <= 2e-3 * abs(loss_ref.item())
    refp = dict(ref.named_parameters())
    got_all, want_all = [], []
    for name, mod in lm.named_modules():
        if getattr(mod, "has_lora", False):
            gw = refp[name + ".weight"].grad.double()
            s, A, B = mod.lora_scale, mod.lora_A.detach().double(), mod.lora_B.detach().double()
            for got, want in ((mod.lora_A.grad, s * B.t() @ gw), (mod.lora_B.grad, s * gw @ A.t())):
                got_all.append(got.double().reshape(-1))
                want_all.append(want.reshape(-1))
                rel = float((got.double() - want).norm() / want.norm())
                assert rel <= 0.25, (name, rel)
    g, w = torch.cat(got_all), torch.cat(want_all)
    assert float((g - w).norm() / w.norm()) <= 5e-2
    for k, p in lm.named_parameters():
        assert (p.grad is not None) == (".lora_" in k), k
    opt = torch.optim.AdamW([p for p in lm.parameters() if p.requires_grad], lr=1e-3)
    for _ in range(3):
        opt.step()
        opt.zero_grad()
        with torch.autocast("cuda", torch.float16, enabled=fp16):
            (lm(mel, ti, pm, targets=ty) * scale).backward()
    for k, p in lm.named_parameters():
        if ".lora_" not in k:
            assert torch.equal(p.detach(), frozen[k]), k


QV = ("encoder.attn.query", "encoder.attn.value", "decoder.attn.query", "decoder.attn.value")
MEDIUM_TARGETS = QV + ("decoder.cross_attn.key", "decoder.cross_attn.value", "encoder.mlp.2", "decoder.mlp.0")


def _lora_medium(depth):
    from tests.test_model_gpu import _build_width
    from olmoasr_b200.lora import add_lora

    m, sd, dims, OM, mel, ti, ty, pm = _build_width("medium", depth)
    add_lora(m, 32, 64, targets=MEDIUM_TARGETS)
    torch.manual_seed(3)
    _randomize_b(m)
    merged = dict(sd)
    for name, mod in m.named_modules():
        if getattr(mod, "has_lora", False):
            merged[name + ".weight"] = (mod.weight.detach().double() + mod.lora_scale * mod.lora_B.detach().double()
                                        @ mod.lora_A.detach().double()).float().cpu()
    return m, merged, dims, OM, mel, ti, ty, pm


def test_medium_adapter_gradients_against_the_fp32_oracle(golden_dir):
    """Medium widths at depth 2+2 over subset slabs: loss and adapter gradients against the fp32 oracle with the merged
    weights W + s B A (dA = s B^T dW, dB = s dW A^T), at the training parity tests' tolerances: an adapter's gradient
    is as close as max(1.5 x, 2e-2) the reference's own bf16 error on its base weight's gradient (a projection of it)."""
    noise = torch.load(golden_dir / "model_medium_2x2.pt", weights_only=False)["grad_noise"]
    m, merged, dims, OM, mel, ti, ty, pm = _lora_medium((2, 2))
    sl = m.use_slabs()
    p = {k: v.clone().requires_grad_(k != "encoder.positional_embedding") for k, v in merged.items()}
    loss_ref = OM.token_ce(OM.model_forward(p, dims, mel, ti, pm, train_model=True), ty)
    loss_ref.backward()
    sl.zero_grad()
    loss = m(mel.cuda(), ti.cuda(), pm.cuda(), targets=ty.cuda())
    loss.backward()
    assert abs(loss.item() - loss_ref.item()) <= 1e-3 * abs(loss_ref.item()), (loss.item(), loss_ref.item())
    worst = []
    for name, mod in m.named_modules():
        if getattr(mod, "has_lora", False):
            gw = p[name + ".weight"].grad.double()
            s, A, B = mod.lora_scale, mod.lora_A.detach().double().cpu(), mod.lora_B.detach().double().cpu()
            for ab, got, want in (("A", mod.lora_A.grad, s * B.t() @ gw), ("B", mod.lora_B.grad, s * gw @ A.t())):
                worst.append((float((got.double().cpu() - want).norm() / want.norm()), name))
    worst.sort(reverse=True)
    print("largest adapter gradient rel-L2 errors:", worst[:4])
    for r, k in worst:
        assert r <= max(1.5 * noise[k + ".weight"], 2e-2), (k, r, noise[k + ".weight"])


def test_medium_full_depth_lora_steps_over_slabs():
    """Full-depth medium with adapters: the loss against the fp32 oracle with merged weights (1e-3 relative, as the
    full-depth parity test), then FusedAdamW steps over subset slabs change the adapters and no frozen byte."""
    import olmoasr_b200 as ob
    from olmoasr_b200.optim import FusedAdamW

    depth = (ob.VARIANT_TO_DIMS["medium"].n_audio_layer, ob.VARIANT_TO_DIMS["medium"].n_text_layer)
    m, merged, dims, OM, mel, ti, ty, pm = _lora_medium(depth)
    with torch.no_grad():
        loss_ref = OM.token_ce(OM.model_forward(merged, dims, mel, ti, pm, train_model=True), ty).item()
    frozen = {k: p.detach().clone() for k, p in m.named_parameters() if not p.requires_grad}
    lora0 = {k: p.detach().clone() for k, p in m.named_parameters() if p.requires_grad}
    sl = m.use_slabs()
    assert sl.numel == sum((p.numel() + 63) // 64 * 64 for p in m.parameters() if p.requires_grad)
    opt = FusedAdamW([p for p in m.parameters() if p.requires_grad], lr=1e-3, slabs=sl)
    mel, ti, ty, pm = mel.cuda(), ti.cuda(), ty.cuda(), pm.cuda()
    losses = []
    for _ in range(4):
        loss = m(mel, ti, pm, targets=ty)
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(loss.item())
    assert abs(losses[0] - loss_ref) <= 1e-3 * abs(loss_ref), (losses[0], loss_ref)
    assert losses[-1] < losses[0]
    for k, p in m.named_parameters():
        if k in frozen:
            assert torch.equal(p.detach(), frozen[k]), k
        else:
            assert not torch.equal(p.detach(), lora0[k]), k


@pytest.mark.parametrize("mode", ["greedy", "beam", "timestamps"])
def test_adapted_model_decodes_like_its_merge(mode):
    """Adapters in both stacks at the decode tests' sharpened weights: decode() of the adapted model (encoder through the
    tail GEMM, decoder with the engine's effective weights and the hook path's tail GEMM) gives the merged model's ids."""
    from olmoasr_b200 import synthetic
    from olmoasr_b200.decoding import DecodingOptions, decode
    from olmoasr_b200.lora import add_lora, merge_lora
    from oracle import logmel
    from tests.test_decode_engine_gpu import SHARPEN, _build

    m = _build("tiny", emb_scale=SHARPEN["tiny"][0], pos_scale=SHARPEN["tiny"][1])[0]
    mel = torch.from_numpy(logmel.log_mel_spectrogram(synthetic.waveforms(3).numpy())).cuda()
    add_lora(m, 32, 64, targets=ALL)
    torch.manual_seed(5)
    _randomize_b(m, 0.01)
    opts = {"greedy": DecodingOptions(language="en", without_timestamps=True, sample_len=24, fp16=False),
            "beam": DecodingOptions(language="en", beam_size=3, without_timestamps=True, sample_len=24, fp16=False),
            "timestamps": DecodingOptions(language="en", without_timestamps=False, sample_len=24, fp16=False)}[mode]
    adapted = [r.tokens for r in decode(m, mel, opts)]
    merged = [r.tokens for r in decode(merge_lora(m), mel, opts)]
    assert adapted == merged


def test_merge_lora_after_training_keeps_loss_and_decode():
    import olmoasr_b200 as ob
    from olmoasr_b200.decoding import DecodingOptions, decode
    from olmoasr_b200.lora import add_lora, merge_lora

    m = _model()
    ref_keys = set(m.state_dict())
    mel, ti, ty, pm, lens = _batch()
    lm = add_lora(m, 32, 64, targets=("decoder.attn.query", "decoder.attn.value", "decoder.cross_attn.key",
                                     "decoder.cross_attn.value", "decoder.mlp.2"))
    opt = torch.optim.AdamW([p for p in lm.parameters() if p.requires_grad], lr=1e-3)
    for _ in range(3):
        lm(mel, ti, pm, targets=ty).backward()
        opt.step()
        opt.zero_grad()
    assert any(float(p.abs().max()) > 0 for n, p in lm.named_parameters() if n.endswith("lora_B"))
    with torch.no_grad():
        before = lm(mel, ti, pm, targets=ty).item()
    opts = [DecodingOptions(language="en", without_timestamps=True, sample_len=16, fp16=False)]
    mel30 = ob.pad_or_trim(mel, 3000)
    toks_before = [[r.tokens for r in decode(lm, mel30, o)] for o in opts]
    merged = merge_lora(lm)
    assert set(merged.state_dict()) == ref_keys
    with torch.no_grad():
        after = merged(mel, ti, pm, targets=ty).item()
    assert abs(after - before) <= 2e-3 * abs(before)
    # the decode engine casts W + s B A with the merge kernel: identical weights, identical tokens
    toks_after = [[r.tokens for r in decode(merged, mel30, o)] for o in opts]
    assert toks_before == toks_after
