"""End-to-end parity of the CUDA model against the oracle (the reference's own arithmetic, pinned in
tests/test_oracle_pin.py) on the seeded synthetic batch of SURVEY.md section 8(d).

Tolerances (north_star: "logits/loss within 1e-3 relative in bf16"):
  * loss: |ours - ref_bf16| <= 1e-3 * |ref_bf16|  (ref_bf16 = oracle under torch.autocast(bfloat16));
  * logits: bf16 end-to-end noise of the REFERENCE ITSELF against its fp32 run is ~8e-3 relative L2 (tiny), so the
    elementwise 1e-3 cannot hold between any two bf16 executions; we require ours to be as close to the fp32 oracle
    as the reference's bf16 path is (<= 1.5x its error) and within 1e-2 relative L2 of the bf16 oracle;
  * gradients: relative L2 per tensor against the fp32 oracle.
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def setup():
    import olmoasr_b200 as ob
    from olmoasr_b200.model import OLMoASR
    from oracle import logmel, synth
    from oracle import model as OM

    dims_o = OM.variant_dims("tiny")
    sd = OM.init_state_dict(dims_o, seed=0, train=True)
    torch.manual_seed(0)
    m = OLMoASR(ob.VARIANT_TO_DIMS["tiny"])
    assert all(torch.equal(m.state_dict()[k], sd[k]) for k in sd)  # same seed -> the reference's initial weights
    m = m.cuda()
    B = 2
    wav = synth.waveforms(B)
    mel_cpu = torch.from_numpy(logmel.log_mel_spectrogram(wav.numpy()))
    ti, ty, pm, lens = synth.text_batch(B)
    return dict(m=m, sd=sd, dims=dims_o, OM=OM, wav=wav, mel=mel_cpu, ti=ti, ty=ty, pm=pm)


def _rel(a, b):
    return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-30))


def test_forward_logits_and_loss(setup, golden_dir):
    s = setup
    OM = s["OM"]
    with torch.no_grad():
        ref32 = OM.model_forward(s["sd"], s["dims"], s["mel"], s["ti"], s["pm"], train_model=True)
        refbf = OM.model_forward(s["sd"], s["dims"], s["mel"], s["ti"], s["pm"], train_model=True, autocast_dtype=torch.bfloat16)
        got = s["m"](s["mel"].cuda(), s["ti"].cuda(), s["pm"].cuda()).cpu()
    assert got.shape == ref32.shape == (2, 448, 51865) and got.dtype == torch.float32
    e_ref = _rel(refbf, ref32)
    e_our = _rel(got, ref32)
    e_pair = _rel(got, refbf)
    print(f"rel-L2 vs fp32 oracle: reference-bf16 {e_ref:.3e}, ours {e_our:.3e}; ours vs reference-bf16 {e_pair:.3e}")
    assert e_our <= 1.5 * e_ref
    assert e_pair <= 1e-2
    loss_ref = OM.token_ce(refbf, s["ty"]).item()
    loss_got = F.cross_entropy(got.view(-1, got.shape[-1]), s["ty"].view(-1), ignore_index=51864).item()
    assert abs(loss_got - loss_ref) <= 1e-3 * abs(loss_ref)
    # outputs of the unmodified reference: the fp32 record is host-independent; the bf16 record (CPU-dependent bit
    # pattern) only serves as the yardstick of the reference's own bf16 error
    g = torch.load(golden_dir / "model_tiny.pt", weights_only=False)
    noise = _rel(g["logits_bf16_sample"], g["logits_fp32_sample"])
    assert abs(loss_got - g["loss_fp32"]) <= 1e-3 * abs(g["loss_fp32"])
    assert _rel(got[:, ::16, ::997], g["logits_fp32_sample"]) <= 1.5 * noise


def test_fused_loss_and_gradients(setup, golden_dir):
    s = setup
    OM, m = s["OM"], s["m"]
    p = {k: v.clone().requires_grad_(k != "encoder.positional_embedding") for k, v in s["sd"].items()}
    loss_ref = OM.token_ce(OM.model_forward(p, s["dims"], s["mel"], s["ti"], s["pm"], train_model=True), s["ty"])
    loss_ref.backward()
    m.zero_grad(set_to_none=True)
    loss = m.loss(s["mel"].cuda(), s["ti"].cuda(), s["ty"].cuda(), s["pm"].cuda())
    loss.backward()
    assert abs(loss.item() - loss_ref.item()) <= 2e-3 * abs(loss_ref.item())
    worst = []
    for k, prm in m.named_parameters():
        gref = p[k].grad
        r = _rel(prm.grad.cpu(), gref)
        worst.append((r, k))
    worst.sort(reverse=True)
    print("largest gradient rel-L2 errors:", [(f"{r:.3e}", k) for r, k in worst[:6]])
    # yardstick: the reference's OWN bf16-autocast gradients against its fp32 gradients (tools/make_golden.py);
    # e.g. cross-attention query weights carry ~11 % bf16 noise at initialisation in the reference itself
    noise = torch.load(golden_dir / "grad_noise_tiny.pt", weights_only=False)
    for r, k in worst:
        assert r <= max(1.5 * noise[k], 2e-2), (k, r, noise[k])
    assert sum(r for r, _ in worst) / len(worst) <= 1.5 * sum(noise.values()) / len(noise)
    assert m.decoder.token_embedding.weight.grad[51864].abs().max().item() <= 1e-6 + m.decoder.token_embedding.weight.grad.abs().max().item()
    # drop-in path (fp32 logits + F.cross_entropy + autograd) gives the same gradients as the fused head
    g_fused = {k: q.grad.clone() for k, q in m.named_parameters()}
    m.zero_grad(set_to_none=True)
    logits = m(s["mel"].cuda(), s["ti"].cuda(), s["pm"].cuda())
    F.cross_entropy(logits.view(-1, logits.shape[-1]), s["ty"].cuda().view(-1), ignore_index=51864).backward()
    for k, q in m.named_parameters():
        assert _rel(q.grad, g_fused[k]) <= 2e-2, k


def test_waveform_to_loss_pipeline(setup):
    """mel computed on the GPU from the waveform == mel computed by the oracle, through to the loss."""
    import olmoasr_b200 as ob
    s = setup
    mel_gpu = ob.log_mel_spectrogram(s["wav"].cuda())
    assert (mel_gpu.cpu() - s["mel"]).abs().max().item() < 1e-4
    with torch.no_grad():
        a = s["m"].loss(mel_gpu, s["ti"].cuda(), s["ty"].cuda(), s["pm"].cuda()).item()
        b = s["m"].loss(s["mel"].cuda(), s["ti"].cuda(), s["ty"].cuda(), s["pm"].cuda()).item()
    assert abs(a - b) <= 1e-3 * abs(b)


def test_no_padding_mask_path_and_error_behaviour(setup):
    s = setup
    OM, m = s["OM"], s["m"]
    with torch.no_grad():
        ref = OM.model_forward(s["sd"], s["dims"], s["mel"], s["ti"][:, :20], None, train_model=True, autocast_dtype=torch.bfloat16)
        got = m(s["mel"].cuda(), s["ti"][:, :20].cuda()).cpu()
    assert _rel(got, ref) <= 1e-2
    with pytest.raises(AssertionError, match="incorrect audio shape"):   # model.py:601
        m.encoder(torch.zeros(1, 80, 2000, device="cuda"))


# =====================================================================================================================
# The benchmarked variants (BASELINE.json configs 2, 3, 5): real width / head count, so the kernels run the tile shapes,
# grids and vector widths of the benchmark (N = 1024 / 3072 / 4096 GEMM tiles, 16 heads, d = 1024 LayerNorm rows,
# K = 3000-row split-K wgrads, the M-fastest logits raster), at depth 2+2 so that the fp32 oracle finishes in seconds.
# Tolerances, as for tiny: loss within 1e-3 relative (north_star); logits and gradients as close to the fp32 oracle as the
# REFERENCE'S OWN bf16-autocast run is (yardsticks recorded from the reference in tests/golden/model_<v>_2x2.pt).
# =====================================================================================================================
def _build_width(name, depth):
    from dataclasses import replace

    import olmoasr_b200 as ob
    from olmoasr_b200.model import OLMoASR
    from oracle import logmel, synth
    from oracle import model as OM

    dims_o = replace(OM.variant_dims(name), n_audio_layer=depth[0], n_text_layer=depth[1])
    sd = OM.init_state_dict(dims_o, seed=0, train=True)
    m = OLMoASR(replace(ob.VARIANT_TO_DIMS[name], n_audio_layer=depth[0], n_text_layer=depth[1]))
    m.load_state_dict(sd)
    wav = synth.waveforms(2)
    mel = torch.from_numpy(logmel.log_mel_spectrogram(wav.numpy()))
    ti, ty, pm, _ = synth.text_batch(2)
    return m.cuda(), sd, dims_o, OM, mel, ti, ty, pm


@pytest.mark.parametrize("name", ["base", "small", "medium"])
@pytest.mark.parametrize("slab", [False, True])
def test_benchmark_widths_forward_and_gradients(name, slab, golden_dir):
    m, sd, dims, OM, mel, ti, ty, pm = _build_width(name, (2, 2))
    g = torch.load(golden_dir / f"model_{name}_2x2.pt", weights_only=False)
    if slab:
        m.use_slabs()
    # fp32 oracle, live on the host cores (pinned to the reference by tests/test_oracle_pin.py at these widths)
    p = {k: v.clone().requires_grad_(k != "encoder.positional_embedding") for k, v in sd.items()}
    ref32 = OM.model_forward(p, dims, mel, ti, pm, train_model=True)
    loss_ref = OM.token_ce(ref32, ty)
    loss_ref.backward()
    assert abs(loss_ref.item() - g["loss_fp32"]) <= 1e-5 * g["loss_fp32"]
    with torch.no_grad():
        got = m(mel.cuda(), ti.cuda(), pm.cuda()).cpu()
    e_our, e_ref = _rel(got, ref32.detach()), g["logits_bf16_noise"]
    print(f"{name}: logits rel-L2 vs fp32 oracle: ours {e_our:.3e}, reference-bf16 {e_ref:.3e}")
    assert e_our <= 1.5 * e_ref
    assert _rel(got[:, ::16, ::997], g["logits_fp32_sample"]) <= 2.0 * e_ref          # vs the unmodified reference's record
    loss = m(mel.cuda(), ti.cuda(), pm.cuda(), targets=ty.cuda())
    if slab:
        m._slabs.zero_grad()
    loss.backward()
    assert abs(loss.item() - loss_ref.item()) <= 1e-3 * abs(loss_ref.item()), (loss.item(), loss_ref.item())
    assert abs(loss.item() - g["loss_bf16"]) <= 1e-3 * abs(g["loss_bf16"])
    noise = g["grad_noise"]
    worst = sorted(((_rel(prm.grad.cpu(), p[k].grad), k) for k, prm in m.named_parameters()), reverse=True)
    print(f"{name}: largest gradient rel-L2 errors:", [(f"{r:.3e}", k, f"ref {noise[k]:.3e}") for r, k in worst[:4]])
    for r, k in worst:
        assert r <= max(1.5 * noise[k], 2e-2), (k, r, noise[k])
    assert sum(r for r, _ in worst) / len(worst) <= 1.5 * sum(noise.values()) / len(noise)


@pytest.mark.parametrize("name", ["base", "medium"])
def test_full_depth_loss_matches_fp32_oracle(name):
    """BASELINE.json configs 2 and 3 at FULL depth (6+6 / 24+24 layers): the fused loss against the fp32 oracle's, within
    north_star's 1e-3 relative.  (Accumulated bf16 noise over 48 blocks is the thing this adds over the 2+2 tests.)"""
    import olmoasr_b200 as ob
    from oracle import model as OM
    depth = (ob.VARIANT_TO_DIMS[name].n_audio_layer, ob.VARIANT_TO_DIMS[name].n_text_layer)
    m, sd, dims, OM, mel, ti, ty, pm = _build_width(name, depth)
    with torch.no_grad():
        loss_ref = OM.token_ce(OM.model_forward(sd, dims, mel, ti, pm, train_model=True), ty).item()
        got = m(mel.cuda(), ti.cuda(), pm.cuda(), targets=ty.cuda()).item()
    print(f"{name} full depth: loss {got:.6f} vs fp32 oracle {loss_ref:.6f}")
    assert abs(got - loss_ref) <= 1e-3 * abs(loss_ref)
