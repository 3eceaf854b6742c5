"""The training step under torch.autocast("cuda", torch.float16) with torch.amp.GradScaler, the reference trainer's
default configuration (scripts/training/train_timestamps.py:1414, :2128, :2349).

Accuracy is measured against the oracle (the reference's arithmetic on the CPU) in fp32, with the reference's own fp16
autocast error as the yardstick: bf16 arithmetic is about 8x further from fp32 than fp16 and cannot pass these bounds.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

LOSS_SCALE = 2.0 ** 16      # GradScaler's default initial scale


def _rel(a, b):
    return float((a.detach().float() - b.detach().float()).norm() / (b.detach().float().norm() + 1e-30))


@pytest.fixture(scope="module")
def setup():
    import olmoasr_b200 as ob
    from olmoasr_b200.model import OLMoASR
    from oracle import logmel, synth
    from oracle import model as OM

    dims_o = OM.variant_dims("tiny")
    sd = OM.init_state_dict(dims_o, seed=0, train=True)
    torch.manual_seed(0)
    m = OLMoASR(ob.VARIANT_TO_DIMS["tiny"]).cuda()
    B = 2
    wav = synth.waveforms(B)
    mel = torch.from_numpy(logmel.log_mel_spectrogram(wav.numpy()))
    ti, ty, pm, _ = synth.text_batch(B)
    return dict(m=m, sd=sd, dims=dims_o, OM=OM, mel=mel, ti=ti, ty=ty, pm=pm, ob=ob)


def test_fp16_logits_and_loss_match_the_reference_fp16_path(setup):
    s = setup
    OM = s["OM"]
    with torch.no_grad():
        ref32 = OM.model_forward(s["sd"], s["dims"], s["mel"], s["ti"], s["pm"], train_model=True)
        ref16 = OM.model_forward(s["sd"], s["dims"], s["mel"], s["ti"], s["pm"], train_model=True, autocast_dtype=torch.float16)
        with torch.autocast("cuda", dtype=torch.float16):
            got = s["m"](s["mel"].cuda(), s["ti"].cuda(), s["pm"].cuda()).cpu()
        got_bf = s["m"](s["mel"].cuda(), s["ti"].cuda(), s["pm"].cuda()).cpu()
    assert got.dtype == torch.float32
    e_ref, e_our, e_bf = _rel(ref16, ref32), _rel(got, ref32), _rel(got_bf, ref32)
    print(f"rel-L2 vs fp32 oracle: reference fp16 {e_ref:.3e}, ours fp16 {e_our:.3e}, ours bf16 {e_bf:.3e}")
    assert e_our <= 1.5 * e_ref
    assert e_bf > 1.5 * e_ref            # the bound tells the two 16-bit types apart
    loss_ref = OM.token_ce(ref16, s["ty"]).item()
    with torch.autocast("cuda", dtype=torch.float16):
        loss = s["m"].loss(s["mel"].cuda(), s["ti"].cuda(), s["ty"].cuda(), s["pm"].cuda())
    assert loss.dtype == torch.float32 and loss.dim() == 0
    assert abs(loss.item() - loss_ref) <= 1e-3 * abs(loss_ref)


def test_fp16_gradients_within_the_reference_fp16_noise(setup):
    s = setup
    OM, m = s["OM"], s["m"]
    grads = {}
    for dt in (None, torch.float16):
        p = {k: v.clone().requires_grad_(k != "encoder.positional_embedding") for k, v in s["sd"].items()}
        with torch.autocast("cpu", dtype=torch.float16, enabled=dt is not None):
            logits = OM.model_forward(p, s["dims"], s["mel"], s["ti"], s["pm"], train_model=True)
        OM.token_ce(logits.float(), s["ty"]).backward()
        grads[dt] = {k: v.grad for k, v in p.items() if v.grad is not None}
    m.zero_grad(set_to_none=True)
    with torch.autocast("cuda", dtype=torch.float16):
        loss = m.loss(s["mel"].cuda(), s["ti"].cuda(), s["ty"].cuda(), s["pm"].cuda())
    loss.backward()
    # The CPU reference keeps attention's P and dS in fp32; the kernels round them to fp16 for the tensor cores (as GPU
    # flash attention does), which adds noise to the gradients of the projections that feed attention (query, key,
    # value).  Those are bounded by 2x the reference's own fp16 noise, every other tensor by 1.5x.
    ratios = []
    for k, prm in m.named_parameters():
        g32 = grads[None][k]
        noise = _rel(grads[torch.float16][k], g32)
        ours = _rel(prm.grad.cpu(), g32)
        ratios.append(((ours + 1e-6) / (noise + 1e-6), k, ours, noise))
    ratios.sort()
    print("worst ratios to the reference fp16 noise:", ratios[-3:])
    for r, k, ours, noise in ratios:
        feeds_attention = any(f"attn.{n}." in k for n in ("query", "key", "value"))
        assert r <= (2.0 if feeds_attention else 1.5), (k, ours, noise)


def _batch(s, B=2):
    return s["mel"].cuda(), s["ti"].cuda(), s["ty"].cuda(), s["pm"].cuda()


def _fresh_model(s, slabs):
    from olmoasr_b200.model import OLMoASR
    torch.manual_seed(0)
    m = OLMoASR(s["ob"].VARIANT_TO_DIMS["tiny"]).cuda()
    sl = m.use_slabs() if slabs else None
    return m, sl


def _reference_loop(m, opt, scaler, batch, steps=3):
    mel, ti, ty, pm = batch
    for _ in range(steps):
        opt.zero_grad()
        with torch.autocast("cuda", dtype=torch.float16):
            loss = m.loss(mel, ti, ty, pm)
        scaler.scale(loss).backward()
        scaler.unscale_(opt)
        torch.nn.utils.clip_grad_norm_(m.parameters(), 1.0)
        scaler.step(opt)
        scaler.update()
    return loss


def test_reference_loop_with_torch_adamw_hand_over_mode(setup):
    m, _ = _fresh_model(setup, slabs=False)
    opt = torch.optim.AdamW(m.parameters(), lr=1e-4)
    scaler = torch.amp.GradScaler("cuda")
    before = [p.detach().clone() for p in m.parameters()]
    loss = _reference_loop(m, opt, scaler, _batch(setup))
    assert torch.isfinite(loss) and scaler.get_scale() == 65536.0
    assert all(not torch.equal(a, p) for a, p in zip(before, m.parameters()))


def test_fused_adamw_under_grad_scaler_matches_explicit_inv_scale(setup):
    from olmoasr_b200.optim import FusedAdamW

    batch = _batch(setup)
    mel, ti, ty, pm = batch
    m1, sl1 = _fresh_model(setup, slabs=True)
    m2, sl2 = _fresh_model(setup, slabs=True)
    o1, o2 = FusedAdamW(m1.parameters(), lr=1e-4, slabs=sl1), FusedAdamW(m2.parameters(), lr=1e-4, slabs=sl2)
    scaler = torch.amp.GradScaler("cuda")
    scale = scaler.get_scale()
    for step in range(3):
        for m, o in ((m1, o1), (m2, o2)):
            o.zero_grad()
            with torch.autocast("cuda", dtype=torch.float16):
                loss = m.loss(mel, ti, ty, pm)
            (loss * scale if o is o2 else scaler.scale(loss)).backward()
        torch.cuda.synchronize()
        with _SyncDebug():          # scaler.step never waits for the host in slab mode
            scaler.step(o1)
        scaler.update()
        o2.step(inv_scale=1.0 / scale)
        assert scaler.get_scale() == scale
    assert sl1.S_dtype == torch.float16
    assert torch.equal(sl1.P, sl2.P) and torch.equal(sl1.S, sl2.S) and torch.equal(sl1.M, sl2.M)
    assert o1.applied_steps() == 3
    # a bf16 forward (e.g. in-loop evaluation) re-casts the shadows; the next fp16 step casts them back
    with torch.no_grad():
        m1.loss(mel, ti, ty, pm)
    assert sl1.S_dtype == torch.bfloat16 and torch.equal(sl1.S, sl1.P.bfloat16())


class _SyncDebug:
    def __enter__(self):
        self.prev = torch.cuda.get_sync_debug_mode()
        torch.cuda.set_sync_debug_mode("error")

    def __exit__(self, *exc):
        torch.cuda.set_sync_debug_mode(self.prev)


def test_overflowing_scale_skips_the_step_and_halves_the_scale(setup):
    from olmoasr_b200.optim import FusedAdamW

    mel, ti, ty, pm = _batch(setup)
    m, sl = _fresh_model(setup, slabs=True)
    opt = FusedAdamW(m.parameters(), lr=1e-4, slabs=sl)
    scaler = torch.amp.GradScaler("cuda", init_scale=2.0 ** 40)
    opt.zero_grad()
    with torch.autocast("cuda", dtype=torch.float16):
        loss = m.loss(mel, ti, ty, pm)
    assert torch.isfinite(loss)
    P0, S0 = sl.P.clone(), sl.S.clone()
    scaler.scale(loss).backward()       # d(logits) * 2^40 overflows fp16 to inf
    with _SyncDebug():
        scaler.step(opt)
    scaler.update()
    assert not bool(torch.isfinite(sl.G).all())
    assert torch.equal(sl.P, P0) and torch.equal(sl.S, S0)
    assert opt.applied_steps() == 0
    assert scaler.get_scale() == 2.0 ** 39


def test_reference_loop_with_fused_adamw_over_slabs(setup):
    """The reference's order -- scaler.unscale_(opt); clip_grad_norm_; scaler.step(opt) -- with FusedAdamW over slabs: the
    step gets grad_scale None and GradScaler's found_inf, and must equal the same operations done by hand."""
    from olmoasr_b200.optim import FusedAdamW

    mel, ti, ty, pm = _batch(setup)
    m1, sl1 = _fresh_model(setup, slabs=True)
    m2, sl2 = _fresh_model(setup, slabs=True)
    o1 = FusedAdamW(m1.parameters(), lr=1e-4, slabs=sl1, max_grad_norm=None)
    o2 = FusedAdamW(m2.parameters(), lr=1e-4, slabs=sl2, max_grad_norm=None)
    scaler = torch.amp.GradScaler("cuda")
    scale = scaler.get_scale()
    loss = _reference_loop(m1, o1, scaler, (mel, ti, ty, pm))
    for _ in range(3):
        o2.zero_grad()
        with torch.autocast("cuda", dtype=torch.float16):
            loss2 = m2.loss(mel, ti, ty, pm)
        (loss2 * scale).backward()
        sl2.G.mul_(1.0 / scale)
        torch.nn.utils.clip_grad_norm_(m2.parameters(), 1.0)
        o2.step()
    assert torch.equal(loss, loss2)
    assert o1.applied_steps() == 3 and scaler.get_scale() == scale
    assert torch.equal(sl1.P, sl2.P) and torch.equal(sl1.S, sl2.S)


def test_reference_loop_hand_over_matches_manual_scaling(setup):
    """Hand-over mode (no slabs, torch AdamW): GradScaler's loop equals scaling, unscaling and clipping by hand."""
    mel, ti, ty, pm = _batch(setup)
    m1, _ = _fresh_model(setup, slabs=False)
    m2, _ = _fresh_model(setup, slabs=False)
    o1, o2 = torch.optim.AdamW(m1.parameters(), lr=1e-4), torch.optim.AdamW(m2.parameters(), lr=1e-4)
    scaler = torch.amp.GradScaler("cuda")
    scale = scaler.get_scale()
    _reference_loop(m1, o1, scaler, (mel, ti, ty, pm))
    for _ in range(3):
        o2.zero_grad()
        with torch.autocast("cuda", dtype=torch.float16):
            loss2 = m2.loss(mel, ti, ty, pm)
        (loss2 * scale).backward()
        for p in m2.parameters():
            p.grad.mul_(1.0 / scale)
        torch.nn.utils.clip_grad_norm_(m2.parameters(), 1.0)
        o2.step()
    assert all(torch.equal(a, b) for a, b in zip(m1.parameters(), m2.parameters()))


def test_hook_decode_path_in_slab_mode_after_an_fp16_step(setup):
    """The kv-cache (hook) decoder under fp16 autocast reads the weights in the type the shadow slab holds."""
    from olmoasr_b200.model import OLMoASR

    mel, ti, ty, pm = _batch(setup)
    m, sl = _fresh_model(setup, slabs=True)
    ref = OLMoASR(setup["ob"].VARIANT_TO_DIMS["tiny"]).cuda()
    ref.load_state_dict(m.state_dict())
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        m.loss(mel, ti, ty, pm)                     # the slab now holds fp16 shadows
        assert sl.S_dtype == torch.float16
        outs = []
        for model in (m, ref):
            xa = model.encoder(mel)
            cache, hooks = model.install_kv_cache_hooks()
            logits = model.decoder(ti[:, :3], xa, kv_cache=cache)
            logits2 = model.decoder(ti[:, 3:4], xa, kv_cache=cache)
            for h in hooks:
                h.remove()
            outs.append((logits, logits2))
    for a, b in zip(*outs):
        assert torch.isfinite(a).all()
        assert torch.equal(a, b)


@pytest.mark.parametrize("name", ["base", "small", "medium"])
@pytest.mark.parametrize("slab", [False, True])
def test_benchmark_widths_fp16(name, slab, golden_dir):
    """The benchmarked widths at depth 2+2 (the tile shapes, LayerNorm widths and head counts of the benchmark) in fp16:
    logits as close to the fp32 oracle as the reference's own fp16 forward is (computed live), loss within 1e-3 of the
    fp32 oracle's, and every gradient within half the reference's recorded bf16 noise (fp16 keeps 3 more mantissa bits).
    The fp16 oracle's own gradients are not computed here: fp16 matmuls on the host take minutes at these widths."""
    from tests.test_model_gpu import _build_width

    m, sd, dims, OM, mel, ti, ty, pm = _build_width(name, (2, 2))
    g = torch.load(golden_dir / f"model_{name}_2x2.pt", weights_only=False)
    if slab:
        m.use_slabs()
    p = {k: v.clone().requires_grad_(k != "encoder.positional_embedding") for k, v in sd.items()}
    ref32 = OM.model_forward(p, dims, mel, ti, pm, train_model=True)
    loss_ref = OM.token_ce(ref32, ty)
    loss_ref.backward()
    with torch.no_grad():
        ref16 = OM.model_forward(sd, dims, mel, ti, pm, train_model=True, autocast_dtype=torch.float16)
        with torch.autocast("cuda", dtype=torch.float16):
            got = m(mel.cuda(), ti.cuda(), pm.cuda()).cpu()
    e_our, e_ref = _rel(got, ref32), _rel(ref16, ref32)
    print(f"{name}: logits rel-L2 vs fp32 oracle: ours fp16 {e_our:.3e}, reference fp16 {e_ref:.3e}")
    assert e_our <= 1.5 * e_ref
    with torch.autocast("cuda", dtype=torch.float16):
        loss = m(mel.cuda(), ti.cuda(), pm.cuda(), targets=ty.cuda())
    if slab:
        m._slabs.zero_grad()
    # scaled as GradScaler scales it: unscaled, the encoder's attention gradients at these widths lie below fp16's range
    (loss * LOSS_SCALE).backward()
    for prm in m.parameters():
        prm.grad.mul_(1.0 / LOSS_SCALE)
    assert abs(loss.item() - loss_ref.item()) <= 1e-3 * abs(loss_ref.item()), (loss.item(), loss_ref.item())
    noise = g["grad_noise"]           # the reference's bf16-autocast gradient error, per tensor
    errs = {k: _rel(prm.grad.cpu(), p[k].grad) for k, prm in m.named_parameters()}
    worst = sorted(((e / noise[k], k, e) for k, e in errs.items()), reverse=True)
    print(f"{name}: largest fp16 gradient errors relative to the reference's bf16 noise:", worst[:3])
    for r, k, e in worst:
        assert e <= 0.5 * noise[k], (k, e, noise[k])


@pytest.mark.parametrize("name", ["base", "medium"])
def test_full_depth_fp16_loss_matches_fp32_oracle(name):
    """Full depth (6+6 / 24+24 layers) in fp16: the fused loss within 1e-3 of the fp32 oracle's.  The residual stream
    keeps fp16 range through 48 blocks."""
    import olmoasr_b200 as ob
    from tests.test_model_gpu import _build_width

    depth = (ob.VARIANT_TO_DIMS[name].n_audio_layer, ob.VARIANT_TO_DIMS[name].n_text_layer)
    m, sd, dims, OM, mel, ti, ty, pm = _build_width(name, depth)
    with torch.no_grad():
        loss_ref = OM.token_ce(OM.model_forward(sd, dims, mel, ti, pm, train_model=True), ty).item()
        with torch.autocast("cuda", dtype=torch.float16):
            got = m(mel.cuda(), ti.cuda(), pm.cuda(), targets=ty.cuda()).item()
    print(f"{name} full depth fp16: loss {got:.6f} vs fp32 oracle {loss_ref:.6f}")
    assert abs(got - loss_ref) <= 1e-3 * abs(loss_ref)
