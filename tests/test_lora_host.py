"""Host logic of LoRA fine-tuning (olmoasr_b200/lora.py and the adapter sites of the fused blocks) on the CPU:
tests/cpu_backend.py stands in for the dense kernels, and the tail GEMM, the scaled cast and the merge are stood in for
below.  The tail stand-in is the dense GEMM over the concatenated reduction [A | A2] [B | B2]^T, which is what the kernel
accumulates.  The kernels themselves are checked on the GPU in tests/test_lora_gpu.py."""
import copy

import pytest
import torch

from tests import cpu_backend
from oracle import logmel, synth

BF = torch.bfloat16


def gemm_lowrank(a, b, a2, b2, M, N, K, K2, *, b_mn=False, out=None, out2=None, bias=None, aux=None, epi=0, block_n=0):
    A = torch.cat([a, a2], 1)
    B = torch.cat([b, b2], 0 if b_mn else 1)
    return cpu_backend.gemm(A, B, M, N, K + K2, b_mn=b_mn, out=out, out2=out2, bias=bias, aux=aux, epi=epi)


def cast_scaled16(src, scale, dst):
    dst.copy_((scale * src).to(dst.dtype))
    return dst


def lora_merge(w, b, a, scale, out=None):
    r = w + scale * (b @ a)
    if out is not None:
        out.copy_(r)
        return out
    return r


def layernorm_bwd(dy, x, weight, mean, rstd, dweight, dbias, dresidual=None):
    """The kernel skips the reduction of a null dweight / dbias (a frozen affine)."""
    d = x.shape[1]
    dweight = torch.zeros(d) if dweight is None else dweight
    dbias = torch.zeros(d) if dbias is None else dbias
    return cpu_backend.layernorm_bwd(dy, x, weight, mean, rstd, dweight, dbias, dresidual)


def _dims():
    from olmoasr_b200.config.model_dims import ModelDimensions
    return ModelDimensions(80, 1500, 64, 1, 2, 51864, 448, 64, 1, 2)


@pytest.fixture()
def setup(monkeypatch):
    from olmoasr_b200 import kernels
    from olmoasr_b200.model import OLMoASR

    cpu_backend.install(monkeypatch)
    for fn in (gemm_lowrank, cast_scaled16, lora_merge, layernorm_bwd):
        monkeypatch.setattr(kernels, fn.__name__, fn)
    torch.manual_seed(0)
    m = OLMoASR(_dims())
    mel = torch.from_numpy(logmel.log_mel_spectrogram(synth.waveforms(2).numpy()))
    ti, ty, pm, lens = synth.text_batch(2)
    return m, mel, ti, ty, pm, lens


ALL = ("encoder.attn.query", "encoder.attn.key", "encoder.attn.value", "encoder.attn.out", "encoder.mlp.0", "encoder.mlp.2",
       "decoder.attn.query", "decoder.attn.value", "decoder.cross_attn.query", "decoder.cross_attn.key",
       "decoder.cross_attn.out", "decoder.mlp.2")


def _randomize_b(m):
    with torch.no_grad():
        for n, p in m.named_parameters():
            if n.endswith("lora_B"):
                p.copy_(0.05 * torch.randn_like(p))


def test_add_lora_names_shapes_freezing_and_round_trip(setup):
    from olmoasr_b200.lora import add_lora
    from olmoasr_b200.model import OLMoASR

    m = setup[0]
    ref_keys = set(m.state_dict())
    add_lora(m, 8, 16)
    lora = {k: p for k, p in m.named_parameters() if ".lora_" in k}
    assert set(lora) == {f"{s}.blocks.{i}.attn.{n}.lora_{ab}" for s in ("encoder", "decoder") for i in range(2)
                         for n in ("query", "value") for ab in "AB"}
    for k, p in m.named_parameters():
        assert p.requires_grad == (".lora_" in k), k
        if k.endswith("lora_A"):
            assert p.shape == (8, 64) and p.abs().max() > 0
        elif k.endswith("lora_B"):
            assert p.shape == (64, 8) and p.abs().max() == 0
    assert m.encoder.blocks[0].attn.query.lora_scale == 2.0
    sd = m.state_dict()
    assert set(sd) == ref_keys | set(lora)
    _randomize_b(m)
    fresh = add_lora(OLMoASR(_dims()), 8, 16)
    fresh.load_state_dict(m.state_dict())
    for k, v in m.state_dict().items():
        assert torch.equal(fresh.state_dict()[k], v), k


@pytest.mark.parametrize("case", ["r4", "r12", "r200", "enc_cross", "bad_name", "bad_stack", "twice", "slabs", "too_wide",
                                  "half"])
def test_add_lora_errors(setup, case):
    from olmoasr_b200.lora import add_lora

    m = setup[0]
    kw = dict(r=8, alpha=8)
    if case == "r4":
        kw["r"] = 4
    elif case == "r12":
        kw["r"] = 12
    elif case == "r200":
        kw.update(r=200, targets=("decoder.mlp.0",))
    elif case == "half":
        m.half()
    elif case == "enc_cross":
        kw["targets"] = ("encoder.cross_attn.query",)
    elif case == "bad_name":
        kw["targets"] = ("decoder.attn.qkv",)
    elif case == "bad_stack":
        kw["targets"] = ("text.attn.query",)
    elif case == "twice":
        add_lora(m, 8, 8)
    elif case == "slabs":
        m.use_slabs()
    elif case == "too_wide":
        kw.update(r=72, targets=("decoder.attn.query", "decoder.attn.key", "decoder.attn.value"))
    with pytest.raises(ValueError):
        add_lora(m, **kw)


@pytest.mark.parametrize("extra", [None, "ln_and_query"])
def test_subset_slabs_hold_the_trainable_parameters_and_match_autograd(setup, extra):
    """use_slabs() after add_lora lays out the trainable parameters only, in backward-completion order, and direct
    slab gradients equal the autograd hand-over's.  "ln_and_query" re-enables the LayerNorms and one member of the
    fused q / k / v weight, so that group is only partly trainable."""
    from olmoasr_b200 import slab
    from olmoasr_b200.lora import add_lora

    m, mel, ti, ty, pm, lens = setup
    add_lora(m, 8, 16, targets=ALL)
    _randomize_b(m)
    if extra:
        for blk in list(m.encoder.blocks) + list(m.decoder.blocks):
            for p in blk.attn_ln.parameters():
                p.requires_grad_(True)
            blk.attn.query.weight.requires_grad_(True)
    ref = copy.deepcopy(m)
    train = [p for p in m.parameters() if p.requires_grad]
    sl = m.use_slabs()
    assert len(sl.params) == len(train) and {id(p) for p in sl.params} == {id(p) for p in train}
    assert sl.numel == sum((p.numel() + slab.ALIGN - 1) // slab.ALIGN * slab.ALIGN for p in train)
    assert sl.numel < sum(p.numel() for p in m.parameters()) // 10
    order = {pid: i for i, pid in enumerate(sl.layout_order)}   # units partition the layout into runs, in order
    assert [i for ps, _ in m.grad_units() for i in sorted(order[id(p)] for p in ps)] == list(range(len(order)))
    sl.zero_grad()
    m(mel, ti, pm, targets=ty).backward()
    ref(mel, ti, pm, targets=ty).backward()
    refp = dict(ref.named_parameters())
    for k, p in m.named_parameters():
        if not p.requires_grad:
            assert refp[k].grad is None, k
            continue
        assert p.grad.data_ptr() == sl.grad(p).data_ptr(), k
        g, w = p.grad, refp[k].grad
        assert float((g - w).norm() / (w.norm() + 1e-30)) <= 1e-5, k


def test_frozen_encoder_keeps_no_graph(setup):
    """Adapters in the decoder only: the encoder's output takes no gradient, so autograd records nothing in the
    encoder and its blocks keep no activations for a backward."""
    from olmoasr_b200.lora import add_lora

    m, mel, ti, ty, pm, lens = setup
    add_lora(m, 8, 16, targets=("decoder.attn.query", "decoder.attn.value"))
    xa = m.encoder(mel)
    assert xa.grad_fn is None and not xa.requires_grad


def _merged_reference(m, lora_model, mel, ti, ty, pm):
    """Loss and d(loss)/d(W_eff) of the plain model whose weights are W + s B A."""
    ref = copy.deepcopy(m)
    sd = {k: v for k, v in lora_model.state_dict().items() if ".lora_" not in k}
    for name, mod in lora_model.named_modules():
        if getattr(mod, "has_lora", False):
            sd[name + ".weight"] = mod.weight.detach() + mod.lora_scale * mod.lora_B.detach() @ mod.lora_A.detach()
    ref.load_state_dict(sd)
    loss = ref(mel, ti, pm, targets=ty)
    loss.backward()
    return loss, ref


@pytest.mark.parametrize("packed", [False, True])
def test_adapter_gradients_equal_autograd_through_the_merged_weight(setup, packed, monkeypatch):
    from olmoasr_b200 import kernels
    from olmoasr_b200.lora import add_lora
    from tests import test_packed_decoder_host as P

    m, mel, ti, ty, pm, lens = setup
    for fn in (P.attention_fwd_varlen, P.attention_bwd_varlen, P.embed_fwd_packed, P.embed_bwd_packed):
        monkeypatch.setattr(kernels, fn.__name__, fn)
    base = copy.deepcopy(m)
    add_lora(m, 8, 16, targets=ALL)
    _randomize_b(m)
    loss = m(mel, ti, targets=ty, text_lens=lens) if packed else m(mel, ti, pm, targets=ty)
    loss.backward()
    loss_ref, ref = _merged_reference(base, m, mel, ti, ty, pm)
    assert abs(loss.item() - loss_ref.item()) <= 2e-3 * abs(loss_ref.item())
    refp = dict(ref.named_parameters())
    checked = 0
    for name, mod in m.named_modules():
        if not getattr(mod, "has_lora", False):
            continue
        gw = refp[name + ".weight"].grad.double()
        s, A, B = mod.lora_scale, mod.lora_A.detach().double(), mod.lora_B.detach().double()
        for got, want in ((mod.lora_A.grad, s * B.t() @ gw), (mod.lora_B.grad, s * gw @ A.t())):
            rel = float((got.double() - want).norm() / want.norm())
            # both sides round activations to bf16 independently (1-3 % here); a wrong scale or sign is >= 50 %
            assert rel <= 5e-2, (name, rel)
        checked += 1
        assert mod.weight.grad is None and (mod.bias is None or mod.bias.grad is None)
    assert checked == 2 * 6 + 2 * 6


def test_linear_hook_path_uses_the_effective_weight(setup):
    from olmoasr_b200.lora import add_lora

    m = add_lora(setup[0], 8, 16)
    _randomize_b(m)
    lin = m.decoder.blocks[0].attn.value
    x = torch.randn(3, 5, 64).to(BF)
    with torch.no_grad():
        y = lin(x).float()
        w = lin.weight + lin.lora_scale * lin.lora_B @ lin.lora_A
        want = torch.nn.functional.linear(x.float(), w, lin.bias)
    assert float((y - want).norm() / want.norm()) <= 1e-2


def test_frozen_parameters_get_no_gradient_work(setup, monkeypatch):
    """Only adapters trainable: every wgrad is an adapter's (no base, tied-logits or stem wgrad), and with the adapters
    in the decoder only, no d(loss)/d(encoder output) and no encoder backward at all."""
    from olmoasr_b200 import _core
    from olmoasr_b200.lora import add_lora

    m, mel, ti, ty, pm, lens = setup
    add_lora(m, 8, 16, targets=("decoder.attn.query", "decoder.attn.value", "decoder.cross_attn.key"))
    _randomize_b(m)
    wgrads, dgrads = [], []
    real_wgrad, real_dgrad = _core.linear_wgrad, _core.lora_dgrad

    def rec_wgrad(dy, x, n_valid=None, side=None, out=None):
        wgrads.append((dy.shape[1] if n_valid is None else n_valid, x.shape[1]))
        return real_wgrad(dy, x, n_valid, side, out)

    def rec_dgrad(dy, w, ops, v, **kw):
        dgrads.append(tuple(dy.shape))
        return real_dgrad(dy, w, ops, v, **kw)

    monkeypatch.setattr(_core, "linear_wgrad", rec_wgrad)
    monkeypatch.setattr(_core, "lora_dgrad", rec_dgrad)
    loss = m(mel, ti, pm, targets=ty)
    loss.backward()
    assert wgrads and set(wgrads) <= {(8, 64), (64, 8)}, set(wgrads)
    assert len(wgrads) == 2 * 3 * 2                     # 2 layers x 3 adapters x (dA, dB)
    assert (2 * 1500, 128) not in dgrads                 # no dxa through the cross K / V weights
    assert all(rows != 2 * 1500 for rows, _ in dgrads)   # nothing of the encoder's backward ran
    for k, p in m.named_parameters():
        assert (p.grad is not None) == (".lora_" in k), k


def test_re_enabled_parameters_take_gradients(setup):
    from olmoasr_b200.lora import add_lora

    m, mel, ti, ty, pm, lens = setup
    add_lora(m, 8, 16)
    for blk in m.decoder.blocks:
        for p in blk.mlp_ln.parameters():
            p.requires_grad_(True)
    m.decoder.blocks[1].mlp[2].bias.requires_grad_(True)
    loss = m(mel, ti, pm, targets=ty)
    loss.backward()
    for k, p in m.named_parameters():
        want = ".lora_" in k or ".mlp_ln." in k and k.startswith("decoder") or k == "decoder.blocks.1.mlp.2.bias"
        assert (p.grad is not None) == want, k


def test_merge_lora_restores_the_reference_key_set(setup):
    from olmoasr_b200.lora import add_lora, merge_lora

    m, mel, ti, ty, pm, lens = setup
    ref_keys = set(m.state_dict())
    add_lora(m, 8, 16, targets=ALL)
    _randomize_b(m)
    with torch.no_grad():
        before = m(mel, ti, pm, targets=ty).item()
    lin = m.encoder.blocks[0].mlp[0]
    want = lin.weight.detach() + lin.lora_scale * lin.lora_B.detach() @ lin.lora_A.detach()
    merge_lora(m)
    assert set(m.state_dict()) == ref_keys
    assert torch.equal(lin.weight.detach(), want)
    assert all(p.requires_grad for p in m.parameters())
    with torch.no_grad():
        after = m(mel, ti, pm, targets=ty).item()
    assert abs(after - before) <= 2e-3 * abs(before)


def test_merge_lora_restores_the_flags_set_before_add_lora(setup):
    from olmoasr_b200.lora import add_lora, merge_lora

    m = setup[0]
    m.encoder.conv1.weight.requires_grad_(False)
    merge_lora(add_lora(m, 8, 16))
    assert [n for n, p in m.named_parameters() if not p.requires_grad] == ["encoder.conv1.weight"]
