"""Packed decoder training on the GPU: the varlen attention kernels and the packed embedding against the dense kernels
run on one sample at a time (bit for bit) and against the fp64 attention reference, then the packed model route against
the dense route and the fp32 oracle, and its determinism over optimizer steps at full medium depth."""
import gc

import pytest
import torch

from tests import attention_reference as ar

pytestmark = pytest.mark.gpu

HD = 64
DTYPES = [torch.bfloat16, torch.float16]
DT_ID = {torch.bfloat16: "bf16", torch.float16: "fp16"}
EDGE_LENS = [1, 31, 127, 128, 129, 255, 256, 448]     # around the 64- and 128-row tiles, next to each other
LOSS_SCALE = 2.0 ** 16


def _synthetic_lens():
    from olmoasr_b200 import synthetic
    return synthetic.text_batch(16)[3].tolist()


LENS = {"edges": EDGE_LENS, "synthetic": None}


def _rel(a, b):
    return float((a.float() - b.float()).norm() / (b.float().norm() + 1e-30))


def _nan(shape, dtype):
    return torch.full(shape, float("nan"), device="cuda", dtype=dtype)


def _single_key(n, Tkv, causal):
    """Query / key rows of one sample whose dS is exactly zero (a query that sees one key), as in the dense parity test."""
    vis = ar.visibility(n, Tkv, causal, Tkv if not causal else n, "cuda")
    one = vis.sum(dim=1) == 1
    return one, vis.any(dim=0) & ~(vis & ~one[:, None]).any(dim=0)


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("H", [16, 20])
@pytest.mark.parametrize("form", ["self", "cross"])
@pytest.mark.parametrize("batch", ["edges", "synthetic"])
def test_varlen_attention_equals_each_sample_alone(batch, form, H, dtype):
    from olmoasr_b200 import kernels as K
    from olmoasr_b200._core import PackedBatch

    lens = LENS[batch] or _synthetic_lens()
    B, S = len(lens), max(lens)
    pk = PackedBatch(lens, S, "cuda")
    N, W = pk.N, H * HD
    Ta = None if form == "self" else 1500
    kv_rows = N if Ta is None else B * Ta
    g = torch.Generator(device="cuda").manual_seed(7)
    q, do = (torch.randn(N, W, device="cuda", generator=g).to(dtype) for _ in range(2))
    k, v = (torch.randn(kv_rows, W, device="cuda", generator=g).to(dtype) for _ in range(2))
    o = _nan((N, W), dtype)
    o, lse = K.attention_fwd_varlen(q, k, v, pk, H, Tkv=Ta, out=o)
    dq, dk, dv = _nan((N, W), dtype), _nan((kv_rows, W), dtype), _nan((kv_rows, W), dtype)
    K.attention_bwd_varlen(q, k, v, o, do, lse, pk, H, Tkv=Ta, dq=dq, dk=dk, dv=dv)
    torch.cuda.synchronize()
    for t in (o, lse, dq, dk, dv):
        assert not t.isnan().any(), "a row was left unwritten"
    cu = pk.cu.tolist()
    for b, n in enumerate(lens):
        qr = slice(cu[b], cu[b + 1])
        kr = qr if Ta is None else slice(b * Ta, (b + 1) * Ta)
        tkv = n if Ta is None else Ta
        causal = Ta is None
        o1, lse1 = K.attention_fwd(q[qr], k[kr], v[kr], 1, H, n, tkv, causal=causal)
        dq1, dk1, dv1 = K.attention_bwd(q[qr], k[kr], v[kr], o1, do[qr], lse1, 1, H, n, tkv, causal=causal)
        assert torch.equal(o[qr], o1), (b, n, "o")
        assert torch.equal(lse[:, qr], lse1[0]), (b, n, "lse")
        assert torch.equal(dq[qr], dq1), (b, n, "dq")
        assert torch.equal(dk[kr], dk1), (b, n, "dk")
        assert torch.equal(dv[kr], dv1), (b, n, "dv")
        # and within the fp64 reference's tolerances of the dense attention tests
        ref = ar.reference(q[qr], k[kr], v[kr], do[qr], 1, H, n, tkv, causal=causal)
        emu = ar.reference(q[qr], k[kr], v[kr], do[qr], 1, H, n, tkv, causal=causal, emulate=dtype)
        single_q, single_k = _single_key(n, tkv, causal)
        got = {"o": o[qr], "dq": dq[qr], "dk": dk[kr], "dv": dv[kr]}
        rows = {"o": None, "dq": ~single_q, "dk": ~single_k, "dv": None}
        for key in ("dq", "dk"):
            noise = got[key][single_q if key == "dq" else single_k]
            assert noise.numel() == 0 or float(noise.abs().max()) <= 1e-3, (b, n, key)
        for key in ("o", "dq", "dk", "dv"):
            if rows[key] is None or rows[key].any():
                ar.check(got[key], ref[key], emu[key], rows=rows[key], name=f"{key} sample {b} len {n}")
        ar.check_lse(lse[:, qr][None], ref, name=f"lse sample {b} len {n}")


@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("batch", ["edges", "synthetic"])
def test_packed_embedding_equals_the_dense_rows(batch, dtype):
    from olmoasr_b200 import kernels as K
    from olmoasr_b200._core import PackedBatch

    lens = LENS[batch] or _synthetic_lens()
    B, S, d, V = len(lens), 448, 1024, 51865
    pk = PackedBatch(lens, S, "cuda")
    g = torch.Generator(device="cuda").manual_seed(3)
    ids = torch.randint(0, 400, (B, S), device="cuda", generator=g)     # few ids: many rows share one
    ids[0, 0] = 51864                                                      # padding_idx gets no gradient
    emb = torch.randn(V, d, device="cuda", generator=g)
    pos = torch.randn(S, d, device="cuda", generator=g)
    dense = K.embed_fwd(ids, emb, pos, 0, dtype=dtype)
    packed = K.embed_fwd_packed(ids, emb, pos, pk, dtype)
    rows = pk.rows.long()
    assert torch.equal(packed, dense[rows])
    dx = torch.zeros(B * S, d, device="cuda", dtype=dtype)                 # padded rows carry no gradient
    dx[rows] = torch.randn(pk.N, d, device="cuda", generator=g).to(dtype)
    demb_d, dpos_d = torch.zeros(V, d, device="cuda"), torch.zeros(S, d, device="cuda")
    demb_p, dpos_p = torch.zeros(V, d, device="cuda"), torch.zeros(S, d, device="cuda")
    K.embed_bwd(ids, dx, demb_d, dpos_d, 51864)
    K.embed_bwd_packed(ids, dx[rows].contiguous(), demb_p, dpos_p, pk, 51864)
    assert torch.equal(demb_p, demb_d) and torch.equal(dpos_p, dpos_d)


# ---------------------------------------------------------------------------------------------------- model
_ORACLE = {}


def _model_case(name):
    """(model, fp32 oracle loss, oracle gradients, the reference's bf16 gradient noise, inputs) for a benchmarked width
    at depth 2+2, or tiny at full depth."""
    from tests.test_model_gpu import _build_width
    from pathlib import Path

    golden = Path(__file__).resolve().parent / "golden"
    m, sd, dims, OM, mel, ti, ty, pm = _build_width(name, (4, 4) if name == "tiny" else (2, 2))
    if name not in _ORACLE:
        p = {k: v.clone().requires_grad_(k != "encoder.positional_embedding") for k, v in sd.items()}
        loss_ref = OM.token_ce(OM.model_forward(p, dims, mel, ti, pm, train_model=True), ty)
        loss_ref.backward()
        noise = torch.load(golden / ("grad_noise_tiny.pt" if name == "tiny" else f"model_{name}_2x2.pt"), weights_only=False)
        _ORACLE[name] = (loss_ref.item(), {k: v.grad for k, v in p.items() if v.grad is not None},
                         noise if name == "tiny" else noise["grad_noise"])
    return (m,) + _ORACLE[name] + ((mel.cuda(), ti.cuda(), ty.cuda(), pm.cuda()),)


def _step(m, inputs, dtype, lens=None):
    mel, ti, ty, pm = inputs
    if getattr(m, "_slabs", None) is not None:
        m._slabs.zero_grad()
    else:
        m.zero_grad(set_to_none=True)
    with torch.autocast("cuda", dtype=dtype):
        loss = m(mel, ti, targets=ty, text_lens=lens) if lens is not None else m(mel, ti, pm, targets=ty)
    scale = LOSS_SCALE if dtype == torch.float16 else 1.0   # unscaled, fp16 encoder attention gradients underflow
    (loss * scale).backward()
    return loss.item(), {k: p.grad.float().cpu() / scale for k, p in m.named_parameters()}


@pytest.mark.parametrize("slab", [False, True], ids=["autograd", "slab"])
@pytest.mark.parametrize("dtype", DTYPES, ids=DT_ID.get)
@pytest.mark.parametrize("name", ["tiny", "base", "small", "medium"])
def test_packed_model_matches_dense_and_oracle(name, dtype, slab):
    from olmoasr_b200 import synthetic

    m, loss_ref, g_ref, noise, inputs = _model_case(name)
    if slab:
        m.use_slabs()
    lens = synthetic.text_batch(2)[3]
    loss_d, g_d = _step(m, inputs, dtype)
    loss_p, g_p = _step(m, inputs, dtype, lens)
    assert abs(loss_p - loss_d) <= 1e-4 * abs(loss_d), (loss_p, loss_d)
    assert abs(loss_p - loss_ref) <= 1e-3 * abs(loss_ref), (loss_p, loss_ref)
    for k in g_d:
        e_pd, e_do, e_po = _rel(g_p[k], g_d[k]), _rel(g_d[k], g_ref[k]), _rel(g_p[k], g_ref[k])
        assert e_pd <= e_do, (k, e_pd, e_do)
        # the oracle tolerance of BASELINE.md that tests/test_model_gpu.py asserts
        assert e_po <= max(1.5 * noise[k], 2e-2), (k, e_po, noise[k])


def test_cuda_text_lens_are_refused():
    import olmoasr_b200 as ob
    from olmoasr_b200.model import OLMoASR
    from olmoasr_b200 import synthetic

    m = OLMoASR(ob.VARIANT_TO_DIMS["tiny"]).cuda()
    ti, ty, _, lens = synthetic.text_batch(2)
    mel = torch.zeros(2, 80, 3000, device="cuda")
    with pytest.raises(ValueError, match="host data"):
        m(mel, ti.cuda(), targets=ty.cuda(), text_lens=lens.cuda())


def test_full_depth_medium_three_adamw_steps():
    """Three FusedAdamW steps per route from the same weights on bench's 16-clip batch: losses within 1e-3 of each other
    at every step, and two packed runs bit-identical in losses and gradient slabs."""
    import olmoasr_b200 as ob
    from olmoasr_b200 import synthetic as synth
    from olmoasr_b200.model import OLMoASR
    from olmoasr_b200.optim import FusedAdamW

    dev = torch.device("cuda")
    B = 16
    mel = ob.log_mel_spectrogram(synth.waveforms(B, int16=True).to(dev))
    ti, ty, pm, lens = synth.text_batch(B)
    ti, ty, pm = ti.to(dev), ty.to(dev), pm.to(dev)

    def run(packed, ref_grads=None):
        torch.manual_seed(0)        # the same initial weights in every run
        with torch.device(dev):
            m = OLMoASR(ob.VARIANT_TO_DIMS["medium"])
        slabs = m.use_slabs()
        opt = FusedAdamW(m.parameters(), lr=1.5e-3, betas=(0.9, 0.98), eps=1e-6, weight_decay=0.1, max_grad_norm=1.0,
                         slabs=slabs)
        losses, grads = [], []
        for step in range(3):
            loss = m(mel, ti, targets=ty, text_lens=lens) if packed else m(mel, ti, pm, targets=ty)
            opt.zero_grad()
            loss.backward()
            if ref_grads is None:
                grads.append(slabs.G.cpu())
            else:
                assert torch.equal(slabs.G.cpu(), ref_grads[step]), f"gradient slab of step {step} differs between packed runs"
            opt.step()
            losses.append(loss.item())
        del m, opt, slabs, loss
        gc.collect()
        torch.cuda.empty_cache()     # the GEMM's split-K scratch is allocated outside torch's caching allocator
        return losses, grads

    dense, _ = run(False)
    packed, g1 = run(True)
    again, _ = run(True, g1)
    for a, b in zip(packed, dense):
        assert abs(a - b) <= 1e-3 * abs(b), (packed, dense)
    assert packed == again
