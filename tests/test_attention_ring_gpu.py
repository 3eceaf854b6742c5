"""Attention forward / backward at shapes where the loops meet the three-stage TMA rings' edges: key-tile and query-step
counts below, equal to and one past the ring depth (the forward and the dQ kernel step over 128-key tiles, the dK / dV
kernel over 64-query tiles), and a causal problem whose key lengths are shorter than one tile."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _sdpa_ref(q, k, v, B, H, Tq, Tkv, causal, kv_len):
    qh, kh, vh = (t.view(B, -1, H, 64).permute(0, 2, 1, 3) for t in (q, k, v))
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


def _close(got, want, rtol):
    atol = rtol * (want.abs().max().item() + 1e-12)
    err = (got.float() - want.float()).abs().max().item()
    assert err <= atol, f"max err {err} > {atol}"


@pytest.mark.parametrize("B,H,Tq,Tkv,causal,kv_len", [
    (1, 2, 256, 256, False, None),      # 2 key tiles, 4 query steps
    (1, 2, 384, 384, False, None),      # 3 key tiles (= ring depth), 6 query steps
    (2, 2, 385, 385, False, None),      # 4 key tiles (ring depth + 1), 7 query steps, ragged
    (2, 1, 192, 385, False, None),      # 3 query steps (= ring depth) against 4 key tiles
    (1, 1, 129, 200, False, None),      # 3 query steps, 2 key tiles, one-row tail
    (2, 2, 300, 300, True, [40, 100]),  # causal, every sample's keys within the first tile
])
def test_attention_ring_edges(B, H, Tq, Tkv, causal, kv_len):
    from olmoasr_b200 import kernels as K

    torch.manual_seed(5)
    d = H * 64
    q = torch.randn(B * Tq, d, device="cuda").bfloat16()
    kv = torch.randn(B * Tkv, 2 * d, device="cuda").bfloat16()   # K / V as column views of a fused buffer (ld = 2d)
    k, v = kv[:, :d], kv[:, d:]
    lens = torch.tensor(kv_len, device="cuda", dtype=torch.int32) if kv_len is not None else None
    o, lse = K.attention_fwd(q, k, v, B, H, Tq, Tkv, causal=causal, kv_len=lens)
    qr, kr, vr = (t.float().clone().requires_grad_(True) for t in (q, k, v))
    oref = _sdpa_ref(qr, kr, vr, B, H, Tq, Tkv, causal, kv_len)
    _close(o, oref.detach(), rtol=1.0 / 64)
    dout = torch.randn(B * Tq, d, device="cuda").bfloat16()
    oref.backward(dout.float())
    dq, dk, dv = K.attention_bwd(q, k, v, o, dout, lse, B, H, Tq, Tkv, causal=causal, kv_len=lens)
    _close(dq, qr.grad, rtol=1.0 / 48)
    _close(dk, kr.grad, rtol=1.0 / 48)
    _close(dv, vr.grad, rtol=1.0 / 48)
    if kv_len is not None:   # keys past a sample's length get exactly zero gradient
        for i, n in enumerate(kv_len):
            rows = slice(i * Tkv + n, (i + 1) * Tkv)
            assert not dk[rows].any() and not dv[rows].any()
