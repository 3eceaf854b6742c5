"""fp64 reference of the training attention kernels and the tolerance rule their tests use (TEST INFRASTRUCTURE).

Plain torch, on whichever device the inputs live; no import of olmoasr_b200.  Tensors are in the kernels' layout
(include/oasr_b200.h): q / o / dout / dq are (B*Tq, H*64), k / v / dk / dv are (B*Tkv, H*64), lse is (B, H, Tq).

`reference(..., emulate=None)` states the operation in fp64 from the exact 16-bit inputs: the scaled scores masked by
`causal` (key <= query) and `kv_len` (keys >= kv_len[b] hidden, kv_len clamped to [1, Tkv] as the kernels do), O,
the natural-log lse, and the backward as explicit formulas (D = rowsum(dO o O), dS = P o (dP - D), dQ = scale dS K,
dK = scale dS^T Q, dV = P^T dO).  One sample at a time, so B = 16 at T = 1500 never holds more than one sample's
(H, Tq, Tkv) fp64 matrices.

`reference(..., emulate=dtype)` is the rounding-point yardstick: the same computation in fp32, rounded to the 16-bit
type where any 16-bit flash implementation has to round -- the unnormalised P before P V, P before dV, dS before the
dQ and dK products, and each output once.  Its distance from fp64 is what 16-bit storage alone costs.

`check(got, ref64, emu, rows)` compares per row -- one (query, head) for O and dQ, one (key, head) for dK and dV --
the relative L2 error, each row's norm floored at FLOOR x the tensor's RMS row norm (not the median: where most rows
are exactly zero, such as dQ of queries that see a single key, a median floor would vanish and every zero row would
divide fp32 noise by nothing).  A reference that is identically zero is compared exactly.  It passes when

    max row error (kernel)  <= ALPHA x max row error (yardstick) + BETA x u
    mean row error (kernel) <= ALPHA x mean row error (yardstick)

with u = 2^-8 for bf16 and 2^-11 for fp16.  The lse has no 16-bit rounding point; `check_lse` bounds the kernel's
error by LSE_TOL x (1 + max |scaled score| of the row), the scale of the fp32 score sums it is computed from.

With OASR_ATTN_REPORT set to a file name, check() and check_lse() append one JSON line per call to that file;
tools/attention_error_table.py runs tests/test_attention_parity_gpu.py that way and prints the table below.

Measured on an H100 SXM (80 GB HBM3, 700 W power limit) over tests/test_attention_parity_gpu.py: kernel / yardstick
ratios, max-row ratio / mean-row ratio, the largest over the cases of each group:

    group            dtype   O            dQ           dK           dV
    production       bf16    1.02 / 1.00  1.10 / 1.00  1.04 / 1.00  1.02 / 1.00
                     fp16    1.03 / 1.00  1.08 / 1.00  1.04 / 1.00  1.14 / 1.00
    mask edges       bf16    1.01 / 1.00  1.00 / 1.00  1.00 / 1.00  1.00 / 1.00
                     fp16    1.01 / 1.00  1.01 / 1.00  1.04 / 1.00  1.06 / 1.00
    score regimes    bf16    1.00 / 1.00  1.92 / 1.49  1.57 / 1.51  1.00 / 1.00
                     fp16    1.00 / 1.00  1.00 / 1.01  1.27 / 1.01  1.00 / 1.00
    scale            bf16    1.00 / 1.00  1.00 / 1.01  1.01 / 1.00  1.00 / 1.00
                     fp16    1.02 / 1.00  1.00 / 1.00  0.97 / 1.00  1.00 / 1.00

The kernels round where the yardstick does, so their error tracks it.  The largest ratio, 1.92, is dQ of a peaked bf16
row, where dS = P o (dP - D) cancels and the kernel's and the yardstick's independent 1-ulp roundings of O (through D)
decide the worst row; ALPHA = 2.5 leaves 30% above it.  No case needed the absolute term, so BETA = 0.  The kernels'
worst lse error was 0.35 x LSE_TOL.  Every deliberately wrong problem of tests/test_attention_reference_host.py fails
by a ratio of 9 or more, and the kernels fed kv_len - 1 by 27.5 or more.
"""
from __future__ import annotations

import json
import os
from typing import Dict, NamedTuple, Optional

import torch

HD = 64
U = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
ALPHA = 2.5
BETA = 0.0
FLOOR = 1.0 / 8
LSE_TOL = 2.0 ** -20


def n_visible(kv_len, b: int, Tkv: int) -> int:
    """Keys of sample b the kernels attend to: kv_len[b] clamped to [1, Tkv] (all Tkv without kv_len)."""
    if kv_len is None:
        return Tkv
    return min(max(int(kv_len[b]), 1), Tkv)


def visibility(Tq: int, Tkv: int, causal: bool, n_valid: int, device) -> torch.Tensor:
    """(Tq, Tkv) bool: key j is visible to query i."""
    j = torch.arange(Tkv, device=device)
    vis = (j < n_valid).expand(Tq, Tkv)
    if causal:
        vis = vis & (j[None, :] <= torch.arange(Tq, device=device)[:, None])
    return vis


def _heads(x: torch.Tensor, b: int, T: int, H: int, dt) -> torch.Tensor:
    """Rows of sample b as (H, T, 64) in type dt."""
    return x[b * T:(b + 1) * T, :H * HD].to(dt).reshape(T, H, HD).transpose(0, 1)


def _rows(x: torch.Tensor) -> torch.Tensor:
    """(H, T, 64) -> (T, H*64), the kernels' layout."""
    return x.transpose(0, 1).reshape(x.shape[1], -1)


def sample_fp64(q, k, v, dout, vis, scale) -> Dict[str, torch.Tensor]:
    """fp64 attention of one sample: q (H, Tq, 64), k / v (H, Tkv, 64), dout (H, Tq, 64) or None, vis (Tq, Tkv)."""
    s = (q @ k.transpose(1, 2)) * scale
    s = s.masked_fill(~vis, float("-inf"))
    lse = torch.logsumexp(s, dim=-1)
    p = torch.exp(s - lse[..., None])
    o = p @ v
    out = {"o": o, "lse": lse, "smax": s.masked_fill(~vis, 0.0).abs().amax(dim=-1)}
    if dout is not None:
        dlt = (dout * o).sum(dim=-1)
        dp = dout @ v.transpose(1, 2)
        ds = p * (dp - dlt[..., None])
        out["dq"] = scale * (ds @ k)
        out["dk"] = scale * (ds.transpose(1, 2) @ q)
        out["dv"] = p.transpose(1, 2) @ dout
    return out


def sample_emulated(q, k, v, dout, vis, scale, dtype) -> Dict[str, torch.Tensor]:
    """fp32 attention of one sample rounded to `dtype` at a flash kernel's rounding points (arguments as sample_fp64)."""
    rnd = lambda x: x.to(dtype).float()   # noqa: E731
    s = (q @ k.transpose(1, 2)) * scale
    s = s.masked_fill(~vis, float("-inf"))
    m = s.amax(dim=-1, keepdim=True)
    pu = torch.exp(s - m)
    l = pu.sum(dim=-1, keepdim=True)
    o = rnd((rnd(pu) @ v) / l)
    lse = (m + torch.log(l))[..., 0]
    out = {"o": o, "lse": lse}
    if dout is not None:
        p = torch.exp(s - lse[..., None])
        dlt = (dout * o).sum(dim=-1)
        dp = dout @ v.transpose(1, 2)
        ds = rnd(p * (dp - dlt[..., None]))
        out["dq"] = rnd(scale * (ds @ k))
        out["dk"] = rnd(scale * (ds.transpose(1, 2) @ q))
        out["dv"] = rnd(rnd(p).transpose(1, 2) @ dout)
    return out


def reference(q, k, v, dout, B, H, Tq, Tkv, causal=False, kv_len=None, scale=None, emulate=None, vis_fn=None):
    """Attention forward (and backward when dout is given) in the kernels' layout: o, lse (natural log), smax (the
    row's largest |scaled score|; fp64 only), dq, dk, dv.  fp64 when emulate is None, else the rounding-point yardstick
    for the 16-bit type `emulate`.  vis_fn(b, vis) -> vis may alter a sample's visibility (tests of the tests)."""
    scale = HD ** -0.5 if scale is None else scale
    dt = torch.float64 if emulate is None else torch.float32
    kv_len = kv_len.tolist() if torch.is_tensor(kv_len) else kv_len
    parts = {}
    for b in range(B):
        vis = visibility(Tq, Tkv, causal, n_visible(kv_len, b, Tkv), q.device)
        if vis_fn is not None:
            vis = vis_fn(b, vis)
        args = [_heads(q, b, Tq, H, dt), _heads(k, b, Tkv, H, dt), _heads(v, b, Tkv, H, dt),
                None if dout is None else _heads(dout, b, Tq, H, dt), vis, scale]
        res = sample_fp64(*args) if emulate is None else sample_emulated(*args, emulate)
        for key, val in res.items():
            parts.setdefault(key, []).append(val if key in ("lse", "smax") else _rows(val))
    return {key: torch.stack(val) if key in ("lse", "smax") else torch.cat(val) for key, val in parts.items()}


class RowErrors(NamedTuple):
    worst: float        # kernel's largest row error
    mean: float         # kernel's mean row error
    emu_worst: float    # the same for the yardstick
    emu_mean: float
    worst_ratio: float  # worst / emu_worst
    mean_ratio: float   # mean / emu_mean


def row_errors(got, ref64, emu, rows: Optional[torch.Tensor] = None) -> RowErrors:
    """Relative L2 error per 64-wide row (one position of one head).  rows: optional bool (n,) over the positions
    (the tensors' first dimension) that take part."""
    ref = ref64.double()
    g, e = got.double(), emu.double()
    if rows is not None:
        ref, g, e = ref[rows], g[rows], e[rows]
    ref, g, e = (t.reshape(-1, HD) for t in (ref, g, e))
    norm = ref.norm(dim=1)
    floor = FLOOR * float(norm.square().mean().sqrt())
    assert floor > 0, "row_errors: the reference is identically zero"
    denom = norm.clamp_min(floor)
    eg = (g - ref).norm(dim=1) / denom
    ee = (e - ref).norm(dim=1) / denom
    worst, mean = float(eg.max()), float(eg.mean())
    ew, em = float(ee.max()), float(ee.mean())
    return RowErrors(worst, mean, ew, em, worst / max(ew, 1e-300), mean / max(em, 1e-300))


def _report(**fields) -> None:
    path = os.environ.get("OASR_ATTN_REPORT")
    if path:
        with open(path, "a") as f:
            f.write(json.dumps({"test": os.environ.get("PYTEST_CURRENT_TEST", ""), **fields}) + "\n")


def check(got, ref64, emu, rows: Optional[torch.Tensor] = None, *, dtype=None, name: str = "") -> Optional[RowErrors]:
    """Assert the tolerance rule of the module docstring; dtype (default got's) picks u.  Where the reference's rows
    are all exactly zero the kernel's must be too."""
    dtype = dtype or got.dtype
    sel = (lambda t: t) if rows is None else (lambda t: t[rows])   # noqa: E731
    if not sel(ref64).any():
        assert not sel(got).any(), f"{name}: the reference is zero, the result is not"
        return None
    r = row_errors(got, ref64, emu, rows)
    _report(kind="rows", name=name, dtype=str(dtype).removeprefix("torch."), **r._asdict())
    ok = r.worst <= ALPHA * r.emu_worst + BETA * U[dtype] and r.mean <= ALPHA * r.emu_mean
    assert ok, f"{name}: {r}"
    return r


def check_lse(got_log2, ref, rows: Optional[torch.Tensor] = None, name: str = "lse") -> float:
    """Kernel lse (log2 domain) x ln 2 against the fp64 natural-log lse; returns the worst error in LSE_TOL units.
    rows: optional bool (Tq,) of the query positions that take part."""
    err = (got_log2.double() * 0.6931471805599453 - ref["lse"].double()).abs() / (1.0 + ref["smax"].double())
    if rows is not None:
        err = err[..., rows]
    worst = float(err.max()) / LSE_TOL
    _report(kind="lse", name=name, lse_tol_units=worst)
    assert worst <= 1.0, f"{name}: lse error {worst:.3g} x LSE_TOL"
    return worst
